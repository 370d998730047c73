// Road centre lines for `rs features --type road` (DESIGN.md §8): Zhang-Suen thinning of halo'd binary planes, the m-degree of
// every skeleton pixel, the one-pass spur pruning, and the chain lists of the pruned skeleton.
//
// thin_kernel: one CTA per plane. The plane lives bit-packed in shared memory for every iteration (bit j of word k of a row is
// column 32 k + j). Each thread computes the new words of up to THIN_WORDS words 32 pixels at a time: B (the foreground count of
// P2..P9) with word-wide adders, A (the 0 -> 1 transitions of P2, P3, ..., P9, P2) with an at-least-one / at-least-two pair. The
// new words wait in registers between two barriers, so every deletion of a sub-iteration is decided on the state at its start
// with one buffer. __syncthreads_or ends the loop after the first full iteration that deleted nothing.
//
// Graph: pixels are m-adjacent when they are 4-neighbours, or diagonal neighbours with no common 4-neighbour in the skeleton.
// degree_kernel writes each skeleton pixel's m-degree (-1 off the skeleton). prune_kernel walks from every endpoint, at most
// min_length steps, and clears the spurs and short isolated pieces it decides on the input graph. Chains of the pruned graph:
// a node (degree != 2) starts a walk toward each m-neighbour and keeps it when it ends at a larger node, or back at itself through
// a larger last pixel than its second (so each chain is kept from exactly one of its two ends); a node-free cycle starts at its
// smallest pixel, which rsb_label_components gives as the root of its 8-connected component (m- and 8-connected components are
// the same), toward the smaller of its two neighbours. count_kernel (one CTA per plane row) counts chains and pixels per pixel,
// scan_kernel turns the row sums into row offsets and tile totals, and write_kernel walks again and writes the pixel lists.

#include <stdint.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr int THIN_THREADS = 1024;
constexpr int THIN_WORDS = RSB_ROAD_MAX_WORDS / THIN_THREADS;  // words per thread, held in registers
constexpr int PASS_THREADS = 256;
constexpr int ROW_THREADS = 256;
constexpr int SCAN_THREADS = 1024;
constexpr int CHAIN_SHIFT = 28;  // packed per-pixel counts: chains << CHAIN_SHIFT | pixels

static_assert(RSB_ROAD_MAX_WORDS % THIN_THREADS == 0, "words per thread");

__device__ __forceinline__ uint32_t word_at(const uint32_t* S, int H, int nw, int r, int k) {
    return (r < 0 || r >= H || k < 0 || k >= nw) ? 0u : S[r * nw + k];
}

// new value of word w after one Zhang-Suen sub-iteration (sub 0 or 1) on the shared plane
__device__ __forceinline__ uint32_t zs_word(const uint32_t* S, int H, int nw, int w, int sub) {
    const int r = w / nw, k = w - r * nw;
    const uint32_t c = S[w];
    if (!c) return 0u;
    const uint32_t n = word_at(S, H, nw, r - 1, k), s = word_at(S, H, nw, r + 1, k);
    const uint32_t nl = word_at(S, H, nw, r - 1, k - 1), nr = word_at(S, H, nw, r - 1, k + 1);
    const uint32_t cl = word_at(S, H, nw, r, k - 1), cr = word_at(S, H, nw, r, k + 1);
    const uint32_t sl = word_at(S, H, nw, r + 1, k - 1), sr = word_at(S, H, nw, r + 1, k + 1);
    // column c - 1 of bit j is bit j - 1: (x << 1) | (left word >> 31); column c + 1: (x >> 1) | (right word << 31)
    const uint32_t p2 = n, p3 = (n >> 1) | (nr << 31), p4 = (c >> 1) | (cr << 31), p5 = (s >> 1) | (sr << 31);
    const uint32_t p6 = s, p7 = (s << 1) | (sl >> 31), p8 = (c << 1) | (cl >> 31), p9 = (n << 1) | (nl >> 31);
    const uint32_t P[8] = {p2, p3, p4, p5, p6, p7, p8, p9};
    uint32_t b0 = 0, b1 = 0, b2 = 0, b3 = 0, one = 0, two = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t x = P[i];
        const uint32_t c0 = b0 & x;
        b0 ^= x;
        const uint32_t c1 = b1 & c0;
        b1 ^= c0;
        const uint32_t c2 = b2 & c1;
        b2 ^= c1;
        b3 |= c2;
        const uint32_t t = ~x & P[(i + 1) & 7];
        two |= one & t;
        one |= t;
    }
    const uint32_t b_ok = (b1 | b2 | b3) & ~(b3 | (b2 & b1 & b0));  // 2 <= B <= 6
    const uint32_t a_ok = one & ~two;                               // A == 1
    const uint32_t keep = sub == 0 ? ~(p2 & p4 & p6) & ~(p4 & p6 & p8) : ~(p2 & p4 & p8) & ~(p2 & p6 & p8);
    return c & ~(b_ok & a_ok & keep);
}

__global__ void __launch_bounds__(THIN_THREADS) thin_kernel(const uint8_t* __restrict__ planes, int64_t image_stride, int H, int W,
                                                            uint8_t* __restrict__ skel, int32_t* __restrict__ iterations) {
    extern __shared__ uint32_t S[];
    const int nw = (W + 31) >> 5, total = H * nw;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NWARPS = THIN_THREADS / 32;
    const uint8_t* img = planes + static_cast<int64_t>(blockIdx.x) * image_stride;
    for (int w = warp; w < total; w += NWARPS) {
        const int r = w / nw, x = (w - r * nw) * 32 + lane;
        const uint32_t b = __ballot_sync(0xffffffffu, x < W && img[static_cast<int64_t>(r) * W + x] != 0);
        if (lane == 0) S[w] = b;
    }
    __syncthreads();

    int it = 0;
    while (true) {
        int changed = 0;
        for (int sub = 0; sub < 2; ++sub) {
            uint32_t nv[THIN_WORDS];
#pragma unroll
            for (int j = 0; j < THIN_WORDS; ++j) {
                const int w = threadIdx.x + j * THIN_THREADS;
                nv[j] = w < total ? zs_word(S, H, nw, w, sub) : 0u;
            }
            __syncthreads();
#pragma unroll
            for (int j = 0; j < THIN_WORDS; ++j) {
                const int w = threadIdx.x + j * THIN_THREADS;
                if (w < total && nv[j] != S[w]) {
                    S[w] = nv[j];
                    changed = 1;
                }
            }
            if (sub == 0) __syncthreads();
        }
        ++it;
        if (!__syncthreads_or(changed)) break;
    }

    uint8_t* out = skel + static_cast<int64_t>(blockIdx.x) * H * W;
    for (int w = warp; w < total; w += NWARPS) {
        const int r = w / nw, x = (w - r * nw) * 32 + lane;
        if (x < W) out[static_cast<int64_t>(r) * W + x] = (S[w] >> lane) & 1u;
    }
    if (threadIdx.x == 0) iterations[blockIdx.x] = it;
}

__device__ __forceinline__ bool on(const uint8_t* s, int H, int W, int y, int x) {
    return y >= 0 && y < H && x >= 0 && x < W && s[y * W + x];
}

// the m-neighbours of skeleton pixel (y, x) in increasing pixel index -> their count
__device__ __forceinline__ int m_neighbours(const uint8_t* s, int H, int W, int y, int x, int* out) {
    int n = 0;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            if (dy == 0 && dx == 0) continue;
            if (!on(s, H, W, y + dy, x + dx)) continue;
            if (dy != 0 && dx != 0 && (on(s, H, W, y + dy, x) || on(s, H, W, y, x + dx))) continue;
            out[n++] = (y + dy) * W + x + dx;
        }
    return n;
}

// the m-neighbour of degree-2 pixel p other than prev
__device__ __forceinline__ int other(const uint8_t* s, int H, int W, int p, int prev) {
    int nb[8];
    m_neighbours(s, H, W, p / W, p % W, nb);
    return nb[0] == prev ? nb[1] : nb[0];
}

__global__ void __launch_bounds__(PASS_THREADS) degree_kernel(const uint8_t* __restrict__ skel, int H, int W, int8_t* __restrict__ deg) {
    const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
    if (i >= H * W) return;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * H * W;
    const uint8_t* s = skel + base;
    int nb[8];
    deg[base + i] = s[i] ? static_cast<int8_t>(m_neighbours(s, H, W, i / W, i % W, nb)) : static_cast<int8_t>(-1);
}

// one thread per pixel; endpoints walk at most min_length steps and clear what the rule removes in out (a copy of skel)
__global__ void __launch_bounds__(PASS_THREADS) prune_kernel(const uint8_t* __restrict__ skel, const int8_t* __restrict__ deg, int H, int W,
                                                             int min_length, uint8_t* __restrict__ out) {
    const int e = blockIdx.x * PASS_THREADS + threadIdx.x;
    if (e >= H * W) return;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * H * W;
    const uint8_t* s = skel + base;
    const int8_t* d = deg + base;
    if (d[e] != 1) return;
    int nb[8];
    m_neighbours(s, H, W, e / W, e % W, nb);
    int k = 1, prev = e, cur = nb[0], remove = 0;
    while (k < min_length) {
        const int dc = d[cur];
        if (dc >= 3) {  // a spur of k pixels, not counting the junction
            remove = k;
            break;
        }
        if (dc == 1) {  // endpoint to endpoint, k + 1 pixels
            remove = k + 1 < min_length ? k + 1 : 0;
            break;
        }
        ++k;
        const int next = other(s, H, W, cur, prev);
        prev = cur;
        cur = next;
    }
    prev = -1;
    cur = e;
    for (int j = 0; j < remove; ++j) {
        out[base + cur] = 0;
        if (j + 1 == remove) break;
        const int next = j == 0 ? nb[0] : other(s, H, W, cur, prev);
        prev = cur;
        cur = next;
    }
}

// nodes mark their component's root: areas[root] = 0 means "has a node" (areas of roots are otherwise >= 1)
__global__ void __launch_bounds__(PASS_THREADS) node_flag_kernel(const int8_t* __restrict__ deg, const int32_t* __restrict__ labels, int HW,
                                                                 int32_t* areas) {
    const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
    if (i >= HW) return;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * HW;
    const int d = deg[base + i];
    if (d >= 0 && d != 2) areas[base + labels[base + i]] = 0;
}

// walks from p through q until a node, or back to p; writes the pixels to out when given -> length; end, before_end
__device__ __forceinline__ int walk(const uint8_t* s, const int8_t* d, int H, int W, int p, int q, int32_t* out, int& end, int& before_end) {
    int prev = p, cur = q, len = 2;
    if (out) {
        out[0] = p;
        out[1] = q;
    }
    while (cur != p && d[cur] == 2) {
        const int next = other(s, H, W, cur, prev);
        prev = cur;
        cur = next;
        if (out) out[len] = cur;
        ++len;
    }
    end = cur;
    before_end = prev;
    return len;
}

// the chains pixel p starts: visits (second pixel, length) of each in order of the second pixel; returns their count
template <typename F>
__device__ __forceinline__ int chains_of(const uint8_t* s, const int8_t* d, const int32_t* labels, const int32_t* flags, int H, int W, int p, F visit) {
    const int dp = d[p];
    if (dp < 0) return 0;
    int nb[8];
    const int n = m_neighbours(s, H, W, p / W, p % W, nb);
    if (dp != 2) {
        int c = 0;
        for (int j = 0; j < n; ++j) {
            int e, b;
            const int len = walk(s, d, H, W, p, nb[j], nullptr, e, b);
            if (e > p || (e == p && nb[j] < b)) {
                visit(nb[j], len);
                ++c;
            }
        }
        return c;
    }
    if (labels[p] != p || flags[p] == 0) return 0;
    int e, b;
    visit(nb[0], walk(s, d, H, W, p, nb[0], nullptr, e, b));  // nb[0] is the smaller neighbour
    return 1;
}

__device__ __forceinline__ int64_t block_sum(int64_t v, int64_t* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    int64_t t = 0;
    if (threadIdx.x == 0)
        for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) t += red[i];
    __syncthreads();
    return t;
}

// exclusive prefix of v over the block (in thread order) -> the prefix; total = the block's sum
__device__ __forceinline__ int64_t block_exclusive(int64_t v, int64_t* red, int64_t& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int64_t x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) red[warp] = x;
    __syncthreads();
    int64_t before = 0;
    total = 0;
    for (int i = 0; i < nwarps; ++i) {
        if (i < warp) before += red[i];
        total += red[i];
    }
    __syncthreads();
    return before + x - v;
}

// grid (H, N): counts[p] = chains << CHAIN_SHIFT | pixels of the chains p starts; row_sums[n][y] = the row's (chains << 32 | pixels)
__global__ void __launch_bounds__(ROW_THREADS) count_kernel(const uint8_t* __restrict__ skel, const int8_t* __restrict__ deg,
                                                            const int32_t* __restrict__ labels, const int32_t* __restrict__ flags, int H, int W,
                                                            int32_t* __restrict__ counts, int64_t* __restrict__ row_sums) {
    __shared__ int64_t red[ROW_THREADS / 32];
    const int y = blockIdx.x;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * H * W;
    int64_t sum = 0;
    for (int x = threadIdx.x; x < W; x += ROW_THREADS) {
        const int p = y * W + x;
        int pixels = 0;
        const int c = chains_of(skel + base, deg + base, labels + base, flags + base, H, W, p, [&](int, int len) { pixels += len; });
        counts[base + p] = (c << CHAIN_SHIFT) | pixels;
        sum += (static_cast<int64_t>(c) << 32) + pixels;
    }
    const int64_t t = block_sum(sum, red);
    if (threadIdx.x == 0) row_sums[static_cast<int64_t>(blockIdx.y) * H + y] = t;
}

// one CTA per plane: row_sums become exclusive row offsets; totals[n] = the plane's (chains << 32 | pixels)
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(int64_t* row_sums, int H, int64_t* __restrict__ totals) {
    __shared__ int64_t red[SCAN_THREADS / 32];
    int64_t* rs = row_sums + static_cast<int64_t>(blockIdx.x) * H;
    int64_t carry = 0;
    for (int y0 = 0; y0 < H; y0 += SCAN_THREADS) {
        const int y = y0 + threadIdx.x;
        const int64_t v = y < H ? rs[y] : 0;
        int64_t total;
        const int64_t ex = block_exclusive(v, red, total);
        if (y < H) rs[y] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

// grid (H, N): writes the chains each pixel of row y starts at its place in the batch's lists
__global__ void __launch_bounds__(ROW_THREADS) write_kernel(const uint8_t* __restrict__ skel, const int8_t* __restrict__ deg,
                                                            const int32_t* __restrict__ labels, const int32_t* __restrict__ flags, int H, int W,
                                                            const int32_t* __restrict__ counts, const int64_t* __restrict__ row_offsets,
                                                            const int64_t* __restrict__ chain_base, const int64_t* __restrict__ pixel_base,
                                                            int64_t* __restrict__ chain_offsets, int32_t* __restrict__ pixels) {
    __shared__ int64_t red[ROW_THREADS / 32];
    const int y = blockIdx.x, n = blockIdx.y;
    const int64_t base = static_cast<int64_t>(n) * H * W;
    const int64_t row = row_offsets[static_cast<int64_t>(n) * H + y];
    int64_t next_chain = chain_base[n] + (row >> 32), next_pixel = pixel_base[n] + (row & 0xffffffffll);
    const uint8_t* s = skel + base;
    const int8_t* d = deg + base;
    for (int x0 = 0; x0 < W; x0 += ROW_THREADS) {
        const int x = x0 + threadIdx.x, p = y * W + x;
        const int32_t c = x < W ? counts[base + p] : 0;
        const int64_t v = (static_cast<int64_t>(c >> CHAIN_SHIFT) << 32) + (c & ((1 << CHAIN_SHIFT) - 1));
        int64_t total;
        const int64_t ex = block_exclusive(v, red, total);
        if (c != 0) {
            int64_t ci = next_chain + (ex >> 32), pi = next_pixel + (ex & 0xffffffffll);
            chains_of(s, d, labels + base, flags + base, H, W, p, [&](int q, int len) {
                int e, b;
                chain_offsets[ci++] = pi;
                walk(s, d, H, W, p, q, pixels + pi, e, b);
                pi += len;
            });
        }
        next_chain += total >> 32;
        next_pixel += total & 0xffffffffll;
    }
}

int check_shape(const char* what, int N, int H, int W) {
    if (N < 1 || N > 65535 || H < 1 || W < 1 || H > RSB_ROAD_MAX_SIZE || W > RSB_ROAD_MAX_SIZE)
        return set_error(RSB_E_UNSUPPORTED, "%s: N=%d H=%d W=%d (need 1 <= N <= 65535 and 1 <= H, W <= %d)", what, N, H, W, RSB_ROAD_MAX_SIZE);
    return RSB_OK;
}

dim3 pass_grid(int N, int H, int W) { return dim3(static_cast<unsigned>((H * W + PASS_THREADS - 1) / PASS_THREADS), static_cast<unsigned>(N)); }

int launched(const char* what) {
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, what);
}

}  // namespace

extern "C" int rsb_road_thin(const uint8_t* planes, int64_t image_stride, int32_t N, int32_t H, int32_t W, uint8_t* skel, int32_t* iterations,
                             void* stream) {
    if (!planes || !skel || !iterations) return set_error(RSB_E_INVALID, "road_thin: null pointer");
    int rc = check_shape("road_thin", N, H, W);
    if (rc != RSB_OK) return rc;
    const int64_t words = static_cast<int64_t>(H) * ((W + 31) / 32);
    if (words > RSB_ROAD_MAX_WORDS)
        return set_error(RSB_E_UNSUPPORTED, "road_thin: a %d x %d plane takes %lld 32-bit row words, more than the %d that fit the kernel's shared memory",
                         H, W, (long long)words, RSB_ROAD_MAX_WORDS);
    if (image_stride < static_cast<int64_t>(H) * W)
        return set_error(RSB_E_INVALID, "road_thin: image_stride %lld < H*W = %lld", (long long)image_stride, (long long)H * W);
    rc = rsb_device_ok();
    if (rc != RSB_OK) return rc;
    const int smem = static_cast<int>(words * 4);
    cudaError_t e = cudaFuncSetAttribute(thin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RSB_ROAD_MAX_WORDS * 4);
    if (e != cudaSuccess) return set_cuda_error(e, "road_thin: shared memory attribute");
    thin_kernel<<<N, THIN_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(planes, image_stride, H, W, skel, iterations);
    return launched("road_thin launch");
}

extern "C" int rsb_road_degree(const uint8_t* skel, int32_t N, int32_t H, int32_t W, int8_t* deg, void* stream) {
    if (!skel || !deg) return set_error(RSB_E_INVALID, "road_degree: null pointer");
    int rc = check_shape("road_degree", N, H, W);
    if (rc != RSB_OK) return rc;
    rc = rsb_device_ok();
    if (rc != RSB_OK) return rc;
    degree_kernel<<<pass_grid(N, H, W), PASS_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(skel, H, W, deg);
    return launched("road_degree launch");
}

extern "C" int rsb_road_prune(const uint8_t* skel, const int8_t* deg, int32_t N, int32_t H, int32_t W, int32_t min_length, uint8_t* out, void* stream) {
    if (!skel || !deg || !out) return set_error(RSB_E_INVALID, "road_prune: null pointer");
    int rc = check_shape("road_prune", N, H, W);
    if (rc != RSB_OK) return rc;
    if (min_length < 0) return set_error(RSB_E_INVALID, "road_prune: min_length %d (need >= 0)", min_length);
    if (out == skel) return set_error(RSB_E_INVALID, "road_prune: out must not alias skel");
    rc = rsb_device_ok();
    if (rc != RSB_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const cudaError_t e = cudaMemcpyAsync(out, skel, static_cast<size_t>(N) * H * W, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return set_cuda_error(e, "road_prune: copy");
    prune_kernel<<<pass_grid(N, H, W), PASS_THREADS, 0, st>>>(skel, deg, H, W, min_length, out);
    return launched("road_prune launch");
}

extern "C" int rsb_road_chain_count(const uint8_t* skel, const int8_t* deg, const int32_t* labels, int32_t* flags, int32_t N, int32_t H, int32_t W,
                                    int32_t* counts, int64_t* row_offsets, int64_t* totals, void* stream) {
    if (!skel || !deg || !labels || !flags || !counts || !row_offsets || !totals) return set_error(RSB_E_INVALID, "road_chain_count: null pointer");
    int rc = check_shape("road_chain_count", N, H, W);
    if (rc != RSB_OK) return rc;
    if (labels == flags) return set_error(RSB_E_INVALID, "road_chain_count: labels and flags must not alias");
    rc = rsb_device_ok();
    if (rc != RSB_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    node_flag_kernel<<<pass_grid(N, H, W), PASS_THREADS, 0, st>>>(deg, labels, H * W, flags);
    count_kernel<<<dim3(H, N), ROW_THREADS, 0, st>>>(skel, deg, labels, flags, H, W, counts, row_offsets);
    scan_kernel<<<N, SCAN_THREADS, 0, st>>>(row_offsets, H, totals);
    return launched("road_chain_count launch");
}

extern "C" int rsb_road_chain_write(const uint8_t* skel, const int8_t* deg, const int32_t* labels, const int32_t* flags, int32_t N, int32_t H, int32_t W,
                                    const int32_t* counts, const int64_t* row_offsets, const int64_t* chain_base, const int64_t* pixel_base,
                                    int64_t* chain_offsets, int32_t* pixels, void* stream) {
    if (!skel || !deg || !labels || !flags || !counts || !row_offsets || !chain_base || !pixel_base || !chain_offsets || !pixels)
        return set_error(RSB_E_INVALID, "road_chain_write: null pointer");
    int rc = check_shape("road_chain_write", N, H, W);
    if (rc != RSB_OK) return rc;
    rc = rsb_device_ok();
    if (rc != RSB_OK) return rc;
    write_kernel<<<dim3(H, N), ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(skel, deg, labels, flags, H, W, counts, row_offsets, chain_base,
                                                                                  pixel_base, chain_offsets, pixels);
    return launched("road_chain_write launch");
}
