// `rs compare` (robosat/tools/compare.py): per-pixel work of the side-by-side review images.
//
// rsb_compare_count: for every (tile, mask) the non-zero count of the mask (the coverage filter's numerator) and the confusion
// counts against the tile's label, "foreground" meaning index != 0. A CTA owns one 16 KB chunk of every plane of one tile and
// reads it with 16-byte loads; the non-zero bytes of a 32-bit word are found with one add and two logic ops and counted with
// popc. Each CTA reduces its counts in shared memory and adds them to the tile's int64 counters: integer sums, so the result
// does not depend on the grid. A second launch turns (non-zero, both non-zero, label non-zero) into (tp, fp, fn, tn).
//
// rsb_compare_compose: the RGB composite image | label | mask 0 | ... of kept tiles, written in one pass straight into the
// output buffer (pinned host memory through its device mapping, so no device copy of the composite exists). The tile's
// 256-entry palettes are staged in shared memory. A thread makes 16 consecutive output pixels (48 bytes, three 16-byte stores),
// walking rows and columns incrementally.

#include <stdint.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr int COUNT_THREADS = 256;
constexpr int COUNT_VECS = 4;                                      // 16-byte vectors per thread and plane
constexpr int64_t COUNT_CHUNK = int64_t(COUNT_THREADS) * COUNT_VECS * 16;  // plane bytes per CTA
constexpr int COMPOSE_THREADS = 256;
constexpr int COMPOSE_PIX = 16;                                     // output pixels per thread

// bit 7 of each byte of the result is set iff that byte of w is non-zero
__device__ __forceinline__ uint32_t nonzero_bytes(uint32_t w) { return (((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) | w) & 0x80808080u; }

__device__ __forceinline__ void count_word(uint32_t m, uint32_t l, uint32_t& nz, uint32_t& tp, uint32_t& lb) {
    const uint32_t a = nonzero_bytes(m), b = nonzero_bytes(l);
    nz += __popc(a);
    tp += __popc(a & b);
    lb += __popc(b);
}

// raw[(n * M + m) * 4 + {0, 1, 2}] += (mask non-zero, both non-zero, label non-zero) over this CTA's chunk
__global__ void __launch_bounds__(COUNT_THREADS) compare_count_kernel(const uint8_t* __restrict__ masks, const uint8_t* __restrict__ labels, int M,
                                                                       int64_t hw, int64_t pitch, unsigned long long* __restrict__ raw) {
    __shared__ uint32_t part[COUNT_THREADS / 32][3];
    const int n = blockIdx.y;
    const int64_t begin = int64_t(blockIdx.x) * COUNT_CHUNK;
    const int64_t end = min(begin + COUNT_CHUNK, hw);
    const uint8_t* lab = labels ? labels + int64_t(n) * pitch : nullptr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int m = 0; m < M; ++m) {
        const uint8_t* mk = masks + (int64_t(n) * M + m) * pitch;
        uint32_t nz = 0, tp = 0, lb = 0;
        for (int64_t off = begin + int64_t(threadIdx.x) * 16; off < end; off += COUNT_THREADS * 16) {
            if (off + 16 <= end) {
                const uint4 a = __ldg(reinterpret_cast<const uint4*>(mk + off));
                const uint4 b = lab ? __ldg(reinterpret_cast<const uint4*>(lab + off)) : make_uint4(0, 0, 0, 0);
                count_word(a.x, b.x, nz, tp, lb);
                count_word(a.y, b.y, nz, tp, lb);
                count_word(a.z, b.z, nz, tp, lb);
                count_word(a.w, b.w, nz, tp, lb);
            } else {
                for (int64_t i = off; i < end; ++i) count_word(mk[i], lab ? lab[i] : 0u, nz, tp, lb);
            }
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            nz += __shfl_xor_sync(0xffffffffu, nz, s);
            tp += __shfl_xor_sync(0xffffffffu, tp, s);
            lb += __shfl_xor_sync(0xffffffffu, lb, s);
        }
        if (lane == 0) {
            part[warp][0] = nz;
            part[warp][1] = tp;
            part[warp][2] = lb;
        }
        __syncthreads();
        if (threadIdx.x < 3) {
            unsigned long long sum = 0;
            for (int w = 0; w < COUNT_THREADS / 32; ++w) sum += part[w][threadIdx.x];
            if (sum) atomicAdd(raw + (int64_t(n) * M + m) * 4 + threadIdx.x, sum);
        }
        __syncthreads();
    }
}

// in place: (non-zero, both, label, -) -> (tp, fp, fn, tn)
__global__ void compare_finalize_kernel(int64_t* counts, int64_t pairs, int64_t hw) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= pairs) return;
    int64_t* c = counts + i * 4;
    const int64_t nz = c[0], tp = c[1], lb = c[2];
    c[0] = tp;
    c[1] = nz - tp;
    c[2] = lb - tp;
    c[3] = hw - nz - lb + tp;
}

__global__ void __launch_bounds__(COMPOSE_THREADS) compare_compose_kernel(const uint8_t* __restrict__ images, const uint8_t* __restrict__ planes,
                                                                           const uint32_t* __restrict__ palettes, int P, int H, int W,
                                                                           int64_t pitch, uint8_t* __restrict__ out, int64_t out_stride) {
    extern __shared__ uint32_t pal[];  // [P][256]
    const int n = blockIdx.y;
    for (int i = threadIdx.x; i < P * 256; i += COMPOSE_THREADS) pal[i] = palettes[int64_t(n) * P * 256 + i];
    __syncthreads();
    const int64_t CW = int64_t(1 + P) * W;
    const int64_t total = CW * H;
    const int64_t p0 = (int64_t(blockIdx.x) * COMPOSE_THREADS + threadIdx.x) * COMPOSE_PIX;
    if (p0 >= total) return;
    int64_t y = p0 / CW;
    const int col = int(p0 - y * CW);
    int j = col / W, x = col - j * W;
    const uint8_t* image = images + int64_t(n) * H * W * 3;
    const uint8_t* plane0 = planes + int64_t(n) * P * pitch;
    uint32_t word[COMPOSE_PIX * 3 / 4];
#pragma unroll
    for (int k = 0; k < COMPOSE_PIX * 3 / 4; ++k) word[k] = 0;
#pragma unroll
    for (int k = 0; k < COMPOSE_PIX; ++k) {
        uint32_t rgb = 0;
        if (y < H) {  // false only past the last pixel of the tile
            const int64_t at = y * W + x;
            if (j == 0) {
                const uint8_t* px = image + at * 3;
                rgb = uint32_t(px[0]) | (uint32_t(px[1]) << 8) | (uint32_t(px[2]) << 16);
            } else {
                rgb = pal[(j - 1) * 256 + plane0[int64_t(j - 1) * pitch + at]];
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int b = 3 * k + c;  // compile-time byte position after unrolling
            word[b >> 2] |= ((rgb >> (8 * c)) & 0xffu) << (8 * (b & 3));
        }
        if (++x == W) {
            x = 0;
            if (++j == 1 + P) {
                j = 0;
                ++y;
            }
        }
    }
    uint8_t* dst = out + int64_t(n) * out_stride + p0 * 3;
    if (p0 + COMPOSE_PIX <= total) {
        uint4* v = reinterpret_cast<uint4*>(dst);
        v[0] = make_uint4(word[0], word[1], word[2], word[3]);
        v[1] = make_uint4(word[4], word[5], word[6], word[7]);
        v[2] = make_uint4(word[8], word[9], word[10], word[11]);
    } else {
        const int bytes = int(total - p0) * 3;
#pragma unroll
        for (int b = 0; b < COMPOSE_PIX * 3; ++b)  // unrolled so that `word` stays in registers
            if (b < bytes) dst[b] = uint8_t(word[b >> 2] >> (8 * (b & 3)));
    }
}

// the pointer the device uses for `p`: device memory as is, pinned host memory through its mapping; anything else is an error
int device_view(const void* p, const char* what, void** dev) {
    cudaPointerAttributes attr;
    cudaError_t e = cudaPointerGetAttributes(&attr, p);
    if (e != cudaSuccess) return set_cuda_error(e, what);
    if ((attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged || attr.type == cudaMemoryTypeHost) && attr.devicePointer) {
        *dev = attr.devicePointer;
        return RSB_OK;
    }
    return set_error(RSB_E_INVALID, "%s is neither device memory nor pinned host memory", what);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int rsb_compare_count(const uint8_t* masks, const uint8_t* labels, int32_t N, int32_t M, int64_t hw, int64_t pitch, int64_t* counts,
                                 void* stream) {
    if (!masks || !counts || N < 0 || M < 1 || M >= RSB_COMPARE_MAX_PLANES || hw < 1 || pitch < hw || pitch % 16)
        return set_error(RSB_E_INVALID, "compare_count: bad arguments (N %d, M %d, hw %lld, pitch %lld)", N, M, (long long)hw, (long long)pitch);
    if (!aligned16(masks) || (labels && !aligned16(labels))) return set_error(RSB_E_INVALID, "compare_count: planes must be 16-byte aligned");
    if (N > 65535) return set_error(RSB_E_UNSUPPORTED, "compare_count: %d tiles in one launch (at most 65535)", N);
    const int64_t chunks = (hw + COUNT_CHUNK - 1) / COUNT_CHUNK;
    if (chunks > 0x7fffffff) return set_error(RSB_E_UNSUPPORTED, "compare_count: %lld chunks per plane", (long long)chunks);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    if (N == 0) return RSB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t pairs = int64_t(N) * M;
    cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(int64_t) * 4 * pairs, st);
    if (e != cudaSuccess) return set_cuda_error(e, "compare_count: clear counts");
    compare_count_kernel<<<dim3(unsigned(chunks), unsigned(N)), COUNT_THREADS, 0, st>>>(masks, labels, M, hw, pitch,
                                                                                        reinterpret_cast<unsigned long long*>(counts));
    e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "compare_count launch");
    compare_finalize_kernel<<<unsigned((pairs + 255) / 256), 256, 0, st>>>(counts, pairs, hw);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "compare_count finalize launch");
}

extern "C" int rsb_compare_compose(const uint8_t* images, const uint8_t* planes, const uint32_t* palettes, int32_t N, int32_t P, int32_t H, int32_t W,
                                   int64_t pitch, uint8_t* out, int64_t out_stride, void* stream) {
    if (!images || !planes || !palettes || !out || N < 0 || P < 1 || P >= RSB_COMPARE_MAX_PLANES || H < 1 || W < 1 || pitch < int64_t(H) * W)
        return set_error(RSB_E_INVALID, "compare_compose: bad arguments (N %d, P %d, %dx%d, pitch %lld)", N, P, W, H, (long long)pitch);
    const int64_t out_bytes = int64_t(H) * W * (1 + P) * 3;
    if (out_stride < out_bytes || out_stride % 16 || !aligned16(out))
        return set_error(RSB_E_INVALID, "compare_compose: out must be 16-byte aligned with a 16-byte multiple stride of at least %lld bytes (got %lld)",
                         (long long)out_bytes, (long long)out_stride);
    if (N > 65535) return set_error(RSB_E_UNSUPPORTED, "compare_compose: %d tiles in one launch (at most 65535)", N);
    const int64_t blocks = (int64_t(H) * W * (1 + P) + int64_t(COMPOSE_THREADS) * COMPOSE_PIX - 1) / (int64_t(COMPOSE_THREADS) * COMPOSE_PIX);
    if (blocks > 0x7fffffff) return set_error(RSB_E_UNSUPPORTED, "compare_compose: %lld CTAs per tile", (long long)blocks);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    if (N == 0) return RSB_OK;
    void* out_dev = nullptr;
    const int rc = device_view(out, "compare_compose: out", &out_dev);
    if (rc != RSB_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    compare_compose_kernel<<<dim3(unsigned(blocks), unsigned(N)), COMPOSE_THREADS, size_t(P) * 256 * 4, st>>>(
        images, planes, palettes, P, H, W, pitch, static_cast<uint8_t*>(out_dev), out_stride);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "compare_compose launch");
}
