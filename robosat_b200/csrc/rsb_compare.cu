// `rs compare` (robosat/tools/compare.py): per-pixel work of the side-by-side review images.
//
// rsb_compare_count: for every (tile, mask) the non-zero count of the mask (the coverage filter's numerator) and the confusion
// counts against the tile's label, "foreground" meaning index != 0. A CTA owns one 16 KB chunk of every plane of one tile and
// reads it with 16-byte loads; the non-zero bytes of a 32-bit word are found with one add and two logic ops and counted with
// popc. Each CTA reduces its counts in shared memory and adds them to the tile's int64 counters: integer sums, so the result
// does not depend on the grid. A second launch turns (non-zero, both non-zero, label non-zero) into (tp, fp, fn, tn).
//
// rsb_compare_class_counts: the same chunks and loads, but per class: histograms of the label, of every mask and of the pixels
// where label == mask, plus the count of values >= C per plane. Each CTA keeps 256-bin histograms in shared memory (any uint8
// value has a bin), feeds them from per-thread runs of equal values and flushes the non-zero bins once per mask with int64
// atomics; bins >= C go to the out-of-range count.
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

// One run of equal values per thread and histogram, kept in registers: a pixel equal to the run's value adds to its count,
// any other value flushes the run into the CTA's shared histogram with one atomic and starts a new run. A thread walks 16
// consecutive bytes of a plane at a time and label planes hold long runs (background above all), so the one bin most pixels
// fall in sees one shared atomic per run rather than one per pixel, with no warp-wide vote on the common path; a 16-byte
// vector of one value in both planes is fed as one step of 16.
__device__ __forceinline__ void run_feed(uint32_t v, uint32_t n, uint32_t& cur, uint32_t& cnt, uint32_t* hist) {
    if (v == cur) {
        cnt += n;
    } else {
        if (cnt) atomicAdd(hist + cur, cnt);
        cur = v;
        cnt = n;
    }
}

// true iff the 16 bytes of v all equal its first byte
__device__ __forceinline__ bool uniform16(const uint4& v) {
    const uint32_t s = (v.x & 0xffu) * 0x01010101u;
    return v.x == s && v.y == s && v.z == s && v.w == s;
}

constexpr int CLASS_BINS = 256;                 // every uint8 value has a bin; bins >= C are the out-of-range count
constexpr uint32_t NOT_BOTH = CLASS_BINS;       // the both-histogram's bin for label != mask, never flushed to the output
static_assert(COUNT_THREADS == CLASS_BINS, "compare_class_kernel clears and flushes one bin per thread");
static_assert(RSB_COMPARE_MAX_CLASSES <= CLASS_BINS, "a class index is a uint8 value");

// per (tile n, chunk): histograms of label n (mask 0's pass only), of every mask m and of label == mask m, flushed once per mask
__global__ void __launch_bounds__(COUNT_THREADS) compare_class_kernel(const uint8_t* __restrict__ masks, const uint8_t* __restrict__ labels, int M,
                                                                       int C, int64_t hw, int64_t pitch, unsigned long long* __restrict__ label_hist,
                                                                       unsigned long long* __restrict__ mask_hist,
                                                                       unsigned long long* __restrict__ both_hist,
                                                                       unsigned long long* __restrict__ out_of_range) {
    __shared__ uint32_t lab_h[CLASS_BINS], msk_h[CLASS_BINS], both_h[CLASS_BINS + 1];
    const int n = blockIdx.y;
    const int64_t begin = int64_t(blockIdx.x) * COUNT_CHUNK;
    const int64_t end = min(begin + COUNT_CHUNK, hw);
    const uint8_t* lab = labels ? labels + int64_t(n) * pitch : nullptr;
    const int t = threadIdx.x;  // COUNT_THREADS == CLASS_BINS: thread t clears and flushes bin t
    for (int m = 0; m < M; ++m) {
        const bool first = m == 0;
        lab_h[t] = 0;
        msk_h[t] = 0;
        both_h[t] = 0;
        if (t == 0) both_h[NOT_BOTH] = 0;
        __syncthreads();
        const uint8_t* mk = masks + (int64_t(n) * M + m) * pitch;
        uint32_t lc = 0, ln = 0, mc = 0, mn = 0, bc = 0, bn = 0;
        for (int64_t off = begin + int64_t(t) * 16; off < end; off += COUNT_THREADS * 16) {
            if (off + 16 <= end) {
                const uint4 a = __ldg(reinterpret_cast<const uint4*>(mk + off));
                const uint4 b = lab ? __ldg(reinterpret_cast<const uint4*>(lab + off)) : make_uint4(0, 0, 0, 0);
                if (uniform16(a) && uniform16(b)) {  // most vectors of a label-like plane: one step for all 16 pixels
                    const uint32_t mv = a.x & 0xffu, lv = b.x & 0xffu;
                    if (first) run_feed(lv, 16, lc, ln, lab_h);
                    run_feed(mv, 16, mc, mn, msk_h);
                    run_feed(lv == mv ? mv : NOT_BOTH, 16, bc, bn, both_h);
                    continue;
                }
                const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    const uint32_t mv = (aw[k >> 2] >> (8 * (k & 3))) & 0xffu, lv = (bw[k >> 2] >> (8 * (k & 3))) & 0xffu;
                    if (first) run_feed(lv, 1, lc, ln, lab_h);
                    run_feed(mv, 1, mc, mn, msk_h);
                    run_feed(lv == mv ? mv : NOT_BOTH, 1, bc, bn, both_h);
                }
            } else {
                for (int64_t i = off; i < end; ++i) {
                    const uint32_t mv = mk[i], lv = lab ? lab[i] : 0u;
                    if (first) run_feed(lv, 1, lc, ln, lab_h);
                    run_feed(mv, 1, mc, mn, msk_h);
                    run_feed(lv == mv ? mv : NOT_BOTH, 1, bc, bn, both_h);
                }
            }
        }
        if (ln) atomicAdd(lab_h + lc, ln);
        if (mn) atomicAdd(msk_h + mc, mn);
        if (bn) atomicAdd(both_h + bc, bn);
        __syncthreads();
        const int64_t oor = int64_t(n) * (1 + M);
        if (first && lab_h[t]) atomicAdd(t < C ? label_hist + int64_t(n) * C + t : out_of_range + oor, (unsigned long long)lab_h[t]);
        if (msk_h[t]) atomicAdd(t < C ? mask_hist + (int64_t(n) * M + m) * C + t : out_of_range + oor + 1 + m, (unsigned long long)msk_h[t]);
        if (t < C && both_h[t]) atomicAdd(both_hist + (int64_t(n) * M + m) * C + t, (unsigned long long)both_h[t]);
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

extern "C" int rsb_compare_class_counts(const uint8_t* masks, const uint8_t* labels, int32_t N, int32_t M, int32_t C, int64_t hw, int64_t pitch,
                                        int64_t* label_hist, int64_t* mask_hist, int64_t* both_hist, int64_t* out_of_range, void* stream) {
    if (!masks || !label_hist || !mask_hist || !both_hist || !out_of_range || N < 0 || M < 1 || M >= RSB_COMPARE_MAX_PLANES || C < 2 ||
        C > RSB_COMPARE_MAX_CLASSES || hw < 1 || pitch < hw || pitch % 16)
        return set_error(RSB_E_INVALID, "compare_class_counts: bad arguments (N %d, M %d, C %d, hw %lld, pitch %lld)", N, M, C, (long long)hw,
                         (long long)pitch);
    if (!aligned16(masks) || (labels && !aligned16(labels))) return set_error(RSB_E_INVALID, "compare_class_counts: planes must be 16-byte aligned");
    if (N > 65535) return set_error(RSB_E_UNSUPPORTED, "compare_class_counts: %d tiles in one launch (at most 65535)", N);
    const int64_t chunks = (hw + COUNT_CHUNK - 1) / COUNT_CHUNK;
    if (chunks > 0x7fffffff) return set_error(RSB_E_UNSUPPORTED, "compare_class_counts: %lld chunks per plane", (long long)chunks);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    if (N == 0) return RSB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t pairs = int64_t(N) * M;
    const struct { void* p; int64_t count; } outs[4] = {{label_hist, int64_t(N) * C}, {mask_hist, pairs * C}, {both_hist, pairs * C},
                                                        {out_of_range, int64_t(N) * (1 + M)}};
    for (const auto& o : outs) {
        const cudaError_t e = cudaMemsetAsync(o.p, 0, sizeof(int64_t) * o.count, st);
        if (e != cudaSuccess) return set_cuda_error(e, "compare_class_counts: clear the histograms");
    }
    compare_class_kernel<<<dim3(unsigned(chunks), unsigned(N)), COUNT_THREADS, 0, st>>>(
        masks, labels, M, C, hw, pitch, reinterpret_cast<unsigned long long*>(label_hist), reinterpret_cast<unsigned long long*>(mask_hist),
        reinterpret_cast<unsigned long long*>(both_hist), reinterpret_cast<unsigned long long*>(out_of_range));
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "compare_class_counts launch");
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
