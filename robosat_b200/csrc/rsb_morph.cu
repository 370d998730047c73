// Fused binary morphology for `rs features` (robosat/features/core.py:65-92 denoise + grow): a chain of up to four erosions and
// dilations of (labels == class_index) with OpenCV's semantics, computed on bit-packed rows in shared memory.
//
// One CTA computes a band of BH output rows of one tile. It loads the band plus the chain's vertical reach above and below as
// 32-pixel words (W <= 1024, so a row is at most 32 words: lane c of a warp owns word c of the row it works on). Each op then
// shrinks the valid row range by its own reach. Per op and output row, the element's rows are grouped by their span: the rows of
// one group are combined vertically (AND for erode, OR for dilate), and the result is run horizontally over the span with
// log-step doubling on funnel-shifted neighbour words (shuffles). Pixels outside the image are the identity of the op that reads
// them (1 for erode, 0 for dilate), as OpenCV's default border value, so every op re-fills them for the next one.

#include <stdint.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int MORPH_THREADS = 256;

struct MorphStage {
    int32_t dilate, ay, lo, hi, ngroups;
    int8_t rows[RSB_MORPH_MAX_K];        // element rows with a non-empty span, grouped by span
    uint8_t gstart[RSB_MORPH_MAX_K + 1]; // group g owns rows[gstart[g] .. gstart[g+1])
    int8_t d0[RSB_MORPH_MAX_K];          // group g's span as pixel offsets d0 .. d0 + len - 1 from the anchor column
    uint8_t len[RSB_MORPH_MAX_K];
    uint8_t pad_[3];
};

struct alignas(16) MorphParams {
    MorphStage op[RSB_MORPH_MAX_OPS];
    int32_t nops, pad_[3];
};
static_assert(sizeof(MorphParams) % 16 == 0, "MorphParams is copied to shared memory in 16-byte words");

__device__ __forceinline__ uint32_t combine(uint32_t a, uint32_t b, int dilate) { return dilate ? (a | b) : (a & b); }

// word of pixels x + d for x in this lane's word; lanes outside the row read `border`
__device__ __forceinline__ uint32_t shifted(uint32_t v, int d, uint32_t border, int lane) {
    const int s0 = lane + (d >> 5), s1 = s0 + 1;
    uint32_t w0 = __shfl_sync(FULL, v, s0 & 31);
    uint32_t w1 = __shfl_sync(FULL, v, s1 & 31);
    if (static_cast<unsigned>(s0) > 31u) w0 = border;
    if (static_cast<unsigned>(s1) > 31u) w1 = border;
    return __funnelshift_r(w0, w1, d & 31);
}

// min / max of v over pixel offsets a .. b, a <= b, all of one sign. A doubled word T_p covers p pixels; read only at positions
// where, outside the row, it covers outside pixels alone (so the border fill is exact): runs forward (x .. x + p - 1) for
// offsets >= 0, which are read at x + offset >= 0, and backward (x - p + 1 .. x) for offsets < 0, read at x + offset < 1024.
__device__ __forceinline__ uint32_t one_sided_run(uint32_t v, int a, int b, int dilate, int lane) {
    const uint32_t border = dilate ? 0u : FULL;
    const int len = b - a + 1;
    const int dir = a >= 0 ? 1 : -1;
    int p = 1;
    while (2 * p <= len) {
        v = combine(v, shifted(v, dir * p, border, lane), dilate);
        p *= 2;
    }
    // forward: T_p(x + a) and T_p(x + b - p + 1); backward: T_p(x + b) and T_p(x + a + p - 1)
    uint32_t r = shifted(v, dir > 0 ? a : b, border, lane);
    if (p != len) r = combine(r, shifted(v, dir > 0 ? b - p + 1 : a + p - 1, border, lane), dilate);
    return r;
}

// min / max of v over pixel offsets d0 .. d0 + len - 1 (len <= 64, |offsets| <= 63)
__device__ __forceinline__ uint32_t horizontal_run(uint32_t v, int d0, int len, int dilate, int lane) {
    const int d1 = d0 + len - 1;
    if (d0 >= 0 || d1 < 0) return one_sided_run(v, d0, d1, dilate, lane);
    return combine(one_sided_run(v, d0, -1, dilate, lane), one_sided_run(v, 0, d1, dilate, lane), dilate);
}

__global__ void __launch_bounds__(MORPH_THREADS) morph_binary_kernel(const uint8_t* __restrict__ labels, int64_t image_stride, int H, int W,
                                                                     int cls, MorphParams params, int BH, int bands,
                                                                     uint8_t* __restrict__ out, int32_t* __restrict__ counts) {
    extern __shared__ __align__(16) uint32_t smem[];
    MorphParams& p = *reinterpret_cast<MorphParams*>(smem);
    {
        const uint4* src = reinterpret_cast<const uint4*>(&params);
        uint4* dst = reinterpret_cast<uint4*>(smem);
        for (int i = threadIdx.x; i < static_cast<int>(sizeof(MorphParams) / 16); i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();

    const int n = blockIdx.x / bands;
    const int y0 = (blockIdx.x % bands) * BH;
    const int y1 = min(y0 + BH, H);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int nops = p.nops;
    int reach_lo = 0, reach_hi = 0;
    for (int k = 0; k < nops; ++k) {
        reach_lo += p.op[k].lo;
        reach_hi += p.op[k].hi;
    }
    const int base = y0 - reach_lo;                  // image row of buffer row 0
    const int R = (y1 - y0) + reach_lo + reach_hi;   // buffer rows
    uint32_t* buf0 = smem + sizeof(MorphParams) / 4;
    uint32_t* buf1 = buf0 + R * 32;
    const int words = (W + 31) >> 5;
    const uint32_t valid = lane < (W >> 5) ? FULL : (lane == (W >> 5) ? ((1u << (W & 31)) - 1u) : 0u);

    // labels -> packed (labels == cls), rows outside the image = op 0's identity
    {
        const uint32_t border = p.op[0].dilate ? 0u : FULL;
        const uint8_t* img = labels + static_cast<int64_t>(n) * image_stride;
        for (int r = warp; r < R; r += nwarps) {
            const int y = base + r;
            uint32_t w = border;
            if (y >= 0 && y < H) {
                const uint8_t* row = img + static_cast<int64_t>(y) * W;
                uint32_t mine = 0;
                for (int c = 0; c < words; ++c) {
                    const int x = c * 32 + lane;
                    const uint32_t b = __ballot_sync(FULL, x < W && row[x] == cls);
                    if (lane == c) mine = b;
                }
                w = (mine & valid) | (border & ~valid);
            }
            buf0[r * 32 + lane] = w;
        }
    }
    __syncthreads();

    int lo_done = 0, hi_done = 0, fg = 0;
    for (int k = 0; k < nops; ++k) {
        const MorphStage& s = p.op[k];
        const int dilate = s.dilate;
        lo_done += s.lo;
        hi_done += s.hi;
        const uint32_t* src = (k & 1) ? buf1 : buf0;
        uint32_t* dst = (k & 1) ? buf0 : buf1;
        const bool last = k == nops - 1;
        const uint32_t next_border = (!last && p.op[k + 1].dilate) ? 0u : FULL;
        for (int r = lo_done + warp; r < R - hi_done; r += nwarps) {
            const int y = base + r;
            if (y < 0 || y >= H) {  // only halo rows of inner ops get here
                dst[r * 32 + lane] = next_border;
                continue;
            }
            uint32_t acc = dilate ? 0u : FULL;
            for (int g = 0; g < s.ngroups; ++g) {
                uint32_t v = dilate ? 0u : FULL;
                for (int t = s.gstart[g]; t < s.gstart[g + 1]; ++t) v = combine(v, src[(r + s.rows[t] - s.ay) * 32 + lane], dilate);
                acc = combine(acc, horizontal_run(v, s.d0[g], s.len[g], dilate, lane), dilate);
            }
            if (!last) {
                dst[r * 32 + lane] = (acc & valid) | (next_border & ~valid);
                continue;
            }
            acc &= valid;
            fg += __popc(acc);
            uint8_t* orow = out + (static_cast<int64_t>(n) * H + y) * W;
            for (int c = 0; c < words; ++c) {
                const uint32_t wc = __shfl_sync(FULL, acc, c);
                const int x = c * 32 + lane;
                if (x < W) orow[x] = static_cast<uint8_t>((wc >> lane) & 1u);
            }
        }
        if (!last) __syncthreads();
    }
    for (int o = 16; o > 0; o >>= 1) fg += __shfl_xor_sync(FULL, fg, o);
    if (lane == 0 && fg) atomicAdd(&counts[n], fg);
}

}  // namespace

extern "C" int rsb_morph_binary(const uint8_t* labels, int64_t image_stride, int32_t N, int32_t H, int32_t W, int32_t class_index,
                                const rsb_morph_op* ops_host, int32_t nops, uint8_t* out, int32_t* fg_counts, void* stream) {
    if (!labels || !ops_host || !out || !fg_counts) return set_error(RSB_E_INVALID, "morph_binary: null pointer");
    if (N < 1 || H < 1 || W < 1 || H > 1024 || W > 1024)
        return set_error(RSB_E_UNSUPPORTED, "morph_binary: N=%d H=%d W=%d (need N >= 1 and 1 <= H, W <= 1024)", N, H, W);
    if (image_stride < static_cast<int64_t>(H) * W)
        return set_error(RSB_E_INVALID, "morph_binary: image_stride %lld < H*W = %lld", (long long)image_stride, (long long)H * W);
    if (class_index < 0 || class_index > 255) return set_error(RSB_E_INVALID, "morph_binary: class_index %d is not a uint8 label", class_index);
    if (nops < 1 || nops > RSB_MORPH_MAX_OPS) return set_error(RSB_E_UNSUPPORTED, "morph_binary: nops=%d (need 1..%d)", nops, RSB_MORPH_MAX_OPS);

    MorphParams params = {};
    params.nops = nops;
    int halo = 0;
    for (int k = 0; k < nops; ++k) {
        const rsb_morph_op& o = ops_host[k];
        MorphStage& s = params.op[k];
        if (o.dilate != 0 && o.dilate != 1) return set_error(RSB_E_INVALID, "morph_binary: op %d: dilate must be 0 or 1", k);
        if (o.kh < 1 || o.kw < 1 || o.kh > RSB_MORPH_MAX_K || o.kw > RSB_MORPH_MAX_K)
            return set_error(RSB_E_UNSUPPORTED, "morph_binary: op %d: element %dx%d (need 1..%d)", k, o.kh, o.kw, RSB_MORPH_MAX_K);
        if (o.ay < 0 || o.ay >= o.kh || o.ax < 0 || o.ax >= o.kw)
            return set_error(RSB_E_INVALID, "morph_binary: op %d: anchor (%d, %d) outside the %dx%d element", k, o.ay, o.ax, o.kh, o.kw);
        s.dilate = o.dilate;
        s.ay = o.ay;
        s.lo = o.ay;
        s.hi = o.kh - 1 - o.ay;
        // group the element's rows by span, in order of first appearance
        int nrows = 0;
        bool used[RSB_MORPH_MAX_K] = {};
        for (int i = 0; i < o.kh; ++i) {
            const int j0 = o.span[i][0], j1 = o.span[i][1];
            if (j0 >= j1) continue;
            if (j0 < 0 || j1 > o.kw) return set_error(RSB_E_INVALID, "morph_binary: op %d: row %d span [%d, %d) outside [0, %d)", k, i, j0, j1, o.kw);
            if (used[i]) continue;
            s.gstart[s.ngroups] = static_cast<uint8_t>(nrows);
            s.d0[s.ngroups] = static_cast<int8_t>(j0 - o.ax);
            s.len[s.ngroups] = static_cast<uint8_t>(j1 - j0);
            for (int i2 = i; i2 < o.kh; ++i2) {
                if (o.span[i2][0] == j0 && o.span[i2][1] == j1) {
                    used[i2] = true;
                    s.rows[nrows++] = static_cast<int8_t>(i2);
                }
            }
            ++s.ngroups;
        }
        s.gstart[s.ngroups] = static_cast<uint8_t>(nrows);
        if (nrows == 0) return set_error(RSB_E_INVALID, "morph_binary: op %d: the structuring element has no set cell", k);
        halo += o.kh - 1;
    }
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;

    // bands of BH rows: the largest power of two up to 128 that still gives every SM two CTAs
    int BH = 128;
    while (BH > 8 && static_cast<int64_t>(N) * ((H + BH - 1) / BH) < 2 * num_sms()) BH /= 2;
    if (BH > H) BH = H;
    const int bands = (H + BH - 1) / BH;
    const int64_t blocks = static_cast<int64_t>(N) * bands;
    if (blocks > 0x7fffffff) return set_error(RSB_E_UNSUPPORTED, "morph_binary: %lld CTAs", (long long)blocks);
    const size_t smem = sizeof(MorphParams) + static_cast<size_t>(BH + halo) * 32 * 4 * 2;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaFuncSetAttribute(morph_binary_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return set_cuda_error(e, "morph_binary: shared memory attribute");
    e = cudaMemsetAsync(fg_counts, 0, sizeof(int32_t) * N, st);
    if (e != cudaSuccess) return set_cuda_error(e, "morph_binary: clear fg_counts");
    morph_binary_kernel<<<static_cast<unsigned>(blocks), MORPH_THREADS, smem, st>>>(labels, image_stride, H, W, class_index, params, BH, bands, out,
                                                                                      fg_counts);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "morph_binary launch");
}
