// The band rule of `rs tile` and `rs segment` (DESIGN.md §8): a decoded window of an 8- or 16-bit raster, [rows][cols][k] samples
// (the selected bands, then the alpha band when there is one), rendered to the 8-bit RGBA rows that rsb_tile_warp and
// rsb_tile_average take with spp 4, and the per-band histograms of the valid pixels that `--stretch` picks its percentiles from.
//
// Both kernels read the window as one flat array of pixels, four consecutive pixels per thread and step: their 4 k samples are
// 4 k * sizeof(T) bytes at a multiple of that offset, so they come in as 16-, 8- or 4-byte vector loads (the window must start
// 16-byte aligned). The few pixels past the last whole group are read one by one.
//
// render_kernel: v = floor((510 t + d) / (2 d)) with d = HI - LO and t = clamp(s, LO, HI) - LO, in 32-bit integers (510 * 65535 fits);
// A = 0 when the alpha sample is 0 or every selected band equals nodata (the raw samples, before scaling). One 32-bit store per pixel.
//
// hist8_kernel: 8-bit bins of every selected band in shared memory per CTA (at most 3 x 256 counters), flushed with one global
// atomic per non-zero bin. hist16_kernel: 65 536 bins per band do not fit one CTA, so a cluster of four CTAs holds them in
// distributed shared memory, CTA r the values [r 16384, (r + 1) 16384) of every band; a sample's count goes to its owner with a
// (possibly remote) shared atomic, and after a cluster barrier each CTA flushes the non-zero bins it owns.

#include <cooperative_groups.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/rsb200.h"
#include "rsb_host.h"

namespace cg = cooperative_groups;
using namespace rsb;

namespace {

constexpr int THREADS = 256;
constexpr int HIST16_THREADS = 1024;  // few CTAs fit an SM with 64 KB of bins per band: they bring the warps
constexpr int HIST16_CLUSTER = 4;
constexpr int HIST16_BINS = 65536 / HIST16_CLUSTER;  // per CTA and band

struct BandParams {
    const void* src;
    int64_t pixels, cols;  // rows * cols pixels, cols per row
    int32_t nodata;        // -1: none
    int32_t lo[3], d[3];   // render only
    uint8_t* out;
    int64_t out_pitch;
    unsigned long long* hist;  // histogram only: [nsel][2^bits]
};

// the 4 K samples of pixels 4 g .. 4 g + 3, as vector loads of the widest size that divides their byte count
template <typename T, int K>
__device__ __forceinline__ void load_group(const T* src, int64_t g, T (&s)[4 * K]) {
    constexpr int BYTES = 4 * K * int(sizeof(T));
    const char* base = reinterpret_cast<const char*>(src) + g * BYTES;
    if constexpr (BYTES % 16 == 0) {
#pragma unroll
        for (int i = 0; i < BYTES / 16; ++i) reinterpret_cast<uint4*>(s)[i] = __ldg(reinterpret_cast<const uint4*>(base) + i);
    } else if constexpr (BYTES % 8 == 0) {
#pragma unroll
        for (int i = 0; i < BYTES / 8; ++i) reinterpret_cast<uint2*>(s)[i] = __ldg(reinterpret_cast<const uint2*>(base) + i);
    } else {
#pragma unroll
        for (int i = 0; i < BYTES / 4; ++i) reinterpret_cast<uint32_t*>(s)[i] = __ldg(reinterpret_cast<const uint32_t*>(base) + i);
    }
}

// whether a pixel (its K samples at s) is valid: the alpha sample (the last, when K is 2 or 4) is not 0, and not every selected
// band equals nodata
template <typename T, int K>
__device__ __forceinline__ bool valid(const T* s, int32_t nodata) {
    constexpr int NSEL = K >= 3 ? 3 : 1;
    constexpr bool ALPHA = K == 2 || K == 4;
    bool all = nodata >= 0;
#pragma unroll
    for (int b = 0; b < NSEL; ++b) all = all && int32_t(s[b]) == nodata;
    return !all && (!ALPHA || s[K - 1] != 0);
}

__device__ __forceinline__ uint32_t scale(uint32_t s, int32_t lo, int32_t d) {
    const int32_t t = min(max(int32_t(s), lo), lo + d) - lo;
    return uint32_t(510 * t + d) / uint32_t(2 * d);
}

template <typename T, int K>
__device__ __forceinline__ uint32_t rgba(const T* s, const BandParams& p) {
    constexpr int NSEL = K >= 3 ? 3 : 1;
    const uint32_t a = valid<T, K>(s, p.nodata) ? 0xff000000u : 0u;
    if (NSEL == 1) {
        const uint32_t v = scale(s[0], p.lo[0], p.d[0]);
        return v | (v << 8) | (v << 16) | a;
    }
    return scale(s[0], p.lo[0], p.d[0]) | (scale(s[1], p.lo[1], p.d[1]) << 8) | (scale(s[2], p.lo[2], p.d[2]) << 16) | a;
}

template <typename T, int K>
__global__ void __launch_bounds__(THREADS) render_kernel(const BandParams p) {
    const T* src = static_cast<const T*>(p.src);
    const int64_t groups = p.pixels / 4;
    for (int64_t g = int64_t(blockIdx.x) * THREADS + threadIdx.x; g < groups; g += int64_t(gridDim.x) * THREADS) {
        T s[4 * K];
        load_group<T, K>(src, g, s);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t px = 4 * g + i, r = px / p.cols, c = px - r * p.cols;
            *reinterpret_cast<uint32_t*>(p.out + r * p.out_pitch + 4 * c) = rgba<T, K>(s + K * i, p);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < p.pixels - 4 * groups) {
        const int64_t px = 4 * groups + threadIdx.x, r = px / p.cols, c = px - r * p.cols;
        T s[K];
#pragma unroll
        for (int b = 0; b < K; ++b) s[b] = src[px * K + b];
        *reinterpret_cast<uint32_t*>(p.out + r * p.out_pitch + 4 * c) = rgba<T, K>(s, p);
    }
}

// the counts of pixel s (K samples) into `bins` of the selected bands: count(band, value) is called for a valid pixel
template <typename T, int K, typename F>
__device__ __forceinline__ void count_window(const BandParams& p, int64_t first, int64_t stride, F&& count) {
    constexpr int NSEL = K >= 3 ? 3 : 1;
    const T* src = static_cast<const T*>(p.src);
    const int64_t groups = p.pixels / 4;
    for (int64_t g = first; g < groups; g += stride) {
        T s[4 * K];
        load_group<T, K>(src, g, s);
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (valid<T, K>(s + K * i, p.nodata)) {
#pragma unroll
                for (int b = 0; b < NSEL; ++b) count(b, uint32_t(s[K * i + b]));
            }
    }
    if (first < p.pixels - 4 * groups) {  // the last pixels, one per thread of the first threads
        const int64_t px = 4 * groups + first;
        T s[K];
#pragma unroll
        for (int b = 0; b < K; ++b) s[b] = src[px * K + b];
        if (valid<T, K>(s, p.nodata)) {
#pragma unroll
            for (int b = 0; b < NSEL; ++b) count(b, uint32_t(s[b]));
        }
    }
}

template <int K>
__global__ void __launch_bounds__(THREADS) hist8_kernel(const BandParams p) {
    constexpr int NSEL = K >= 3 ? 3 : 1;
    __shared__ uint32_t bins[NSEL * 256];
    for (int i = threadIdx.x; i < NSEL * 256; i += THREADS) bins[i] = 0;
    __syncthreads();
    count_window<uint8_t, K>(p, int64_t(blockIdx.x) * THREADS + threadIdx.x, int64_t(gridDim.x) * THREADS,
                             [&](int b, uint32_t v) { atomicAdd(&bins[b * 256 + v], 1u); });
    __syncthreads();
    for (int i = threadIdx.x; i < NSEL * 256; i += THREADS)
        if (bins[i]) atomicAdd(p.hist + i, static_cast<unsigned long long>(bins[i]));
}

template <int K>
__global__ void __cluster_dims__(HIST16_CLUSTER, 1, 1) __launch_bounds__(HIST16_THREADS) hist16_kernel(const BandParams p) {
    constexpr int NSEL = K >= 3 ? 3 : 1;
    extern __shared__ uint32_t bins[];  // [NSEL][HIST16_BINS]: the values this CTA owns
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned rank = cluster.block_rank();
    for (int i = threadIdx.x; i < NSEL * HIST16_BINS; i += HIST16_THREADS) bins[i] = 0;
    cluster.sync();  // every CTA's bins are clear before any count arrives
    uint32_t* const o0 = cluster.map_shared_rank(bins, 0);
    uint32_t* const o1 = cluster.map_shared_rank(bins, 1);
    uint32_t* const o2 = cluster.map_shared_rank(bins, 2);
    uint32_t* const o3 = cluster.map_shared_rank(bins, 3);
    count_window<uint16_t, K>(p, int64_t(blockIdx.x) * HIST16_THREADS + threadIdx.x, int64_t(gridDim.x) * HIST16_THREADS, [&](int b, uint32_t v) {
        const uint32_t r = v / HIST16_BINS;  // the owner, selected without a local array
        uint32_t* const o = r == 0 ? o0 : r == 1 ? o1 : r == 2 ? o2 : o3;
        atomicAdd(o + b * HIST16_BINS + (v % HIST16_BINS), 1u);
    });
    cluster.sync();  // every count has landed
    for (int i = threadIdx.x; i < NSEL * HIST16_BINS; i += HIST16_THREADS)
        if (bins[i]) atomicAdd(p.hist + (i / HIST16_BINS) * 65536 + rank * HIST16_BINS + i % HIST16_BINS, static_cast<unsigned long long>(bins[i]));
}

// checks common to both entry points (`fn` names the entry point in the message)
int validate(const char* fn, const void* src, int64_t rows, int64_t cols, int32_t bits, int32_t nsel, int32_t alpha, int32_t nodata) {
    if (!src) return set_error(RSB_E_INVALID, "%s: null pointer", fn);
    if (reinterpret_cast<uintptr_t>(src) % 16) return set_error(RSB_E_INVALID, "%s: the window is not 16-byte aligned", fn);
    if (bits != 8 && bits != 16) return set_error(RSB_E_INVALID, "%s: %d bits per sample (need 8 or 16)", fn, bits);
    if ((nsel != 1 && nsel != 3) || (alpha != 0 && alpha != 1)) return set_error(RSB_E_INVALID, "%s: %d bands, alpha %d (need 1 or 3 bands, alpha 0 or 1)", fn, nsel, alpha);
    if (nodata < -1 || nodata >= (1 << bits)) return set_error(RSB_E_INVALID, "%s: nodata %d (need -1 or 0..%d)", fn, nodata, (1 << bits) - 1);
    if (rows < 1 || cols < 1 || rows > (int64_t(1) << 31) || cols > (int64_t(1) << 31))
        return set_error(RSB_E_INVALID, "%s: window of %lld x %lld pixels", fn, (long long)cols, (long long)rows);
    return RSB_OK;
}

int grid_for(int64_t groups, int per_sm) {
    const int64_t want = (groups + THREADS - 1) / THREADS;
    return int(std::max<int64_t>(1, std::min<int64_t>(want, int64_t(num_sms()) * per_sm)));
}

template <typename T>
void render_launch(const BandParams& p, int k, int grid, cudaStream_t st) {
    if (k == 1) render_kernel<T, 1><<<grid, THREADS, 0, st>>>(p);
    else if (k == 2) render_kernel<T, 2><<<grid, THREADS, 0, st>>>(p);
    else if (k == 3) render_kernel<T, 3><<<grid, THREADS, 0, st>>>(p);
    else render_kernel<T, 4><<<grid, THREADS, 0, st>>>(p);
}

template <int K>
cudaError_t hist16_launch(const BandParams& p, int64_t groups, cudaStream_t st) {
    constexpr int NSEL = K >= 3 ? 3 : 1;
    const int smem = NSEL * HIST16_BINS * int(sizeof(uint32_t));
    cudaError_t e = cudaFuncSetAttribute(hist16_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    // clusters fill the SMs once (one CTA per SM with three bands' 192 KB, two with one band's 64 KB), and never more than the window needs
    const int per_sm = NSEL == 3 ? 1 : 2;
    int grid = int(std::max<int64_t>(1, std::min<int64_t>((groups + HIST16_THREADS - 1) / HIST16_THREADS, int64_t(num_sms()) * per_sm)));
    grid = (grid + HIST16_CLUSTER - 1) / HIST16_CLUSTER * HIST16_CLUSTER;
    hist16_kernel<K><<<grid, HIST16_THREADS, smem, st>>>(p);
    return cudaGetLastError();
}

}  // namespace

extern "C" int rsb_tile_render(const void* src, int64_t rows, int64_t cols, int32_t bits, int32_t nsel, int32_t alpha, int32_t nodata,
                               const int32_t* scale_host, uint8_t* out, int64_t out_pitch, void* stream) {
    int rc = validate("tile_render", src, rows, cols, bits, nsel, alpha, nodata);
    if (rc != RSB_OK) return rc;
    if (!scale_host || !out) return set_error(RSB_E_INVALID, "tile_render: null pointer");
    if (out_pitch < 4 * cols || out_pitch % 4 || reinterpret_cast<uintptr_t>(out) % 4)
        return set_error(RSB_E_INVALID, "tile_render: output pitch %lld for %lld columns (need a multiple of 4, at least 4 per column, 4-byte aligned)",
                         (long long)out_pitch, (long long)cols);
    BandParams p = {};
    for (int b = 0; b < nsel; ++b) {
        const int32_t lo = scale_host[2 * b], hi = scale_host[2 * b + 1];
        if (lo < 0 || hi <= lo || hi >= (1 << bits))
            return set_error(RSB_E_INVALID, "tile_render: scale %d,%d of band %d (need 0 <= LO < HI <= %d)", lo, hi, b, (1 << bits) - 1);
        p.lo[b] = lo;
        p.d[b] = hi - lo;
    }
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    p.src = src;
    p.pixels = rows * cols;
    p.cols = cols;
    p.nodata = nodata;
    p.out = out;
    p.out_pitch = out_pitch;
    const int grid = grid_for(p.pixels / 4 + 1, 8);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (bits == 8) render_launch<uint8_t>(p, nsel + alpha, grid, st);
    else render_launch<uint16_t>(p, nsel + alpha, grid, st);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "tile_render launch");
}

extern "C" int rsb_band_histogram(const void* src, int64_t rows, int64_t cols, int32_t bits, int32_t nsel, int32_t alpha, int32_t nodata,
                                  int64_t* hist, void* stream) {
    int rc = validate("band_histogram", src, rows, cols, bits, nsel, alpha, nodata);
    if (rc != RSB_OK) return rc;
    if (!hist || reinterpret_cast<uintptr_t>(hist) % 8) return set_error(RSB_E_INVALID, "band_histogram: null or unaligned histogram");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    BandParams p = {};
    p.src = src;
    p.pixels = rows * cols;
    p.cols = cols;
    p.nodata = nodata;
    p.hist = reinterpret_cast<unsigned long long*>(hist);
    const int k = nsel + alpha;
    const int64_t groups = p.pixels / 4 + 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e;
    if (bits == 8) {
        const int grid = grid_for(groups, 8);
        if (k == 1) hist8_kernel<1><<<grid, THREADS, 0, st>>>(p);
        else if (k == 2) hist8_kernel<2><<<grid, THREADS, 0, st>>>(p);
        else if (k == 3) hist8_kernel<3><<<grid, THREADS, 0, st>>>(p);
        else hist8_kernel<4><<<grid, THREADS, 0, st>>>(p);
        e = cudaGetLastError();
    } else {
        e = k == 1 ? hist16_launch<1>(p, groups, st) : k == 2 ? hist16_launch<2>(p, groups, st) : k == 3 ? hist16_launch<3>(p, groups, st)
                                                                                                      : hist16_launch<4>(p, groups, st);
    }
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "band_histogram launch");
}
