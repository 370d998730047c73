// Reprojection and resampling of `rs mosaic` (DESIGN.md §8): slippy-map index tiles sampled back onto one output raster grid.
//
// `rs tile`'s rule with the roles swapped. The tile set is a raster of 2^z S square pixels in EPSG:3857 (the "world"); a global
// pixel is valid when its tile's file exists. The host computes the exact global pixel coordinates (gx, gy) of the centres of
// output pixels (kG, lG) of a lattice every G output pixels (G a power of two); here every output pixel interpolates them
// bilinearly inside its lattice cell with the weights (i - kG) / G, which are exact binary fractions, and every float64 operation
// is a separately rounded __d*_rn in the order of tests/mosaic_reference.py, so the device and the restatement agree bit for bit.
//
// warp_kernel: one CTA per (band of BAND output rows, segment of SEG output columns) of the window. The lattice nodes of the CTA are
// staged in shared memory first (at most 9 x 257 when G = 1). Each thread then produces runs of four consecutive pixels of a row
// and writes them as one 32-bit store when the layout allows. A sample's tile is looked up through the slot table of the window's
// tile range (__ldg; -1: no file) and its index byte read from the stack of decoded planes. A pixel is covered when the global
// pixel containing (gx, gy) lies in the world and is valid; covered pixels are counted per CTA and added with one int64 atomic. A
// sample outside the slot table's tile range, or a pixel whose lattice cell lies outside the uploaded nodes, is a planning error
// of the host: it is counted in `misses`, never read.

#include <stdint.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr int THREADS = 256;
constexpr int BAND = 8;    // output rows of a CTA
constexpr int SEG = 256;   // output columns of a CTA
constexpr int NODE_ROWS = BAND + 1, NODE_COLS = SEG + 1;  // the lattice nodes of a CTA when G = 1 (fewer for larger G)

struct MosaicParams {
    const uint8_t* planes;
    int64_t plane_stride;
    int32_t num_planes;
    const int32_t* slots;
    int64_t tx0, ty0;          // the slot table covers tiles [tx0, tx0 + tiles_w) x [ty0, ty0 + tiles_h)
    int32_t tiles_w, tiles_h, size;
    int64_t span_w, span_h;    // tiles_w * size, tiles_h * size
    double world;              // 2^z size
    int64_t last;              // world - 1
    const double2* nodes;
    int64_t node_x0, node_y0;
    int32_t nodes_w, nodes_h, log2g;
    double inv_g;
    int64_t col0, row0;        // the window's first output column and row
    int32_t cols, rows, segs, nodata;
    uint8_t* out;
    int64_t out_pitch;
    int32_t vector_stores;
    unsigned long long* covered;
    unsigned long long* misses;
};

// global pixel (i, j), inside the world -> whether its tile has a file, its index byte in v; outside the table sets `miss`
__device__ __forceinline__ bool load(const MosaicParams& p, int64_t i, int64_t j, uint32_t& v, bool& miss) {
    const int64_t li = i - p.tx0 * p.size, lj = j - p.ty0 * p.size;
    if (li < 0 || lj < 0 || li >= p.span_w || lj >= p.span_h) {
        miss = true;
        return false;
    }
    const int32_t ci = int32_t(li), cj = int32_t(lj);  // span_w, span_h < 2^31 (checked by the host entry)
    const int32_t tx = ci / p.size, ty = cj / p.size;
    const int32_t slot = __ldg(p.slots + int64_t(ty) * p.tiles_w + tx);
    if (slot < 0) return false;
    if (slot >= p.num_planes) {
        miss = true;
        return false;
    }
    v = __ldg(p.planes + int64_t(slot) * p.plane_stride + int64_t(cj - ty * p.size) * p.size + (ci - tx * p.size));
    return true;
}

__device__ __forceinline__ double lerp(double a, double b, double t) { return __dadd_rn(a, __dmul_rn(t, __dsub_rn(b, a))); }

template <bool BILINEAR>
__global__ void __launch_bounds__(THREADS) warp_kernel(const MosaicParams p) {
    __shared__ double2 nodes[NODE_ROWS * NODE_COLS];
    __shared__ unsigned long long sums[2][THREADS / 32];
    const int band = blockIdx.x / p.segs, seg = blockIdx.x % p.segs;
    const int r0 = band * BAND, r1 = min(p.rows, r0 + BAND), c0 = seg * SEG, c1 = min(p.cols, c0 + SEG);
    const int64_t kx0 = (p.col0 + c0) >> p.log2g, kx1 = ((p.col0 + c1 - 1) >> p.log2g) + 1;
    const int64_t ky0 = (p.row0 + r0) >> p.log2g, ky1 = ((p.row0 + r1 - 1) >> p.log2g) + 1;
    const int nw = int(kx1 - kx0 + 1), nh = int(ky1 - ky0 + 1);
    const int64_t lx = kx0 - p.node_x0, ly = ky0 - p.node_y0;
    if (lx < 0 || ly < 0 || lx + nw > p.nodes_w || ly + nh > p.nodes_h) {  // the lattice does not reach this CTA: a host error
        if (threadIdx.x == 0) atomicAdd(p.misses, static_cast<unsigned long long>(r1 - r0) * static_cast<unsigned long long>(c1 - c0));
        return;
    }
    for (int i = threadIdx.x; i < nw * nh; i += THREADS) nodes[i] = p.nodes[(ly + i / nw) * p.nodes_w + lx + i % nw];
    __syncthreads();

    unsigned long long covered = 0, misses = 0;
    const int quads = (c1 - c0 + 3) / 4;
    const int64_t gmask = (int64_t(1) << p.log2g) - 1;
    for (int q = threadIdx.x; q < (r1 - r0) * quads; q += THREADS) {
        const int r = r0 + q / quads, c = c0 + (q % quads) * 4;
        const int64_t oy = p.row0 + r;
        const int iy = int((oy >> p.log2g) - ky0);
        const double fy = __dmul_rn(double(oy & gmask), p.inv_g);
        uint32_t px[4] = {uint32_t(p.nodata), uint32_t(p.nodata), uint32_t(p.nodata), uint32_t(p.nodata)};
        const int cn = min(4, c1 - c);
        for (int k = 0; k < cn; ++k) {
            const int64_t ox = p.col0 + c + k;
            const int ix = int((ox >> p.log2g) - kx0);
            const double fx = __dmul_rn(double(ox & gmask), p.inv_g);
            const double2 n00 = nodes[iy * nw + ix], n10 = nodes[iy * nw + ix + 1];
            const double2 n01 = nodes[(iy + 1) * nw + ix], n11 = nodes[(iy + 1) * nw + ix + 1];
            const double gx = lerp(lerp(n00.x, n10.x, fx), lerp(n01.x, n11.x, fx), fy);
            const double gy = lerp(lerp(n00.y, n10.y, fx), lerp(n01.y, n11.y, fx), fy);
            if (!(gx >= 0.0 && gx < p.world && gy >= 0.0 && gy < p.world)) continue;  // NaN fails too
            bool miss = false;
            uint32_t v;
            if (!load(p, int64_t(gx), int64_t(gy), v, miss)) {
                misses += miss;
                continue;
            }
            if (BILINEAR) {
                const double a = __dsub_rn(gx, 0.5), b = __dsub_rn(gy, 0.5);
                const double fa0 = floor(a), fb0 = floor(b);
                const double fa = __dsub_rn(a, fa0), fb = __dsub_rn(b, fb0);
                const double ga = __dsub_rn(1.0, fa), gb = __dsub_rn(1.0, fb);
                const int64_t i0 = int64_t(fa0), j0 = int64_t(fb0);
                const int64_t ia = max(int64_t(0), min(p.last, i0)), ib = max(int64_t(0), min(p.last, i0 + 1));
                const int64_t ja = max(int64_t(0), min(p.last, j0)), jb = max(int64_t(0), min(p.last, j0 + 1));
                const int64_t ti[4] = {ia, ib, ia, ib}, tj[4] = {ja, ja, jb, jb};
                const double tw[4] = {__dmul_rn(ga, gb), __dmul_rn(fa, gb), __dmul_rn(ga, fb), __dmul_rn(fa, fb)};
                double acc = 0.0, ws = 0.0;
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    uint32_t tv;
                    if (!load(p, ti[t], tj[t], tv, miss)) continue;
                    acc = __dadd_rn(acc, __dmul_rn(tw[t], double(tv)));
                    ws = __dadd_rn(ws, tw[t]);
                }
                if (miss) {
                    ++misses;
                    continue;
                }
                const double qv = floor(__dadd_rn(__ddiv_rn(acc, ws), 0.5));
                v = qv <= 0.0 ? 0u : qv >= 255.0 ? 255u : uint32_t(qv);
            }
            px[k] = v;
            ++covered;
        }
        uint8_t* o = p.out + int64_t(r) * p.out_pitch + c;
        if (p.vector_stores && cn == 4) {
            *reinterpret_cast<unsigned int*>(o) = px[0] | (px[1] << 8) | (px[2] << 16) | (px[3] << 24);
        } else {
            for (int k = 0; k < cn; ++k) o[k] = uint8_t(px[k]);
        }
    }
    for (int off = 16; off > 0; off >>= 1) {
        covered += __shfl_down_sync(0xffffffffu, covered, off);
        misses += __shfl_down_sync(0xffffffffu, misses, off);
    }
    if ((threadIdx.x & 31) == 0) {
        sums[0][threadIdx.x >> 5] = covered;
        sums[1][threadIdx.x >> 5] = misses;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long cs = 0, m = 0;
        for (int w = 0; w < THREADS / 32; ++w) {
            cs += sums[0][w];
            m += sums[1][w];
        }
        if (cs) atomicAdd(p.covered, cs);
        if (m) atomicAdd(p.misses, m);
    }
}

}  // namespace

extern "C" int rsb_mosaic_warp(const uint8_t* planes, int64_t plane_stride, int32_t num_planes, const int32_t* slots, int64_t tile_x0,
                               int64_t tile_y0, int32_t tiles_w, int32_t tiles_h, int32_t zoom, int32_t size, const double* nodes,
                               int64_t node_x0, int64_t node_y0, int32_t nodes_w, int32_t nodes_h, int32_t grid_step, int64_t out_col0,
                               int64_t out_row0, int32_t out_cols, int32_t out_rows, int32_t resampling, int32_t nodata, uint8_t* out,
                               int64_t out_pitch, int64_t* covered, int64_t* misses, void* stream) {
    if (!planes || !slots || !nodes || !out || !covered || !misses) return set_error(RSB_E_INVALID, "mosaic_warp: null pointer");
    if (zoom < 0 || zoom > RSB_COVER_MAX_ZOOM || size < 1 || size > RSB_TILE_MAX_SIZE)
        return set_error(RSB_E_INVALID, "mosaic_warp: zoom %d, size %d (need 0..%d, 1..%d)", zoom, size, RSB_COVER_MAX_ZOOM, RSB_TILE_MAX_SIZE);
    if (num_planes < 1 || plane_stride < int64_t(size) * size)
        return set_error(RSB_E_INVALID, "mosaic_warp: %d planes of stride %lld for %d x %d tiles", num_planes, (long long)plane_stride, size, size);
    const int64_t tiles = int64_t(1) << zoom;
    if (tiles_w < 1 || tiles_h < 1 || tile_x0 < 0 || tile_y0 < 0 || tile_x0 + tiles_w > tiles || tile_y0 + tiles_h > tiles ||
        int64_t(tiles_w) * size > INT32_MAX || int64_t(tiles_h) * size > INT32_MAX)
        return set_error(RSB_E_INVALID, "mosaic_warp: slot table of %d x %d tiles at (%lld, %lld) at zoom %d, size %d", tiles_w, tiles_h,
                         (long long)tile_x0, (long long)tile_y0, zoom, size);
    if (grid_step < 1 || grid_step > RSB_TILE_MAX_STEP || (grid_step & (grid_step - 1)))
        return set_error(RSB_E_INVALID, "mosaic_warp: lattice step %d (need a power of two in 1..%d)", grid_step, RSB_TILE_MAX_STEP);
    if (nodes_w < 2 || nodes_h < 2 || node_x0 < 0 || node_y0 < 0 || reinterpret_cast<uintptr_t>(nodes) % 16)
        return set_error(RSB_E_INVALID, "mosaic_warp: lattice of %d x %d nodes at (%lld, %lld)", nodes_w, nodes_h, (long long)node_x0, (long long)node_y0);
    if (out_cols < 1 || out_rows < 1 || out_col0 < 0 || out_row0 < 0 || out_pitch < out_cols ||
        (int64_t(out_rows) + BAND - 1) / BAND * ((int64_t(out_cols) + SEG - 1) / SEG) > INT32_MAX)
        return set_error(RSB_E_INVALID, "mosaic_warp: output window %d x %d at (%lld, %lld), pitch %lld", out_cols, out_rows, (long long)out_col0,
                         (long long)out_row0, (long long)out_pitch);
    if (resampling != 0 && resampling != 1) return set_error(RSB_E_INVALID, "mosaic_warp: resampling %d (0 nearest, 1 bilinear)", resampling);
    if (nodata < 0 || nodata > 255) return set_error(RSB_E_INVALID, "mosaic_warp: nodata %d (need 0..255)", nodata);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(covered, 0, sizeof(int64_t), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(misses, 0, sizeof(int64_t), st);
    if (e != cudaSuccess) return set_cuda_error(e, "mosaic_warp: clear counts");
    int log2g = 0;
    while ((1 << log2g) < grid_step) ++log2g;
    MosaicParams p;
    p.planes = planes;
    p.plane_stride = plane_stride;
    p.num_planes = num_planes;
    p.slots = slots;
    p.tx0 = tile_x0;
    p.ty0 = tile_y0;
    p.tiles_w = tiles_w;
    p.tiles_h = tiles_h;
    p.size = size;
    p.span_w = int64_t(tiles_w) * size;
    p.span_h = int64_t(tiles_h) * size;
    p.world = double(tiles * size);
    p.last = tiles * size - 1;
    p.nodes = reinterpret_cast<const double2*>(nodes);
    p.node_x0 = node_x0;
    p.node_y0 = node_y0;
    p.nodes_w = nodes_w;
    p.nodes_h = nodes_h;
    p.log2g = log2g;
    p.inv_g = 1.0 / grid_step;
    p.col0 = out_col0;
    p.row0 = out_row0;
    p.cols = out_cols;
    p.rows = out_rows;
    p.segs = (out_cols + SEG - 1) / SEG;
    p.nodata = nodata;
    p.out = out;
    p.out_pitch = out_pitch;
    p.vector_stores = out_pitch % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0;
    p.covered = reinterpret_cast<unsigned long long*>(covered);
    p.misses = reinterpret_cast<unsigned long long*>(misses);
    const dim3 grid(unsigned(((out_rows + BAND - 1) / BAND) * p.segs));
    if (resampling) warp_kernel<true><<<grid, THREADS, 0, st>>>(p);
    else warp_kernel<false><<<grid, THREADS, 0, st>>>(p);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "mosaic_warp launch");
}
