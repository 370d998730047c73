// Reprojection and resampling of `rs tile` (DESIGN.md §8): slippy-map RGB tiles sampled from a window of a GeoTIFF.
//
// The host computes the exact source coordinates (u, v) of the pixel centres gx = kG, gy = lG of a global lattice (every G tile
// pixels of the zoom level, G a power of two); here every output pixel interpolates them bilinearly inside its lattice cell with
// the weights (gx - kG) / G, which are exact binary fractions, and every float64 operation is a separately rounded __d*_rn in the
// order of tests/tile_reference.py, so the device and the restatement agree bit for bit.
//
// warp_kernel: one CTA per (tile, band of BAND rows, segment of SEG columns). The lattice nodes the CTA's pixels need are staged
// in shared memory first (at most (BAND - 1) / G + 2 rows of (SEG - 1) / G + 2 nodes, so 9 x 257 when G = 1). Each thread then
// produces runs of four consecutive pixels of a row and writes their 12 RGB bytes as three 32-bit stores when the layout allows.
// Source pixels are read through the read-only path. A pixel is covered when the source pixel that contains (u, v) lies in the
// raster and is valid; covered pixels are counted per CTA and added to the tile's int64 count with one atomic. A source pixel
// inside the raster but outside the uploaded window is a planning error of the host: it is counted in `misses`, never read.
//
// average_kernel (`--resampling average`): the same CTAs over a lattice of pixel corners; each pixel sums the source pixels under the
// bounding box of its four corners (see the comment above the kernel).

#include <stdint.h>
#include <stdio.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr int THREADS = 256;
constexpr int BAND = 8;    // output rows of a CTA
constexpr int SEG = 256;   // output columns of a CTA
constexpr int NODE_ROWS = BAND + 1, NODE_COLS = SEG + 1;  // the lattice nodes of a CTA when G = 1 (fewer for larger G)

struct WarpParams {
    const uint8_t* src;
    int64_t src_pitch, row0, col0, rows, cols;  // the window: raster rows [row0, row0 + rows), columns [col0, col0 + cols)
    double width, height;                       // the raster
    int64_t last_col, last_row;
    int32_t alpha, nodata;
    const double2* nodes;
    int64_t node_x0, node_y0;
    int32_t nodes_w, nodes_h, log2g;
    double inv_g;
    const int64_t* tiles;
    int32_t size, segs;
    uint8_t* out;
    int64_t image_stride;
    int32_t vector_stores;
    unsigned long long* covered;
    unsigned long long* misses;
};

// pixel (i, j) of the raster -> whether it is valid, its RGB in r, g, b; a pixel outside the window sets `miss`
template <int SPP>
__device__ __forceinline__ bool load(const WarpParams& p, int64_t i, int64_t j, uint32_t& r, uint32_t& g, uint32_t& b, bool& miss) {
    const int64_t li = i - p.col0, lj = j - p.row0;
    if (li < 0 || lj < 0 || li >= p.cols || lj >= p.rows) {
        miss = true;
        return false;
    }
    const uint8_t* px = p.src + lj * p.src_pitch + li * SPP;
    bool valid = true;
    if (SPP == 1) {
        r = g = b = __ldg(px);
    } else if (SPP == 3) {
        r = __ldg(px);
        g = __ldg(px + 1);
        b = __ldg(px + 2);
    } else {
        const uint32_t w = __ldg(reinterpret_cast<const unsigned int*>(px));
        r = w & 0xff;
        g = (w >> 8) & 0xff;
        b = (w >> 16) & 0xff;
        valid = !p.alpha || (w >> 24) != 0;
    }
    return valid && !(int32_t(r) == p.nodata && int32_t(g) == p.nodata && int32_t(b) == p.nodata);
}

__device__ __forceinline__ double lerp(double a, double b, double t) { return __dadd_rn(a, __dmul_rn(t, __dsub_rn(b, a))); }

__device__ __forceinline__ uint32_t quantize(double acc, double wsum) {
    const double q = floor(__dadd_rn(__ddiv_rn(acc, wsum), 0.5));
    return q <= 0.0 ? 0u : q >= 255.0 ? 255u : uint32_t(q);
}

template <int SPP, bool BILINEAR>
__global__ void __launch_bounds__(THREADS) warp_kernel(const WarpParams p) {
    __shared__ double2 nodes[NODE_ROWS * NODE_COLS];
    __shared__ unsigned long long sums[2][THREADS / 32];
    const int n = blockIdx.y;
    const int band = blockIdx.x / p.segs, seg = blockIdx.x % p.segs;
    const int S = p.size;
    const int r0 = band * BAND, r1 = min(S, r0 + BAND), c0 = seg * SEG, c1 = min(S, c0 + SEG);
    const int64_t tx = p.tiles[2 * n], ty = p.tiles[2 * n + 1];
    const int64_t kx0 = (tx * S + c0) >> p.log2g, kx1 = ((tx * S + c1 - 1) >> p.log2g) + 1;
    const int64_t ky0 = (ty * S + r0) >> p.log2g, ky1 = ((ty * S + r1 - 1) >> p.log2g) + 1;
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
    for (int q = threadIdx.x; q < (r1 - r0) * quads; q += THREADS) {
        const int r = r0 + q / quads, c = c0 + (q % quads) * 4;
        const int64_t gy = ty * S + r;
        const int iy = int((gy >> p.log2g) - ky0);
        const double fy = __dmul_rn(double(gy & ((int64_t(1) << p.log2g) - 1)), p.inv_g);
        uint32_t px[4] = {0u, 0u, 0u, 0u};  // 0x00BBGGRR per pixel
        const int cn = min(4, c1 - c);
        for (int k = 0; k < cn; ++k) {
            const int64_t gx = tx * S + c + k;
            const int ix = int((gx >> p.log2g) - kx0);
            const double fx = __dmul_rn(double(gx & ((int64_t(1) << p.log2g) - 1)), p.inv_g);
            const double2 n00 = nodes[iy * nw + ix], n10 = nodes[iy * nw + ix + 1];
            const double2 n01 = nodes[(iy + 1) * nw + ix], n11 = nodes[(iy + 1) * nw + ix + 1];
            const double u = lerp(lerp(n00.x, n10.x, fx), lerp(n01.x, n11.x, fx), fy);
            const double v = lerp(lerp(n00.y, n10.y, fx), lerp(n01.y, n11.y, fx), fy);
            if (!(u >= 0.0 && u < p.width && v >= 0.0 && v < p.height)) continue;  // NaN fails too
            bool miss = false;
            uint32_t cr, cg, cb;
            if (!load<SPP>(p, int64_t(u), int64_t(v), cr, cg, cb, miss)) {
                misses += miss;
                continue;
            }
            if (BILINEAR) {
                const double a = __dsub_rn(u, 0.5), b = __dsub_rn(v, 0.5);
                const double fa0 = floor(a), fb0 = floor(b);
                const double fa = __dsub_rn(a, fa0), fb = __dsub_rn(b, fb0);
                const double ga = __dsub_rn(1.0, fa), gb = __dsub_rn(1.0, fb);
                const int64_t i0 = int64_t(fa0), j0 = int64_t(fb0);
                const int64_t ia = max(int64_t(0), min(p.last_col, i0)), ib = max(int64_t(0), min(p.last_col, i0 + 1));
                const int64_t ja = max(int64_t(0), min(p.last_row, j0)), jb = max(int64_t(0), min(p.last_row, j0 + 1));
                const int64_t ti[4] = {ia, ib, ia, ib}, tj[4] = {ja, ja, jb, jb};
                const double tw[4] = {__dmul_rn(ga, gb), __dmul_rn(fa, gb), __dmul_rn(ga, fb), __dmul_rn(fa, fb)};
                double ar = 0.0, ag = 0.0, ab = 0.0, ws = 0.0;
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    uint32_t tr, tg, tb;
                    if (!load<SPP>(p, ti[t], tj[t], tr, tg, tb, miss)) continue;
                    ar = __dadd_rn(ar, __dmul_rn(tw[t], double(tr)));
                    ag = __dadd_rn(ag, __dmul_rn(tw[t], double(tg)));
                    ab = __dadd_rn(ab, __dmul_rn(tw[t], double(tb)));
                    ws = __dadd_rn(ws, tw[t]);
                }
                if (miss) {
                    ++misses;
                    continue;
                }
                cr = quantize(ar, ws);
                cg = quantize(ag, ws);
                cb = quantize(ab, ws);
            }
            px[k] = cr | (cg << 8) | (cb << 16);
            ++covered;
        }
        uint8_t* o = p.out + n * p.image_stride + (int64_t(r) * S + c) * 3;
        if (p.vector_stores && cn == 4) {
            unsigned int* o4 = reinterpret_cast<unsigned int*>(o);
            o4[0] = px[0] | (px[1] << 24);
            o4[1] = (px[1] >> 8) | (px[2] << 16);
            o4[2] = (px[2] >> 16) | (px[3] << 8);
        } else {
            for (int k = 0; k < cn; ++k) {
                o[3 * k] = uint8_t(px[k]);
                o[3 * k + 1] = uint8_t(px[k] >> 8);
                o[3 * k + 2] = uint8_t(px[k] >> 16);
            }
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
        unsigned long long c = 0, m = 0;
        for (int w = 0; w < THREADS / 32; ++w) {
            c += sums[0][w];
            m += sums[1][w];
        }
        if (c) atomicAdd(p.covered + n, c);
        if (m) atomicAdd(p.misses, m);
    }
}

template <int SPP>
void launch(const WarpParams& p, int N, int resampling, cudaStream_t st) {
    const dim3 grid(unsigned(((p.size + BAND - 1) / BAND) * p.segs), unsigned(N));
    if (resampling) warp_kernel<SPP, true><<<grid, THREADS, 0, st>>>(p);
    else warp_kernel<SPP, false><<<grid, THREADS, 0, st>>>(p);
}

// Area averaging (DESIGN.md §8, `rs tile --resampling average`): the nodes hold (u, v) at global pixel corners (kG, lG). A pixel
// interpolates its four corners, each in the lattice cell that contains it, and sums the source pixels its corners' bounding box
// overlaps, row by row: r = sum_i wx_i p(i, j) over the row's valid pixels, then A += wy_j r, every operation rounded separately.
// The CTA's nodes (at most BAND / G + 2 rows of SEG / G + 2, so 10 x 258 when G = 1) are staged in shared memory; one thread per
// pixel, consecutive threads on consecutive columns, so a warp's loads of one footprint row fall into a few cache lines.
constexpr int AVG_NODE_ROWS = BAND + 2, AVG_NODE_COLS = SEG + 2;

template <int SPP>
__global__ void __launch_bounds__(THREADS) average_kernel(const WarpParams p) {
    __shared__ double2 nodes[AVG_NODE_ROWS * AVG_NODE_COLS];
    __shared__ unsigned long long sums[2][THREADS / 32];
    const int n = blockIdx.y;
    const int band = blockIdx.x / p.segs, seg = blockIdx.x % p.segs;
    const int S = p.size;
    const int r0 = band * BAND, r1 = min(S, r0 + BAND), c0 = seg * SEG, c1 = min(S, c0 + SEG);
    const int64_t tx = p.tiles[2 * n], ty = p.tiles[2 * n + 1];
    // corners tx S + c0 .. tx S + c1 (inclusive) and the same in y
    const int64_t kx0 = (tx * S + c0) >> p.log2g, kx1 = ((tx * S + c1) >> p.log2g) + 1;
    const int64_t ky0 = (ty * S + r0) >> p.log2g, ky1 = ((ty * S + r1) >> p.log2g) + 1;
    const int nw = int(kx1 - kx0 + 1), nh = int(ky1 - ky0 + 1);
    const int64_t lx = kx0 - p.node_x0, ly = ky0 - p.node_y0;
    if (lx < 0 || ly < 0 || lx + nw > p.nodes_w || ly + nh > p.nodes_h) {  // the lattice does not reach this CTA: a host error
        if (threadIdx.x == 0) atomicAdd(p.misses, static_cast<unsigned long long>(r1 - r0) * static_cast<unsigned long long>(c1 - c0));
        return;
    }
    for (int i = threadIdx.x; i < nw * nh; i += THREADS) nodes[i] = p.nodes[(ly + i / nw) * p.nodes_w + lx + i % nw];
    __syncthreads();

    const int64_t gmask = (int64_t(1) << p.log2g) - 1;
    // (u, v) of global corner (gx, gy), interpolated in the cell that contains it
    auto corner = [&](int64_t gx, int64_t gy) {
        const int ix = int((gx >> p.log2g) - kx0), iy = int((gy >> p.log2g) - ky0);
        const double fx = __dmul_rn(double(gx & gmask), p.inv_g), fy = __dmul_rn(double(gy & gmask), p.inv_g);
        const double2 n00 = nodes[iy * nw + ix], n10 = nodes[iy * nw + ix + 1];
        const double2 n01 = nodes[(iy + 1) * nw + ix], n11 = nodes[(iy + 1) * nw + ix + 1];
        return make_double2(lerp(lerp(n00.x, n10.x, fx), lerp(n01.x, n11.x, fx), fy), lerp(lerp(n00.y, n10.y, fx), lerp(n01.y, n11.y, fx), fy));
    };

    unsigned long long covered = 0, misses = 0;
    const int cols = c1 - c0;
    for (int q = threadIdx.x; q < (r1 - r0) * cols; q += THREADS) {
        const int r = r0 + q / cols, c = c0 + q % cols;
        const int64_t gx = tx * S + c, gy = ty * S + r;
        const double2 p00 = corner(gx, gy), p10 = corner(gx + 1, gy), p01 = corner(gx, gy + 1), p11 = corner(gx + 1, gy + 1);
        uint32_t px = 0;  // 0x00BBGGRR
        do {
            if (isnan(p00.x + p10.x + p01.x + p11.x + p00.y + p10.y + p01.y + p11.y)) break;  // a NaN corner: uncovered
            const double u0 = fmin(fmin(p00.x, p10.x), fmin(p01.x, p11.x)), u1 = fmax(fmax(p00.x, p10.x), fmax(p01.x, p11.x));
            const double v0 = fmin(fmin(p00.y, p10.y), fmin(p01.y, p11.y)), v1 = fmax(fmax(p00.y, p10.y), fmax(p01.y, p11.y));
            const double a0 = fmax(u0, 0.0), a1 = fmin(u1, p.width), b0 = fmax(v0, 0.0), b1 = fmin(v1, p.height);
            if (!(a0 < a1 && b0 < b1)) break;
            if (__dsub_rn(u1, u0) > double(RSB_TILE_MAX_FOOTPRINT) || __dsub_rn(v1, v0) > double(RSB_TILE_MAX_FOOTPRINT)) {  // the host refuses these
                ++misses;
                break;
            }
            const int64_t i0 = int64_t(floor(a0)), i1 = int64_t(ceil(a1)), j0 = int64_t(floor(b0)), j1 = int64_t(ceil(b1));
            double ar = 0.0, ag = 0.0, ab = 0.0, ws = 0.0;
            bool miss = false;
            for (int64_t j = j0; j < j1; ++j) {
                const double wy = __dsub_rn(fmin(double(j + 1), b1), fmax(double(j), b0));
                double rr = 0.0, rg = 0.0, rb = 0.0, rw = 0.0;
                for (int64_t i = i0; i < i1; ++i) {
                    uint32_t cr, cg, cb;
                    if (!load<SPP>(p, i, j, cr, cg, cb, miss)) continue;
                    const double wx = __dsub_rn(fmin(double(i + 1), a1), fmax(double(i), a0));
                    rr = __dadd_rn(rr, __dmul_rn(wx, double(cr)));
                    rg = __dadd_rn(rg, __dmul_rn(wx, double(cg)));
                    rb = __dadd_rn(rb, __dmul_rn(wx, double(cb)));
                    rw = __dadd_rn(rw, wx);
                }
                ar = __dadd_rn(ar, __dmul_rn(wy, rr));
                ag = __dadd_rn(ag, __dmul_rn(wy, rg));
                ab = __dadd_rn(ab, __dmul_rn(wy, rb));
                ws = __dadd_rn(ws, __dmul_rn(wy, rw));
            }
            if (miss) {
                ++misses;
                break;
            }
            if (!(ws > 0.0)) break;
            px = quantize(ar, ws) | (quantize(ag, ws) << 8) | (quantize(ab, ws) << 16);
            ++covered;
        } while (false);
        uint8_t* o = p.out + n * p.image_stride + (int64_t(r) * S + c) * 3;
        o[0] = uint8_t(px);
        o[1] = uint8_t(px >> 8);
        o[2] = uint8_t(px >> 16);
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
        unsigned long long c = 0, m = 0;
        for (int w = 0; w < THREADS / 32; ++w) {
            c += sums[0][w];
            m += sums[1][w];
        }
        if (c) atomicAdd(p.covered + n, c);
        if (m) atomicAdd(p.misses, m);
    }
}

// the checks both entry points make before the device check (`fn` names the entry point in the message)
int validate(const char* fn, const uint8_t* src, int64_t src_pitch, int64_t win_row0, int64_t win_col0, int64_t win_rows, int64_t win_cols,
             int64_t raster_w, int64_t raster_h, int32_t spp, int32_t alpha, int32_t nodata, const double* nodes, int64_t node_x0, int64_t node_y0,
             int32_t nodes_w, int32_t nodes_h, int32_t grid_step, const int64_t* tiles, int32_t N, int32_t size, const uint8_t* out,
             const int64_t* covered, const int64_t* misses) {
    if (!src || !nodes || !tiles || !out || !covered || !misses) return set_error(RSB_E_INVALID, "%s: null pointer", fn);
    if (spp != 1 && spp != 3 && spp != 4) return set_error(RSB_E_INVALID, "%s: %d samples per pixel (need 1, 3 or 4)", fn, spp);
    if ((alpha != 0 && alpha != 1) || (alpha && spp != 4)) return set_error(RSB_E_INVALID, "%s: alpha %d with %d samples", fn, alpha, spp);
    if (nodata < -1 || nodata > 255) return set_error(RSB_E_INVALID, "%s: nodata %d (need -1 or 0..255)", fn, nodata);
    if (raster_w < 1 || raster_h < 1 || win_rows < 1 || win_cols < 1 || win_row0 < 0 || win_col0 < 0 || win_row0 + win_rows > raster_h ||
        win_col0 + win_cols > raster_w || src_pitch < win_cols * spp || (spp == 4 && (src_pitch % 4 || reinterpret_cast<uintptr_t>(src) % 4)))
        return set_error(RSB_E_INVALID, "%s: window rows [%lld, +%lld) cols [%lld, +%lld) pitch %lld of a %lld x %lld raster", fn,
                         (long long)win_row0, (long long)win_rows, (long long)win_col0, (long long)win_cols, (long long)src_pitch,
                         (long long)raster_w, (long long)raster_h);
    if (grid_step < 1 || grid_step > RSB_TILE_MAX_STEP || (grid_step & (grid_step - 1)))
        return set_error(RSB_E_INVALID, "%s: lattice step %d (need a power of two in 1..%d)", fn, grid_step, RSB_TILE_MAX_STEP);
    if (nodes_w < 2 || nodes_h < 2 || node_x0 < 0 || node_y0 < 0 || reinterpret_cast<uintptr_t>(nodes) % 16)
        return set_error(RSB_E_INVALID, "%s: lattice of %d x %d nodes at (%lld, %lld)", fn, nodes_w, nodes_h, (long long)node_x0, (long long)node_y0);
    if (N < 1 || N > 65535 || size < 1 || size > RSB_TILE_MAX_SIZE) return set_error(RSB_E_INVALID, "%s: N %d, size %d", fn, N, size);
    return RSB_OK;
}

// clears the counts and fills the launch parameters (everything but vector_stores)
int prepare(const char* fn, WarpParams& p, const uint8_t* src, int64_t src_pitch, int64_t win_row0, int64_t win_col0, int64_t win_rows,
            int64_t win_cols, int64_t raster_w, int64_t raster_h, int32_t alpha, int32_t nodata, const double* nodes, int64_t node_x0,
            int64_t node_y0, int32_t nodes_w, int32_t nodes_h, int32_t grid_step, const int64_t* tiles, int32_t N, int32_t size, uint8_t* out,
            int64_t image_stride, int64_t* covered, int64_t* misses, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(covered, 0, sizeof(int64_t) * size_t(N), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(misses, 0, sizeof(int64_t), st);
    if (e != cudaSuccess) {
        char what[64];
        snprintf(what, sizeof what, "%s: clear counts", fn);
        return set_cuda_error(e, what);
    }
    int log2g = 0;
    while ((1 << log2g) < grid_step) ++log2g;
    p.src = src;
    p.src_pitch = src_pitch;
    p.row0 = win_row0;
    p.col0 = win_col0;
    p.rows = win_rows;
    p.cols = win_cols;
    p.width = double(raster_w);
    p.height = double(raster_h);
    p.last_col = raster_w - 1;
    p.last_row = raster_h - 1;
    p.alpha = alpha;
    p.nodata = nodata;
    p.nodes = reinterpret_cast<const double2*>(nodes);
    p.node_x0 = node_x0;
    p.node_y0 = node_y0;
    p.nodes_w = nodes_w;
    p.nodes_h = nodes_h;
    p.log2g = log2g;
    p.inv_g = 1.0 / grid_step;
    p.tiles = tiles;
    p.size = size;
    p.segs = (size + SEG - 1) / SEG;
    p.out = out;
    p.image_stride = image_stride;
    p.vector_stores = 0;
    p.covered = reinterpret_cast<unsigned long long*>(covered);
    p.misses = reinterpret_cast<unsigned long long*>(misses);
    return RSB_OK;
}

}  // namespace

extern "C" int rsb_tile_warp(const uint8_t* src, int64_t src_pitch, int64_t win_row0, int64_t win_col0, int64_t win_rows, int64_t win_cols,
                             int64_t raster_w, int64_t raster_h, int32_t spp, int32_t alpha, int32_t nodata, const double* nodes, int64_t node_x0,
                             int64_t node_y0, int32_t nodes_w, int32_t nodes_h, int32_t grid_step, const int64_t* tiles, int32_t N, int32_t size,
                             int32_t resampling, uint8_t* out, int64_t image_stride, int64_t* covered, int64_t* misses, void* stream) {
    int rc = validate("tile_warp", src, src_pitch, win_row0, win_col0, win_rows, win_cols, raster_w, raster_h, spp, alpha, nodata, nodes, node_x0,
                      node_y0, nodes_w, nodes_h, grid_step, tiles, N, size, out, covered, misses);
    if (rc != RSB_OK) return rc;
    if (resampling != 0 && resampling != 1) return set_error(RSB_E_INVALID, "tile_warp: resampling %d (0 nearest, 1 bilinear)", resampling);
    if (image_stride < int64_t(size) * size * 3) return set_error(RSB_E_INVALID, "tile_warp: image stride %lld < %d", (long long)image_stride, size * size * 3);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    WarpParams p;
    rc = prepare("tile_warp", p, src, src_pitch, win_row0, win_col0, win_rows, win_cols, raster_w, raster_h, alpha, nodata, nodes, node_x0, node_y0,
                 nodes_w, nodes_h, grid_step, tiles, N, size, out, image_stride, covered, misses, st);
    if (rc != RSB_OK) return rc;
    p.vector_stores = size % 4 == 0 && image_stride % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0;
    if (spp == 1) launch<1>(p, N, resampling, st);
    else if (spp == 3) launch<3>(p, N, resampling, st);
    else launch<4>(p, N, resampling, st);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "tile_warp launch");
}

extern "C" int rsb_tile_average(const uint8_t* src, int64_t src_pitch, int64_t win_row0, int64_t win_col0, int64_t win_rows, int64_t win_cols,
                                int64_t raster_w, int64_t raster_h, int32_t spp, int32_t alpha, int32_t nodata, const double* nodes, int64_t node_x0,
                                int64_t node_y0, int32_t nodes_w, int32_t nodes_h, int32_t grid_step, const int64_t* tiles, int32_t N, int32_t size,
                                uint8_t* out, int64_t image_stride, int64_t* covered, int64_t* misses, void* stream) {
    int rc = validate("tile_average", src, src_pitch, win_row0, win_col0, win_rows, win_cols, raster_w, raster_h, spp, alpha, nodata, nodes, node_x0,
                      node_y0, nodes_w, nodes_h, grid_step, tiles, N, size, out, covered, misses);
    if (rc != RSB_OK) return rc;
    if (image_stride < int64_t(size) * size * 3)
        return set_error(RSB_E_INVALID, "tile_average: image stride %lld < %d", (long long)image_stride, size * size * 3);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    WarpParams p;
    rc = prepare("tile_average", p, src, src_pitch, win_row0, win_col0, win_rows, win_cols, raster_w, raster_h, alpha, nodata, nodes, node_x0,
                 node_y0, nodes_w, nodes_h, grid_step, tiles, N, size, out, image_stride, covered, misses, st);
    if (rc != RSB_OK) return rc;
    const dim3 grid(unsigned(((size + BAND - 1) / BAND) * p.segs), unsigned(N));
    if (spp == 1) average_kernel<1><<<grid, THREADS, 0, st>>>(p);
    else if (spp == 3) average_kernel<3><<<grid, THREADS, 0, st>>>(p);
    else average_kernel<4><<<grid, THREADS, 0, st>>>(p);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "tile_average launch");
}
