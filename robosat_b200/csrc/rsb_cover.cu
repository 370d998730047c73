// Tile covers for `rs cover` (robosat/tools/cover.py: supermercado's burntiles.burn, i.e. rasterio.features.rasterize with
// all_touched=True on each feature's own tile grid), and the 64-bit key sort + unique that merges the covers of all features.
//
// A feature's grid is W x H tiles; the host computes it (DESIGN.md §8). The batch's cells live in one global bitmap, one bit per
// tile, rows of ceil(W / 32) words, restricted to a row window [row_lo, row_lo + rows) per feature so that a feature larger than
// the memory budget can be covered in row bands. A cell is set when
//   (a) the scanline fill of `rs rasterize` sets it (row centre r + 0.5, even-odd per polygon, spans [floor(a + 0.5), floor(b + 0.5))), or
//   (b) GDAL's all-touched line walk over some edge of some ring burns it.
// The walk is a sequential float64 recurrence along one edge, so it cannot be split: one thread walks one edge from its own
// clipped start, exactly as the restatement does (tests/cover_reference.py), and sets bits with atomicOr in the global bitmap.
// A long edge is therefore walked once, not once per band of the fill; edges, not bands, carry the walk's parallelism. The fill
// then runs one CTA per (feature, band of rows) with fill_band (rsb_geom.cuh) on rows of up to RSB_COVER_MAX_WIDTH columns, and
// ORs its rows into the same bitmap (the bands of a launch are disjoint, and the walk kernel has finished, so plain stores
// suffice). Bits are OR-ed, so the bitmap does not depend on the order of anything.
//
// Keys are (x << zoom) | y, so ascending keys are tiles in (x, y) order. rsb_cover_emit_keys writes one key per set bit in an
// unspecified order; rsb_sort_unique_u64 sorts them with a stable LSD radix sort of ceil(key_bits / 8) 8-bit passes (the
// histogram / scan / warp-ranked scatter design of the Lovász sort in rsb_loss.cu, for 64-bit keys without payload) and drops
// adjacent duplicates, so the result is identical from run to run.
//
// Every float64 operation of the transform, the crossings and the walk uses an explicitly rounded intrinsic: nvcc would otherwise
// contract a * b + c into an FMA and the walk would leave the restatement's float sequence.

#include <stdint.h>

#include <algorithm>

#include "../../include/rsb200.h"
#include "rsb_geom.cuh"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int FILL_THREADS = 256;
constexpr int WALK_THREADS = 128;
constexpr int EMIT_THREADS = 256;
constexpr int SORT_THREADS = 256;
constexpr int SORT_ITEMS = 16;
constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;  // keys per CTA of the sort
constexpr int SORT_WARPS = SORT_THREADS / 32;

// grid row of a feature: xmin, ymin, W, H, row_lo, rows
struct CoverGrid {
    int64_t xmin, ymin, W, H, row_lo, rows;
};

__device__ __forceinline__ CoverGrid load_grid(const int64_t* __restrict__ g, int f) {
    const int64_t* p = g + 6 * static_cast<int64_t>(f);
    return CoverGrid{p[0], p[1], p[2], p[3], p[4], p[5]};
}

__device__ __forceinline__ void burn_cell(uint32_t* __restrict__ bm, const CoverGrid& g, int64_t words, int64_t ix, int64_t iy) {
    const int64_t r = iy - g.row_lo;
    if (r < 0 || r >= g.rows) return;
    atomicOr(&bm[r * words + (ix >> 5)], 1u << (ix & 31));
}

// GDAL's GDALdllImageLineAllTouched for one edge, as restated in DESIGN.md §8. Returns false when the step bound was exceeded.
__device__ bool walk_edge(double x0, double y0, double x1, double y1, const CoverGrid& g, int64_t words, uint32_t* __restrict__ bm) {
    const double Wd = static_cast<double>(g.W), Hd = static_cast<double>(g.H);
    if ((y0 < 0.0 && y1 < 0.0) || (y0 > Hd && y1 > Hd) || (x0 < 0.0 && x1 < 0.0) || (x0 > Wd && x1 > Wd)) return true;
    if (x0 > x1) {
        double t = x0;
        x0 = x1;
        x1 = t;
        t = y0;
        y0 = y1;
        y1 = t;
    }
    if (floor(x0) == floor(x1) || fabs(__dsub_rn(x0, x1)) < 0.01) {  // near-vertical: one column
        const double ix = floor(x1);
        if (ix < 0.0 || ix >= Wd) return true;
        const int64_t first = static_cast<int64_t>(fmax(floor(fmin(y0, y1)), 0.0));
        const int64_t last = static_cast<int64_t>(fmin(floor(fmax(y0, y1)), Hd - 1.0));
        const int64_t lo = max(first, g.row_lo), hi = min(last, g.row_lo + g.rows - 1);
        for (int64_t iy = lo; iy <= hi; ++iy) burn_cell(bm, g, words, static_cast<int64_t>(ix), iy);
        return true;
    }
    if (floor(y0) == floor(y1) || fabs(__dsub_rn(y0, y1)) < 0.01) {  // near-horizontal: one row
        const double iy = floor(y0);
        if (iy < 0.0 || iy >= Hd) return true;
        const int64_t r = static_cast<int64_t>(iy) - g.row_lo;
        if (r < 0 || r >= g.rows) return true;
        const int64_t c0 = static_cast<int64_t>(fmax(floor(x0), 0.0));
        const int64_t c1 = static_cast<int64_t>(fmin(floor(x1), Wd - 1.0));
        for (int64_t w = c0 >> 5; w <= (c1 >> 5); ++w) {  // whole words at a time
            const int lo = w == (c0 >> 5) ? static_cast<int>(c0 & 31) : 0;
            const int hi = w == (c1 >> 5) ? static_cast<int>(c1 & 31) : 31;
            const uint32_t mask = (hi == 31 ? FULL : ((1u << (hi + 1)) - 1u)) & (FULL << lo);
            atomicOr(&bm[r * words + w], mask);
        }
        return true;
    }
    const double slope = __ddiv_rn(__dsub_rn(y1, y0), __dsub_rn(x1, x0));
    if (x1 > Wd) {
        y1 = __dsub_rn(y1, __dmul_rn(__dsub_rn(x1, Wd), slope));
        x1 = Wd;
    }
    if (x0 < 0.0) {
        y0 = __dadd_rn(y0, __dmul_rn(__dsub_rn(0.0, x0), slope));
        x0 = 0.0;
    }
    if (y1 > y0) {
        if (y0 < 0.0) {
            x0 = __dadd_rn(x0, __ddiv_rn(__dsub_rn(0.0, y0), slope));
            y0 = 0.0;
        }
        if (y1 >= Hd) x1 = __dsub_rn(x1, __ddiv_rn(__dsub_rn(y1, Hd), slope));
    } else {
        if (y0 >= Hd) {
            x0 = __dadd_rn(x0, __ddiv_rn(__dsub_rn(Hd, y0), slope));
            y0 = Hd;
        }
        if (y1 < 0.0) x1 = __dsub_rn(x1, __ddiv_rn(__dsub_rn(y1, 0.0), slope));
    }
    // every step reaches a column or row border or moves y by 1e-9, so a walk inside the grid takes about W + H steps; the
    // bound only turns a walk that cannot finish (coordinates beyond float64's resolution of 1e-9) into an error
    int64_t budget = 4 * (g.W + g.H) + 1024;
    while (x0 >= 0.0 && x0 < x1) {
        if (--budget < 0) return false;
        const double ix = floor(x0), iy = floor(y0);
        if (iy >= 0.0 && iy < Hd) burn_cell(bm, g, words, static_cast<int64_t>(ix), static_cast<int64_t>(iy));
        double step_x = __dsub_rn(floor(__dadd_rn(x0, 1.0)), x0);
        double step_y = __dmul_rn(step_x, slope);
        if (floor(__dadd_rn(y0, step_y)) == iy) {
            x0 = __dadd_rn(x0, step_x);
            y0 = __dadd_rn(y0, step_y);
        } else if (slope < 0.0) {
            step_y = __dsub_rn(iy, y0);
            if (step_y > -0.000000001) step_y = -0.000000001;
            step_x = __ddiv_rn(step_y, slope);
            x0 = __dadd_rn(x0, step_x);
            y0 = __dadd_rn(y0, step_y);
        } else {
            step_y = __dsub_rn(__dadd_rn(iy, 1.0), y0);
            if (step_y < 0.000000001) step_y = 0.000000001;
            step_x = __ddiv_rn(step_y, slope);
            x0 = __dadd_rn(x0, step_x);
            y0 = __dadd_rn(y0, step_y);
        }
    }
    return true;
}

// one thread per edge of the batch; vertex_offsets [F + 1] is the prefix of the features' vertex counts
__global__ void __launch_bounds__(WALK_THREADS) cover_walk_kernel(const double* __restrict__ vertices, const int64_t* __restrict__ ring_offsets,
                                                                  const int32_t* __restrict__ poly_rings, const int32_t* __restrict__ feature_polys,
                                                                  const int64_t* __restrict__ vertex_offsets, const double* __restrict__ transforms,
                                                                  const int64_t* __restrict__ grids, const int64_t* __restrict__ bitmap_offsets, int F,
                                                                  uint32_t* __restrict__ bitmap, int64_t* __restrict__ status) {
    const int64_t total = vertex_offsets[F];
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int f = static_cast<int>(upper_bound(vertex_offsets, 0, F + 1, t) - 1);
        const CoverGrid g = load_grid(grids, f);
        if (g.rows <= 0) continue;
        const int64_t ring_lo = poly_rings[feature_polys[f]], ring_hi = poly_rings[feature_polys[f + 1]];
        const int64_t i = ring_offsets[ring_lo] + (t - vertex_offsets[f]);
        const int64_t ring = upper_bound(ring_offsets, ring_lo, ring_hi + 1, i) - 1;
        const int64_t v0 = ring_offsets[ring], v1 = ring_offsets[ring + 1];
        const double c0 = transforms[4 * f + 0], c1 = transforms[4 * f + 1], r0 = transforms[4 * f + 2], r1 = transforms[4 * f + 3];
        const double2 a = to_pixels(vertices, i, c0, c1, r0, r1);
        const double2 b = to_pixels(vertices, i + 1 < v1 ? i + 1 : v0, c0, c1, r0, r1);
        const int64_t words = (g.W + 31) >> 5;
        if (!walk_edge(a.x, a.y, b.x, b.y, g, words, bitmap + bitmap_offsets[f])) atomicOr(reinterpret_cast<unsigned long long*>(&status[1]), 1ull);
    }
}

// one CTA per band: bands[3 * b] = (feature, first row of the band within the feature's window, rows <= BH)
__global__ void __launch_bounds__(FILL_THREADS) cover_fill_kernel(const double* __restrict__ vertices, const int64_t* __restrict__ ring_offsets,
                                                                  const int32_t* __restrict__ poly_rings, const int32_t* __restrict__ feature_polys,
                                                                  const double* __restrict__ transforms, const int64_t* __restrict__ grids,
                                                                  const int64_t* __restrict__ bitmap_offsets, const int32_t* __restrict__ bands,
                                                                  uint32_t* __restrict__ bitmap) {
    extern __shared__ __align__(16) uint32_t tog[];
    const int f = bands[3 * blockIdx.x], band_row = bands[3 * blockIdx.x + 1], rows = bands[3 * blockIdx.x + 2];
    const CoverGrid g = load_grid(grids, f);
    const int words = static_cast<int>((g.W + 31) >> 5);
    uint32_t* out = bitmap + bitmap_offsets[f] + static_cast<int64_t>(band_row) * words;
    for (int i = threadIdx.x; i < rows * words; i += blockDim.x) tog[i] = 0u;
    fill_band(
        vertices, ring_offsets, poly_rings, feature_polys[f], feature_polys[f + 1], [](int k) { return k; }, transforms[4 * f + 0], transforms[4 * f + 1],
        transforms[4 * f + 2], transforms[4 * f + 3], g.W, g.row_lo + band_row, rows, tog, [&](int r, int w, uint32_t bits) {
            if (bits) out[static_cast<int64_t>(r) * words + w] |= bits;
        });
}

// popcount of the batch's bitmap into status[0]; with keys, also one key per set bit at slots taken from status[2]
__global__ void __launch_bounds__(EMIT_THREADS) cover_emit_kernel(const uint32_t* __restrict__ bitmap, const int64_t* __restrict__ bitmap_offsets,
                                                                  const int64_t* __restrict__ grids, int F, int zoom, int64_t* __restrict__ keys,
                                                                  int64_t capacity, int64_t* __restrict__ status) {
    const int64_t total = bitmap_offsets[F];
    const int lane = threadIdx.x & 31;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    unsigned long long mine = 0;
    for (int64_t base = static_cast<int64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~31); base < total; base += stride) {
        const int64_t w = base + lane;
        const uint32_t bits = w < total ? bitmap[w] : 0u;
        if (!keys) {
            mine += __popc(bits);
            continue;
        }
        const int n = __popc(bits);
        int incl = n;
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(FULL, incl, o);
            if (lane >= o) incl += u;
        }
        unsigned long long slot = 0;
        if (lane == 31 && incl) slot = atomicAdd(reinterpret_cast<unsigned long long*>(&status[2]), static_cast<unsigned long long>(incl));
        slot = __shfl_sync(FULL, slot, 31) + static_cast<unsigned long long>(incl - n);
        if (!n) continue;
        const int f = static_cast<int>(upper_bound(bitmap_offsets, 0, F + 1, w) - 1);
        const CoverGrid g = load_grid(grids, f);
        const int64_t words = (g.W + 31) >> 5;
        const int64_t local = w - bitmap_offsets[f];
        const int64_t y = g.ymin + g.row_lo + local / words;
        const int64_t xb = g.xmin + (local % words) * 32;
        for (uint32_t m = bits; m; m &= m - 1, ++slot) {
            const int64_t x = xb + (__ffs(m) - 1);
            if (static_cast<int64_t>(slot) < capacity) keys[slot] = (x << zoom) | y;
        }
    }
    if (!keys) {
        for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(FULL, mine, o);
        if (lane == 0 && mine) atomicAdd(reinterpret_cast<unsigned long long*>(&status[0]), mine);
    }
}

// ---- 64-bit key sort + unique ----

// per-tile digit histogram: hist[digit][tile]
__global__ void __launch_bounds__(SORT_THREADS) sort_hist_kernel(const uint64_t* __restrict__ keys, uint32_t* __restrict__ hist, int shift, int tiles) {
    __shared__ uint32_t sh[256];
    const int tile = blockIdx.x;
    sh[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t* k = keys + static_cast<int64_t>(tile) * SORT_TILE;
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) atomicAdd(&sh[(k[j * SORT_THREADS + threadIdx.x] >> shift) & 255u], 1u);
    __syncthreads();
    hist[static_cast<int64_t>(threadIdx.x) * tiles + tile] = sh[threadIdx.x];
}

// exclusive scan of n counters in place by one CTA; the total goes to *total when given
__global__ void __launch_bounds__(1024) sort_scan_kernel(uint32_t* __restrict__ h, int64_t n, int64_t* __restrict__ total) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += blockDim.x) {
        const int64_t i = base + threadIdx.x;
        const uint32_t v = i < n ? h[i] : 0;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, incl, o);
            if ((threadIdx.x & 31) >= o) incl += t;
        }
        if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            const uint32_t w = threadIdx.x < (blockDim.x >> 5) ? warp_tot[threadIdx.x] : 0;
            uint32_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(FULL, wi, o);
                if (threadIdx.x >= o) wi += t;
            }
            warp_tot[threadIdx.x] = wi - w;
        }
        __syncthreads();
        const uint32_t carry = carry_s;
        if (i < n) h[i] = carry + warp_tot[threadIdx.x >> 5] + incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry_s = carry + warp_tot[threadIdx.x >> 5] + incl;
        __syncthreads();
    }
    if (total && threadIdx.x == 0) *total = carry_s;
}

// stable scatter of one tile: warp w owns the contiguous 512-key slice [w * 512, w * 512 + 512) of the tile
__global__ void __launch_bounds__(SORT_THREADS) sort_scatter_kernel(const uint64_t* __restrict__ keys_in, uint64_t* __restrict__ keys_out,
                                                                    const uint32_t* __restrict__ hist, int shift, int tiles) {
    __shared__ uint32_t cnt[SORT_WARPS][256];
    const int tile = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < SORT_WARPS * 256; i += blockDim.x) (&cnt[0][0])[i] = 0;
    __syncthreads();
    const int64_t base = static_cast<int64_t>(tile) * SORT_TILE + warp * (32 * SORT_ITEMS);
    uint64_t k[SORT_ITEMS];
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) k[j] = keys_in[base + j * 32 + lane];
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        const uint32_t d = static_cast<uint32_t>(k[j] >> shift) & 255u;
        const uint32_t peers = __match_any_sync(FULL, d);
        if (lane == (__ffs(peers) - 1)) cnt[warp][d] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    {
        const int d = threadIdx.x;
        uint32_t run = hist[static_cast<int64_t>(d) * tiles + tile];
#pragma unroll
        for (int w = 0; w < SORT_WARPS; ++w) {
            const uint32_t c = cnt[w][d];
            cnt[w][d] = run;
            run += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; ++j) {
        const uint32_t d = static_cast<uint32_t>(k[j] >> shift) & 255u;
        const uint32_t peers = __match_any_sync(FULL, d);
        const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
        const uint32_t off = cnt[warp][d] + rank;
        __syncwarp();
        if (lane == (__ffs(peers) - 1)) cnt[warp][d] += __popc(peers);
        __syncwarp();
        keys_out[off] = k[j];
    }
}

// keys a thread owns in the unique pass: SORT_ITEMS consecutive ones
__device__ __forceinline__ bool is_first(const uint64_t* __restrict__ k, int64_t i, int64_t n) { return i < n && (i == 0 || k[i] != k[i - 1]); }

__device__ uint32_t block_exclusive_sum(uint32_t v, uint32_t* warp_tot) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = lane < SORT_WARPS ? warp_tot[lane] : 0;
        uint32_t wi = w;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, wi, o);
            if (lane >= o) wi += t;
        }
        if (lane < SORT_WARPS) warp_tot[lane] = wi - w;
    }
    __syncthreads();
    return warp_tot[warp] + incl - v;
}

__global__ void __launch_bounds__(SORT_THREADS) unique_count_kernel(const uint64_t* __restrict__ keys, int64_t n, uint32_t* __restrict__ tile_counts) {
    __shared__ uint32_t warp_tot[SORT_WARPS];
    const int64_t first = static_cast<int64_t>(blockIdx.x) * SORT_TILE + threadIdx.x * SORT_ITEMS;
    uint32_t c = 0;
    for (int j = 0; j < SORT_ITEMS; ++j) c += is_first(keys, first + j, n);
    const uint32_t excl = block_exclusive_sum(c, warp_tot);
    if (threadIdx.x == SORT_THREADS - 1) tile_counts[blockIdx.x] = excl + c;
}

__global__ void __launch_bounds__(SORT_THREADS) unique_scatter_kernel(const uint64_t* __restrict__ keys, int64_t n, const uint32_t* __restrict__ tile_offsets,
                                                                      uint64_t* __restrict__ out) {
    __shared__ uint32_t warp_tot[SORT_WARPS];
    const int64_t first = static_cast<int64_t>(blockIdx.x) * SORT_TILE + threadIdx.x * SORT_ITEMS;
    uint32_t c = 0;
    for (int j = 0; j < SORT_ITEMS; ++j) c += is_first(keys, first + j, n);
    int64_t o = static_cast<int64_t>(tile_offsets[blockIdx.x]) + block_exclusive_sum(c, warp_tot);
    for (int j = 0; j < SORT_ITEMS; ++j)
        if (is_first(keys, first + j, n)) out[o++] = keys[first + j];
}

int64_t sort_tiles(int64_t n) { return (n + SORT_TILE - 1) / SORT_TILE; }

}  // namespace

extern "C" int rsb_cover_polygons(const double* vertices, const int64_t* ring_offsets, const int32_t* poly_rings, int32_t num_polys,
                                  const int32_t* feature_polys, const int64_t* vertex_offsets, const double* transforms, const int64_t* grids,
                                  const int64_t* bitmap_offsets, int32_t F, int64_t num_vertices, const int32_t* bands, int32_t num_bands,
                                  int32_t band_rows, int32_t max_words, uint32_t* bitmap, int64_t bitmap_words, int64_t* status, void* stream) {
    if (!feature_polys || !vertex_offsets || !transforms || !grids || !bitmap_offsets || !bands || !status)
        return set_error(RSB_E_INVALID, "cover_polygons: null pointer");
    if (F < 1) return set_error(RSB_E_INVALID, "cover_polygons: F=%d (need F >= 1)", F);
    if (num_polys < 1 || !vertices || !ring_offsets || !poly_rings)
        return set_error(RSB_E_INVALID, "cover_polygons: need at least one polygon and its arrays (num_polys=%d)", num_polys);
    if ((reinterpret_cast<uintptr_t>(vertices) & 15) != 0) return set_error(RSB_E_INVALID, "cover_polygons: vertices must be 16-byte aligned");
    if (num_vertices < 0 || num_bands < 0) return set_error(RSB_E_INVALID, "cover_polygons: num_vertices=%lld num_bands=%d", (long long)num_vertices, num_bands);
    if (max_words < 1 || max_words > RSB_COVER_MAX_WIDTH / 32)
        return set_error(RSB_E_INVALID, "cover_polygons: max_words=%d (need 1..%d: grids of at most %d columns)", max_words, RSB_COVER_MAX_WIDTH / 32,
                         RSB_COVER_MAX_WIDTH);
    if (band_rows < 1 || static_cast<int64_t>(band_rows) * max_words > RSB_COVER_MAX_WIDTH / 32)
        return set_error(RSB_E_INVALID, "cover_polygons: band_rows=%d x max_words=%d exceeds %d shared-memory words", band_rows, max_words,
                         RSB_COVER_MAX_WIDTH / 32);
    if (num_bands > 0 && !bitmap) return set_error(RSB_E_INVALID, "cover_polygons: null bitmap");
    if (bitmap_words < 0) return set_error(RSB_E_INVALID, "cover_polygons: bitmap_words=%lld", (long long)bitmap_words);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = static_cast<size_t>(band_rows) * max_words * 4;
    cudaError_t e = cudaFuncSetAttribute(cover_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return set_cuda_error(e, "cover_polygons: shared memory attribute");
    e = cudaMemsetAsync(status, 0, 4 * sizeof(int64_t), st);
    if (e == cudaSuccess && bitmap_words > 0) e = cudaMemsetAsync(bitmap, 0, static_cast<size_t>(bitmap_words) * 4, st);
    if (e != cudaSuccess) return set_cuda_error(e, "cover_polygons: clear");
    if (num_vertices > 0) {
        const int64_t blocks = std::min<int64_t>((num_vertices + WALK_THREADS - 1) / WALK_THREADS, 32 * num_sms());
        cover_walk_kernel<<<static_cast<unsigned>(blocks), WALK_THREADS, 0, st>>>(vertices, ring_offsets, poly_rings, feature_polys, vertex_offsets, transforms,
                                                                                   grids, bitmap_offsets, F, bitmap, status);
    }
    if (num_bands > 0)
        cover_fill_kernel<<<static_cast<unsigned>(num_bands), FILL_THREADS, smem, st>>>(vertices, ring_offsets, poly_rings, feature_polys, transforms, grids,
                                                                                        bitmap_offsets, bands, bitmap);
    if (bitmap_words > 0) {
        const int64_t blocks = std::min<int64_t>((bitmap_words + EMIT_THREADS - 1) / EMIT_THREADS, 8 * num_sms());
        cover_emit_kernel<<<static_cast<unsigned>(blocks), EMIT_THREADS, 0, st>>>(bitmap, bitmap_offsets, grids, F, 0, nullptr, 0, status);
    }
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "cover_polygons launch");
}

extern "C" int rsb_cover_emit_keys(const uint32_t* bitmap, int64_t bitmap_words, const int64_t* bitmap_offsets, const int64_t* grids, int32_t F,
                                   int32_t zoom, int64_t* keys, int64_t capacity, int64_t* status, void* stream) {
    if (!bitmap || !bitmap_offsets || !grids || !keys || !status) return set_error(RSB_E_INVALID, "cover_emit_keys: null pointer");
    if (F < 1 || bitmap_words < 1 || capacity < 0) return set_error(RSB_E_INVALID, "cover_emit_keys: F=%d bitmap_words=%lld capacity=%lld", F,
                                                                      (long long)bitmap_words, (long long)capacity);
    if (zoom < 0 || zoom > RSB_COVER_MAX_ZOOM) return set_error(RSB_E_INVALID, "cover_emit_keys: zoom %d (need 0..%d)", zoom, RSB_COVER_MAX_ZOOM);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(status + 2, 0, sizeof(int64_t), st);
    if (e != cudaSuccess) return set_cuda_error(e, "cover_emit_keys: clear");
    const int64_t blocks = std::min<int64_t>((bitmap_words + EMIT_THREADS - 1) / EMIT_THREADS, 8 * num_sms());
    cover_emit_kernel<<<static_cast<unsigned>(blocks), EMIT_THREADS, 0, st>>>(bitmap, bitmap_offsets, grids, F, zoom, keys, capacity, status);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "cover_emit_keys launch");
}

extern "C" int64_t rsb_sort_unique_workspace_bytes(int64_t n) {
    if (n < 0) return -1;
    const int64_t tiles = sort_tiles(n);
    return 2 * tiles * SORT_TILE * 8 + (256 * tiles + tiles) * 4;
}

extern "C" int rsb_sort_unique_u64(int64_t* keys, int64_t n, int32_t key_bits, void* workspace, int64_t workspace_bytes, int64_t* unique_count, void* stream) {
    if (!keys || !unique_count) return set_error(RSB_E_INVALID, "sort_unique_u64: null pointer");
    if (n < 0 || key_bits < 0 || key_bits > 64) return set_error(RSB_E_INVALID, "sort_unique_u64: n=%lld key_bits=%d", (long long)n, key_bits);
    const int64_t tiles = sort_tiles(n);
    if (256 * tiles > 0x7fffffffLL) return set_error(RSB_E_INVALID, "sort_unique_u64: n=%lld keys is too many for one sort", (long long)n);
    if (n > 0 && (!workspace || workspace_bytes < rsb_sort_unique_workspace_bytes(n)))
        return set_error(RSB_E_INVALID, "sort_unique_u64: workspace of %lld bytes < %lld", (long long)workspace_bytes, (long long)rsb_sort_unique_workspace_bytes(n));
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaSuccess;
    if (n == 0) {
        e = cudaMemsetAsync(unique_count, 0, sizeof(int64_t), st);
        return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "sort_unique_u64: clear");
    }
    // the passes ping-pong between two buffers of whole tiles in the workspace; the padding is all ones and sorts last
    const int64_t np = tiles * SORT_TILE;
    uint64_t* buf[2] = {static_cast<uint64_t*>(workspace), static_cast<uint64_t*>(workspace) + np};
    uint32_t* hist = reinterpret_cast<uint32_t*>(buf[1] + np);
    uint32_t* tile_counts = hist + 256 * tiles;
    e = cudaMemcpyAsync(buf[0], keys, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && np > n) e = cudaMemsetAsync(buf[0] + n, 0xff, static_cast<size_t>(np - n) * 8, st);
    if (e != cudaSuccess) return set_cuda_error(e, "sort_unique_u64: stage");
    int cur = 0;
    const int passes = (key_bits + 7) / 8;
    for (int pass = 0; pass < passes; ++pass) {
        const int shift = 8 * pass;
        sort_hist_kernel<<<static_cast<unsigned>(tiles), SORT_THREADS, 0, st>>>(buf[cur], hist, shift, static_cast<int>(tiles));
        sort_scan_kernel<<<1, 1024, 0, st>>>(hist, 256 * tiles, nullptr);
        sort_scatter_kernel<<<static_cast<unsigned>(tiles), SORT_THREADS, 0, st>>>(buf[cur], buf[cur ^ 1], hist, shift, static_cast<int>(tiles));
        cur ^= 1;
    }
    unique_count_kernel<<<static_cast<unsigned>(tiles), SORT_THREADS, 0, st>>>(buf[cur], n, tile_counts);
    sort_scan_kernel<<<1, 1024, 0, st>>>(tile_counts, tiles, unique_count);
    unique_scatter_kernel<<<static_cast<unsigned>(tiles), SORT_THREADS, 0, st>>>(buf[cur], n, tile_counts, reinterpret_cast<uint64_t*>(keys));
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "sort_unique_u64 launch");
}
