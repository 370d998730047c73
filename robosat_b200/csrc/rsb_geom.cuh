// Device helpers shared by the geometry kernels: the vertex transform, a binary search over offset arrays, and the one polygon
// fill of `rs rasterize`, `rs cover` and `rs merge`.
//
// fill_band is GDAL's scanline rule (all_touched=False, DESIGN.md §8, restated in tests/rasterize_reference.py) on one band of
// rows of a W-column grid, held in shared memory as bit-packed rows of 32-column words. For each polygon, the threads stride over
// its edges. Each crossing of an edge with a row's centre line yc = r + 0.5 (y1 <= yc < y2 with y1 <= y2) at x XORs the toggle
// bit of column clamp(floor(x + 0.5), 0, W); a toggle at W is dropped. Rounding is monotone, so the sorted crossings map to
// sorted columns, and the prefix XOR of a row's toggles is exactly the union of GDAL's pair spans [floor(a + 0.5), floor(b + 0.5))
// (even-odd within the polygon). A warp takes a row: the prefix XOR runs within a word by shift-XOR doubling and across words by
// a warp scan of the word parities. The row goes to the caller, which ORs it into its output (polygons are unioned, not XOR-ed),
// and its toggles are cleared for the next polygon. Only the rows a polygon crossed in this band are scanned.
//
// Every float64 operation of the transform and the crossing uses an explicitly rounded intrinsic: nvcc would otherwise contract
// a * b + c into an FMA and disagree with the numpy restatement at near-ties.
#pragma once

#include <stdint.h>

namespace rsb {

// vertex i -> grid coordinates (c0 + X * c1, r0 + Y * r1); vertices are 16-byte aligned (x, y) pairs
__device__ __forceinline__ double2 to_pixels(const double* __restrict__ v, int64_t i, double c0, double c1, double r0, double r1) {
    const double2 m = reinterpret_cast<const double2*>(v)[i];
    return make_double2(__dadd_rn(c0, __dmul_rn(m.x, c1)), __dadd_rn(r0, __dmul_rn(m.y, r1)));
}

// first index in [lo, hi) with a[index] > v (hi when none)
__device__ __forceinline__ int64_t upper_bound(const int64_t* __restrict__ a, int64_t lo, int64_t hi, int64_t v) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] <= v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// Fills grid rows [y0, y0 + rows) of a W-column grid with the union of polygons poly_at(k), k in [k0, k1), under the transform
// (c0, c1, r0, r1). Called by the whole CTA. poly_at returns -1 to skip an entry; the CTA still passes that entry's barriers.
// W and y0 keep the caller's integer types (int for a tile, int64_t for a cover grid), so the column and row arithmetic is no
// wider than the caller's. tog holds rows * ceil(W / 32) shared words, zero on entry (the caller's zeroing needs no barrier of
// its own: the first one here orders it) and zero again on return. Each finished word w of band row r (0 <= r < rows) goes to
// emit(r, w, bits), zero words included, with the bits past column W cleared. One thread emits a given word per polygon and a
// barrier separates the polygons, so emit may OR without atomics.
template <class Cols, class Row, class PolyAt, class Emit>
__device__ __forceinline__ void fill_band(const double* __restrict__ vertices, const int64_t* __restrict__ ring_offsets, const int32_t* __restrict__ poly_rings,
                                          int k0, int k1, PolyAt poly_at, double c0, double c1, double r0, double r1, Cols W, Row y0, int rows,
                                          uint32_t* tog, Emit emit) {
    constexpr unsigned FULL = 0xffffffffu;
    __shared__ int s_rmin, s_rmax;
    const int words = static_cast<int>((W + 31) >> 5);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    if (tid == 0) {
        s_rmin = INT32_MAX;
        s_rmax = -1;
    }
    const double band_lo = static_cast<double>(y0), band_hi = static_cast<double>(y0 + rows), Wd = static_cast<double>(W);
    __syncthreads();

    for (int k = k0; k < k1; ++k) {
        const int p = poly_at(k);
        int rlo = INT32_MAX, rhi = -1;
        const int ring_lo = p < 0 ? 0 : poly_rings[p], ring_hi = p < 0 ? 0 : poly_rings[p + 1];
        for (int ring = ring_lo; ring < ring_hi; ++ring) {
            const int64_t v0 = ring_offsets[ring], v1 = ring_offsets[ring + 1];
            for (int64_t i = v0 + tid; i < v1; i += blockDim.x) {
                double2 a = to_pixels(vertices, i, c0, c1, r0, r1);
                double2 b = to_pixels(vertices, i + 1 < v1 ? i + 1 : v0, c0, c1, r0, r1);
                if (a.y > b.y) {
                    const double2 t = a;
                    a = b;
                    b = t;
                }
                // rows with y1 <= r + 0.5 < y2 inside the band; start one row early and test exactly
                if (!(a.y < band_hi && b.y > band_lo && a.y < b.y)) continue;
                const double start = fmax(floor(a.y - 0.5), band_lo);
                const double dx = __dsub_rn(b.x, a.x), dy = __dsub_rn(b.y, a.y);
                for (int r = static_cast<int>(start - band_lo); r < rows; ++r) {
                    const double yc = static_cast<double>(y0 + r) + 0.5;
                    if (!(yc < b.y)) break;
                    if (!(a.y <= yc)) continue;
                    const double x = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(yc, a.y), dx), dy), a.x);
                    const double c = fmin(fmax(floor(__dadd_rn(x, 0.5)), 0.0), Wd);
                    const Cols col = static_cast<Cols>(c);
                    if (col < W) atomicXor(&tog[r * words + static_cast<int>(col >> 5)], 1u << (col & 31));
                    rlo = min(rlo, r);
                    rhi = max(rhi, r);
                }
            }
        }
        const int hit = rhi >= 0;
        if (hit) {
            atomicMin(&s_rmin, rlo);
            atomicMax(&s_rmax, rhi);
        }
        if (!__syncthreads_or(hit)) continue;
        const int lo = s_rmin, hi = s_rmax;
        __syncthreads();
        if (tid == 0) {
            s_rmin = INT32_MAX;
            s_rmax = -1;
        }
        for (int r = lo + warp; r <= hi; r += nwarps) {
            uint32_t carry = 0;  // parity of all toggles left of this chunk
            for (int cw = 0; cw < words; cw += 32) {
                const int w = cw + lane;
                uint32_t t = 0;
                if (w < words) {
                    t = tog[r * words + w];
                    tog[r * words + w] = 0u;
                }
                // inclusive prefix XOR within the word (bit j = XOR of bits 0..j)
                t ^= t << 1;
                t ^= t << 2;
                t ^= t << 4;
                t ^= t << 8;
                t ^= t << 16;
                // exclusive scan of the word parities (bit 31 of the prefixed word) across the warp
                uint32_t par = t >> 31;
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t u = __shfl_up_sync(FULL, par, o);
                    if (lane >= o) par ^= u;
                }
                const uint32_t excl = (par ^ (t >> 31)) ^ carry;
                // bits past column W cleared (a toggle at W was dropped, so the row's parity may leave them set)
                if (w < words) emit(r, w, (excl ? ~t : t) & (32 * w + 32 <= W ? FULL : ~(FULL << (W & 31))));
                carry = __shfl_sync(FULL, par, 31) ^ carry;
            }
        }
        __syncthreads();
    }
}

}  // namespace rsb
