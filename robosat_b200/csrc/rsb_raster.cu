// Polygon fill for `rs rasterize` (robosat/tools/rasterize.py:64-83: rasterio.features.rasterize, all_touched=False, burn value
// 1, merge "replace"): GeoJSON polygons in EPSG:3857 burned into {0, 1} tile masks with GDAL's scanline rule.
//
// One CTA fills a band of BH rows of one tile. Shared memory holds two bit-packed bands of 32-pixel words: toggles and the
// accumulated mask. For each polygon of the tile's list, threads stride over its edges. Each crossing of an edge with a row's
// centre line yc = r + 0.5 (y1 <= yc < y2 with y1 <= y2) at x XORs the toggle bit of column clamp(floor(x + 0.5), 0, size); a
// toggle at `size` is dropped. Rounding is monotone, so the sorted crossings map to sorted columns, and the prefix XOR of a row's
// toggles is exactly the union of GDAL's pair spans [floor(a + 0.5), floor(b + 0.5)). A warp takes a row: the prefix XOR runs
// within a word by shift-XOR doubling and across words by a warp scan of the word parities. The row is OR-ed into the
// accumulator (polygons are unioned, not XOR-ed) and its toggles are cleared for the next polygon. Only rows a polygon crossed
// in this band are scanned. At the end the bits are expanded to bytes and the foreground is counted.
//
// Every float64 operation of the vertex transform and the crossing uses an explicitly rounded intrinsic: nvcc would otherwise
// contract a * b + c into an FMA and disagree with the numpy restatement (tests/rasterize_reference.py) at near-ties.

#include <stdint.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int RASTER_THREADS = 256;

__device__ __forceinline__ double2 to_pixels(const double* __restrict__ v, int64_t i, double c0, double c1, double r0, double r1) {
    const double2 m = reinterpret_cast<const double2*>(v)[i];
    return make_double2(__dadd_rn(c0, __dmul_rn(m.x, c1)), __dadd_rn(r0, __dmul_rn(m.y, r1)));
}

__global__ void __launch_bounds__(RASTER_THREADS) rasterize_kernel(const double* __restrict__ vertices, const int64_t* __restrict__ ring_offsets,
                                                                   const int32_t* __restrict__ poly_rings, int32_t num_polys,
                                                                   const int32_t* __restrict__ tile_poly_offsets, const int32_t* __restrict__ tile_polys,
                                                                   const double* __restrict__ tile_transforms, int size, int BH, int bands,
                                                                   uint8_t* __restrict__ out, int64_t image_stride, int32_t* __restrict__ counts) {
    extern __shared__ __align__(16) uint32_t smem[];
    __shared__ int s_rmin, s_rmax;
    const int words = (size + 31) >> 5;
    const int n = blockIdx.x / bands;
    const int y0 = (blockIdx.x % bands) * BH;
    const int rows = min(BH, size - y0);
    uint32_t* tog = smem;
    uint32_t* acc = smem + BH * words;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    for (int i = tid; i < 2 * BH * words; i += blockDim.x) smem[i] = 0u;
    if (tid == 0) {
        s_rmin = INT32_MAX;
        s_rmax = -1;
    }
    const double c0 = tile_transforms[4 * n + 0], c1 = tile_transforms[4 * n + 1];
    const double r0 = tile_transforms[4 * n + 2], r1 = tile_transforms[4 * n + 3];
    const int p_begin = tile_poly_offsets[n], p_end = tile_poly_offsets[n + 1];
    const double band_lo = static_cast<double>(y0), band_hi = static_cast<double>(y0 + rows);
    __syncthreads();

    for (int k = p_begin; k < p_end; ++k) {
        const int p = tile_polys[k];
        int rlo = INT32_MAX, rhi = -1;
        if (p >= 0 && p < num_polys) {
            for (int ring = poly_rings[p]; ring < poly_rings[p + 1]; ++ring) {
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
                    for (int r = static_cast<int>(start) - y0; r < rows; ++r) {
                        const double yc = static_cast<double>(y0 + r) + 0.5;
                        if (!(yc < b.y)) break;
                        if (!(a.y <= yc)) continue;
                        const double x = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(yc, a.y), dx), dy), a.x);
                        const double c = fmin(fmax(floor(__dadd_rn(x, 0.5)), 0.0), static_cast<double>(size));
                        const int col = static_cast<int>(c);
                        if (col < size) atomicXor(&tog[r * words + (col >> 5)], 1u << (col & 31));
                        rlo = min(rlo, r);
                        rhi = max(rhi, r);
                    }
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
            for (int c0w = 0; c0w < words; c0w += 32) {
                const int w = c0w + lane;
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
                if (w < words) acc[r * words + w] |= excl ? ~t : t;
                carry = __shfl_sync(FULL, par, 31) ^ carry;
            }
        }
        __syncthreads();
    }

    // bits -> bytes, count. Four pixels per thread, stored as one 32-bit word when the row is 4-byte aligned.
    uint8_t* img = out + static_cast<int64_t>(n) * image_stride;
    const bool wide = (size & 3) == 0 && (image_stride & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0;
    const int quads = (size + 3) >> 2;
    int fg = 0;
    for (int idx = tid; idx < rows * quads; idx += blockDim.x) {
        const int r = idx / quads, q = idx - r * quads;
        const int x = 4 * q;
        const uint32_t word = acc[r * words + (x >> 5)];
        uint32_t nib = (word >> (x & 31)) & 0xfu;
        if (x + 4 > size) nib &= (1u << (size - x)) - 1u;
        fg += __popc(nib);
        uint8_t* row = img + static_cast<int64_t>(y0 + r) * size;
        const uint32_t bytes = (nib * 0x00204081u) & 0x01010101u;
        if (wide) {
            *reinterpret_cast<uint32_t*>(row + x) = bytes;
        } else {
            for (int j = 0; j < 4 && x + j < size; ++j) row[x + j] = static_cast<uint8_t>((bytes >> (8 * j)) & 1u);
        }
    }
    for (int o = 16; o > 0; o >>= 1) fg += __shfl_xor_sync(FULL, fg, o);
    if (lane == 0 && fg) atomicAdd(&counts[n], fg);
}

}  // namespace

extern "C" int rsb_rasterize_polygons(const double* vertices, const int64_t* ring_offsets, const int32_t* poly_rings, int32_t num_polys,
                                      const int32_t* tile_poly_offsets, const int32_t* tile_polys, const double* tile_transforms, int32_t N, int32_t size, uint8_t* out, int64_t image_stride,
                                      int32_t* fg_counts, void* stream) {
    if (!tile_poly_offsets || !tile_polys || !tile_transforms || !out || !fg_counts) return set_error(RSB_E_INVALID, "rasterize_polygons: null pointer");
    if (N < 1) return set_error(RSB_E_INVALID, "rasterize_polygons: N=%d (need N >= 1)", N);
    if (size < 1 || size > RSB_RASTER_MAX_SIZE)
        return set_error(RSB_E_INVALID, "rasterize_polygons: size %d (need 1 <= size <= %d)", size, RSB_RASTER_MAX_SIZE);
    if (image_stride < static_cast<int64_t>(size) * size)
        return set_error(RSB_E_INVALID, "rasterize_polygons: image_stride %lld < size*size = %lld", (long long)image_stride,
                         (long long)size * size);
    if (num_polys < 0) return set_error(RSB_E_INVALID, "rasterize_polygons: num_polys=%d", num_polys);
    if (num_polys > 0 && (!vertices || !ring_offsets || !poly_rings))
        return set_error(RSB_E_INVALID, "rasterize_polygons: null polygon array with %d polygons", num_polys);
    if (vertices && (reinterpret_cast<uintptr_t>(vertices) & 15) != 0)
        return set_error(RSB_E_INVALID, "rasterize_polygons: vertices must be 16-byte aligned");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;

    // bands of BH rows: at most 128 rows and 48 KB of shared memory, halved while the grid gives fewer than two CTAs per SM
    const int words = (size + 31) / 32;
    int BH = 128;
    while (BH > 1 && static_cast<size_t>(BH) * words * 8 > 48 * 1024) BH /= 2;
    while (BH > 16 && static_cast<int64_t>(N) * ((size + BH - 1) / BH) < 2 * num_sms()) BH /= 2;
    if (BH > size) BH = size;
    const int bands = (size + BH - 1) / BH;
    const int64_t blocks = static_cast<int64_t>(N) * bands;
    if (blocks > 0x7fffffff) return set_error(RSB_E_INVALID, "rasterize_polygons: %lld CTAs", (long long)blocks);
    const size_t smem = static_cast<size_t>(BH) * words * 4 * 2;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaFuncSetAttribute(rasterize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return set_cuda_error(e, "rasterize_polygons: shared memory attribute");
    e = cudaMemsetAsync(fg_counts, 0, sizeof(int32_t) * N, st);
    if (e != cudaSuccess) return set_cuda_error(e, "rasterize_polygons: clear fg_counts");
    rasterize_kernel<<<static_cast<unsigned>(blocks), RASTER_THREADS, smem, st>>>(vertices, ring_offsets, poly_rings, num_polys, tile_poly_offsets,
                                                                                  tile_polys, tile_transforms, size, BH, bands, out, image_stride,
                                                                                  fg_counts);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "rasterize_polygons launch");
}
