// Polygon fill for `rs rasterize` (robosat/tools/rasterize.py:64-83: rasterio.features.rasterize, all_touched=False, burn value
// 1, merge "replace"): GeoJSON polygons in EPSG:3857 burned into {0, 1} tile masks with GDAL's scanline rule.
//
// One CTA fills a band of BH rows of one tile with fill_band (rsb_geom.cuh, which explains the scheme) over the tile's polygon
// list, OR-ing the finished rows into a bit-packed accumulator in shared memory next to the toggles. At the end the bits are
// expanded to bytes and the foreground is counted.

#include <stdint.h>

#include "../../include/rsb200.h"
#include "rsb_geom.cuh"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int RASTER_THREADS = 256;

__global__ void __launch_bounds__(RASTER_THREADS) rasterize_kernel(const double* __restrict__ vertices, const int64_t* __restrict__ ring_offsets,
                                                                   const int32_t* __restrict__ poly_rings, int32_t num_polys,
                                                                   const int32_t* __restrict__ tile_poly_offsets, const int32_t* __restrict__ tile_polys,
                                                                   const double* __restrict__ tile_transforms, int size, int BH, int bands,
                                                                   uint8_t* __restrict__ out, int64_t image_stride, int32_t* __restrict__ counts) {
    extern __shared__ __align__(16) uint32_t smem[];
    const int words = (size + 31) >> 5;
    const int n = blockIdx.x / bands;
    const int y0 = (blockIdx.x % bands) * BH;
    const int rows = min(BH, size - y0);
    uint32_t* tog = smem;
    uint32_t* acc = smem + BH * words;
    const int tid = threadIdx.x, lane = tid & 31;
    for (int i = tid; i < 2 * BH * words; i += blockDim.x) smem[i] = 0u;
    const double c0 = tile_transforms[4 * n + 0], c1 = tile_transforms[4 * n + 1];
    const double r0 = tile_transforms[4 * n + 2], r1 = tile_transforms[4 * n + 3];
    fill_band(
        vertices, ring_offsets, poly_rings, tile_poly_offsets[n], tile_poly_offsets[n + 1],
        [&](int k) {
            const int p = tile_polys[k];
            return p >= 0 && p < num_polys ? p : -1;
        },
        c0, c1, r0, r1, size, y0, rows, tog, [&](int r, int w, uint32_t bits) { acc[r * words + w] |= bits; });

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
