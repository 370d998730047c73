// `rs merge` (robosat/tools/merge.py, robosat/graph/core.py): link features that lie within d metres of each other, find the
// connected components, and close the union of each component's cells with a disk (DESIGN.md §8).
//
// rsb_merge_near: one warp per candidate pair (i, j) of one feature set on EPSG:3395 vertices (RsbShapes, as packed by
// robosat_b200/dedupe.py). The pair is near when some vertex of one lies within d of some edge of the other, with the
// point-to-segment distance t = clamp(((p - a).(b - a)) / |b - a|^2, 0, 1), q = a + t (b - a), |p - q|^2 <= d * d, every
// operation rounded on its own (__d*_rn, no FMA contraction), so tests/merge_reference.py reproduces every flag. Every vertex
// starts exactly one edge, so testing (start of e, f) and (start of f, e) for every edge pair covers every (vertex, edge) pair.
// The lanes split the larger feature's edges; an edge scans the other feature only when its box, widened by a pad a little
// larger than d, meets that feature's box (a point within d of the edge lies in the widened box, so the filter never drops a
// pair the formula links). The result is an "any", so the early exit is deterministic.
//
// rsb_merge_components: union-find over the linked pairs. One thread per pair hooks the larger of the two roots to the smaller
// with atomicCAS and retries until both ends share a root; a root only ever moves to a smaller index, so the final root of a
// component is its smallest member. A second pass follows each node's pointers to its root. labels[i] is therefore the
// smallest index of i's component on every run.
//
// rsb_merge_fill: one CTA per (component, band of rows) sets the cells whose centres the component's polygons cover, with the
// scanline fill of rsb_geom.cuh (even-odd per polygon, union across polygons) on bit-packed rows.
//
// rsb_merge_close: one CTA per (component, tile of 32 rows x 32 words) computes erode(dilate(fill)) with the digital disk
// {(i, j): i^2 + j^2 <= K^2}: the tile's rows plus 2K halo rows and 2 halo words on each side are staged in shared memory,
// dilated into the tile plus K rows and 1 word, then eroded into the tile. Each disk row i is a horizontal run of half-width
// floor(sqrt(K^2 - i^2)), applied with funnel shifts of the neighbouring words. Cells outside the grid are 0 for both ops; the
// host's margin of K + 2 cells keeps the dilation off the grid edge, so this is the closing on the unbounded lattice. Grids have
// no width limit beyond the fill's (a band row in shared memory). The set cells of each component are counted.

#include <stdint.h>

#include <algorithm>

#include "../../include/rsb200.h"
#include "rsb_geom.cuh"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int NEAR_THREADS = 128;
constexpr int UF_THREADS = 256;
constexpr int FILL_THREADS = 256;
constexpr int CLOSE_THREADS = 256;
constexpr int TILE_ROWS = 32;   // output rows of a closing tile
constexpr int TILE_WORDS = 32;  // output words of a closing tile
constexpr int IN_ROWS = TILE_ROWS + 4 * RSB_MERGE_MAX_RADIUS;
constexpr int IN_WORDS = TILE_WORDS + 4;
constexpr int DIL_ROWS = TILE_ROWS + 2 * RSB_MERGE_MAX_RADIUS;
constexpr int DIL_WORDS = TILE_WORDS + 2;

struct Set {
    const double2* __restrict__ v;
    const int32_t* __restrict__ next;
    const int64_t* __restrict__ fv;
    const double* __restrict__ box;
};

// |p - q|^2 <= dd, q the point of segment ab nearest to p (ab has positive length)
__device__ __forceinline__ bool within(double2 p, double2 a, double2 b, double dd) {
    const double dx = __dsub_rn(b.x, a.x), dy = __dsub_rn(b.y, a.y);
    const double len2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
    const double num = __dadd_rn(__dmul_rn(__dsub_rn(p.x, a.x), dx), __dmul_rn(__dsub_rn(p.y, a.y), dy));
    double t = len2 > 0.0 ? __ddiv_rn(num, len2) : 0.0;
    t = fmin(fmax(t, 0.0), 1.0);
    const double qx = __dadd_rn(a.x, __dmul_rn(t, dx)), qy = __dadd_rn(a.y, __dmul_rn(t, dy));
    const double ex = __dsub_rn(p.x, qx), ey = __dsub_rn(p.y, qy);
    return __dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)) <= dd;
}

__global__ void __launch_bounds__(NEAR_THREADS) merge_near_kernel(Set S, const int32_t* __restrict__ pairs, int64_t n, double d, double pad,
                                                                  uint8_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const double dd = __dmul_rn(d, d);
    const int64_t warps = static_cast<int64_t>(gridDim.x) * (NEAR_THREADS / 32);
    for (int64_t w = (static_cast<int64_t>(blockIdx.x) * NEAR_THREADS + threadIdx.x) >> 5; w < n; w += warps) {
        int a = pairs[2 * w], b = pairs[2 * w + 1];
        if (S.fv[b + 1] - S.fv[b] > S.fv[a + 1] - S.fv[a]) {  // lanes stride over the larger feature's edges
            const int t = a;
            a = b;
            b = t;
        }
        const int64_t s0 = S.fv[a], s1 = S.fv[a + 1], t0 = S.fv[b], t1 = S.fv[b + 1];
        const double* tb = S.box + 4 * static_cast<int64_t>(b);
        bool found = false;
        for (int64_t base = s0; base < s1 && !found; base += 32) {
            bool hit = false;
            const int64_t v = base + lane;
            if (v < s1) {
                const double2 c = S.v[v], g = S.v[S.next[v]];
                const bool meets = !(fmax(c.x, g.x) + pad < tb[0] || tb[2] < fmin(c.x, g.x) - pad || fmax(c.y, g.y) + pad < tb[1] || tb[3] < fmin(c.y, g.y) - pad);
                if (meets)
                    for (int64_t u = t0; u < t1 && !hit; ++u) {
                        const double2 e = S.v[u], f = S.v[S.next[u]];
                        hit = within(c, e, f, dd) || within(e, c, g, dd);
                    }
            }
            found = __any_sync(FULL, hit);
        }
        if (lane == 0) out[w] = found ? 1 : 0;
    }
}

__device__ __forceinline__ int find_root(int32_t* parent, int x) {
    int p = static_cast<int>(atomicAdd(reinterpret_cast<unsigned*>(&parent[x]), 0u));
    while (p != x) {
        x = p;
        p = static_cast<int>(atomicAdd(reinterpret_cast<unsigned*>(&parent[x]), 0u));
    }
    return x;
}

__global__ void __launch_bounds__(UF_THREADS) uf_init_kernel(int32_t* __restrict__ parent, int32_t n) {
    for (int i = blockIdx.x * UF_THREADS + threadIdx.x; i < n; i += gridDim.x * UF_THREADS) parent[i] = i;
}

__global__ void __launch_bounds__(UF_THREADS) uf_hook_kernel(const int32_t* __restrict__ pairs, const uint8_t* __restrict__ linked, int64_t m, int32_t* parent) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * UF_THREADS;
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * UF_THREADS + threadIdx.x; k < m; k += stride) {
        if (!linked[k]) continue;
        int a = pairs[2 * k], b = pairs[2 * k + 1];
        while (true) {
            a = find_root(parent, a);
            b = find_root(parent, b);
            if (a == b) break;
            const int hi = max(a, b), lo = min(a, b);
            if (atomicCAS(&parent[hi], hi, lo) == hi) break;  // hi was still a root: hooked
            a = hi;
            b = lo;
        }
    }
}

__global__ void __launch_bounds__(UF_THREADS) uf_jump_kernel(int32_t* parent, int32_t n, int32_t* __restrict__ labels) {
    for (int i = blockIdx.x * UF_THREADS + threadIdx.x; i < n; i += gridDim.x * UF_THREADS) labels[i] = find_root(parent, i);
}

// ---- fill ----

// one CTA per band: bands[3 * b] = (component, first row, rows); grids[2 * c] = (W, H)
__global__ void __launch_bounds__(FILL_THREADS, 1) merge_fill_kernel(const double* __restrict__ vertices, const int64_t* __restrict__ ring_offsets,
                                                                  const int32_t* __restrict__ poly_rings, const int32_t* __restrict__ comp_poly_offsets,
                                                                  const int32_t* __restrict__ comp_polys, const double* __restrict__ transforms,
                                                                  const int64_t* __restrict__ grids, const int64_t* __restrict__ bitmap_offsets,
                                                                  const int32_t* __restrict__ bands, uint32_t* __restrict__ bitmap) {
    extern __shared__ __align__(16) uint32_t tog[];
    const int c = bands[3 * blockIdx.x], band_row = bands[3 * blockIdx.x + 1], rows = bands[3 * blockIdx.x + 2];
    const int64_t W = grids[2 * c];
    const int words = static_cast<int>((W + 31) >> 5);
    uint32_t* out = bitmap + bitmap_offsets[c] + static_cast<int64_t>(band_row) * words;
    for (int i = threadIdx.x; i < rows * words; i += blockDim.x) tog[i] = 0u;
    fill_band(
        vertices, ring_offsets, poly_rings, comp_poly_offsets[c], comp_poly_offsets[c + 1], [&](int k) { return comp_polys[k]; }, transforms[4 * c + 0],
        transforms[4 * c + 1], transforms[4 * c + 2], transforms[4 * c + 3], W, band_row, rows, tog,
        [&](int r, int w, uint32_t bits) {
            if (bits) out[static_cast<int64_t>(r) * words + w] |= bits;
        });
}

// ---- closing ----

__device__ __forceinline__ int disk_span(int K, int i) {  // floor(sqrt(K^2 - i^2))
    const int r2 = K * K - i * i;
    int s = 0;
    while ((s + 1) * (s + 1) <= r2) ++s;
    return s;
}

// OR (dilate) or AND (erode) of the word `cur` over horizontal offsets -s .. s, with its neighbours prev and next
__device__ __forceinline__ uint32_t run(uint32_t prev, uint32_t cur, uint32_t next, int s, bool dilate) {
    uint32_t h = cur;
    for (int j = 1; j <= s; ++j) {
        const uint32_t l = __funnelshift_l(prev, cur, j), r = __funnelshift_r(cur, next, j);
        h = dilate ? (h | l | r) : (h & l & r);
    }
    return h;
}

// one CTA per tile: tiles[3 * t] = (component, first row, first word)
__global__ void __launch_bounds__(CLOSE_THREADS) merge_close_kernel(const uint32_t* __restrict__ fill, const int64_t* __restrict__ grids,
                                                                    const int64_t* __restrict__ bitmap_offsets, const int32_t* __restrict__ tiles, int K,
                                                                    uint32_t* __restrict__ out, unsigned long long* __restrict__ counts) {
    __shared__ uint32_t in[IN_ROWS][IN_WORDS];
    __shared__ uint32_t dil[DIL_ROWS][DIL_WORDS];
    const int c = tiles[3 * blockIdx.x];
    const int64_t row0 = tiles[3 * blockIdx.x + 1], word0 = tiles[3 * blockIdx.x + 2];
    const int64_t W = grids[2 * c], H = grids[2 * c + 1];
    const int64_t words = (W + 31) >> 5;
    const uint32_t tail = (W & 31) ? (1u << (W & 31)) - 1u : FULL;
    const uint32_t* src = fill + bitmap_offsets[c];
    const int in_rows = TILE_ROWS + 4 * K, dil_rows = TILE_ROWS + 2 * K;
    // stage rows row0 - 2K .. and words word0 - 2 ..; outside the grid is 0
    for (int i = threadIdx.x; i < in_rows * IN_WORDS; i += CLOSE_THREADS) {
        const int r = i / IN_WORDS, w = i % IN_WORDS;
        const int64_t gr = row0 - 2 * K + r, gw = word0 - 2 + w;
        in[r][w] = (gr >= 0 && gr < H && gw >= 0 && gw < words) ? src[gr * words + gw] : 0u;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < dil_rows * DIL_WORDS; i += CLOSE_THREADS) {
        const int r = i / DIL_WORDS, w = i % DIL_WORDS;  // dil[r][w] is grid row row0 - K + r, word word0 - 1 + w
        const int64_t gr = row0 - K + r, gw = word0 - 1 + w;
        uint32_t acc = 0u;
        if (gr >= 0 && gr < H && gw >= 0 && gw < words) {
            for (int di = -K; di <= K; ++di) {
                const uint32_t* row = in[r + K + di];
                acc |= run(row[w], row[w + 1], row[w + 2], disk_span(K, di), true);
            }
            if (gw == words - 1) acc &= tail;
        }
        dil[r][w] = acc;
    }
    __syncthreads();
    unsigned long long n = 0;
    for (int i = threadIdx.x; i < TILE_ROWS * TILE_WORDS; i += CLOSE_THREADS) {
        const int r = i / TILE_WORDS, w = i % TILE_WORDS;
        const int64_t gr = row0 + r, gw = word0 + w;
        if (gr >= H || gw >= words) continue;
        uint32_t acc = FULL;
        for (int di = -K; di <= K; ++di) {
            const uint32_t* row = dil[r + K + di];
            acc &= run(row[w], row[w + 1], row[w + 2], disk_span(K, di), false);
        }
        if (gw == words - 1) acc &= tail;
        out[bitmap_offsets[c] + gr * words + gw] = acc;
        n += __popc(acc);
    }
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(FULL, n, o);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(&counts[c], n);
}

}  // namespace

extern "C" int rsb_merge_near(const RsbShapes* shapes, const int32_t* pairs, int64_t num_pairs, double threshold, uint8_t* out, void* stream) {
    if (!shapes || !shapes->vertices || !shapes->next || !shapes->feature_vertices || !shapes->boxes || shapes->num_features < 1 || shapes->num_vertices < 1)
        return set_error(RSB_E_INVALID, "merge_near: shapes need at least one feature, one vertex and their arrays");
    if ((reinterpret_cast<uintptr_t>(shapes->vertices) & 15) != 0) return set_error(RSB_E_INVALID, "merge_near: vertices must be 16-byte aligned");
    if (num_pairs < 0 || (num_pairs > 0 && (!pairs || !out))) return set_error(RSB_E_INVALID, "merge_near: num_pairs=%lld with null pairs or out", (long long)num_pairs);
    if (!(threshold > 0.0) || !(threshold < 1e300)) return set_error(RSB_E_INVALID, "merge_near: threshold %g (need a positive finite distance)", threshold);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    if (num_pairs == 0) return RSB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Set S{reinterpret_cast<const double2*>(shapes->vertices), shapes->next, shapes->feature_vertices, shapes->boxes};
    const double pad = threshold * (1.0 + 1e-6) + 1e-3;  // wider than any rounding of the distance test
    const int64_t blocks = std::min<int64_t>((num_pairs + NEAR_THREADS / 32 - 1) / (NEAR_THREADS / 32), 64 * num_sms());
    merge_near_kernel<<<static_cast<unsigned>(blocks), NEAR_THREADS, 0, st>>>(S, pairs, num_pairs, threshold, pad, out);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "merge_near launch");
}

extern "C" int rsb_merge_components(const int32_t* pairs, const uint8_t* linked, int64_t num_pairs, int32_t n, int32_t* parent, int32_t* labels, void* stream) {
    if (n < 1 || !parent || !labels) return set_error(RSB_E_INVALID, "merge_components: n=%d (need n >= 1) or null parent / labels", n);
    if (num_pairs < 0 || (num_pairs > 0 && (!pairs || !linked))) return set_error(RSB_E_INVALID, "merge_components: num_pairs=%lld with null arrays", (long long)num_pairs);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned nb = static_cast<unsigned>(std::min<int64_t>((n + UF_THREADS - 1) / UF_THREADS, 16 * num_sms()));
    uf_init_kernel<<<nb, UF_THREADS, 0, st>>>(parent, n);
    if (num_pairs > 0) {
        const unsigned pb = static_cast<unsigned>(std::min<int64_t>((num_pairs + UF_THREADS - 1) / UF_THREADS, 16 * num_sms()));
        uf_hook_kernel<<<pb, UF_THREADS, 0, st>>>(pairs, linked, num_pairs, parent);
    }
    uf_jump_kernel<<<nb, UF_THREADS, 0, st>>>(parent, n, labels);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "merge_components launch");
}

extern "C" int rsb_merge_fill(const double* vertices, const int64_t* ring_offsets, const int32_t* poly_rings, int32_t num_polys,
                              const int32_t* comp_poly_offsets, const int32_t* comp_polys, const double* transforms, const int64_t* grids,
                              const int64_t* bitmap_offsets, int32_t C, const int32_t* bands, int32_t num_bands, int32_t band_rows, int32_t max_words,
                              uint32_t* bitmap, int64_t bitmap_words, void* stream) {
    if (!comp_poly_offsets || !comp_polys || !transforms || !grids || !bitmap_offsets || !bands || !bitmap)
        return set_error(RSB_E_INVALID, "merge_fill: null pointer");
    if (C < 1 || num_polys < 1 || !vertices || !ring_offsets || !poly_rings)
        return set_error(RSB_E_INVALID, "merge_fill: C=%d num_polys=%d (need at least one component and one polygon)", C, num_polys);
    if ((reinterpret_cast<uintptr_t>(vertices) & 15) != 0) return set_error(RSB_E_INVALID, "merge_fill: vertices must be 16-byte aligned");
    if (num_bands < 1 || bitmap_words < 1) return set_error(RSB_E_INVALID, "merge_fill: num_bands=%d bitmap_words=%lld", num_bands, (long long)bitmap_words);
    if (max_words < 1 || max_words > RSB_COVER_MAX_WIDTH / 32 || band_rows < 1 || static_cast<int64_t>(band_rows) * max_words > RSB_COVER_MAX_WIDTH / 32)
        return set_error(RSB_E_INVALID, "merge_fill: band_rows=%d x max_words=%d (need at most %d shared-memory words)", band_rows, max_words,
                         RSB_COVER_MAX_WIDTH / 32);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = static_cast<size_t>(band_rows) * max_words * 4;
    cudaError_t e = cudaFuncSetAttribute(merge_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return set_cuda_error(e, "merge_fill: shared memory attribute");
    e = cudaMemsetAsync(bitmap, 0, static_cast<size_t>(bitmap_words) * 4, st);
    if (e != cudaSuccess) return set_cuda_error(e, "merge_fill: clear");
    merge_fill_kernel<<<static_cast<unsigned>(num_bands), FILL_THREADS, smem, st>>>(vertices, ring_offsets, poly_rings, comp_poly_offsets, comp_polys,
                                                                                    transforms, grids, bitmap_offsets, bands, bitmap);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "merge_fill launch");
}

extern "C" int rsb_merge_close(const uint32_t* fill, const int64_t* grids, const int64_t* bitmap_offsets, int32_t C, const int32_t* tiles, int32_t num_tiles,
                               int32_t radius, uint32_t* out, int64_t* counts, void* stream) {
    if (!fill || !grids || !bitmap_offsets || !tiles || !out || !counts) return set_error(RSB_E_INVALID, "merge_close: null pointer");
    if (C < 1 || num_tiles < 1) return set_error(RSB_E_INVALID, "merge_close: C=%d num_tiles=%d", C, num_tiles);
    if (radius < 1 || radius > RSB_MERGE_MAX_RADIUS) return set_error(RSB_E_INVALID, "merge_close: radius %d (need 1..%d)", radius, RSB_MERGE_MAX_RADIUS);
    if (fill == out) return set_error(RSB_E_INVALID, "merge_close: out must not alias fill");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(counts, 0, static_cast<size_t>(C) * 8, st);
    if (e != cudaSuccess) return set_cuda_error(e, "merge_close: clear counts");
    merge_close_kernel<<<static_cast<unsigned>(num_tiles), CLOSE_THREADS, 0, st>>>(fill, grids, bitmap_offsets, tiles, radius, out,
                                                                                   reinterpret_cast<unsigned long long*>(counts));
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "merge_close launch");
}
