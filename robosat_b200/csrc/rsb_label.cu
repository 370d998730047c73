// Connected components of binary planes for `rs features --type building` (DESIGN.md §8): union-find labels, per-component areas
// and border flags, and the speck-drop / hole-fill passes of the building rule.
//
// Labels are image-local linear indices y * W + x, and the root of a component is its smallest pixel index, so labels do not
// depend on the launch shape or on the order in which threads run. Every parent pointer is smaller than its child (values only
// ever go down, by atomicMin, starting from the pixel's own index), so the root of a tree is its smallest member and merging two
// trees under the smaller root keeps that true.
//
// label_local_kernel: one CTA per 32 x 32 tile of one image. The tile's foreground bits are ballots in shared memory; each pixel
// unites with its earlier neighbours inside the tile (left, up, and for 8-connectivity up-left and up-right) on a shared-memory
// parent array, the trees are flattened, and the tile-local component sizes and border flags are summed with shared atomics. Tile
// row-major order agrees with image row-major order, so the tile-local root is the component's smallest pixel within the tile.
// Every pixel gets its tile root's image index (or -1); the tile root alone carries its tile-local area and border bit in stats.
//
// label_merge_kernel: one thread per pixel along a tile boundary unites the pairs that cross it, in global memory, hooking the
// larger root under the smaller with atomicMin (rsb_merge_components hooks the same way).
//
// label_finish_kernel: each tile root points straight at its root and, when it is no longer a root itself, adds its area and
// border bit to its root's stats with int32 atomics (one atomic per tile piece of a component, not one per pixel). Every other
// pixel still points at its tile root, so the passes after it find a pixel's root in two reads, without walking the trees.

#include <stdint.h>

#include <algorithm>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int TILE = 32;             // a CTA labels TILE x TILE pixels; lane x owns column x
constexpr int LOCAL_THREADS = 256;   // 8 warps, each takes rows warp, warp + 8, ...
constexpr int PASS_THREADS = 256;
constexpr int32_t BORDER = 1 << 30;  // stats bit: the component touches the image border
constexpr int32_t AREA = BORDER - 1; // stats bits: the component's area (H * W <= 2^26)

__device__ __forceinline__ int find_root(const volatile int32_t* L, int i) {
    int p = L[i];
    while (p != i) {
        i = p;
        p = L[i];
    }
    return i;
}

// joins the trees of a and b: the larger root is hooked under the smaller; a hook that finds its target no longer a root
// (another thread hooked it first) retries from the parent it found
__device__ __forceinline__ void unite(volatile int32_t* L, int a, int b) {
    while (true) {
        a = find_root(L, a);
        b = find_root(L, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(const_cast<int32_t*>(&L[b]), a);
        if (old == b) return;
        b = old;
    }
}

__global__ void __launch_bounds__(LOCAL_THREADS) label_local_kernel(const uint8_t* __restrict__ planes, int64_t image_stride, int H, int W, int value,
                                                                    int conn8, int tiles_x, int tiles_per_image, int32_t* __restrict__ labels,
                                                                    int32_t* __restrict__ stats) {
    __shared__ int32_t parent[TILE * TILE];
    __shared__ int32_t cnt[TILE * TILE];
    __shared__ uint32_t bits[TILE];
    const int n = blockIdx.x / tiles_per_image, t = blockIdx.x % tiles_per_image;
    const int x0 = (t % tiles_x) * TILE, y0 = (t / tiles_x) * TILE;
    const int lx = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NW = LOCAL_THREADS / 32;
    const uint8_t* img = planes + static_cast<int64_t>(n) * image_stride;
    const int x = x0 + lx;

    for (int ly = warp; ly < TILE; ly += NW) {
        const int y = y0 + ly, i = ly * TILE + lx;
        const bool fg = x < W && y < H && img[static_cast<int64_t>(y) * W + x] == value;
        const uint32_t b = __ballot_sync(FULL, fg);
        if (lx == 0) bits[ly] = b;
        parent[i] = fg ? i : -1;
        cnt[i] = 0;
    }
    __syncthreads();

    volatile int32_t* P = parent;
    for (int ly = warp; ly < TILE; ly += NW) {
        const int i = ly * TILE + lx;
        if (!((bits[ly] >> lx) & 1u)) continue;
        if (lx > 0 && ((bits[ly] >> (lx - 1)) & 1u)) unite(P, i, i - 1);
        if (ly > 0) {
            const uint32_t up = bits[ly - 1];
            if ((up >> lx) & 1u) unite(P, i, i - TILE);
            if (conn8) {
                if (lx > 0 && ((up >> (lx - 1)) & 1u)) unite(P, i, i - TILE - 1);
                if (lx < TILE - 1 && ((up >> (lx + 1)) & 1u)) unite(P, i, i - TILE + 1);
            }
        }
    }
    __syncthreads();

    for (int ly = warp; ly < TILE; ly += NW) {
        const int i = ly * TILE + lx, y = y0 + ly;
        if (!((bits[ly] >> lx) & 1u)) continue;
        const int r = find_root(P, i);
        P[i] = r;
        atomicAdd(&cnt[r], 1);
        if (x == 0 || y == 0 || x == W - 1 || y == H - 1) atomicOr(&cnt[r], BORDER);
    }
    __syncthreads();

    if (x >= W) return;
    const int64_t base = static_cast<int64_t>(n) * H * W;
    for (int ly = warp; ly < TILE && y0 + ly < H; ly += NW) {
        const int i = ly * TILE + lx;
        const int64_t g = base + static_cast<int64_t>(y0 + ly) * W + x;
        const int r = parent[i];
        labels[g] = r < 0 ? -1 : (y0 + r / TILE) * W + x0 + r % TILE;
        stats[g] = r == i ? cnt[i] : 0;
    }
}

// pairs across the tile boundaries: nv = tiles_x - 1 column boundaries of H pixels, then nh = tiles_y - 1 row boundaries of W
__global__ void __launch_bounds__(PASS_THREADS) label_merge_kernel(int32_t* labels, int H, int W, int conn8, int nv, int nh, int64_t total) {
    const int64_t per_image = static_cast<int64_t>(nv) * H + static_cast<int64_t>(nh) * W;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * PASS_THREADS;
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * PASS_THREADS + threadIdx.x; k < total; k += stride) {
        const int64_t n = k / per_image;
        int64_t j = k % per_image;
        volatile int32_t* L = labels + n * H * W;
        if (j < static_cast<int64_t>(nv) * H) {  // column c - 1 | c
            const int c = static_cast<int>(j / H + 1) * TILE, y = static_cast<int>(j % H);
            const int p = y * W + c, q = p - 1;
            const bool fp = L[p] >= 0, fq = L[q] >= 0;
            if (fp && fq) unite(L, p, q);
            if (conn8 && y > 0) {
                if (fp && L[q - W] >= 0) unite(L, p, q - W);
                if (fq && L[p - W] >= 0) unite(L, q, p - W);
            }
        } else {  // row r - 1 | r
            j -= static_cast<int64_t>(nv) * H;
            const int r = static_cast<int>(j / W + 1) * TILE, x = static_cast<int>(j % W);
            const int p = r * W + x, u = p - W;
            if (L[p] < 0) continue;
            if (L[u] >= 0) unite(L, p, u);
            if (conn8) {
                if (x > 0 && L[u - 1] >= 0) unite(L, p, u - 1);
                if (x < W - 1 && L[u + 1] >= 0) unite(L, p, u + 1);
            }
        }
    }
}

// blockIdx.y = image; only tile roots work: each points itself at its root and, when hooked, adds its area and border bit there.
// Every other pixel still points at its tile root, so root_of() below finds any pixel's root in two reads.
__global__ void __launch_bounds__(PASS_THREADS) label_finish_kernel(int32_t* labels, int32_t* stats, int HW) {
    const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
    if (i >= HW) return;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * HW;
    const int32_t s = stats[base + i];
    if (s == 0) return;  // not a tile root
    volatile int32_t* L = labels + base;
    const int r = find_root(L, i);
    if (r == i) return;
    L[i] = r;
    atomicAdd(&stats[base + r], s & AREA);
    if (s & BORDER) atomicOr(&stats[base + r], BORDER);
}

// the root of pixel i of an image after label_finish_kernel, -1 off the plane
__device__ __forceinline__ int root_of(const int32_t* L, int i) {
    const int t = L[i];
    return t < 0 ? -1 : L[t];
}

// labels[i] = the root of i, areas[i] = the area of i's component (0 off the plane), in place over the stats: a thread rewrites
// only its own pixel, tile roots keep their value, and only roots' stats are read, each keeping its area
__global__ void __launch_bounds__(PASS_THREADS) label_areas_kernel(int32_t* labels, int32_t* stats, int HW) {
    const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
    if (i >= HW) return;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * HW;
    const int l = root_of(labels + base, i);
    labels[base + i] = l;
    stats[base + i] = l < 0 ? 0 : (stats[base + l] & AREA);
}

// out = opened pixels whose 8-connected component has at least min_area pixels
__global__ void __launch_bounds__(PASS_THREADS) drop_specks_kernel(const int32_t* labels, const int32_t* __restrict__ stats, int HW,
                                                                   int min_area, uint8_t* __restrict__ out) {
    const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
    if (i >= HW) return;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * HW;
    const int l = root_of(labels + base, i);
    out[base + i] = (l >= 0 && (stats[base + l] & AREA) >= min_area) ? 1 : 0;
}

// labels / stats of out's background (4-connected): out |= background components that miss the border and have < min_hole_area
// pixels; counts[n] += foreground of the result
__global__ void __launch_bounds__(PASS_THREADS) fill_holes_kernel(const int32_t* labels, const int32_t* __restrict__ stats, int HW,
                                                                  int min_hole_area, uint8_t* __restrict__ out, int32_t* __restrict__ counts) {
    const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
    const int64_t base = static_cast<int64_t>(blockIdx.y) * HW;
    int set = 0;
    if (i < HW) {
        const int l = root_of(labels + base, i);
        if (l < 0) {
            set = 1;
        } else {
            const int32_t s = stats[base + l];
            set = !(s & BORDER) && (s & AREA) < min_hole_area;
            if (set) out[base + i] = 1;
        }
    }
    int c = __popc(__ballot_sync(FULL, set));
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&counts[blockIdx.y], c);
}

struct Shape {
    int tiles_x, tiles_per_image, nv, nh;
    int64_t local_blocks, merge_total;
    dim3 pass_grid;
};

Shape shape_of(int N, int H, int W) {
    Shape s;
    s.tiles_x = (W + TILE - 1) / TILE;
    const int tiles_y = (H + TILE - 1) / TILE;
    s.tiles_per_image = s.tiles_x * tiles_y;
    s.nv = s.tiles_x - 1;
    s.nh = tiles_y - 1;
    s.local_blocks = static_cast<int64_t>(N) * s.tiles_per_image;
    s.merge_total = static_cast<int64_t>(N) * (static_cast<int64_t>(s.nv) * H + static_cast<int64_t>(s.nh) * W);
    s.pass_grid = dim3(static_cast<unsigned>((H * W + PASS_THREADS - 1) / PASS_THREADS), static_cast<unsigned>(N));
    return s;
}

// labels + stats of (plane == value); the caller has validated the arguments
void label(const uint8_t* planes, int64_t image_stride, int N, int H, int W, int value, int conn8, const Shape& s, int32_t* labels, int32_t* stats,
           cudaStream_t st) {
    label_local_kernel<<<static_cast<unsigned>(s.local_blocks), LOCAL_THREADS, 0, st>>>(planes, image_stride, H, W, value, conn8, s.tiles_x,
                                                                                       s.tiles_per_image, labels, stats);
    if (s.merge_total > 0) {
        const int64_t blocks = std::min<int64_t>((s.merge_total + PASS_THREADS - 1) / PASS_THREADS, 64 * static_cast<int64_t>(num_sms()));
        label_merge_kernel<<<static_cast<unsigned>(blocks), PASS_THREADS, 0, st>>>(labels, H, W, conn8, s.nv, s.nh, s.merge_total);
    }
    label_finish_kernel<<<s.pass_grid, PASS_THREADS, 0, st>>>(labels, stats, H * W);
}

int check_shape(const char* what, int64_t image_stride, int N, int H, int W) {
    if (N < 1 || N > 65535 || H < 1 || W < 1 || H > RSB_LABEL_MAX_SIZE || W > RSB_LABEL_MAX_SIZE)
        return set_error(RSB_E_UNSUPPORTED, "%s: N=%d H=%d W=%d (need 1 <= N <= 65535 and 1 <= H, W <= %d)", what, N, H, W, RSB_LABEL_MAX_SIZE);
    if (image_stride < static_cast<int64_t>(H) * W)
        return set_error(RSB_E_INVALID, "%s: image_stride %lld < H*W = %lld", what, (long long)image_stride, (long long)H * W);
    return RSB_OK;
}

}  // namespace

extern "C" int rsb_label_components(const uint8_t* planes, int64_t image_stride, int32_t N, int32_t H, int32_t W, int32_t value, int32_t connectivity,
                                    int32_t* labels, int32_t* areas, void* stream) {
    if (!planes || !labels || !areas) return set_error(RSB_E_INVALID, "label_components: null pointer");
    const int rc = check_shape("label_components", image_stride, N, H, W);
    if (rc != RSB_OK) return rc;
    if (value < 0 || value > 255) return set_error(RSB_E_INVALID, "label_components: value %d is not a uint8", value);
    if (connectivity != 4 && connectivity != 8) return set_error(RSB_E_INVALID, "label_components: connectivity %d (need 4 or 8)", connectivity);
    if (labels == areas) return set_error(RSB_E_INVALID, "label_components: labels and areas must not alias");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Shape s = shape_of(N, H, W);
    label(planes, image_stride, N, H, W, value, connectivity == 8, s, labels, areas, st);
    label_areas_kernel<<<s.pass_grid, PASS_THREADS, 0, st>>>(labels, areas, H * W);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "label_components launch");
}

extern "C" int rsb_building_clean(const uint8_t* opened, int64_t image_stride, int32_t N, int32_t H, int32_t W, int32_t min_area, int32_t min_hole_area,
                                  int32_t* labels, int32_t* stats, uint8_t* out, int32_t* fg_counts, void* stream) {
    if (!opened || !labels || !stats || !out || !fg_counts) return set_error(RSB_E_INVALID, "building_clean: null pointer");
    const int rc = check_shape("building_clean", image_stride, N, H, W);
    if (rc != RSB_OK) return rc;
    if (min_area < 0 || min_hole_area < 0) return set_error(RSB_E_INVALID, "building_clean: min_area %d / min_hole_area %d (need >= 0)", min_area, min_hole_area);
    if (labels == stats) return set_error(RSB_E_INVALID, "building_clean: labels and stats must not alias");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Shape s = shape_of(N, H, W);
    cudaError_t e = cudaMemsetAsync(fg_counts, 0, sizeof(int32_t) * N, st);
    if (e != cudaSuccess) return set_cuda_error(e, "building_clean: clear fg_counts");
    label(opened, image_stride, N, H, W, 1, 1, s, labels, stats, st);
    drop_specks_kernel<<<s.pass_grid, PASS_THREADS, 0, st>>>(labels, stats, H * W, min_area, out);
    label(out, static_cast<int64_t>(H) * W, N, H, W, 0, 0, s, labels, stats, st);
    fill_holes_kernel<<<s.pass_grid, PASS_THREADS, 0, st>>>(labels, stats, H * W, min_hole_area, out, fg_counts);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "building_clean launch");
}
