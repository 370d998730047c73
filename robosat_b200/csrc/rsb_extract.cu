// `rs extract` (robosat/tools/extract.py, robosat/osm/*.py) on the device: DenseNodes decode, the node-location join and the ring
// validity check (DESIGN.md §8).
//
// rsb_pbf_dense_nodes: one CTA per DenseNodes group. Each of the packed id / lat / lon fields is read in tiles of DENSE_THREADS
// bytes, one byte per thread, each tile starting at a value boundary. A byte with a clear continuation bit ends a value; ballots
// and a CTA prefix give every terminator its value's rank, and its thread assembles the value from the (at most 10) bytes before
// it in shared memory. The zigzag-decoded deltas then go through an int64 CTA-wide inclusive scan, plus the running sum carried
// from the previous tile, so a group of any size straddles warps and tiles freely. The next tile starts after the tile's last
// terminator. lat / lon are converted to 1e-7 degree units in the same pass.
//
// rsb_extract_locate: one thread per decoded node, binary search of its biased id in the sorted unique refs; atomicMax of its
// global ordinal into the slot, then a second launch writes the location where that ordinal won, so the later node of a
// duplicated id wins on every run. rsb_extract_gather: one thread per way ref.
//
// rsb_extract_valid: one warp per ring compacts it (closing vertex and consecutive repeats dropped), checks >= 3 distinct positions
// and a non-zero doubled area (int128 sum), and for rings of at most RSB_EXTRACT_WARP_RING vertices tests every pair of edges.
// Longer rings are tested by a second kernel in 64 x 64 edge tiles, one CTA per tile. Orientations are exact: coordinate
// differences take 33 bits, so the cross products are formed in __int128.

#include <stdint.h>

#include <algorithm>

#include "../../include/rsb200.h"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int DENSE_THREADS = 256;
constexpr int DENSE_WARPS = DENSE_THREADS / 32;
constexpr int JOIN_THREADS = 256;
constexpr int RING_THREADS = 128;
constexpr int PAIR_TILE = 64;
constexpr int PAIR_THREADS = 256;
constexpr int64_t LON_LIMIT = 1800000000LL, LAT_LIMIT = 900000000LL;

__device__ __forceinline__ int32_t to_fixed(int64_t v, int64_t granularity, int64_t offset, int64_t limit) {
    const int64_t f = (offset + granularity * v) / 100;
    return (f < -limit || f > limit) ? INT32_MIN : static_cast<int32_t>(f);
}

__device__ __forceinline__ int64_t warp_inclusive_sum(int64_t v, int lane) {
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t u = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += u;
    }
    return v;
}

// field 0: id -> ids; 1: lat -> xy[.][1]; 2: lon -> xy[.][0]
__global__ void __launch_bounds__(DENSE_THREADS) dense_nodes_kernel(const uint8_t* __restrict__ blocks, const int64_t* __restrict__ block_offsets,
                                                                    const int64_t* __restrict__ segs, int64_t* __restrict__ ids, int32_t* __restrict__ xy,
                                                                    int32_t* __restrict__ status) {
    __shared__ uint8_t bytes[DENSE_THREADS];
    __shared__ int64_t vals[DENSE_THREADS];
    __shared__ int warp_count[DENSE_WARPS];
    __shared__ int64_t warp_sum[DENSE_WARPS];
    __shared__ int s_last;
    const int64_t* s = segs + static_cast<int64_t>(blockIdx.x) * RSB_PBF_SEG_FIELDS;
    if (s[RSB_PBF_SEG_KIND] != 0) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint8_t* base = blocks + block_offsets[s[RSB_PBF_SEG_BLOCK]];
    const int64_t count = s[RSB_PBF_SEG_COUNT], out0 = s[RSB_PBF_SEG_OUT_FIRST], gran = s[RSB_PBF_SEG_GRANULARITY];
    for (int field = 0; field < 3; ++field) {
        const int64_t off = s[RSB_PBF_SEG_ID_OFF + 2 * field], len = s[RSB_PBF_SEG_ID_LEN + 2 * field];
        const int64_t offset = field == 1 ? s[RSB_PBF_SEG_LAT_OFFSET] : s[RSB_PBF_SEG_LON_OFFSET];
        const int64_t limit = field == 1 ? LAT_LIMIT : LON_LIMIT;
        int64_t pos = 0, carry = 0, rank_base = 0;
        bool bad = false;
        while (pos < len) {
            const bool in = pos + tid < len;
            const uint8_t b = in ? base[off + pos + tid] : 0x80;
            bytes[tid] = b;
            const bool term = in && !(b & 0x80);
            const unsigned ballot = __ballot_sync(FULL, term);
            if (lane == 0) warp_count[warp] = __popc(ballot);
            if (tid == 0) s_last = -1;
            __syncthreads();
            if (term) atomicMax(&s_last, tid);
            int before = 0, nv = 0;
            for (int w = 0; w < DENSE_WARPS; ++w) {
                before += w < warp ? warp_count[w] : 0;
                nv += warp_count[w];
            }
            const int rank = before + __popc(ballot & ((1u << lane) - 1));
            if (term) {
                int start = tid;
                while (start > 0 && (bytes[start - 1] & 0x80) && tid - start < 10) --start;
                if (tid - start >= 10) {
                    bad = true;
                } else {
                    uint64_t v = 0;
                    for (int k = start; k <= tid; ++k) v |= static_cast<uint64_t>(bytes[k] & 0x7f) << (7 * (k - start));
                    vals[rank] = static_cast<int64_t>(v >> 1) ^ -static_cast<int64_t>(v & 1);
                }
            }
            __syncthreads();
            const int last = s_last;
            if (last < 0) {  // no terminator in a whole tile: a varint longer than 10 bytes
                bad = true;
                break;
            }
            // inclusive scan of vals[0 .. nv) plus the carry
            int64_t v = tid < nv ? vals[tid] : 0;
            v = warp_inclusive_sum(v, lane);
            if (lane == 31) warp_sum[warp] = v;
            __syncthreads();
            int64_t prefix = carry, total = carry;
            for (int w = 0; w < DENSE_WARPS; ++w) {
                prefix += w < warp ? warp_sum[w] : 0;
                total += warp_sum[w];
            }
            v += prefix;
            if (tid < nv) {
                const int64_t o = rank_base + tid;
                if (o < count) {
                    if (field == 0) ids[out0 + o] = v;
                    else xy[2 * (out0 + o) + (field == 1 ? 1 : 0)] = to_fixed(v, gran, offset, limit);
                }
            }
            carry = total;
            rank_base += nv;
            pos += last + 1;
            __syncthreads();  // bytes / vals / warp sums are rewritten by the next tile
        }
        if (__syncthreads_or(bad) || rank_base != count) {
            if (tid == 0) atomicOr(status, 1);
            return;
        }
    }
}

__device__ __forceinline__ int64_t find_key(const uint64_t* __restrict__ keys, int64_t n, uint64_t k) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && keys[lo] == k ? lo : -1;
}

__device__ __forceinline__ uint64_t bias(int64_t id) { return static_cast<uint64_t>(id) ^ 0x8000000000000000ull; }

__global__ void __launch_bounds__(JOIN_THREADS) locate_mark_kernel(const int64_t* __restrict__ ids, int64_t n, int64_t ordinal_base,
                                                                   const uint64_t* __restrict__ keys, int64_t nk, unsigned long long* best) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * JOIN_THREADS;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * JOIN_THREADS + threadIdx.x; i < n; i += stride) {
        const int64_t k = find_key(keys, nk, bias(ids[i]));
        if (k >= 0) atomicMax(&best[k], static_cast<unsigned long long>(ordinal_base + i + 1));
    }
}

__global__ void __launch_bounds__(JOIN_THREADS) locate_write_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ xy, int64_t n,
                                                                    int64_t ordinal_base, const uint64_t* __restrict__ keys, int64_t nk,
                                                                    const unsigned long long* __restrict__ best, int32_t* __restrict__ loc) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * JOIN_THREADS;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * JOIN_THREADS + threadIdx.x; i < n; i += stride) {
        const int64_t k = find_key(keys, nk, bias(ids[i]));
        if (k >= 0 && best[k] == static_cast<unsigned long long>(ordinal_base + i + 1)) {
            loc[2 * k] = xy[2 * i];
            loc[2 * k + 1] = xy[2 * i + 1];
        }
    }
}

__global__ void __launch_bounds__(JOIN_THREADS) gather_kernel(const int64_t* __restrict__ refs, const int32_t* __restrict__ ref_way, int64_t n,
                                                              const uint64_t* __restrict__ keys, int64_t nk, const unsigned long long* __restrict__ best,
                                                              const int32_t* __restrict__ loc, int32_t* __restrict__ verts, int32_t* flags) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * JOIN_THREADS;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * JOIN_THREADS + threadIdx.x; i < n; i += stride) {
        const int64_t k = find_key(keys, nk, static_cast<uint64_t>(refs[i]));
        int32_t x = INT32_MIN, y = INT32_MIN;
        int flag = 1;
        if (k >= 0 && best[k] != 0ull) {
            x = loc[2 * k];
            y = loc[2 * k + 1];
            flag = (x == INT32_MIN || y == INT32_MIN) ? 2 : 0;
        }
        verts[2 * i] = x;
        verts[2 * i + 1] = y;
        if (flag) atomicOr(&flags[ref_way[i]], flag);
    }
}

// ---- validity ----

struct P {
    int32_t x, y;
};

__device__ __forceinline__ int orient(P a, P b, P c) {
    const __int128 l = static_cast<__int128>(static_cast<int64_t>(b.x) - a.x) * (static_cast<int64_t>(c.y) - a.y);
    const __int128 r = static_cast<__int128>(static_cast<int64_t>(b.y) - a.y) * (static_cast<int64_t>(c.x) - a.x);
    return (l > r) - (l < r);
}

__device__ __forceinline__ bool on_segment(P p, P a, P b) {
    return orient(a, b, p) == 0 && min(a.x, b.x) <= p.x && p.x <= max(a.x, b.x) && min(a.y, b.y) <= p.y && p.y <= max(a.y, b.y);
}

// features._intersect: 0 = disjoint, 1 = one common point, 2 = a common piece of positive length
__device__ __forceinline__ int intersect(P a, P b, P c, P d) {
    const int o1 = orient(a, b, c), o2 = orient(a, b, d), o3 = orient(c, d, a), o4 = orient(c, d, b);
    if (o1 == 0 && o2 == 0 && o3 == 0 && o4 == 0) {
        const bool ax = a.x != b.x || c.x != d.x;
        const int32_t a0 = ax ? a.x : a.y, b0 = ax ? b.x : b.y, c0 = ax ? c.x : c.y, d0 = ax ? d.x : d.y;
        const int32_t lo = max(min(a0, b0), min(c0, d0)), hi = min(max(a0, b0), max(c0, d0));
        return lo > hi ? 0 : (lo == hi ? 1 : 2);
    }
    if (o1 != o2 && o3 != o4) return 1;
    if ((o1 == 0 && on_segment(c, a, b)) || (o2 == 0 && on_segment(d, a, b)) || (o3 == 0 && on_segment(a, c, d)) || (o4 == 0 && on_segment(b, c, d))) return 1;
    return 0;
}

// edges i < j of a ring of m vertices: true when they meet in a way a valid ring does not allow
__device__ __forceinline__ bool bad_pair(const P* __restrict__ v, int64_t m, int64_t i, int64_t j) {
    const P a = v[i], b = v[i + 1 < m ? i + 1 : 0], c = v[j], d = v[j + 1 < m ? j + 1 : 0];
    const int hit = intersect(a, b, c, d);
    const bool adjacent = j == i + 1 || (i == 0 && j == m - 1);
    return hit == 2 || (hit == 1 && !adjacent);
}

__device__ __forceinline__ bool same(P a, P b) { return a.x == b.x && a.y == b.y; }

__global__ void __launch_bounds__(RING_THREADS) valid_ring_kernel(const P* __restrict__ verts, const int64_t* __restrict__ ring_offsets, int32_t R,
                                                                  const int32_t* __restrict__ flags, P* __restrict__ scratch, int32_t* __restrict__ lens,
                                                                  uint8_t* __restrict__ valid) {
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (RING_THREADS / 32);
    for (int r = (blockIdx.x * RING_THREADS + threadIdx.x) >> 5; r < R; r += warps) {
        const int64_t v0 = ring_offsets[r], n = ring_offsets[r + 1] - v0;
        if (flags[r] != 0 || n < 1) {
            if (lane == 0) {
                valid[r] = 0;
                lens[r] = 0;
            }
            continue;
        }
        const P* in = verts + v0;
        P* out = scratch + v0;
        // compaction: keep vertex i when it differs from vertex i - 1 (vertex 0 always kept)
        int64_t m = 0;
        for (int64_t base = 0; base < n; base += 32) {
            const int64_t i = base + lane;
            bool keep = false;
            P p{0, 0};
            if (i < n) {
                p = in[i];
                keep = i == 0 || !same(p, in[i - 1]);
            }
            const unsigned ball = __ballot_sync(FULL, keep);
            if (keep) out[m + __popc(ball & ((1u << lane) - 1))] = p;
            m += __popc(ball);
        }
        __syncwarp();
        // drop trailing copies of the first vertex (the closing vertex)
        const P first = out[0];
        while (m > 1 && same(out[m - 1], first)) --m;
        // >= 3 distinct positions: something other than out[0] and out[1]
        bool third = false;
        for (int64_t i = lane; i < m && m >= 3; i += 32) third |= !same(out[i], out[0]) && !same(out[i], out[1]);
        bool ok = __any_sync(FULL, third);
        if (ok) {
            __int128 area = 0;
            for (int64_t i = lane; i < m; i += 32) {
                const P a = out[i], b = out[i + 1 < m ? i + 1 : 0];
                area += static_cast<__int128>(static_cast<int64_t>(a.x) - first.x) * (static_cast<int64_t>(b.y) - first.y) -
                        static_cast<__int128>(static_cast<int64_t>(b.x) - first.x) * (static_cast<int64_t>(a.y) - first.y);
            }
            uint64_t lo = static_cast<uint64_t>(area), hi = static_cast<uint64_t>(area >> 64);
            for (int o = 16; o > 0; o >>= 1) {
                const uint64_t l2 = __shfl_xor_sync(FULL, lo, o), h2 = __shfl_xor_sync(FULL, hi, o);
                const uint64_t s = lo + l2;
                hi = hi + h2 + (s < lo ? 1 : 0);
                lo = s;
            }
            ok = (lo | hi) != 0;
        }
        if (ok && n <= RSB_EXTRACT_WARP_RING) {
            bool bad = false;
            for (int64_t i = 0; i < m && !bad; ++i) {
                bool b = false;
                for (int64_t j = i + 1 + lane; j < m && !b; j += 32) b = bad_pair(out, m, i, j);
                bad = __any_sync(FULL, b);
            }
            ok = !bad;
        }
        if (lane == 0) {
            valid[r] = ok ? 1 : 0;
            lens[r] = static_cast<int32_t>(m);
        }
    }
}

// one CTA per (long ring, edge tile I, edge tile J), J >= I; clears valid[r] on a bad pair
__global__ void __launch_bounds__(PAIR_THREADS) valid_pairs_kernel(const int64_t* __restrict__ ring_offsets, const int32_t* __restrict__ long_rings,
                                                                   int32_t L, const int64_t* __restrict__ tile_offsets, const P* __restrict__ scratch,
                                                                   const int32_t* __restrict__ lens, uint8_t* valid) {
    __shared__ P ei[PAIR_TILE + 1], ej[PAIR_TILE + 1];
    const int64_t total = tile_offsets[L];
    for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
        int lo = 0, hi = L - 1;  // the ring whose tile range holds t
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (tile_offsets[mid] <= t) lo = mid;
            else hi = mid - 1;
        }
        const int r = long_rings[lo];
        const int64_t local = t - tile_offsets[lo];
        const int64_t n = ring_offsets[r + 1] - ring_offsets[r];
        const int64_t nb = (n + PAIR_TILE - 1) / PAIR_TILE;
        const int64_t I = local / nb, J = local % nb;
        const int64_t m = lens[r];
        if (J < I || I * PAIR_TILE >= m) continue;  // uniform over the CTA
        const P* v = scratch + ring_offsets[r];
        for (int k = threadIdx.x; k <= PAIR_TILE; k += PAIR_THREADS) {
            const int64_t a = I * PAIR_TILE + k, b = J * PAIR_TILE + k;
            if (a <= m) ei[k] = v[a < m ? a : 0];
            if (b <= m) ej[k] = v[b < m ? b : 0];
        }
        __syncthreads();
        bool bad = false;
        for (int p = threadIdx.x; p < PAIR_TILE * PAIR_TILE && !bad; p += PAIR_THREADS) {
            const int64_t i = I * PAIR_TILE + p / PAIR_TILE, j = J * PAIR_TILE + p % PAIR_TILE;
            if (j <= i || j >= m) continue;
            const int li = p / PAIR_TILE, lj = p % PAIR_TILE;
            const int hit = intersect(ei[li], ei[li + 1], ej[lj], ej[lj + 1]);
            const bool adjacent = j == i + 1 || (i == 0 && j == m - 1);
            bad = hit == 2 || (hit == 1 && !adjacent);
        }
        if (bad) valid[r] = 0;
        __syncthreads();
    }
}

unsigned grid_for(int64_t n, int threads, int per_sm) {
    return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, static_cast<int64_t>(per_sm) * num_sms())));
}

}  // namespace

extern "C" int rsb_pbf_dense_nodes(const uint8_t* blocks, const int64_t* block_offsets, const int64_t* segs, int32_t G, int64_t* ids, int32_t* xy,
                                   int32_t* status, void* stream) {
    if (G < 0 || !status || (G > 0 && (!blocks || !block_offsets || !segs || !ids || !xy))) return set_error(RSB_E_INVALID, "pbf_dense_nodes: bad arguments");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int32_t), st);
    if (e != cudaSuccess) return set_cuda_error(e, "pbf_dense_nodes: clear");
    if (G > 0) dense_nodes_kernel<<<static_cast<unsigned>(G), DENSE_THREADS, 0, st>>>(blocks, block_offsets, segs, ids, xy, status);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "pbf_dense_nodes launch");
}

extern "C" int rsb_extract_locate(const int64_t* ids, const int32_t* xy, int64_t n, int64_t ordinal_base, const int64_t* keys, int64_t num_keys, int64_t* best,
                                  int32_t* loc, void* stream) {
    if (n < 0 || num_keys < 0 || ordinal_base < 0 || (n > 0 && (!ids || !xy)) || (num_keys > 0 && (!keys || !best || !loc)))
        return set_error(RSB_E_INVALID, "extract_locate: bad arguments");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    if (n == 0 || num_keys == 0) return RSB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned g = grid_for(n, JOIN_THREADS, 16);
    const uint64_t* k = reinterpret_cast<const uint64_t*>(keys);
    unsigned long long* b = reinterpret_cast<unsigned long long*>(best);
    locate_mark_kernel<<<g, JOIN_THREADS, 0, st>>>(ids, n, ordinal_base, k, num_keys, b);
    locate_write_kernel<<<g, JOIN_THREADS, 0, st>>>(ids, xy, n, ordinal_base, k, num_keys, b, loc);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "extract_locate launch");
}

extern "C" int rsb_extract_gather(const int64_t* refs, const int32_t* ref_way, int64_t num_refs, int32_t num_ways, const int64_t* keys, int64_t num_keys,
                                  const int64_t* best, const int32_t* loc, int32_t* verts, int32_t* flags, void* stream) {
    if (num_refs < 0 || num_ways < 0 || num_keys < 0 || (num_ways > 0 && !flags) || (num_refs > 0 && (!refs || !ref_way || !verts)) ||
        (num_keys > 0 && (!keys || !best || !loc)))
        return set_error(RSB_E_INVALID, "extract_gather: bad arguments");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = num_ways > 0 ? cudaMemsetAsync(flags, 0, static_cast<size_t>(num_ways) * 4, st) : cudaSuccess;
    if (e != cudaSuccess) return set_cuda_error(e, "extract_gather: clear");
    if (num_refs > 0)
        gather_kernel<<<grid_for(num_refs, JOIN_THREADS, 16), JOIN_THREADS, 0, st>>>(refs, ref_way, num_refs, reinterpret_cast<const uint64_t*>(keys), num_keys,
                                                                                   reinterpret_cast<const unsigned long long*>(best), loc, verts, flags);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "extract_gather launch");
}

extern "C" int rsb_extract_valid(const int32_t* verts, const int64_t* ring_offsets, int32_t R, const int32_t* flags, const int32_t* long_rings, int32_t L,
                                 const int64_t* tile_offsets, int32_t* scratch, int32_t* lens, uint8_t* valid, void* stream) {
    if (R < 0 || L < 0 || L > R || (R > 0 && (!verts || !ring_offsets || !flags || !scratch || !lens || !valid)) || (L > 0 && (!long_rings || !tile_offsets)))
        return set_error(RSB_E_INVALID, "extract_valid: bad arguments");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    if (R == 0) return RSB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    valid_ring_kernel<<<grid_for(static_cast<int64_t>(R) * 32, RING_THREADS, 16), RING_THREADS, 0, st>>>(
        reinterpret_cast<const P*>(verts), ring_offsets, R, flags, reinterpret_cast<P*>(scratch), lens, valid);
    if (L > 0)
        valid_pairs_kernel<<<static_cast<unsigned>(64 * num_sms()), PAIR_THREADS, 0, st>>>(ring_offsets, long_rings, L, tile_offsets,
                                                                                          reinterpret_cast<const P*>(scratch), lens, valid);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "extract_valid launch");
}
