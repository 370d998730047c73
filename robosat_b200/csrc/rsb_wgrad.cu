// Weight-gradient contraction on wgmma tensor cores: for a forward convolution described by an rsb_conv_desc,
//   dWp[phase*Cout + co][kb*64 + ci] = sum over tile-space pixels p of  dY_phase[p][co] * X_{segment(kb)}[p + (dh, dw)][ci]
// i.e. exactly the packed weight layout the forward kernel consumes, so the same segment list (parity views for strided
// convs, low-res views + phases for the fused upsample, two views for concat, window views for stem / dec5) drives wgrad.
//
// The contraction index is the PIXEL, which is the slow (row) index of NHWC tiles in shared memory, so both operands
// are "MN-major": A = dY tile [128 px][64 co] (x2 for 128 rows of co), B = X tile [128 px][64 ci]; the descriptors use
// LBO = distance between 64-wide column blocks, SBO = 1024 B (8 pixel rows), and advance 2048 B per K=16 MMA.
//
// Work item = (128 output channels) x (phase) x (group of <= 4 consecutive 64-wide K blocks) x (slice of the pixel tiles).
// Per 128-pixel tile: one dY box (2 x 16 KB) + one X box per K block (16 KB each) by TMA; consumer warpgroup g issues
// 8 MMAs (M64 x N<=256 x K16) for output channels [64 g, 64 g + 64) into register accumulators. Epilogue: plain fp32 stores
// into the packed gradient, or, split-K over pixel slices, into the slice's partial gradient in a scratch buffer, which
// wgrad_reduce_kernel adds up in slice order (bit-identical from run to run).

#include <string.h>

#include <new>
#include <type_traits>

#include "../../include/rsb200.h"
#include "rsb_host.h"
#include "rsb_ptx.cuh"

namespace rsb {

static constexpr int kWgGroup = 4;                     // K blocks per work item
static constexpr int kWgPx = 128;                      // pixels (contraction elements) per pipeline stage
static constexpr int kWgTileBytes = kWgPx * 64 * 2;    // one [128 px][64 ch] fp16 box
static constexpr int kWgStageBytes = (2 + kWgGroup) * kWgTileBytes;  // 96 KB
static constexpr int kWgStages = 2;
static constexpr int kWgSmem = kWgStages * kWgStageBytes + 256 + 1024;
static constexpr int kWgThreads = 384;                 // two consumer warpgroups + one producer warpgroup

struct alignas(64) WgradKParams {
    CUtensorMap tmX[RSB_MAX_SRCS];
    CUtensorMap tmDY[4];  // dY view per phase
    int32_t nseg;
    int32_t seg_src[RSB_MAX_SEGS];
    int32_t seg_dh[RSB_MAX_SEGS];
    int32_t seg_dw[RSB_MAX_SEGS];
    int32_t seg_kb0[RSB_MAX_SEGS + 1];  // first K block of each segment (prefix sum of cblocks)
    int32_t kblocks, kgroups;
    int32_t tiles_w, tiles_h, tiles_n, ptiles;  // pixel tiles per phase
    int32_t slices, tiles_per_slice;
    int32_t co_blocks, phases, total_items;
    int32_t TW, TH, TN;
    int32_t Cout;
    int64_t K;  // packed row length = 64 * kblocks
    float* dw;  // [phases*Cout][K] fp32
    // split-K (slices > 1): slice s stores its partial gradient to partial + s * slice_stride, and wgrad_reduce_kernel adds
    // the slices in index order. Set by rsb_wgrad_plan_set_scratch; a single slice stores straight into dw.
    float* partial;
    int64_t slice_stride;
};

struct WgItem {
    int co_blk, phase, pa, pb, kg, slice;
};

__device__ __forceinline__ WgItem wg_decode(const WgradKParams& p, int id) {
    WgItem it;
    it.co_blk = id % p.co_blocks;
    id /= p.co_blocks;
    it.kg = id % p.kgroups;
    id /= p.kgroups;
    it.phase = id % p.phases;
    id /= p.phases;
    it.slice = id;
    it.pa = it.phase >> 1;
    it.pb = it.phase & 1;
    return it;
}

// MN-major SWIZZLE_128B operand: rows = K index (pixels), 64 M/N elements per 128-byte row
__device__ __forceinline__ uint64_t make_sw128_mnmajor_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
    return make_smem_desc(smem_addr, lbo_bytes, 1024, 1);
}

__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ WgradKParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kWgStages * kWgStageBytes);
    uint64_t* empty_bar = full_bar + kWgStages;
    const int warp_idx = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp_idx == 8 && lane == 0) {
        for (int i = 0; i < RSB_MAX_SRCS; ++i) tma_prefetch_desc(&p.tmX[i]);
        for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.tmDY[i]);
        for (int i = 0; i < kWgStages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp_idx >= 8) {
        setmaxnreg_dec<40>();
        if (warp_idx == 8 && elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
                const WgItem it = wg_decode(p, item);
                const int kb_lo = it.kg * kWgGroup;
                const int nkb = min(kWgGroup, p.kblocks - kb_lo);
                const int t_lo = it.slice * p.tiles_per_slice;
                const int t_hi = min(p.ptiles, t_lo + p.tiles_per_slice);
                for (int t = t_lo; t < t_hi; ++t) {
                    int id = t;
                    const int w0 = (id % p.tiles_w) * p.TW;
                    id /= p.tiles_w;
                    const int h0 = (id % p.tiles_h) * p.TH;
                    const int n0 = (id / p.tiles_h) * p.TN;
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], (2 + nkb) * kWgTileBytes);
                    uint8_t* st = smem + stage * kWgStageBytes;
                    // dY: two 64-channel column blocks (the second is zero-filled by TMA when Cout has no such channels)
                    tma_load_4d(st, &p.tmDY[it.phase], &full_bar[stage], it.co_blk * 128, w0, h0, n0);
                    tma_load_4d(st + kWgTileBytes, &p.tmDY[it.phase], &full_bar[stage], it.co_blk * 128 + 64, w0, h0, n0);
                    int s = 0;
                    for (int j = 0; j < nkb; ++j) {
                        const int kb = kb_lo + j;
                        while (kb >= p.seg_kb0[s + 1]) ++s;
                        tma_load_4d(st + (2 + j) * kWgTileBytes, &p.tmX[p.seg_src[s]], &full_bar[stage], (kb - p.seg_kb0[s]) * 64,
                                    w0 + p.seg_dw[s] + it.pb, h0 + p.seg_dh[s] + it.pa, n0);
                    }
                    if (++stage == kWgStages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        setmaxnreg_inc<232>();
        const int g = warp_idx >> 2;                           // output channels [64 g, 64 g + 64) of the item's 128
        const int r0 = 16 * (warp_idx & 3) + (lane >> 2);      // fragment rows r0, r0 + 8
        const int cq = 2 * (lane & 3);
        const uint64_t da0 = make_sw128_mnmajor_desc(smem_u32(smem + g * kWgTileBytes), kWgTileBytes);
        const uint64_t db0 = make_sw128_mnmajor_desc(smem_u32(smem + 2 * kWgTileBytes), kWgTileBytes);
        int stage = 0;
        uint32_t phase = 0;
        float acc[kWgGroup * 32];
        for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
            const WgItem it = wg_decode(p, item);
            const int kb_lo = it.kg * kWgGroup;
            const int nkb = min(kWgGroup, p.kblocks - kb_lo);
            const int t_lo = it.slice * p.tiles_per_slice;
            const int t_hi = min(p.ptiles, t_lo + p.tiles_per_slice);
            // ONE MMA per K step covers all K blocks of the group: the X tiles sit back to back in the stage, so they form an
            // MN-major B operand of N = 64 * nkb columns with LBO = one tile
            auto run = [&](auto nc) {
                constexpr int N = decltype(nc)::value;
                for (int t = t_lo; t < t_hi; ++t) {
                    mbar_wait(&full_bar[stage], phase);
                    const uint64_t so = static_cast<uint64_t>(stage * (kWgStageBytes >> 4));
                    acc_fence(acc);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < kWgPx / 16; ++k)
                        wgmma<N, 0, 1, 1>(acc, da0 + so + 128 * k, db0 + so + 128 * k, (k > 0 || t > t_lo) ? 1u : 0u);
                    wgmma_commit();
                    acc_fence(acc);
                    wgmma_wait<0>();
                    acc_fence(acc);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[stage]);
                    if (++stage == kWgStages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            };
            switch (nkb) {
                case 1: run(std::integral_constant<int, 64>{}); break;
                case 2: run(std::integral_constant<int, 128>{}); break;
                case 3: run(std::integral_constant<int, 192>{}); break;
                default: run(std::integral_constant<int, 256>{}); break;
            }
            // one writer per element: dw itself for a single slice, else this slice's partial buffer
            float* dbase = p.slices > 1 ? p.partial + static_cast<int64_t>(it.slice) * p.slice_stride : p.dw;
            if (t_lo < p.ptiles) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int co = it.co_blk * 128 + 64 * g + r0 + 8 * hh;
                    if (co >= p.Cout) continue;
                    float* drow = dbase + (static_cast<int64_t>(it.phase) * p.Cout + co) * p.K + static_cast<int64_t>(kb_lo) * 64;
#pragma unroll
                    for (int j = 0; j < kWgGroup * 8; ++j) {
                        if (j < nkb * 8) {
                            *reinterpret_cast<float2*>(drow + 8 * j + cq) = make_float2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
                        }
                    }
                }
            }
        }
    }
}

// dw[i] = partial[0][i] + partial[1][i] + ... in slice order: the deterministic second stage of the split-K reduction
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dw, int64_t n4, int slices, int64_t stride4) {
    const float4* p4 = reinterpret_cast<const float4*>(partial);
    float4* d4 = reinterpret_cast<float4*>(dw);
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float4 a = p4[i];
        for (int s = 1; s < slices; ++s) {
            const float4 b = p4[i + s * stride4];
            a.x += b.x;
            a.y += b.y;
            a.z += b.z;
            a.w += b.w;
        }
        d4[i] = a;
    }
}

}  // namespace rsb

using namespace rsb;

struct rsb_wgrad_plan {
    WgradKParams kp;
    int grid;
    int64_t dw_bytes;
};

extern "C" int rsb_wgrad_plan_create(const rsb_conv_desc* d, const void* dy, float* dw_packed, rsb_wgrad_plan** out_plan) {
    if (!d || !dy || !dw_packed || !out_plan) return set_error(RSB_E_INVALID, "wgrad: null argument");
    *out_plan = nullptr;
    if (d->nsrc < 1 || d->nsrc > RSB_MAX_SRCS || d->nseg < 1 || d->nseg > RSB_MAX_SEGS) return set_error(RSB_E_INVALID, "wgrad: bad source/segment count");
    if (d->TW * d->TH * d->TN != 128) return set_error(RSB_E_INVALID, "wgrad: TW*TH*TN must be 128");
    // a pipeline stage covers kWgPx pixels: the forward's 128-pixel tile box, or half of it
    int bw = d->TW, bh = d->TH, bn = d->TN;
    if (kWgPx == 64) {
        if (bn % 2 == 0) bn /= 2;
        else if (bh % 2 == 0) bh /= 2;
        else bw /= 2;
    }
    if (!(d->phases == 1 || d->phases == 4)) return set_error(RSB_E_INVALID, "wgrad: phases must be 1 or 4");
    int rc = rsb_device_ok();
    if (rc) return rc;
    rsb_wgrad_plan* plan = new (std::nothrow) rsb_wgrad_plan();
    if (!plan) return set_error(RSB_E_INVALID, "wgrad: out of host memory");
    memset(&plan->kp, 0, sizeof(plan->kp));
    WgradKParams& kp = plan->kp;
    for (int i = 0; i < d->nsrc; ++i) {
        const rsb_conv_src& s = d->srcs[i];
        const uint64_t dims[4] = {(uint64_t)s.C, (uint64_t)s.W, (uint64_t)s.H, (uint64_t)s.N};
        const uint64_t strides[3] = {(uint64_t)s.pitch_w * 2, (uint64_t)s.pitch_h * 2, (uint64_t)s.pitch_n * 2};
        const uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
        rc = encode_tiled_f16(&kp.tmX[i], 4, s.ptr, dims, strides, box);
        if (rc) {
            delete plan;
            return rc;
        }
    }
    for (int i = d->nsrc; i < RSB_MAX_SRCS; ++i) kp.tmX[i] = kp.tmX[0];
    {
        const int sy = d->out_sy > 0 ? d->out_sy : 1, sx = d->out_sx > 0 ? d->out_sx : 1;
        const uint64_t dims[4] = {(uint64_t)d->Cout, (uint64_t)d->Wt, (uint64_t)d->Ht, (uint64_t)d->Nt};
        const uint64_t strides[3] = {(uint64_t)sx * d->out_pitch_w * 2, (uint64_t)sy * d->out_pitch_h * 2, (uint64_t)d->out_pitch_n * 2};
        const uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
        for (int ph = 0; ph < 4; ++ph) {
            const int a = ph >> 1, b = ph & 1;
            const __half* base = static_cast<const __half*>(dy) + (ph < d->phases ? a * d->out_pitch_h + b * d->out_pitch_w : 0);
            rc = encode_tiled_f16(&kp.tmDY[ph], 4, base, dims, strides, box);
            if (rc) {
                delete plan;
                return rc;
            }
        }
    }
    kp.nseg = d->nseg;
    int kb = 0;
    for (int s = 0; s < d->nseg; ++s) {
        kp.seg_src[s] = d->segs[s].src;
        kp.seg_dh[s] = d->segs[s].dh;
        kp.seg_dw[s] = d->segs[s].dw;
        kp.seg_kb0[s] = kb;
        kb += d->segs[s].cblocks;
    }
    kp.seg_kb0[d->nseg] = kb;
    kp.kblocks = kb;
    kp.kgroups = (kb + kWgGroup - 1) / kWgGroup;
    kp.TW = bw;
    kp.TH = bh;
    kp.TN = bn;
    kp.tiles_w = (d->Wt + bw - 1) / bw;
    kp.tiles_h = (d->Ht + bh - 1) / bh;
    kp.tiles_n = (d->Nt + bn - 1) / bn;
    kp.ptiles = kp.tiles_w * kp.tiles_h * kp.tiles_n;
    kp.co_blocks = (d->Cout + 127) / 128;
    kp.phases = d->phases;
    kp.Cout = d->Cout;
    kp.K = static_cast<int64_t>(kb) * 64;
    kp.dw = dw_packed;
    // split-K over slices of the pixel tiles: pick the slice count that minimises rounds x (tiles per item + epilogue),
    // rounds = ceil(items / SMs) of the persistent grid (e.g. 160 items on 132 SMs would run two rounds for 28 extra items);
    // every slice adds a full copy of the gradient tile (128 x 256 fp32 partials ~ 8 stage times) to the traffic
    const int sms = num_sms();
    const int base_items = kp.co_blocks * kp.phases * kp.kgroups;
    int64_t best_cost = -1;
    int best_tps = kp.ptiles;
    for (int sl = 1; sl <= kp.ptiles && sl <= 4 * sms; ++sl) {
        const int tps = (kp.ptiles + sl - 1) / sl;
        const int eff = (kp.ptiles + tps - 1) / tps;
        const int64_t rounds = (static_cast<int64_t>(base_items) * eff + sms - 1) / sms;
        const int64_t cost = rounds * (tps + 8);
        if (best_cost < 0 || cost < best_cost) {
            best_cost = cost;
            best_tps = tps;
        }
    }
    kp.tiles_per_slice = best_tps;
    kp.slices = (kp.ptiles + kp.tiles_per_slice - 1) / kp.tiles_per_slice;
    kp.total_items = base_items * kp.slices;
    plan->grid = kp.total_items < sms ? kp.total_items : sms;
    plan->dw_bytes = static_cast<int64_t>(d->phases) * d->Cout * kp.K * 4;
    *out_plan = plan;
    return RSB_OK;
}

extern "C" int64_t rsb_wgrad_plan_scratch_bytes(const rsb_wgrad_plan* plan) {
    if (!plan) return 0;
    return plan->kp.slices > 1 ? plan->dw_bytes * plan->kp.slices : 0;
}

extern "C" int rsb_wgrad_plan_set_scratch(rsb_wgrad_plan* plan, float* scratch, int64_t scratch_bytes) {
    if (!plan) return set_error(RSB_E_INVALID, "wgrad: null plan");
    const int64_t need = rsb_wgrad_plan_scratch_bytes(plan);
    if (need == 0) return RSB_OK;  // a single slice writes every element of dw exactly once
    if (!scratch || scratch_bytes < need || (reinterpret_cast<uintptr_t>(scratch) & 15))
        return set_error(RSB_E_INVALID, "wgrad: split-K needs a 16B-aligned scratch of >= %lld bytes", (long long)need);
    plan->kp.partial = scratch;
    plan->kp.slice_stride = plan->dw_bytes / 4;
    return RSB_OK;
}

extern "C" void rsb_wgrad_plan_destroy(rsb_wgrad_plan* plan) { delete plan; }

extern "C" int rsb_wgrad_run(const rsb_wgrad_plan* plan, void* stream_) {
    if (!plan) return set_error(RSB_E_INVALID, "wgrad: null plan");
    if (plan->kp.slices > 1 && plan->kp.partial == nullptr)
        return set_error(RSB_E_INVALID, "wgrad: a split-K plan (%d slices) needs its scratch from rsb_wgrad_plan_set_scratch", plan->kp.slices);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    static bool attr_set[64] = {};  // per device: one process may drive several GPUs
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (!attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(wgrad)");
        attr_set[dev] = true;
    }
    wgrad_tc_kernel<<<plan->grid, kWgThreads, kWgSmem, stream>>>(plan->kp);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "wgrad_tc_kernel launch");
    if (plan->kp.slices > 1) {
        const int64_t n4 = plan->dw_bytes / 16;
        int blocks = static_cast<int>((n4 + 255) / 256);
        if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
        wgrad_reduce_kernel<<<blocks, 256, 0, stream>>>(plan->kp.partial, plan->kp.dw, n4, plan->kp.slices, plan->kp.slice_stride / 4);
        e = cudaGetLastError();
        if (e != cudaSuccess) return set_cuda_error(e, "wgrad_reduce_kernel launch");
    }
    return RSB_OK;
}
