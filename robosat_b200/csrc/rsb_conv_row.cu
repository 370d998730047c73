// Line-buffer convolution for the high-resolution, small-Cout layers (dec5 + final, dec4, layer1 3x3):
// wgmma / TMA like rsb_conv.cu, but every input row is fetched from L2 ONCE and serves all filter taps.
//
// Why: with Cout <= 64 the generic kernel is bound by L2 -> shared-memory operand traffic: it re-fetches the A box for
// every tap (9x for a 3x3, 16x for the 4 phases x 2x2 taps of the fused upsample).
//
// How: a tile is 128 consecutive output pixels of ONE row. A CTA walks a vertical strip (fixed image n, fixed 128
// columns, a chunk of rows) and keeps the last input rows in a shared-memory ring: each ring slot holds one input row
// segment of 128 + halo pixels per 64-channel block, written by one TMA box load (zero fill outside the image = padding).
// The A operand of tap (kh, kw) is that slot's buffer with the start address advanced by kw pixels -- a K-major swizzled
// operand may start at any pixel row of a TMA-written box with base_offset 0 (the swizzle follows the address bits) -- so the
// horizontal taps cost no traffic, and consecutive output rows reuse the ring for the vertical taps. All weights of
// the unit stay resident in shared memory.
//
// Fused nearest-x2 upsample (dec4): a unit fixes the output row phase a; both column phases b = 0, 1 ("sub-tiles") are
// computed from the same ring rows into two accumulators and stored to the strided output views (2h + a, 2w + b).

#include <string.h>

#include <new>
#include <type_traits>

#include "../../include/rsb200.h"
#include "rsb_host.h"
#include "rsb_ptx.cuh"

namespace rsb {

static constexpr int kRowTile = 128;      // output pixels per tile (one row segment)
static constexpr int kRowMaxSlots = 16;   // ring depth in input rows is chosen per plan (latency hiding vs shared memory)
static constexpr int kRowThreads = 288;   // warps 0-7: two consumer warpgroups (wgmma + epilogue), warp 8: TMA
static constexpr int kRowMaxW = 16;       // weight blocks: nsub * taps * cblocks <= 16

struct alignas(64) RowKParams {
    CUtensorMap tmA;      // source view {Cin, Wsrc, Hsrc, N}, box {CBLK, buf_w, 1, 1}
    CUtensorMap tmB;      // packed weights [phases*Cout][K], box {CBLK, BLOCK_N}
    CUtensorMap tmC[4];   // output view per phase, box = 32 consecutive pixels of a row x chunk channels
    int32_t taps_h, taps_w, cblocks, nsub, nphase_a;
    int32_t dh0, dw0;
    int32_t buf_w;        // pixels per ring row = 128 + taps_w + nsub - 2
    int32_t slot_bytes;   // bytes of one (row, cblock) buffer, multiple of 1024
    int32_t slots;        // ring depth (rows)
    int32_t wblock_bytes; // BLOCK_N * CBLK * 2
    int32_t Wt, Ht, Nt, Cout;
    int32_t wstrips, rchunks, rows_per_unit, total_units;
    int32_t relu;
    const float* bias;    // fp32 [Cout] or NULL (mode 0)
    int32_t head_classes;
    const float* head_w;
    const float* head_b;
    float* head_out;
    float acc_scale;      // strict precision: 2^-e of the weight scaling (1 otherwise)
    int32_t plane_bytes;  // strict precision: byte distance between the hi and lo plane of a ring row (= cblocks * slot_bytes)
};

struct RowUnit {
    int n, w0, h_lo, h_hi, a;
};

__device__ __forceinline__ RowUnit row_decode(const RowKParams& p, int id) {
    // the row phase is the FASTEST index: neighbouring CTAs work on the two row phases of the same strip at the same time
    // (the input rows they share are served by L2), and with an even grid every CTA keeps one phase = one resident weight set
    RowUnit u;
    u.a = id % p.nphase_a;
    id /= p.nphase_a;
    const int ws = id % p.wstrips;
    id /= p.wstrips;
    const int rc = id % p.rchunks;
    u.n = id / p.rchunks;
    u.w0 = ws * kRowTile;
    u.h_lo = rc * p.rows_per_unit;
    u.h_hi = min(p.Ht, u.h_lo + p.rows_per_unit);
    return u;
}

// K-major swizzled operand descriptor: CBLK = 64 -> 128-byte rows / SWIZZLE_128B, CBLK = 32 -> 64-byte rows / SWIZZLE_64B
template <int CBLK>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr) {
    return make_smem_desc(smem_addr, 16, CBLK == 64 ? 1024 : 512, CBLK == 64 ? 1 : 2);
}

template <int CBLK, int BLOCK_N, int MODE>
struct RowCfg {
    static constexpr int kPB = CBLK * 2;                       // bytes per pixel per channel block
    static constexpr int kChunk = BLOCK_N >= 64 ? 64 : 32;     // epilogue staging chunk (channels)
    static constexpr int kWgChunkBytes = 64 * kChunk * 2;      // one warpgroup's 64 pixels x kChunk channels
    static constexpr int kStageBytes = MODE == 0 ? 2 * 2 * kWgChunkBytes : 0;  // 2 warpgroups x 2 store slices
    static constexpr int kBarBytes = 512;   // mbarriers
    static constexpr int kHeadBytes = 1088; // final 1x1 weights [8][32] + bias [8] as fp32 (mode 1)
};

// TAPS: 3 (3x3) or 2 (2x2 taps of the fused upsample); CBLOCKS: channel blocks per pixel; NSUB: column phases per tile.
// Warpgroup g (warps 4g .. 4g+3) computes pixels [64 g, 64 g + 64) of the row segment; warp 8 is the TMA producer.
// SPLIT (strict precision, see rsb_conv.cu): every ring row and every weight block holds a hi and a lo fp16 plane; per K step
// one MMA of width 2*BLOCK_N computes A_hi x [W_hi | W_lo] into [main | cross] columns and a second adds A_lo x W_hi onto the
// cross columns; the epilogue adds main + cross in fp32. Instantiated for dec5 + final (the one strict layer whose resident
// weights and 2-plane ring fit in shared memory).
template <int CBLK, int BLOCK_N, int MODE, int TAPS, int CBLOCKS, int NSUB, bool SPLIT = false>
__global__ void __launch_bounds__(kRowThreads, 1) conv_row_kernel(const __grid_constant__ RowKParams p) {
    using Cfg = RowCfg<CBLK, BLOCK_N, MODE>;
    constexpr int kAcc = SPLIT ? 2 * BLOCK_N : BLOCK_N;  // accumulator columns of one sub-tile
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int row_bytes = p.slot_bytes * p.cblocks * (SPLIT ? 2 : 1);  // one ring slot = all channel blocks (and planes) of a row
    uint8_t* smem_rows = smem;
    uint8_t* smem_w = smem_rows + p.slots * row_bytes;
    const int nwblocks = p.nsub * p.taps_h * p.taps_w * p.cblocks;
    uint8_t* smem_c = smem_w + nwblocks * p.wblock_bytes;      // epilogue staging (mode 0), 1024-aligned by construction
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_c + Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + kRowMaxSlots;
    uint64_t* wfull_bar = empty_bar + kRowMaxSlots;
    uint64_t* wempty_bar = wfull_bar + 1;
    float* smem_head = reinterpret_cast<float*>(smem_c + Cfg::kStageBytes + Cfg::kBarBytes);  // [8][32] weights, then [8] bias

    const int warp_idx = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (MODE == 1) {
        // the head's 1x1 weights are read once per pixel and class: keep them in shared memory (broadcast reads)
        for (int i = threadIdx.x; i < p.head_classes * 32; i += blockDim.x) smem_head[i] = p.head_w[i];
        if (threadIdx.x < p.head_classes) smem_head[256 + threadIdx.x] = p.head_b[threadIdx.x];
    }

    if (warp_idx == 8 && lane == 0) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
        for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.tmC[i]);
        for (int i = 0; i < kRowMaxSlots; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
        }
        mbar_init(wfull_bar, 1);
        mbar_init(wempty_bar, 8);
        mbar_fence_init();
    }
    __syncthreads();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");

    if (warp_idx == 8) {
        // ------------------------------------------------------------------ TMA producer
        if (elect_one()) {
            uint32_t q = 0;  // rows loaded so far (ring position)
            uint32_t wq = 0; // weight sets loaded so far
            int cur_a = -1;
            for (int unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
                const RowUnit u = row_decode(p, unit);
                if (u.a != cur_a) {
                    // resident weights of this row phase: nsub x taps x cblocks blocks of [BLOCK_N][CBLK]
                    cur_a = u.a;
                    mbar_wait(wempty_bar, (wq & 1) ^ 1);
                    mbar_expect_tx(wfull_bar, nwblocks * p.wblock_bytes);
                    for (int s = 0; s < p.nsub; ++s) {
                        const int brow = (u.a * p.nsub + s) * p.Cout;
                        for (int t = 0; t < p.taps_h * p.taps_w; ++t) {
                            for (int cb = 0; cb < p.cblocks; ++cb) {
                                const int blk = (s * p.taps_h * p.taps_w + t) * p.cblocks + cb;
                                if constexpr (SPLIT) tma_load_3d(smem_w + blk * p.wblock_bytes, &p.tmB, wfull_bar, (t * p.cblocks + cb) * CBLK, brow, 0);
                                else tma_load_2d(smem_w + blk * p.wblock_bytes, &p.tmB, wfull_bar, (t * p.cblocks + cb) * CBLK, brow);
                            }
                        }
                    }
                    ++wq;
                }
                // input rows of the strip, in order; each row = cblocks boxes of buf_w pixels
                const int r_first = u.h_lo + p.dh0 + u.a;
                const int r_last = u.h_hi - 1 + p.dh0 + u.a + p.taps_h - 1;
                for (int r = r_first; r <= r_last; ++r, ++q) {
                    const int slot = q % p.slots;
                    mbar_wait(&empty_bar[slot], ((q / p.slots) & 1) ^ 1);
                    mbar_expect_tx(&full_bar[slot], (SPLIT ? 2 : 1) * p.cblocks * p.buf_w * Cfg::kPB);
                    for (int cb = 0; cb < p.cblocks; ++cb) {
                        if constexpr (SPLIT) {
                            tma_load_5d(smem_rows + slot * row_bytes + cb * p.slot_bytes, &p.tmA, &full_bar[slot], cb * CBLK, u.w0 + p.dw0, r, u.n, 0);
                            tma_load_5d(smem_rows + slot * row_bytes + p.plane_bytes + cb * p.slot_bytes, &p.tmA, &full_bar[slot], cb * CBLK, u.w0 + p.dw0, r,
                                        u.n, 1);
                        } else {
                            tma_load_4d(smem_rows + slot * row_bytes + cb * p.slot_bytes, &p.tmA, &full_bar[slot], cb * CBLK, u.w0 + p.dw0, r, u.n);
                        }
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers: wgmma + epilogue
        const int g = warp_idx >> 2;
        const int wtid = threadIdx.x & 127;
        const int r0 = 16 * (warp_idx & 3) + (lane >> 2);  // fragment rows (pixels) r0, r0 + 8 of the warpgroup's 64
        const int cq = 2 * (lane & 3);
        const uint32_t rows_base = smem_u32(smem_rows), w_base = smem_u32(smem_w);
        uint8_t* my_c = smem_c + g * 2 * Cfg::kWgChunkBytes;
        uint32_t qbase = 0, wq = 0, wchunk = 0;
        int cur_a = -1;
        float acc[NSUB * kAcc / 2];
        auto release = [&](uint64_t* bar) {
            __syncwarp();
            if (lane == 0) mbar_arrive(bar);
        };
        for (int unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
            const RowUnit u = row_decode(p, unit);
            if (u.a != cur_a) {
                cur_a = u.a;
                mbar_wait(wfull_bar, wq & 1);
                ++wq;
            }
            const int next_unit = unit + gridDim.x;
            const bool last_of_set = next_unit >= p.total_units || row_decode(p, next_unit).a != u.a;
            const int nrows_in = (u.h_hi - u.h_lo) + p.taps_h - 1;
            for (int h = u.h_lo; h < u.h_hi; ++h) {
                const uint32_t qrow = qbase + (h - u.h_lo);  // ring position of input row (h + dh0 + a)
                // rows h-1 .. were already waited for by the previous output row of this strip: only the newest one can be missing
                for (int th = (h == u.h_lo ? 0 : TAPS - 1); th < TAPS; ++th) {
                    const uint32_t qq = qrow + th;
                    mbar_wait(&full_bar[qq % p.slots], (qq / p.slots) & 1);
                }
                uint32_t slot_addr[TAPS];
#pragma unroll
                for (int th = 0; th < TAPS; ++th) slot_addr[th] = rows_base + ((qrow + th) % p.slots) * row_bytes + g * 64 * Cfg::kPB;
                acc_fence(acc);
                wgmma_fence();
                // sub-tile s accumulates into acc[s * kAcc / 2 ...]: the offset must be a compile-time constant
                auto mma_sub = [&](auto sc) {
                    constexpr int s = decltype(sc)::value;
#pragma unroll
                    for (int th = 0; th < TAPS; ++th) {
#pragma unroll
                        for (int tw = 0; tw < TAPS; ++tw) {
#pragma unroll
                            for (int cb = 0; cb < CBLOCKS; ++cb) {
                                constexpr int kPB = Cfg::kPB;
                                const int blk = ((s * TAPS + th) * TAPS + tw) * CBLOCKS + cb;
                                const uint64_t da = make_kmajor_desc<CBLK>(slot_addr[th] + cb * p.slot_bytes + (tw + s) * kPB);
                                const uint64_t db = make_kmajor_desc<CBLK>(w_base + blk * p.wblock_bytes);
#pragma unroll
                                for (int k = 0; k < CBLK / 16; ++k) {
                                    const uint32_t first = (th | tw | cb | k) != 0 ? 1u : 0u;
                                    if constexpr (SPLIT) {
                                        const uint64_t dal = make_kmajor_desc<CBLK>(slot_addr[th] + p.plane_bytes + cb * p.slot_bytes + (tw + s) * kPB);
                                        wgmma<2 * BLOCK_N, s * kAcc / 2>(acc, da + 2 * k, db + 2 * k, first);               // [main | cross]
                                        wgmma<BLOCK_N, s * kAcc / 2 + BLOCK_N / 2>(acc, dal + 2 * k, db + 2 * k, 1u);     // cross += A_lo W_hi
                                    } else {
                                        wgmma<BLOCK_N, s * kAcc / 2>(acc, da + 2 * k, db + 2 * k, first);
                                    }
                                }
                            }
                        }
                    }
                };
                mma_sub(std::integral_constant<int, 0>{});
                if constexpr (NSUB == 2) mma_sub(std::integral_constant<int, 1>{});
                wgmma_commit();
                acc_fence(acc);
                wgmma_wait<0>();
                acc_fence(acc);
                // the oldest ring row is not needed by later output rows of this strip
                release(&empty_bar[qrow % p.slots]);
                if (h == u.h_hi - 1) {
                    for (int th = 1; th < p.taps_h; ++th) release(&empty_bar[(qrow + th) % p.slots]);
                    if (last_of_set) release(wempty_bar);  // the resident weights may be replaced
                }
#pragma unroll
                for (int s = 0; s < NSUB; ++s) {
                    const int phase = (p.nphase_a * p.nsub > 1) ? (u.a * 2 + s) : 0;
                    if constexpr (MODE == 0) {
#pragma unroll
                        for (int ck = 0; ck < BLOCK_N / Cfg::kChunk; ++ck, ++wchunk) {
                            uint8_t* cbuf = my_c + (wchunk & 1) * Cfg::kWgChunkBytes;
                            if (wtid == 0) tma_store_wait_read<1>();
                            named_bar_sync(1 + g, 128);
#pragma unroll
                            for (int jj = 0; jj < Cfg::kChunk / 8; ++jj) {
                                const int j = ck * (Cfg::kChunk / 8) + jj;
                                const int c = 8 * j + cq;
#pragma unroll
                                for (int hh = 0; hh < 2; ++hh) {
                                    const int r = r0 + 8 * hh;
                                    const int su = Cfg::kChunk == 64 ? (jj ^ (r & 7)) : (jj ^ ((r >> 1) & 3));
                                    float a = acc[s * kAcc / 2 + 4 * j + 2 * hh], b = acc[s * kAcc / 2 + 4 * j + 2 * hh + 1];
                                    if (p.bias) {
                                        a += __ldg(p.bias + c);
                                        b += __ldg(p.bias + c + 1);
                                    }
                                    if (p.relu) {
                                        a = fmaxf(a, 0.0f);
                                        b = fmaxf(b, 0.0f);
                                    }
                                    *reinterpret_cast<__half2*>(cbuf + r * (Cfg::kChunk * 2) + su * 16 + (lane & 3) * 4) = __floats2half2_rn(a, b);
                                }
                            }
                            fence_proxy_async_smem();
                            named_bar_sync(1 + g, 128);
                            if (wtid == 0) {
                                tma_store_4d(&p.tmC[phase], cbuf, ck * Cfg::kChunk, u.w0 + g * 64, h, u.n);
                                tma_store_commit();
                            }
                        }
                    } else {
                        // head: ReLU(acc) [32 ch] -> fp32 1x1 conv to `classes` logits, NCHW fp32 store (unet.py:141); the 32
                        // channels of a pixel are spread over the 4 lanes of a quad
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            const int w = u.w0 + g * 64 + r0 + 8 * hh;
                            float v[8];
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    float a = acc[s * kAcc / 2 + 4 * j + 2 * hh + e];
                                    if constexpr (SPLIT) a = (a + acc[s * kAcc / 2 + BLOCK_N / 2 + 4 * j + 2 * hh + e]) * p.acc_scale;
                                    v[2 * j + e] = p.relu ? fmaxf(a, 0.0f) : a;
                                }
                            }
                            for (int k = 0; k < p.head_classes; ++k) {
                                float sum = 0.f;
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    const float2 wv = *reinterpret_cast<const float2*>(smem_head + k * 32 + 8 * j + cq);
                                    sum = fmaf(wv.x, v[2 * j], sum);
                                    sum = fmaf(wv.y, v[2 * j + 1], sum);
                                }
                                sum += __shfl_xor_sync(0xffffffffu, sum, 1);
                                sum += __shfl_xor_sync(0xffffffffu, sum, 2);
                                if (w < p.Wt && (lane & 3) == 0)
                                    p.head_out[((static_cast<int64_t>(u.n) * p.head_classes + k) * p.Ht + h) * p.Wt + w] = sum + smem_head[256 + k];
                            }
                        }
                    }
                }
            }
            qbase += nrows_in;
        }
        if (MODE == 0 && wtid == 0) tma_store_wait<0>();
    }
}

}  // namespace rsb

using namespace rsb;

struct rsb_rowconv_plan {
    RowKParams kp;
    int cblk, block_n, mode, grid, smem;
    bool split;
};

template <int CBLK, int BLOCK_N, int MODE, int TAPS, int CBLOCKS, int NSUB, bool SPLIT = false>
static int launch_row(const rsb_rowconv_plan* plan, cudaStream_t stream) {
    auto kern = conv_row_kernel<CBLK, BLOCK_N, MODE, TAPS, CBLOCKS, NSUB, SPLIT>;
    static int attr_smem[64] = {};  // per device
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (plan->smem > attr_smem[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, plan->smem);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(conv_row)");
        attr_smem[dev] = plan->smem;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(plan->grid);
    cfg.blockDim = dim3(kRowThreads);
    cfg.dynamicSmemBytes = plan->smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, plan->kp);
    if (e != cudaSuccess) return set_cuda_error(e, "conv_row_kernel launch");
    return RSB_OK;
}

extern "C" int rsb_rowconv_plan_create(const rsb_rowconv_desc* d, rsb_rowconv_plan** out_plan) {
    if (!d || !out_plan) return set_error(RSB_E_INVALID, "rowconv: null argument");
    *out_plan = nullptr;
    if (!(d->cin == 32 || d->cin == 64 || d->cin == 128)) return set_error(RSB_E_INVALID, "rowconv: cin must be 32, 64 or 128");
    if (!(d->Cout == 32 || d->Cout == 64)) return set_error(RSB_E_INVALID, "rowconv: Cout must be 32 or 64");
    if (d->taps_h != d->taps_w || (d->taps_h != 2 && d->taps_h != 3)) return set_error(RSB_E_INVALID, "rowconv: taps must be 3x3 or 2x2");
    if (d->nsub < 1 || d->nsub > 2 || d->nphase_a < 1 || d->nphase_a > 2) return set_error(RSB_E_INVALID, "rowconv: nsub / nphase_a must be 1 or 2");
    const int cblk = d->cin == 32 ? 32 : 64;
    const int cblocks = d->cin / cblk;
    if (d->nsub * d->taps_h * d->taps_w * cblocks > kRowMaxW) return set_error(RSB_E_INVALID, "rowconv: too many weight blocks");
    if (d->Wt < 1 || d->Ht < 1 || d->Nt < 1 || !d->weights || !d->src.ptr) return set_error(RSB_E_INVALID, "rowconv: bad geometry / pointers");
    if (d->mode == 1 && (d->Cout != 32 || d->nsub != 1 || d->nphase_a != 1 || d->head_classes < 1 || d->head_classes > 8 || !d->head_w || !d->head_b || !d->head_out))
        return set_error(RSB_E_INVALID, "rowconv: bad head arguments");
    if (d->mode == 0 && !d->out) return set_error(RSB_E_INVALID, "rowconv: null out");
    const bool split = d->split != 0;
    if (split && !(d->mode == 1 && d->cin == 32 && d->taps_h == 3 && d->src.plane > 0 && (d->src.plane * 2) % 16 == 0))
        return set_error(RSB_E_INVALID, "rowconv: the strict-precision line buffer exists for the 3x3 32 -> 32 head layer only (needs src.plane)");
    const int planes = split ? 2 : 1;
    // shared memory: the resident weights and the epilogue staging are fixed, the ring of input rows takes the rest and needs
    // taps_h + 1 rows (e.g. the fused upsample 128 -> 64 does not fit: its weights alone take 128 KB)
    const int buf_w = kRowTile + d->taps_w + d->nsub - 2;
    const int slot_bytes = ((buf_w * cblk * 2 + 1023) / 1024) * 1024;
    const int wblock_bytes = planes * d->Cout * cblk * 2;
    const int stage = d->mode == 0 ? 2 * 2 * 64 * (d->Cout >= 64 ? 64 : 32) * 2 : 0;
    const int fixed = d->nsub * d->taps_h * d->taps_w * cblocks * wblock_bytes + stage + 512 + 1088 + 1024;
    const int row_bytes = slot_bytes * cblocks * planes;
    const int ctas = 1;  // the two consumer warpgroups of one CTA take the whole register file
    int slots = (232448 / ctas - 1024 - fixed) / row_bytes;
    if (slots > kRowMaxSlots) slots = kRowMaxSlots;
    if (slots < d->taps_h + 1)
        return set_error(RSB_E_INVALID, "rowconv: needs %d bytes of shared memory for a %d-row ring", fixed + (d->taps_h + 1) * row_bytes, d->taps_h + 1);
    int rc = rsb_device_ok();
    if (rc) return rc;

    rsb_rowconv_plan* plan = new (std::nothrow) rsb_rowconv_plan();
    if (!plan) return set_error(RSB_E_INVALID, "rowconv: out of host memory");
    memset(&plan->kp, 0, sizeof(plan->kp));
    RowKParams& kp = plan->kp;
    kp.taps_h = d->taps_h;
    kp.taps_w = d->taps_w;
    kp.cblocks = cblocks;
    kp.nsub = d->nsub;
    kp.nphase_a = d->nphase_a;
    kp.dh0 = d->dh0;
    kp.dw0 = d->dw0;
    kp.buf_w = buf_w;
    kp.slot_bytes = slot_bytes;
    kp.wblock_bytes = wblock_bytes;
    kp.plane_bytes = kp.slot_bytes * cblocks;
    kp.acc_scale = d->acc_scale != 0.f ? d->acc_scale : 1.f;
    kp.Wt = d->Wt;
    kp.Ht = d->Ht;
    kp.Nt = d->Nt;
    kp.Cout = d->Cout;
    kp.wstrips = (d->Wt + kRowTile - 1) / kRowTile;
    kp.rows_per_unit = d->rows_per_unit;  // 0: chosen below, once the number of resident CTAs is known
    kp.relu = d->relu;
    kp.bias = d->bias;
    kp.head_classes = d->head_classes;
    kp.head_w = d->head_w;
    kp.head_b = d->head_b;
    kp.head_out = d->head_out;
    const int swz = cblk * 2;  // 64-byte or 128-byte swizzle
    {
        const rsb_conv_src& s = d->src;
        const uint64_t dims[5] = {(uint64_t)d->cin, (uint64_t)s.W, (uint64_t)s.H, (uint64_t)s.N, 2};
        const uint64_t strides[4] = {(uint64_t)s.pitch_w * 2, (uint64_t)s.pitch_h * 2, (uint64_t)s.pitch_n * 2, (uint64_t)s.plane * 2};
        const uint32_t box[5] = {(uint32_t)cblk, (uint32_t)kp.buf_w, 1, 1, 1};  // strict: one plane per load (each lands 1024-aligned)
        rc = encode_tiled_f16(&kp.tmA, split ? 5 : 4, s.ptr, dims, strides, box, swz);
    }
    if (!rc) {
        const int K = d->taps_h * d->taps_w * d->cin;
        const uint64_t rows = (uint64_t)d->nphase_a * d->nsub * d->Cout;
        const uint64_t dims[3] = {(uint64_t)K, rows, 2};
        const uint64_t strides[2] = {(uint64_t)K * 2, rows * (uint64_t)K * 2};
        const uint32_t box[3] = {(uint32_t)cblk, (uint32_t)d->Cout, 2};  // strict: [W_hi rows | W_lo rows] back to back
        rc = encode_tiled_f16(&kp.tmB, split ? 3 : 2, d->weights, dims, strides, box, swz);
    }
    if (!rc && d->mode == 0) {
        const int sy = d->out_sy > 0 ? d->out_sy : 1, sx = d->out_sx > 0 ? d->out_sx : 1;
        const int chunk = d->Cout >= 64 ? 64 : 32;
        const uint64_t dims[4] = {(uint64_t)d->Cout, (uint64_t)d->Wt, (uint64_t)d->Ht, (uint64_t)d->Nt};
        const uint64_t strides[3] = {(uint64_t)sx * d->out_pitch_w * 2, (uint64_t)sy * d->out_pitch_h * 2, (uint64_t)d->out_pitch_n * 2};
        const uint32_t box[4] = {(uint32_t)chunk, 64, 1, 1};  // one warpgroup's 64 pixels
        const int nph = d->nphase_a * d->nsub > 1 ? 4 : 1;
        for (int ph = 0; ph < 4 && !rc; ++ph) {
            const int a = ph >> 1, b = ph & 1;
            const __half* base = static_cast<const __half*>(d->out) + (ph < nph ? a * d->out_pitch_h + b * d->out_pitch_w : 0);
            rc = encode_tiled_f16(&kp.tmC[ph], 4, base, dims, strides, box, chunk * 2);
        }
    } else if (!rc) {
        for (int ph = 0; ph < 4; ++ph) kp.tmC[ph] = kp.tmA;
    }
    if (rc) {
        delete plan;
        return rc;
    }
    plan->cblk = cblk;
    plan->block_n = d->Cout;
    plan->mode = d->mode;
    plan->split = split;
    kp.slots = slots;
    plan->smem = slots * row_bytes + fixed;
    const int sms = num_sms();
    if (kp.rows_per_unit <= 0) {
        // units of consecutive rows: as long as possible (halo rows, ring refill) while still filling every resident CTA
        kp.rows_per_unit = 8;
        for (int r = 32; r >= 8; r /= 2) {
            const int units = d->Nt * kp.wstrips * ((d->Ht + r - 1) / r) * d->nphase_a;
            if (4 * units >= 3 * ctas * sms) {
                kp.rows_per_unit = r;
                break;
            }
        }
    }
    kp.rchunks = (d->Ht + kp.rows_per_unit - 1) / kp.rows_per_unit;
    kp.total_units = d->Nt * kp.wstrips * kp.rchunks * d->nphase_a;
    plan->grid = kp.total_units < ctas * sms ? kp.total_units : ctas * sms;
    if (d->nphase_a == 2 && plan->grid > 1) plan->grid &= ~1;  // even grid: a CTA's units all have the same row phase
    *out_plan = plan;
    return RSB_OK;
}

extern "C" void rsb_rowconv_plan_destroy(rsb_rowconv_plan* plan) { delete plan; }

extern "C" int rsb_rowconv_run(const rsb_rowconv_plan* plan, void* stream_) {
    if (!plan) return set_error(RSB_E_INVALID, "rowconv: null plan");
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const RowKParams& k = plan->kp;
    const int key = ((((plan->cblk * 100 + plan->block_n) * 10 + plan->mode) * 10 + k.taps_h) * 10 + k.cblocks) * 10 + k.nsub;
    if (plan->split) {
        if (key == 32321311) return launch_row<32, 32, 1, 3, 1, 1, true>(plan, st);  // dec5 + final, strict precision
        return set_error(RSB_E_INVALID, "rowconv: no strict-precision kernel instance for this layer");
    }
    switch (key) {  // CBLK BLOCK_N MODE TAPS CBLOCKS NSUB
        case 32321311: return launch_row<32, 32, 1, 3, 1, 1>(plan, st);  // dec5 + final
        case 64321311: return launch_row<64, 32, 1, 3, 1, 1>(plan, st);
        case 32320311: return launch_row<32, 32, 0, 3, 1, 1>(plan, st);  // 3x3, 32 -> 32
        case 64640311: return launch_row<64, 64, 0, 3, 1, 1>(plan, st);  // layer1 3x3
        case 64320311: return launch_row<64, 32, 0, 3, 1, 1>(plan, st);
        case 64320222: return launch_row<64, 32, 0, 2, 2, 2>(plan, st);  // dec4: fused upsample 128 -> 32
        case 64640212: return launch_row<64, 64, 0, 2, 1, 2>(plan, st);  // fused upsample 64 -> 64
        case 64320212: return launch_row<64, 32, 0, 2, 1, 2>(plan, st);
        // no fused upsample 128 -> 64: its resident weights leave no room for the row ring (rsb_rowconv_plan_create)
    }
    return set_error(RSB_E_INVALID, "rowconv: no kernel instance for cblk %d, Cout %d, mode %d, taps %d, cblocks %d, nsub %d", plan->cblk,
                     plan->block_n, plan->mode, k.taps_h, k.cblocks, k.nsub);
}
