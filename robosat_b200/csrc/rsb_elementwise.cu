// HBM-bound helper kernels around the convolution path: input pre-pass (normalise + space-to-depth),
// NHWC max pooling, the predict head (softmax -> foreground -> quantise -> crop) and a generic softmax.
// All are single-pass, 16-byte vectorised where the layout allows, grid sized from the element count.

#include <cuda_fp16.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

namespace rsb {

struct Norm3 {
    float mean[3];
    float inv_std[3];
    float std[3];
};

// dst fp16 [N][H2][W2 + 4][16]; one thread per (n, hh, padded column)
// SPLIT: also write the lo plane (dst + plane) holding half(x - float(half(x))): the strict-precision operand pair
template <int SRC_KIND, bool SPLIT>
__global__ void prepass_s2d_kernel(const void* __restrict__ src, __half* __restrict__ dst, int64_t plane, int N, int H, int W, Norm3 nm) {
    const int H2 = H / 2, W2 = W / 2, Wp = W2 + 4;
    const int64_t total = static_cast<int64_t>(N) * H2 * Wp;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int wp = static_cast<int>(gid % Wp);
    const int hh = static_cast<int>((gid / Wp) % H2);
    const int n = static_cast<int>(gid / (static_cast<int64_t>(Wp) * H2));
    __align__(16) __half v[16];
    __align__(16) __half l[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = l[i] = __float2half_rn(0.f);
    const int ww = wp - 2;
    if (ww >= 0 && ww < W2) {
#pragma unroll
        for (int ph = 0; ph < 2; ++ph) {
            const int h = 2 * hh + ph;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float x0, x1;
                if (SRC_KIND == 0) {
                    const float* s = static_cast<const float*>(src) + ((static_cast<int64_t>(n) * 3 + c) * H + h) * W + 2 * ww;
                    const float2 f = *reinterpret_cast<const float2*>(s);
                    x0 = f.x;
                    x1 = f.y;
                } else {
                    const uint8_t* s = static_cast<const uint8_t*>(src) + ((static_cast<int64_t>(n) * H + h) * W + 2 * ww) * 3 + c;
                    // ToTensor (u8 / 255) then Normalize ((x - mean) / std), both in fp32 like the reference
                    x0 = (static_cast<float>(s[0]) / 255.0f - nm.mean[c]) / nm.std[c];
                    x1 = (static_cast<float>(s[3]) / 255.0f - nm.mean[c]) / nm.std[c];
                }
                const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
                v[(ph * 2 + 0) * 3 + c] = h0;
                v[(ph * 2 + 1) * 3 + c] = h1;
                if (SPLIT) {
                    l[(ph * 2 + 0) * 3 + c] = __float2half_rn(x0 - __half2float(h0));
                    l[(ph * 2 + 1) * 3 + c] = __float2half_rn(x1 - __half2float(h1));
                }
            }
        }
    }
    uint4* o = reinterpret_cast<uint4*>(dst + gid * 16);
    o[0] = *reinterpret_cast<const uint4*>(&v[0]);
    o[1] = *reinterpret_cast<const uint4*>(&v[8]);
    if (SPLIT) {
        uint4* ol = reinterpret_cast<uint4*>(dst + plane + gid * 16);
        ol[0] = *reinterpret_cast<const uint4*>(&l[0]);
        ol[1] = *reinterpret_cast<const uint4*>(&l[8]);
    }
}

// NHWC fp16 max pool, 8 channels (16 bytes) per thread
__global__ void maxpool_nhwc_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int N, int H, int W, int C,
                                    int k, int s, int p, int OH, int OW) {
    const int C8 = C / 8;
    const int64_t total = static_cast<int64_t>(N) * OH * OW * C8;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int c8 = static_cast<int>(gid % C8);
    int64_t r = gid / C8;
    const int ow = static_cast<int>(r % OW);
    r /= OW;
    const int oh = static_cast<int>(r % OH);
    const int n = static_cast<int>(r / OH);
    __half2 m[4];
    const __half2 ninf = __float2half2_rn(-65504.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) m[i] = ninf;
    for (int dy = 0; dy < k; ++dy) {
        const int h = oh * s - p + dy;
        if (h < 0 || h >= H) continue;
        for (int dx = 0; dx < k; ++dx) {
            const int w = ow * s - p + dx;
            if (w < 0 || w >= W) continue;
            const uint4 q = __ldg(reinterpret_cast<const uint4*>(src + ((static_cast<int64_t>(n) * H + h) * W + w) * C + c8 * 8));
            const __half2* h2 = reinterpret_cast<const __half2*>(&q);
#pragma unroll
            for (int i = 0; i < 4; ++i) m[i] = __hmax2(m[i], h2[i]);
        }
    }
    *reinterpret_cast<uint4*>(dst + ((static_cast<int64_t>(n) * OH + oh) * OW + ow) * C + c8 * 8) = *reinterpret_cast<uint4*>(m);
}

// Strict precision: values are (hi, lo) fp16 pairs; hi + lo is exact in fp32 and order-preserving, so the maximum is taken
// on the fp32 sums and split again (the split of a value that came from a pair reproduces that pair).
__global__ void maxpool_nhwc_split_kernel(const __half* __restrict__ src, int64_t src_plane, __half* __restrict__ dst, int64_t dst_plane,
                                          int N, int H, int W, int C, int k, int s, int p, int OH, int OW) {
    const int C8 = C / 8;
    const int64_t total = static_cast<int64_t>(N) * OH * OW * C8;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int c8 = static_cast<int>(gid % C8);
    int64_t r = gid / C8;
    const int ow = static_cast<int>(r % OW);
    r /= OW;
    const int oh = static_cast<int>(r % OH);
    const int n = static_cast<int>(r / OH);
    float m[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = -3.0e38f;
    for (int dy = 0; dy < k; ++dy) {
        const int h = oh * s - p + dy;
        if (h < 0 || h >= H) continue;
        for (int dx = 0; dx < k; ++dx) {
            const int w = ow * s - p + dx;
            if (w < 0 || w >= W) continue;
            const int64_t off = ((static_cast<int64_t>(n) * H + h) * W + w) * C + c8 * 8;
            const uint4 q = __ldg(reinterpret_cast<const uint4*>(src + off));
            const uint4 ql = __ldg(reinterpret_cast<const uint4*>(src + src_plane + off));
            const __half2* h2 = reinterpret_cast<const __half2*>(&q);
            const __half2* l2 = reinterpret_cast<const __half2*>(&ql);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 a = __half22float2(h2[i]), b = __half22float2(l2[i]);
                m[2 * i] = fmaxf(m[2 * i], a.x + b.x);
                m[2 * i + 1] = fmaxf(m[2 * i + 1], a.y + b.y);
            }
        }
    }
    __align__(16) __half hi[8];
    __align__(16) __half lo[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        hi[i] = __float2half_rn(m[i]);
        lo[i] = __float2half_rn(m[i] - __half2float(hi[i]));
    }
    const int64_t o = ((static_cast<int64_t>(n) * OH + oh) * OW + ow) * C + c8 * 8;
    *reinterpret_cast<uint4*>(dst + o) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(dst + dst_plane + o) = *reinterpret_cast<const uint4*>(lo);
}

// Training-side augmentation on the device (robosat/transforms.py:127-221 as composed by train.py:253-258): per sample an optional
// left-right flip followed by k counter-clockwise quarter turns (PIL's FLIP_LEFT_RIGHT / ROTATE_90), applied identically to the
// RGB tile and its mask. op = flip | (k << 1). One thread per output pixel: 3 image bytes + 1 mask label (widened to int64, the
// dtype the losses take -- MaskToTensor's job in the reference). Tiles are H x W; when H != W only the flip bit of an op is used.
__global__ void augment_dihedral_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask, const int32_t* __restrict__ ops,
                                        uint8_t* __restrict__ out_img, int64_t* __restrict__ out_mask, int N, int H, int W) {
    const int64_t total = static_cast<int64_t>(N) * H * W;
    for (int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; gid < total; gid += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(gid % W);
        const int y = static_cast<int>((gid / W) % H);
        const int n = static_cast<int>(gid / (static_cast<int64_t>(H) * W));
        const int op = ops[n] & (H == W ? 7 : 1);  // a non-square tile can only be flipped
        int sy = y, sx = x;
        for (int k = (op >> 1) & 3; k > 0; --k) {  // undo the quarter turns: ROTATE_90 writes out[y][x] = in[x][S-1-y]
            const int t = sy;
            sy = sx;
            sx = W - 1 - t;
        }
        if (op & 1) sx = W - 1 - sx;               // undo the flip: out[y][x] = in[y][W-1-x]
        const int64_t src = (static_cast<int64_t>(n) * H + sy) * W + sx;
        const uint8_t* s3 = img + src * 3;
        uint8_t* d3 = out_img + gid * 3;
        d3[0] = s3[0];
        d3[1] = s3[1];
        d3[2] = s3[2];
        if (mask) out_mask[gid] = static_cast<int64_t>(mask[src]);
    }
}

// number of anchors of np.linspace(0, 1, 256) that are <= x, compared in float64 like np.digitize does
__device__ __forceinline__ int digitize256(float xf) {
    const double x = static_cast<double>(xf);
    const double step = 1.0 / 255.0;
    int k = static_cast<int>(floor(x * 255.0));
    k = k < 0 ? 0 : (k > 255 ? 255 : k);
    // anchor(j) = j * step for j < 255, anchor(255) = 1.0 exactly (linspace pins the endpoint)
    auto anchor = [&](int j) { return j >= 255 ? 1.0 : static_cast<double>(j) * step; };
    while (k < 255 && anchor(k + 1) <= x) ++k;
    while (k >= 0 && anchor(k) > x) --k;
    return k + 1;  // count of anchors <= x (0 when x < 0, 256 when x >= 1)
}

__global__ void head_quantize_kernel(const float* __restrict__ logits, uint8_t* __restrict__ quant, float* __restrict__ probs_fg,
                                     int N, int H, int W, int o) {
    const int OH = H - 2 * o, OW = W - 2 * o;
    const int64_t total = static_cast<int64_t>(N) * OH * OW;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int x = static_cast<int>(gid % OW);
    const int y = static_cast<int>((gid / OW) % OH);
    const int n = static_cast<int>(gid / (static_cast<int64_t>(OW) * OH));
    const int64_t hw = static_cast<int64_t>(H) * W;
    const int64_t pix = static_cast<int64_t>(y + o) * W + (x + o);
    const float l0 = logits[(static_cast<int64_t>(n) * 2 + 0) * hw + pix];
    const float l1 = logits[(static_cast<int64_t>(n) * 2 + 1) * hw + pix];
    // softmax over 2 classes, max-subtracted like torch.softmax
    const float m = fmaxf(l0, l1);
    const float e0 = expf(l0 - m), e1 = expf(l1 - m);
    const float pfg = e1 / (e0 + e1);
    if (probs_fg) probs_fg[gid] = pfg;
    quant[gid] = static_cast<uint8_t>(digitize256(pfg));  // 256 wraps to 0 exactly like .astype(np.uint8)
}

// Test-time augmentation head. View v of tile b is logits sample v*B + b, computed from the tile transformed by op v
// (rsb_augment_dihedral's encoding), so pixel p of the tile's cropped output sits at forward(op, p) in that view. Probabilities
// are summed as int64 fixed point (one = 2^59): integer addition is associative, so the sum is the same bit for bit whatever
// the order of the views and however they are split over calls.
constexpr double kTtaOne = 576460752303423488.0;  // 2^59

struct TtaOps {
    int32_t op[RSB_TTA_MAX_VIEWS];
};

// where pixel (y, x) of an OH x OW crop lies after a left-right flip (op & 1) and k = op >> 1 counter-clockwise quarter turns.
// The crop is centred, so this is also the map of the whole tile restricted to it. Odd k needs OH == OW.
__device__ __forceinline__ void tta_forward_map(int op, int OH, int OW, int y, int x, int& vy, int& vx) {
    if (op & 1) x = OW - 1 - x;
    switch ((op >> 1) & 3) {
        case 0: vy = y; vx = x; break;
        case 1: vy = OW - 1 - x; vx = y; break;   // ROTATE_90: out[y][x] = in[x][S-1-y]
        case 2: vy = OH - 1 - y; vx = OW - 1 - x; break;
        default: vy = x; vx = OH - 1 - y; break;
    }
}

// One block per TW x TW window of one tile's cropped output. Per view, the block stages the matching TW x TW window of the view's
// logits (all C classes) in shared memory with row-contiguous global reads, so the transposed views read HBM as coalesced as the
// identity view; the padded pitch keeps the transposed shared-memory reads free of bank conflicts. Each thread keeps the sums of
// its own pixels in shared memory across the views and writes them once.
__global__ void head_tta_accumulate_kernel(const float* __restrict__ logits, int64_t* __restrict__ acc, TtaOps ops, int V, int B, int C,
                                           int H, int W, int o, int TW, int accumulate) {
    extern __shared__ __align__(16) unsigned char tta_smem[];
    const int OH = H - 2 * o, OW = W - 2 * o;
    const int pitch = TW + 1, npix = TW * TW;
    int64_t* sum = reinterpret_cast<int64_t*>(tta_smem);     // [C][TW * TW]
    float* win = reinterpret_cast<float*>(sum + C * npix);    // [C][TW][TW + 1]
    const int b = blockIdx.z, Y0 = blockIdx.y * TW, X0 = blockIdx.x * TW;
    const int64_t hw = static_cast<int64_t>(H) * W;
    const int cstride = TW * pitch;
    for (int v = 0; v < V; ++v) {
        const int op = ops.op[v];
        int ay, ax, by, bx;  // the view window is the box spanned by the images of the output window's corners
        tta_forward_map(op, OH, OW, Y0, X0, ay, ax);
        tta_forward_map(op, OH, OW, Y0 + TW - 1, X0 + TW - 1, by, bx);
        const int vy0 = min(ay, by), vx0 = min(ax, bx);
        const float* src = logits + static_cast<int64_t>(v * B + b) * C * hw;
        for (int i = threadIdx.x; i < C * npix; i += blockDim.x) {
            const int c = i / npix, r = (i / TW) % TW, col = i % TW;
            const int vy = vy0 + r, vx = vx0 + col;
            if (vy >= 0 && vy < OH && vx >= 0 && vx < OW) win[c * cstride + r * pitch + col] = src[c * hw + static_cast<int64_t>(vy + o) * W + (vx + o)];
        }
        __syncthreads();
        for (int i = threadIdx.x; i < npix; i += blockDim.x) {
            const int y = Y0 + i / TW, x = X0 + i % TW;
            if (y >= OH || x >= OW) continue;
            int vy, vx;
            tta_forward_map(op, OH, OW, y, x, vy, vx);
            const float* l = win + (vy - vy0) * pitch + (vx - vx0);
            // softmax as head_quantize_kernel / softmax_nchw_kernel compute it (max-subtracted expf; for C = 2, e1 / (e0 + e1))
            float m = l[0];
            for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * cstride]);
            float s = 0.f;
            for (int c = 0; c < C; ++c) s += expf(l[c * cstride] - m);
            for (int c = 0; c < C; ++c) {
                const int64_t q = llrint(static_cast<double>(expf(l[c * cstride] - m) / s) * kTtaOne);
                int64_t& a = sum[c * npix + i];
                a = v == 0 ? q : a + q;
            }
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < npix; i += blockDim.x) {
        const int y = Y0 + i / TW, x = X0 + i % TW;
        if (y >= OH || x >= OW) continue;
        for (int c = 0; c < C; ++c) {
            int64_t* d = acc + (static_cast<int64_t>(b * C + c) * OH + y) * OW + x;
            *d = accumulate ? *d + sum[c * npix + i] : sum[c * npix + i];
        }
    }
}

// mean foreground probability of `views` summed views (class 1 of a 2-class acc [N][2][HW]) -> np.digitize bins
__global__ void head_tta_quantize_kernel(const int64_t* __restrict__ acc, uint8_t* __restrict__ quant, int N, int64_t HW, int views) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int64_t n = gid / HW, pix = gid % HW;
    const float pfg = static_cast<float>(static_cast<double>(acc[(n * 2 + 1) * HW + pix]) * (1.0 / kTtaOne) / views);
    quant[gid] = static_cast<uint8_t>(digitize256(pfg));
}

// class index of the largest summed probability (the largest mean), first maximum wins like np.argmax
__global__ void head_tta_argmax_kernel(const int64_t* __restrict__ acc, uint8_t* __restrict__ mask, int N, int C, int64_t HW) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int64_t n = gid / HW, pix = gid % HW;
    const int64_t* a = acc + n * C * HW + pix;
    int64_t m = a[0];
    int best = 0;
    for (int c = 1; c < C; ++c) {
        const int64_t v = a[c * HW];
        if (v > m) {
            m = v;
            best = c;
        }
    }
    mask[gid] = static_cast<uint8_t>(best);
}

// Halo stitch (robosat/tiles.py:162-227 `buffer_tile_image`): canvas pixel (Y, X) of the (S+2o)^2 buffered tile comes from the
// centre tile or one of its 8 neighbours, all resident in a device tile cache [slot][S][S][3] uint8; a missing neighbour
// (slot < 0) leaves nodata = 0. One thread per 4 canvas bytes of a row (rows are 3*(S+2o) bytes; S, o multiples of 4).
__global__ void stitch_halo_kernel(const uint8_t* __restrict__ cache, const int32_t* __restrict__ slots, uint8_t* __restrict__ out, int B, int S,
                                   int o) {
    const int F = S + 2 * o;
    const int row_words = F * 3 / 4;
    const int64_t total = static_cast<int64_t>(B) * F * row_words;
    for (int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; gid < total; gid += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int wq = static_cast<int>(gid % row_words);
        const int Y = static_cast<int>((gid / row_words) % F);
        const int b = static_cast<int>(gid / (static_cast<int64_t>(row_words) * F));
        const int dy = Y < o ? -1 : (Y < o + S ? 0 : 1);
        const int sy = Y - o - dy * S;
        uint32_t word = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int byte = wq * 4 + k;  // byte inside the canvas row
            const int X = byte / 3, c = byte - X * 3;
            const int dx = X < o ? -1 : (X < o + S ? 0 : 1);
            const int sx = X - o - dx * S;
            const int slot = slots[b * 9 + (dy + 1) * 3 + (dx + 1)];
            uint32_t v = 0;
            if (slot >= 0) v = cache[((static_cast<int64_t>(slot) * S + sy) * S + sx) * 3 + c];
            word |= v << (8 * k);
        }
        reinterpret_cast<uint32_t*>(out)[gid] = word;
    }
}

// Same, 4 pixels (12 bytes = three 32-bit words) per thread: with S and o multiples of 4 a group never straddles two source
// tiles and both addresses are 4-byte aligned.
__global__ void stitch_halo_x4_kernel(const uint8_t* __restrict__ cache, const int32_t* __restrict__ slots, uint8_t* __restrict__ out, int B, int S,
                                      int o) {
    const int F = S + 2 * o;
    const int groups = F / 4;
    const int64_t total = static_cast<int64_t>(B) * F * groups;
    for (int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; gid < total; gid += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int X = static_cast<int>(gid % groups) * 4;
        const int Y = static_cast<int>((gid / groups) % F);
        const int b = static_cast<int>(gid / (static_cast<int64_t>(groups) * F));
        const int dy = Y < o ? -1 : (Y < o + S ? 0 : 1);
        const int dx = X < o ? -1 : (X < o + S ? 0 : 1);
        const int sy = Y - o - dy * S, sx = X - o - dx * S;
        const int slot = slots[b * 9 + (dy + 1) * 3 + (dx + 1)];
        uint32_t w0 = 0, w1 = 0, w2 = 0;
        if (slot >= 0) {
            const uint32_t* src = reinterpret_cast<const uint32_t*>(cache + ((static_cast<int64_t>(slot) * S + sy) * S + sx) * 3);
            w0 = __ldg(src);
            w1 = __ldg(src + 1);
            w2 = __ldg(src + 2);
        }
        uint32_t* dst = reinterpret_cast<uint32_t*>(out + ((static_cast<int64_t>(b) * F + Y) * F + X) * 3);
        dst[0] = w0;
        dst[1] = w1;
        dst[2] = w2;
    }
}

// `rs masks` (robosat/tools/masks.py:42-84): un-quantise K probability maps (`anchors[q]`, anchors = np.linspace(0, 1, 256)),
// weighted-average them (np.average over the model axis) and take the arg-max of [background, foreground]. All arithmetic in
// float64 in numpy's order (products rounded, sequential sum over the K inputs, one division by the weight sum / count), so
// the result is bit-identical, including ties (arg-max returns the first maximum = background).
__global__ void softvote_kernel(const uint8_t* __restrict__ quant, const double* __restrict__ weights, uint8_t* __restrict__ mask, int K, int64_t n) {
    const double step = 1.0 / 255.0;
    double scl = 0.0;
    for (int k = 0; k < K; ++k) scl += weights ? weights[k] : 1.0;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        double fs = 0.0, bs = 0.0;
        for (int k = 0; k < K; ++k) {
            const int q = quant[static_cast<int64_t>(k) * n + i];
            const double f = q >= 255 ? 1.0 : static_cast<double>(q) * step;  // linspace pins its last anchor to 1.0
            const double b = 1.0 - f;
            if (weights) {
                // separate IEEE multiply and add, as numpy does (no FMA contraction: it would change the last bit and flip ties)
                fs = __dadd_rn(fs, __dmul_rn(f, weights[k]));
                bs = __dadd_rn(bs, __dmul_rn(b, weights[k]));
            } else {
                fs += f;
                bs += b;
            }
        }
        mask[i] = (fs / scl > bs / scl) ? 1 : 0;
    }
}

// Softmax of one pixel over C classes, as torch.softmax and head_tta_accumulate_kernel compute it: m = fmaxf over the classes in
// order, s = the class-ordered sum of expf(l_c - m); then p_c = expf(l_c - m) / s (`softmax_prob`). `l` points at class 0 of the
// pixel, classes `cstride` floats apart. For C = 2 this is head_quantize_kernel's e1 / (e0 + e1) bit for bit (0 + e0 == e0).
__device__ __forceinline__ void softmax_pixel(const float* __restrict__ l, int64_t cstride, int C, float& m, float& s) {
    m = __ldg(l);
    for (int c = 1; c < C; ++c) m = fmaxf(m, __ldg(l + c * cstride));
    s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(__ldg(l + c * cstride) - m);
}

__device__ __forceinline__ float softmax_prob(float l, float m, float s) { return expf(l - m) / s; }

// `rs predict` for C classes: softmax -> crop `o` -> np.digitize of every class plane. One thread per 4 adjacent pixels of a cropped
// row: the three class-ordered passes re-read the thread's own logits (cache hits; HBM sees each logit once), and each plane's 4
// bins go out as one 32-bit word when the cropped width is a multiple of 4 (`vec`), else as single bytes.
__global__ void head_quantize_classes_kernel(const float* __restrict__ logits, uint8_t* __restrict__ quant, float* __restrict__ probs, int N,
                                             int C, int H, int W, int o, int vec) {
    const int OH = H - 2 * o, OW = W - 2 * o;
    const int groups = (OW + 3) / 4;
    const int64_t total = static_cast<int64_t>(N) * OH * groups;
    const int64_t hw = static_cast<int64_t>(H) * W, ohw = static_cast<int64_t>(OH) * OW;
    for (int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; gid < total; gid += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int x0 = static_cast<int>(gid % groups) * 4;
        const int y = static_cast<int>((gid / groups) % OH);
        const int n = static_cast<int>(gid / (static_cast<int64_t>(groups) * OH));
        const int npx = min(4, OW - x0);
        const float* l = logits + static_cast<int64_t>(n) * C * hw + static_cast<int64_t>(y + o) * W + (x0 + o);
        float m[4], s[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (j < npx) softmax_pixel(l + j, hw, C, m[j], s[j]);
        const int64_t out0 = static_cast<int64_t>(n) * C * ohw + static_cast<int64_t>(y) * OW + x0;
        for (int c = 0; c < C; ++c) {
            const int64_t out = out0 + c * ohw;
            float p[4];
            uint32_t word = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                p[j] = j < npx ? softmax_prob(__ldg(l + c * hw + j), m[j], s[j]) : 0.f;
                word |= static_cast<uint32_t>(static_cast<uint8_t>(digitize256(p[j]))) << (8 * j);  // 256 wraps to 0 like .astype(np.uint8)
            }
            if (vec) {
                *reinterpret_cast<uint32_t*>(quant + out) = word;
                if (probs) *reinterpret_cast<float4*>(probs + out) = make_float4(p[0], p[1], p[2], p[3]);
            } else {
                for (int j = 0; j < npx; ++j) {
                    quant[out + j] = static_cast<uint8_t>(word >> (8 * j));
                    if (probs) probs[out + j] = p[j];
                }
            }
        }
    }
}

// every class of acc [N][C][HW] summed over `views` views -> np.digitize bins of (float)(acc * 2^-59 / views), as
// head_tta_quantize_kernel bins class 1
__global__ void head_tta_quantize_classes_kernel(const int64_t* __restrict__ acc, uint8_t* __restrict__ quant, int64_t total, int views) {
    for (int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; gid < total; gid += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float p = static_cast<float>(static_cast<double>(acc[gid]) * (1.0 / kTtaOne) / views);
        quant[gid] = static_cast<uint8_t>(digitize256(p));
    }
}

// `rs masks --dataset` for C classes: np.argmax(np.average(anchors[q], axis=0, weights=w), axis=0) over quant [K][C][n], float64 in
// numpy's order like softvote_kernel: per class a sequential sum over the K models (products rounded on their own), one division by
// the weight sum / K, then the first maximum. Dividing before comparing matters: it can round two different sums to one value.
__global__ void softvote_classes_kernel(const uint8_t* __restrict__ quant, const double* __restrict__ weights, uint8_t* __restrict__ mask, int K,
                                        int C, int64_t n) {
    const double step = 1.0 / 255.0;
    double scl = 0.0;
    for (int k = 0; k < K; ++k) scl += weights ? weights[k] : 1.0;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        double best = 0.0;
        int arg = 0;
        for (int c = 0; c < C; ++c) {
            double sum = 0.0;
            for (int k = 0; k < K; ++k) {
                const int q = quant[(static_cast<int64_t>(k) * C + c) * n + i];
                const double p = q >= 255 ? 1.0 : static_cast<double>(q) * step;  // linspace pins its last anchor to 1.0
                sum = weights ? __dadd_rn(sum, __dmul_rn(p, weights[k])) : sum + p;
            }
            const double avg = sum / scl;
            if (c == 0 || avg > best) {
                best = avg;
                arg = c;
            }
        }
        mask[i] = static_cast<uint8_t>(arg);
    }
}

// `rs weights` (robosat/tools/weights.py:39-49): np.bincount of the training masks, per class, accumulated over calls
__global__ void class_histogram_kernel(const uint8_t* __restrict__ labels, int64_t n, int C, unsigned long long* __restrict__ counts) {
    __shared__ unsigned int sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
        atomicAdd(&sh[labels[i]], 1u);
    __syncthreads();
    if (threadIdx.x < C && sh[threadIdx.x]) atomicAdd(&counts[threadIdx.x], static_cast<unsigned long long>(sh[threadIdx.x]));
    // labels >= C are counted in shared memory but dropped here; the host checks the total (np.bincount would grow instead)
}

// per-pixel class index of fp32 NCHW logits (first maximum wins, like np.argmax): the `rs serve` mask, serve.py:150-165
__global__ void head_argmax_kernel(const float* __restrict__ logits, uint8_t* __restrict__ mask, int N, int C, int64_t HW) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int64_t pix = gid % HW;
    const int64_t n = gid / HW;
    const float* l = logits + n * C * HW + pix;
    float m = l[0];
    int best = 0;
    for (int c = 1; c < C; ++c) {
        const float v = l[c * HW];
        if (v > m) {
            m = v;
            best = c;
        }
    }
    mask[gid] = static_cast<uint8_t>(best);
}

__global__ void softmax_nchw_kernel(const float* __restrict__ logits, float* __restrict__ probs, int N, int C, int64_t HW) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    const int64_t gid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int64_t pix = gid % HW;
    const int64_t n = gid / HW;
    const float* l = logits + n * C * HW + pix;
    float m = l[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * HW]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(l[c * HW] - m);
    float* o = probs + n * C * HW + pix;
    for (int c = 0; c < C; ++c) o[c * HW] = expf(l[c * HW] - m) / s;
}

static inline unsigned grid_for(int64_t total, int block) { return static_cast<unsigned>((total + block - 1) / block); }

}  // namespace rsb

using namespace rsb;

static int prepass_common(const void* src, int32_t src_kind, void* dst, int64_t plane, int32_t N, int32_t H, int32_t W,
                          const float* mean3_host, const float* std3_host, void* stream) {
    if (!src || !dst || N <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1)) return set_error(RSB_E_INVALID, "prepass: bad arguments");
    if (src_kind != 0 && src_kind != 1) return set_error(RSB_E_INVALID, "prepass: src_kind must be 0 (f32 NCHW) or 1 (u8 NHWC)");
    if (plane < 0 || (plane * 2) % 16) return set_error(RSB_E_INVALID, "prepass: plane stride must be a non-negative multiple of 8 elements");
    Norm3 nm;
    for (int c = 0; c < 3; ++c) {
        nm.mean[c] = mean3_host ? mean3_host[c] : 0.f;
        nm.std[c] = std3_host ? std3_host[c] : 1.f;
        nm.inv_std[c] = 1.f / nm.std[c];
    }
    const int64_t total = static_cast<int64_t>(N) * (H / 2) * (W / 2 + 4);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    __half* d = static_cast<__half*>(dst);
    if (plane > 0) {
        if (src_kind == 0) prepass_s2d_kernel<0, true><<<grid_for(total, 256), 256, 0, st>>>(src, d, plane, N, H, W, nm);
        else prepass_s2d_kernel<1, true><<<grid_for(total, 256), 256, 0, st>>>(src, d, plane, N, H, W, nm);
    } else {
        if (src_kind == 0) prepass_s2d_kernel<0, false><<<grid_for(total, 256), 256, 0, st>>>(src, d, 0, N, H, W, nm);
        else prepass_s2d_kernel<1, false><<<grid_for(total, 256), 256, 0, st>>>(src, d, 0, N, H, W, nm);
    }
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "prepass_s2d launch");
}

extern "C" int rsb_prepass_s2d(const void* src, int32_t src_kind, void* dst, int32_t N, int32_t H, int32_t W,
                               const float* mean3_host, const float* std3_host, void* stream) {
    return prepass_common(src, src_kind, dst, 0, N, H, W, mean3_host, std3_host, stream);
}

extern "C" int rsb_prepass_s2d_split(const void* src, int32_t src_kind, void* dst, int64_t plane, int32_t N, int32_t H, int32_t W,
                                     const float* mean3_host, const float* std3_host, void* stream) {
    if (plane <= 0) return set_error(RSB_E_INVALID, "prepass_split: plane stride must be positive");
    return prepass_common(src, src_kind, dst, plane, N, H, W, mean3_host, std3_host, stream);
}

extern "C" int rsb_maxpool_nhwc_split(const void* src, int64_t src_plane, void* dst, int64_t dst_plane, int32_t N, int32_t H, int32_t W,
                                      int32_t C, int32_t k, int32_t s, int32_t p, void* stream) {
    if (!src || !dst || N <= 0 || H <= 0 || W <= 0 || C <= 0 || (C % 8) || k < 1 || s < 1 || p < 0 || src_plane <= 0 || dst_plane <= 0 ||
        (src_plane % 8) || (dst_plane % 8))
        return set_error(RSB_E_INVALID, "maxpool_split: bad arguments (C and the plane strides must be multiples of 8)");
    const int OH = (H + 2 * p - k) / s + 1, OW = (W + 2 * p - k) / s + 1;
    const int64_t total = static_cast<int64_t>(N) * OH * OW * (C / 8);
    maxpool_nhwc_split_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __half*>(src), src_plane, static_cast<__half*>(dst), dst_plane, N, H, W, C, k, s, p, OH, OW);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "maxpool_split launch");
}

extern "C" int rsb_maxpool_nhwc(const void* src, void* dst, int32_t N, int32_t H, int32_t W, int32_t C, int32_t k, int32_t s,
                                int32_t p, void* stream) {
    if (!src || !dst || N <= 0 || H <= 0 || W <= 0 || C <= 0 || (C % 8) || k < 1 || s < 1 || p < 0)
        return set_error(RSB_E_INVALID, "maxpool: bad arguments (C must be a multiple of 8)");
    const int OH = (H + 2 * p - k) / s + 1, OW = (W + 2 * p - k) / s + 1;
    const int64_t total = static_cast<int64_t>(N) * OH * OW * (C / 8);
    maxpool_nhwc_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __half*>(src), static_cast<__half*>(dst), N, H, W, C, k, s, p, OH, OW);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "maxpool launch");
}

extern "C" int rsb_augment_dihedral(const uint8_t* img, const uint8_t* mask, const int32_t* ops, uint8_t* out_img, int64_t* out_mask, int32_t N,
                                    int32_t S, void* stream) {
    if (!img || !ops || !out_img || N <= 0 || S <= 0 || (mask && !out_mask)) return set_error(RSB_E_INVALID, "augment_dihedral: bad arguments");
    if (img == out_img) return set_error(RSB_E_INVALID, "augment_dihedral: cannot run in place");
    const int64_t total = static_cast<int64_t>(N) * S * S;
    augment_dihedral_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(img, mask, ops, out_img, out_mask, N, S, S);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "augment_dihedral launch");
}

extern "C" int rsb_augment_flip_rect(const uint8_t* img, const int32_t* ops, uint8_t* out_img, int32_t N, int32_t H, int32_t W, void* stream) {
    if (!img || !ops || !out_img || N <= 0 || H <= 0 || W <= 0) return set_error(RSB_E_INVALID, "augment_flip_rect: bad arguments");
    if (img == out_img) return set_error(RSB_E_INVALID, "augment_flip_rect: cannot run in place");
    const int64_t total = static_cast<int64_t>(N) * H * W;
    augment_dihedral_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(img, nullptr, ops, out_img, nullptr, N, H, W);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "augment_flip_rect launch");
}

// bytes of dynamic shared memory of head_tta_accumulate_kernel for a TW x TW window of C classes
static inline int tta_smem_bytes(int C, int TW) { return C * TW * TW * 8 + C * TW * (TW + 1) * 4; }

extern "C" int rsb_head_tta_accumulate(const float* logits, int64_t* acc, const int32_t* ops_host, int32_t views, int32_t B, int32_t C, int32_t H,
                                       int32_t W, int32_t overlap, int32_t accumulate, void* stream) {
    if (!logits || !acc || !ops_host || views < 1 || views > RSB_TTA_MAX_VIEWS || B <= 0 || C < 1 || C > 255 || overlap < 0 ||
        H - 2 * overlap <= 0 || W - 2 * overlap <= 0 || (accumulate != 0 && accumulate != 1))
        return set_error(RSB_E_INVALID, "head_tta_accumulate: bad arguments");
    TtaOps ops = {};
    for (int v = 0; v < views; ++v) {
        if (ops_host[v] < 0 || ops_host[v] > 7) return set_error(RSB_E_INVALID, "head_tta_accumulate: ops must be in 0..7");
        if (H != W && ((ops_host[v] >> 1) & 1)) return set_error(RSB_E_INVALID, "head_tta_accumulate: quarter turns need a square tile");
        ops.op[v] = ops_host[v];
    }
    // the widest window whose staging fits the default 48 KB of shared memory (32 x 32 up to C = 3)
    int TW = 32;
    while (TW > 1 && tta_smem_bytes(C, TW) > 48 * 1024) TW /= 2;
    const int OH = H - 2 * overlap, OW = W - 2 * overlap;
    const dim3 grid((OW + TW - 1) / TW, (OH + TW - 1) / TW, B);
    head_tta_accumulate_kernel<<<grid, 256, tta_smem_bytes(C, TW), static_cast<cudaStream_t>(stream)>>>(logits, acc, ops, views, B, C, H, W, overlap,
                                                                                                         TW, accumulate);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "head_tta_accumulate launch");
}

extern "C" int rsb_head_tta_quantize(const int64_t* acc, uint8_t* quant, int32_t B, int32_t HW, int32_t views, void* stream) {
    if (!acc || !quant || B <= 0 || HW <= 0 || views < 1) return set_error(RSB_E_INVALID, "head_tta_quantize: bad arguments");
    const int64_t total = static_cast<int64_t>(B) * HW;
    head_tta_quantize_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(acc, quant, B, HW, views);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "head_tta_quantize launch");
}

extern "C" int rsb_head_tta_argmax(const int64_t* acc, uint8_t* mask, int32_t B, int32_t C, int32_t HW, void* stream) {
    if (!acc || !mask || B <= 0 || C <= 0 || C > 255 || HW <= 0) return set_error(RSB_E_INVALID, "head_tta_argmax: bad arguments");
    const int64_t total = static_cast<int64_t>(B) * HW;
    head_tta_argmax_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(acc, mask, B, C, HW);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "head_tta_argmax launch");
}

extern "C" int rsb_head_quantize(const float* logits, uint8_t* quant, float* probs_fg, int32_t N, int32_t H, int32_t W,
                                 int32_t overlap, void* stream) {
    if (!logits || !quant || N <= 0 || overlap < 0 || H - 2 * overlap <= 0 || W - 2 * overlap <= 0)
        return set_error(RSB_E_INVALID, "head_quantize: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * (H - 2 * overlap) * (W - 2 * overlap);
    head_quantize_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(logits, quant, probs_fg, N, H, W, overlap);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "head_quantize launch");
}

extern "C" int rsb_stitch_halo(const uint8_t* cache, const int32_t* slots, uint8_t* out, int32_t B, int32_t S, int32_t overlap, void* stream) {
    if (!cache || !slots || !out || B <= 0 || S <= 0 || overlap < 0 || overlap > S || ((S + 2 * overlap) * 3) % 4)
        return set_error(RSB_E_INVALID, "stitch_halo: bad arguments ((S + 2*overlap)*3 must be a multiple of 4, overlap <= S)");
    const int F = S + 2 * overlap;
    const int64_t total = static_cast<int64_t>(B) * F * (F * 3 / 4);
    int64_t blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (S % 4 == 0 && overlap % 4 == 0 && (reinterpret_cast<uintptr_t>(cache) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0) {
        const int64_t groups = static_cast<int64_t>(B) * F * (F / 4);
        int64_t gblocks = (groups + 255) / 256;
        if (gblocks > 132 * 16) gblocks = 132 * 16;
        stitch_halo_x4_kernel<<<static_cast<unsigned>(gblocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(cache, slots, out, B, S, overlap);
    } else {
        stitch_halo_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(cache, slots, out, B, S, overlap);
    }
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "stitch_halo launch");
}

extern "C" int rsb_softvote(const uint8_t* quant, const double* weights, uint8_t* mask, int32_t K, int64_t n, void* stream) {
    if (!quant || !mask || K < 1 || n <= 0) return set_error(RSB_E_INVALID, "softvote: bad arguments");
    softvote_kernel<<<grid_for(n, 256) > 132 * 16 ? 132 * 16 : grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(quant, weights, mask, K, n);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "softvote launch");
}

extern "C" int rsb_head_quantize_classes(const float* logits, uint8_t* quant, float* probs, int32_t N, int32_t C, int32_t H, int32_t W,
                                         int32_t overlap, void* stream) {
    if (!logits || !quant || N <= 0 || C < 2 || C > 255 || overlap < 0 || H - 2 * overlap <= 0 || W - 2 * overlap <= 0)
        return set_error(RSB_E_INVALID, "head_quantize_classes: bad arguments (C must be 2..255, 2*overlap < H and W)");
    const int OH = H - 2 * overlap, OW = W - 2 * overlap;
    const int vec = OW % 4 == 0 && (reinterpret_cast<uintptr_t>(quant) & 3) == 0 && (reinterpret_cast<uintptr_t>(probs) & 15) == 0;
    const int64_t total = static_cast<int64_t>(N) * OH * ((OW + 3) / 4);
    const unsigned blocks = grid_for(total, 256) > 132 * 32 ? 132 * 32 : grid_for(total, 256);
    head_quantize_classes_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(logits, quant, probs, N, C, H, W, overlap, vec);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "head_quantize_classes launch");
}

extern "C" int rsb_head_tta_quantize_classes(const int64_t* acc, uint8_t* quant, int32_t B, int32_t C, int32_t HW, int32_t views, void* stream) {
    if (!acc || !quant || B <= 0 || C < 2 || C > 255 || HW <= 0 || views < 1) return set_error(RSB_E_INVALID, "head_tta_quantize_classes: bad arguments");
    const int64_t total = static_cast<int64_t>(B) * C * HW;
    const unsigned blocks = grid_for(total, 256) > 132 * 32 ? 132 * 32 : grid_for(total, 256);
    head_tta_quantize_classes_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(acc, quant, total, views);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "head_tta_quantize_classes launch");
}

extern "C" int rsb_softvote_classes(const uint8_t* quant, const double* weights, uint8_t* mask, int32_t K, int32_t C, int64_t n, void* stream) {
    if (!quant || !mask || K < 1 || C < 2 || C > 255 || n <= 0) return set_error(RSB_E_INVALID, "softvote_classes: bad arguments");
    softvote_classes_kernel<<<grid_for(n, 256) > 132 * 16 ? 132 * 16 : grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(quant, weights, mask,
                                                                                                                                  K, C, n);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "softvote_classes launch");
}

extern "C" int rsb_class_histogram(const uint8_t* labels, int64_t n, int32_t C, uint64_t* counts, void* stream) {
    if (!labels || !counts || n <= 0 || C < 1 || C > 256) return set_error(RSB_E_INVALID, "class_histogram: bad arguments");
    class_histogram_kernel<<<grid_for(n, 256) > 132 * 8 ? 132 * 8 : grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        labels, n, C, reinterpret_cast<unsigned long long*>(counts));
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "class_histogram launch");
}

extern "C" int rsb_head_argmax(const float* logits, uint8_t* mask, int32_t N, int32_t C, int32_t HW, void* stream) {
    if (!logits || !mask || N <= 0 || C <= 0 || C > 255 || HW <= 0) return set_error(RSB_E_INVALID, "head_argmax: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * HW;
    head_argmax_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(logits, mask, N, C, HW);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "head_argmax launch");
}

extern "C" int rsb_softmax_nchw(const float* logits, float* probs, int32_t N, int32_t C, int32_t HW, void* stream) {
    if (!logits || !probs || N <= 0 || C <= 0 || HW <= 0) return set_error(RSB_E_INVALID, "softmax: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * HW;
    softmax_nchw_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(logits, probs, N, C, HW);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "softmax launch");
}
