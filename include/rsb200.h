/*
 * rsb200.h -- C ABI of librsb200.so: the H100 (sm_90a) kernels behind RoboSat's segmentation hot path.
 *
 * The reference (mapbox/robosat @ cbb1c73) has no FFI of its own: its "operator interface" for this
 * path is a handful of PyTorch call sites. Every entry point below names the reference call site it
 * replaces (file:line under /root/reference). Host code (robosat_b200/*.py) binds these with ctypes.
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer unless the name ends in _host
 *   - the library never allocates or frees user tensors and never synchronises: all work is enqueued
 *     on the `stream` argument (a cudaStream_t passed as void*)
 *   - return value: 0 on success, negative RSB_E_* on failure; rsb_last_error() gives the message
 *     (thread local). There is NO CPU fallback: without a usable sm_90 device every compute entry fails.
 *   - activations are NHWC fp16 ("channels last"), accumulators fp32; weights are pre-packed fp16
 *   - two precisions: "fast" (one fp16 plane per tensor) and "strict" (hi + lo fp16 planes, see rsb_conv_desc.split)
 */
#ifndef RSB200_H
#define RSB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RSB_OK 0
#define RSB_E_INVALID -1   /* bad argument / unsupported shape */
#define RSB_E_CUDA -2      /* CUDA runtime or driver error */
#define RSB_E_NODEVICE -3  /* no sm_90 device / driver entry point missing */
#define RSB_E_UNSUPPORTED -4 /* (host codecs only) valid input of a kind this entry point does not handle: use another decoder */

#define RSB_MAX_SEGS 16
#define RSB_MAX_SRCS 4

int rsb_version(void);
/* sizeof(rsb_conv_src), sizeof(rsb_conv_seg), sizeof(rsb_conv_desc), sizeof(rsb_rowconv_desc) as compiled into the library,
 * so that a binding (ctypes, cgo, ...) can verify its struct declarations before the first call */
void rsb_abi_layout(int32_t* out4);
const char* rsb_last_error(void);
/* 0 if a compute-capability-9.0 device is current and the TMA driver entry point resolves */
int rsb_device_ok(void);

/* ---------------------------------------------------------------------------------------------
 * Implicit-GEMM convolution on wgmma tensor cores (fp16 x fp16 -> fp32 in registers).
 *
 * Replaces every nn.Conv2d (+ folded eval BatchNorm, + ReLU, + residual add, + nearest x2 upsample,
 * + channel concat) the forward pass runs:
 *   resnet conv1 / layer1-4 Bottleneck convs      robosat/unet.py:122-130 (torchvision resnet.py Bottleneck.forward)
 *   ConvRelu.forward                              robosat/unet.py:44
 *   DecoderBlock.forward (interpolate + ConvRelu) robosat/unet.py:73
 *   torch.cat([enc, dec], dim=1)                  robosat/unet.py:134-137
 *   final 1x1 conv + bias                         robosat/unet.py:141
 *
 * One output tile = 128 "tile-space" pixels (box TW x TH x TN of one source view) x BLOCK_N output
 * channels. The contraction is a list of segments; each segment is one TMA box load per 64-channel
 * block from source view `src` displaced by (dh, dw) pixels, multiplied by the next 64 columns of the
 * packed weight matrix [phases*Cout][K]. Strided convs use parity views of the input, the nearest
 * x2 upsample uses 4 output phases of 2x2 taps on the low-resolution input (pre-summed weights),
 * channel concat uses two sources; none of them materialises an intermediate tensor.
 */
typedef struct rsb_conv_src {
    const void* ptr;      /* fp16 base of the view (already offset for parity / padding) */
    int64_t pitch_w;      /* element strides of the view */
    int64_t pitch_h;
    int64_t pitch_n;
    int32_t C;            /* innermost extent (channels, or window elements for overlapped views) */
    int32_t W, H, N;      /* extents of the view (TMA zero-fills outside) */
    int64_t plane;        /* split precision only: element stride from the hi plane (ptr) to the lo plane of the same view */
} rsb_conv_src;

typedef struct rsb_conv_seg {
    int32_t src;          /* index into srcs[] */
    int32_t dh, dw;       /* displacement in tile-space pixels, for phase (0,0) */
    int32_t cblocks;      /* number of 64-element blocks taken from that source */
} rsb_conv_seg;

typedef struct rsb_conv_desc {
    int32_t nsrc;
    rsb_conv_src srcs[RSB_MAX_SRCS];
    int32_t nseg;
    rsb_conv_seg segs[RSB_MAX_SEGS];

    const void* weights;  /* fp16 [phases * Cout][K], K = 64 * sum(cblocks), K contiguous */
    const float* bias;    /* fp32 [Cout] (folded BatchNorm shift / conv bias) or NULL */
    int32_t Cout;         /* multiple of block_n */
    int32_t block_n;      /* 32, 64, 128 or 256 */
    int32_t phases;       /* 1, or 4 for the fused nearest-x2 upsample (phase p = 2*a+b adds (a,b) to every (dh,dw)) */

    int32_t Wt, Ht, Nt;   /* tile-space extents (the pixels that produce outputs) */
    int32_t TW, TH, TN;   /* tile box, TW*TH*TN == 128 */

    /* output: pixel (n, h, w) of tile space, phase (a, b) -> out + n*pitch_n + (h*sy+a)*pitch_h + (w*sx+b)*pitch_w + c */
    void* out;            /* fp16 (mode 0) */
    int64_t out_pitch_w, out_pitch_h, out_pitch_n;
    int32_t out_sy, out_sx;
    const void* residual; /* fp16, same addressing as out, added before ReLU; or NULL */
    int32_t relu;

    /* mode 1 ("head"): block_n == Cout == 32; ReLU(acc) is contracted in fp32 with head_w [classes][32] + head_b
     * and written as fp32 NCHW logits [N][classes][Ht][Wt] to head_out (final 1x1 conv, unet.py:141) */
    int32_t mode;
    int32_t head_classes; /* <= 8 */
    const float* head_w;
    const float* head_b;
    float* head_out;

    /* 1: compute each pair of neighbouring tiles with a CTA pair (cluster of 2; mode 0,
     * block_n >= 128): each CTA loads half of the shared weight tile and multicasts it to both. Same results; 0 = one CTA per tile. */
    int32_t cta_pair;

    /* Split ("strict") precision: every activation and weight is the unevaluated sum of two fp16 numbers, hi = half(v) and
     * lo = half(v - hi) (22+ significant bits), stored as two planes; the kernel accumulates hi*hi + hi*lo + lo*hi in fp32
     * (3 tensor-core MMAs per K step; the lo*lo term is below fp32 resolution). This is what meets the reference's fp32
     * results (logits 1e-3 rel, argmax identical up to the fp32 noise floor); split == 0 is the fast single-fp16 mode.
     *   srcs[i].plane        element stride between the planes of source i
     *   weights              fp16 [2][phases*Cout][K] (hi plane, then lo plane)
     *   out_plane/res_plane  element stride between the planes of out / residual
     * acc_scale (0 = 1): the fp32 accumulator is multiplied by it before bias/residual; the host pre-scales the weights by
     * its inverse (a power of two) so that the lo parts of small weights stay in fp16's normal range. */
    int32_t split;
    int64_t out_plane;
    int64_t res_plane;
    float acc_scale;

    /* K chunking (mode 0; meant for split precision with long K loops): the tensor core truncates its fp32 accumulator after
     * every MMA, so a tile's K loop is cut into chunks of `kchunk` 64-element K blocks whose results the epilogue adds with
     * round-to-nearest fp32 adds through `scratch` (>= grid x 128 x block_n x 4 bytes, see rsb_conv_scratch_bytes; private to
     * the launch, reusable by the next launch on the same stream). 0: no chunking. */
    int32_t kchunk;
    float* scratch;
    int64_t scratch_bytes;

    /* BatchNorm batch statistics fused into the epilogue (training forward of a conv that feeds nn.BatchNorm2d: torchvision
     * resnet.py Bottleneck.forward bn1-3, robosat/unet.py:122-130 in train mode). mode 0, split 0, no residual, phases 1.
     * For every tile t (flat index ((n-tile * tiles_h) + h-tile) * tiles_w + w-tile) and every 32-row quarter q of it:
     *   stats[(t*4 + q)*2*Cout + c]        = sum   of the fp16 outputs of channel c over the quarter's in-range pixels
     *   stats[(t*4 + q)*2*Cout + Cout + c] = sum of their squares
     * every entry is written exactly once per run (no zeroing needed); rsb_bn_partials_finalize folds them. NULL: off. */
    float* stats;
    int64_t stats_bytes;
} rsb_conv_desc;

typedef struct rsb_conv_plan rsb_conv_plan;

/* upper bound of the scratch a chunked plan with this block_n needs on the current device (SMs x 128 x block_n x 4 bytes) */
int64_t rsb_conv_scratch_bytes(int32_t block_n);
int rsb_conv_plan_create(const rsb_conv_desc* desc, rsb_conv_plan** out_plan);
void rsb_conv_plan_destroy(rsb_conv_plan* plan);
/* number of CTAs / tiles the plan launches (for tests and occupancy accounting) */
int rsb_conv_plan_info(const rsb_conv_plan* plan, int32_t* grid, int32_t* tiles, int32_t* kblocks, int32_t* smem_bytes);
int rsb_conv_run(const rsb_conv_plan* plan, void* stream);
/* same contraction with a plain SIMT kernel reading global memory directly (no TMA / wgmma).
 * Test-only checker used to bisect the tensor-core path on the device; never on the product path. */
int rsb_conv_run_simt_check(const rsb_conv_desc* desc, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Line-buffer variant of the same convolution for stride-1 layers with few output channels at high resolution
 * (dec5 + final, dec4, layer1 3x3; unet.py:127, 138-141): a tile is 128 pixels of one output row, input rows live in a
 * shared-memory ring and are fetched once for all filter taps. Same arithmetic and packed weight layout
 * ([phase*Cout + co][(tap_h, tap_w)][ci]) as rsb_conv_*; see csrc/rsb_conv_row.cu.
 */
typedef struct rsb_rowconv_desc {
    rsb_conv_src src;        /* dense NHWC view of the input (TMA zero-fills outside = padding) */
    int32_t cin;             /* 32, 64 or 128 */
    int32_t taps_h, taps_w;  /* 3x3, or 2x2 for the fused upsample */
    int32_t dh0, dw0;        /* displacement of tap (0,0) for phase (0,0): -1, -1 */
    int32_t nsub;            /* 1, or 2 column phases b (phase b adds b to dw) computed per tile */
    int32_t nphase_a;        /* 1, or 2 row phases a (phase a adds a to dh), one per work unit */
    const void* weights;     /* fp16 [(a*nsub + b)*Cout + co][taps_h*taps_w*cin] */
    const float* bias;       /* fp32 [Cout] or NULL */
    int32_t Cout;            /* 32 or 64 */
    int32_t Wt, Ht, Nt;      /* tile-space extents */
    void* out;               /* fp16, addressed like rsb_conv_desc.out (mode 0) */
    int64_t out_pitch_w, out_pitch_h, out_pitch_n;
    int32_t out_sy, out_sx;
    int32_t relu;
    int32_t mode;            /* 0: fp16 NHWC output; 1: head (Cout 32 -> fp32 NCHW logits through head_w / head_b) */
    int32_t head_classes;
    const float* head_w;
    const float* head_b;
    float* head_out;
    int32_t rows_per_unit;   /* output rows per work unit (0 = default 32) */
    /* strict precision (see rsb_conv_desc.split): mode 1, cin 32, 3x3 only -- src.plane gives the lo plane of the input,
     * weights are fp16 [2][Cout][K] (hi, lo of w * 2^e), acc_scale = 2^-e */
    int32_t split;
    float acc_scale;
} rsb_rowconv_desc;

typedef struct rsb_rowconv_plan rsb_rowconv_plan;
int rsb_rowconv_plan_create(const rsb_rowconv_desc* desc, rsb_rowconv_plan** out_plan);
void rsb_rowconv_plan_destroy(rsb_rowconv_plan* plan);
int rsb_rowconv_run(const rsb_rowconv_plan* plan, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Input pre-pass. Replaces `images.to(device)` + the stem's NCHW read (predict.py:83, train.py:172) and,
 * for uint8 input, ToTensor + Normalize (predict.py:71-73). Writes the space-to-depth view the stem
 * convolution consumes: fp16 [N][H/2][W/2 + 4][16], pixel (hh, ww) at column ww + 2, channel
 * (ph*2 + pw)*3 + c = x[n, c, 2*hh+ph, 2*ww+pw]; channels 12..15 and the pad columns are zero.
 *   src_kind 0: fp32 NCHW, already normalised (the reference API)     src_kind 1: uint8 NHWC raw RGB
 */
int rsb_prepass_s2d(const void* src, int32_t src_kind, void* dst, int32_t N, int32_t H, int32_t W,
                    const float* mean3_host, const float* std3_host, void* stream);

/* strict precision: also writes the lo plane at dst + plane (elements): lo = half(x - float(half(x))) */
int rsb_prepass_s2d_split(const void* src, int32_t src_kind, void* dst, int64_t plane, int32_t N, int32_t H, int32_t W,
                          const float* mean3_host, const float* std3_host, void* stream);

/* NHWC fp16 max pooling. Replaces resnet.maxpool (unet.py:125: k3 s2 p1) and F.max_pool2d(enc4, 2, 2) (unet.py:132).
 * Output pixel pitches are explicit so the result can land inside a padded buffer. */
int rsb_maxpool_nhwc(const void* src, void* dst, int32_t N, int32_t H, int32_t W, int32_t C, int32_t k, int32_t s,
                     int32_t p, void* stream);

/* strict precision: the maximum of the (hi, lo) pairs, i.e. of the exact fp32 sums hi + lo, written as a pair again */
int rsb_maxpool_nhwc_split(const void* src, int64_t src_plane, void* dst, int64_t dst_plane, int32_t N, int32_t H, int32_t W,
                           int32_t C, int32_t k, int32_t s, int32_t p, void* stream);

/* Training-side augmentation (robosat/transforms.py:127-221 as composed in train.py:253-258): per sample an optional left-right flip
 * followed by k counter-clockwise quarter turns, applied to the RGB tile uint8 [N][S][S][3] and its mask uint8 [N][S][S] (mask may be
 * NULL); ops int32 [N] on the device, op = flip | (k << 1). out_mask is int64 (what the losses consume). Not in place. */
int rsb_augment_dihedral(const uint8_t* img, const uint8_t* mask, const int32_t* ops, uint8_t* out_img, int64_t* out_mask, int32_t N, int32_t S,
                         void* stream);

/* Predict head. Replaces softmax(outputs, 1) ... np.digitize(foreground, linspace(0,1,256)).astype(uint8)
 * (predict.py:87, 93, 98-103) for the 2-class case, including the crop of the `overlap` border (datasets.py:133-136).
 * logits fp32 [N][2][H][W] -> quant uint8 [N][H-2o][W-2o]; probs_fg (fp32, same cropped shape) optional. */
int rsb_head_quantize(const float* logits, uint8_t* quant, float* probs_fg, int32_t N, int32_t H, int32_t W,
                      int32_t overlap, void* stream);
/* Predict head for C = 2..255 classes (`rs predict` of a multi-class model; no reference counterpart): per pixel the softmax of
 * rsb_head_tta_accumulate (max over the classes in order, class-ordered sum of expf(l - max), one division), the crop of `overlap`,
 * then np.digitize(p, linspace(0, 1, 256)).astype(uint8) of EVERY class. logits fp32 [N][C][H][W] -> quant uint8
 * [N][C][H-2o][W-2o]; probs (fp32, same shape) optional. For C = 2, plane 1 equals rsb_head_quantize's output bit for bit. */
int rsb_head_quantize_classes(const float* logits, uint8_t* quant, float* probs, int32_t N, int32_t C, int32_t H, int32_t W,
                              int32_t overlap, void* stream);
/* softmax over C for any class count: logits fp32 [N][C][H][W] -> probs fp32 same shape (predict.py:87) */
int rsb_softmax_nchw(const float* logits, float* probs, int32_t N, int32_t C, int32_t HW, void* stream);
/* `buffer_tile_image` (robosat/tiles.py:162-227) on the device: builds B buffered tiles uint8 [B][S+2o][S+2o][3] from a cache of
 * decoded RGB tiles uint8 [slots][S][S][3]. slots: int32 [B][9] (device), row-major over (dy, dx) in {-1,0,1}^2, entry 4 = the
 * centre tile, -1 = no such neighbour (nodata 0, as the reference's Image.new(color=0)). */
int rsb_stitch_halo(const uint8_t* cache, const int32_t* slots, uint8_t* out, int32_t B, int32_t S, int32_t overlap, void* stream);
/* `rs masks` soft vote (robosat/tools/masks.py:42-84): quant uint8 [K][n] probability bins of K models (as written by rs predict),
 * weights float64 [K] on the device or NULL -> mask uint8 [n] = argmax([1 - p, p]) of the weighted average, float64, numpy's order. */
int rsb_softvote(const uint8_t* quant, const double* weights, uint8_t* mask, int32_t K, int64_t n, void* stream);
/* `rs masks --dataset` for C = 2..255 classes: quant uint8 [K][C][n] (per model the C probability planes rs predict writes for a
 * multi-class model), weights float64 [K] on the device or NULL -> mask uint8 [n] = np.argmax(np.average(anchors[quant], axis=0,
 * weights=w), axis=0): float64, sequential sum over K, products and sums rounded separately, one division, first maximum wins. */
int rsb_softvote_classes(const uint8_t* quant, const double* weights, uint8_t* mask, int32_t K, int32_t C, int64_t n, void* stream);
/* `rs weights` histogram (robosat/tools/weights.py:39-49): counts[c] += #(labels == c) for c < C; counts is uint64 [C] on the device */
int rsb_class_histogram(const uint8_t* labels, int64_t n, int32_t C, uint64_t* counts, void* stream);
/* `Predictor.segment` head (robosat/tools/serve.py:150-165): output.argmax(axis=0).astype(uint8) of fp32 NCHW logits
 * -> uint8 [N][H*W] class indices, first maximum wins like np.argmax; C <= 255. */
int rsb_head_argmax(const float* logits, uint8_t* mask, int32_t N, int32_t C, int32_t HW, void* stream);

/* Test-time augmentation (no reference counterpart): average the class probabilities of up to 8 dihedral views of each tile.
 * The views' inputs are made with rsb_augment_dihedral (square tiles) or rsb_augment_flip_rect (flips of any tile).
 * logits fp32 [views*B][C][H][W], view-major (sample v*B + b is view v of tile b); ops_host: `views` ops in rsb_augment_dihedral's
 * encoding (flip | k << 1), passed by value so the launch can be captured in a graph; odd k needs H == W. For every tile, class and
 * pixel of the cropped output, the softmax over C of each view's logit at the pixel the op moved it to, as llrint(p * 2^59), is
 * summed into acc int64 [B][C][H-2o][W-2o] (accumulate = 0 overwrites acc). Integer sums: the result does not depend on the order
 * of the views or on how they are split over calls. C <= 255. */
#define RSB_TTA_MAX_VIEWS 8
int rsb_head_tta_accumulate(const float* logits, int64_t* acc, const int32_t* ops_host, int32_t views, int32_t B, int32_t C, int32_t H,
                            int32_t W, int32_t overlap, int32_t accumulate, void* stream);
/* 2-class acc [B][2][HW] summed over `views` views -> quant uint8 [B][HW]: np.digitize bins of the mean foreground probability
 * (float)(acc[b][1] * 2^-59 / views), as rsb_head_quantize bins a single view */
int rsb_head_tta_quantize(const int64_t* acc, uint8_t* quant, int32_t B, int32_t HW, int32_t views, void* stream);
/* acc int64 [B][C][HW] summed over `views` views -> quant uint8 [B][C][HW]: every class binned as rsb_head_tta_quantize bins
 * class 1, (float)(acc * 2^-59 / views); C = 2..255 */
int rsb_head_tta_quantize_classes(const int64_t* acc, uint8_t* quant, int32_t B, int32_t C, int32_t HW, int32_t views, void* stream);
/* acc int64 [B][C][HW] -> uint8 [B][HW]: class of the largest sum (= largest mean probability), first maximum wins; C <= 255 */
int rsb_head_tta_argmax(const int64_t* acc, uint8_t* mask, int32_t B, int32_t C, int32_t HW, void* stream);
/* rsb_augment_dihedral's image transform for H x W tiles without a mask; when H != W only the flip bit of each op is used */
int rsb_augment_flip_rect(const uint8_t* img, const int32_t* ops, uint8_t* out_img, int32_t N, int32_t H, int32_t W, void* stream);

/* `rs features` mask morphology (robosat/features/core.py:65-92: denoise = MORPH_OPEN, grow = MORPH_CLOSE, OpenCV semantics).
 * A chain of up to RSB_MORPH_MAX_OPS binary erosions / dilations of m = (labels == class_index), fused: each label byte is read
 * once and each output byte written once. Op k: out(y, x) = min (erode) or max (dilate) over the element's set cells (i, j) of
 * in(y + i - ay, x + j - ax), no reflection; pixels outside the image are ignored (1 for erode, 0 for dilate). Row i of the
 * element is the run of columns [span[i][0], span[i][1]), empty if span[i][0] >= span[i][1] (every row of an OpenCV ellipse,
 * rectangle or cross is one run). ops_host is read on the host and passed by value into the launch.
 * labels uint8 [N] images of H x W, image n at labels + n * image_stride -> out uint8 {0, 1} [N][H][W]; fg_counts int32 [N] = number
 * of 1 pixels of each result. 1 <= H, W <= 1024, 1 <= kh, kw <= 64; allocates nothing and does not synchronise. */
#define RSB_MORPH_MAX_OPS 4
#define RSB_MORPH_MAX_K 64
typedef struct rsb_morph_op {
    int32_t dilate;                       /* 0 = erode, 1 = dilate */
    int32_t kh, kw;                       /* element size */
    int32_t ay, ax;                       /* anchor (OpenCV's default is (kh / 2, kw / 2)) */
    int16_t span[RSB_MORPH_MAX_K][2];     /* rows 0 .. kh-1 are used */
} rsb_morph_op;
int rsb_morph_binary(const uint8_t* labels, int64_t image_stride, int32_t N, int32_t H, int32_t W, int32_t class_index,
                     const rsb_morph_op* ops_host, int32_t nops, uint8_t* out, int32_t* fg_counts, void* stream);

/* `rs features --type building` connected components (the rule is DESIGN.md §8). planes uint8 [N] images of H x W, image n at
 * planes + n * image_stride; the outputs are int32 [N][H][W]. 1 <= N <= 65535, 1 <= H, W <= RSB_LABEL_MAX_SIZE. Labels are
 * image-local pixel indices y * W + x: labels[n][y][x] = the smallest index of the pixel's component of (plane == value) under
 * 4- or 8-connectivity (`connectivity` = 4 or 8), -1 off the plane; areas[n][y][x] = the number of pixels of that component, 0 off
 * the plane. Identical on every run. Arguments are validated before the device check; allocates nothing and does not synchronise. */
#define RSB_LABEL_MAX_SIZE 8192
int rsb_label_components(const uint8_t* planes, int64_t image_stride, int32_t N, int32_t H, int32_t W, int32_t value, int32_t connectivity,
                         int32_t* labels, int32_t* areas, void* stream);
/* Speck drop and hole fill of the building rule on `opened` ({0, 1} images laid out as rsb_label_components' planes, e.g. the
 * opening from rsb_morph_binary): D = the pixels of 8-connected foreground components of at least min_area pixels; out uint8
 * {0, 1} [N][H][W] = D plus every 4-connected background component of D that touches no image border and has fewer than
 * min_hole_area pixels; fg_counts int32 [N] = the 1 pixels of each result. labels, stats: int32 [N][H][W] workspaces (not
 * aliased). Same limits and guarantees as rsb_label_components. */
int rsb_building_clean(const uint8_t* opened, int64_t image_stride, int32_t N, int32_t H, int32_t W, int32_t min_area, int32_t min_hole_area,
                       int32_t* labels, int32_t* stats, uint8_t* out, int32_t* fg_counts, void* stream);

/* `rs features --type road` (the rule is DESIGN.md §8): thinning, m-degrees, spur pruning and chain lists of N halo'd planes of
 * H x W. 1 <= N <= 65535, 1 <= H, W <= RSB_ROAD_MAX_SIZE; every output is laid out [N][H][W] (contiguous). Pixel indices are
 * plane-local, y * W + x. Arguments are validated before the device check; nothing allocates or synchronises.
 *
 * rsb_road_thin: Zhang-Suen (1984) of (plane != 0), image n at planes + n * image_stride, pixels outside the plane background,
 * until the first full iteration that deletes nothing -> skel uint8 {0, 1}, iterations int32 [N] (full iterations run, the last
 * one included). One CTA per plane keeps it bit-packed in shared memory, so H * ceil(W / 32) <= RSB_ROAD_MAX_WORDS (a 640 x 640
 * plane takes 12 800 words); a larger plane is refused with RSB_E_UNSUPPORTED.
 * rsb_road_degree: deg int8 = the m-degree of each pixel of skel (4-neighbours, and diagonal neighbours with no common
 * 4-neighbour in skel), -1 off skel.
 * rsb_road_prune: out = skel without every chain of (skel, deg) that runs from an endpoint to a junction (degree >= 3) with fewer
 * than min_length pixels not counting the junction, or from an endpoint to an endpoint with fewer than min_length pixels.
 * rsb_road_chain_count: with deg the degrees of skel and labels / flags the labels / areas rsb_label_components gives for
 * (skel == 1) under 8-connectivity (flags is overwritten): counts int32 [N][H][W] per pixel (workspace), row_offsets int64
 * [N][H] (workspace), totals int64 [N] = each plane's (chain count << 32 | pixel count of its lists).
 * rsb_road_chain_write: the same skel, deg, labels, flags, counts and row_offsets; chain_base / pixel_base int64 [N] the index of
 * plane n's first chain and first pixel in the outputs (prefix sums of totals) -> chain_offsets int64 [chains] the start of each
 * chain in pixels, pixels int32 the chains' pixel indices. A plane's chains come in (first pixel, second pixel) order; each is
 * written from its end with the smaller index (a loop at one node, or a node-free cycle from its smallest pixel, toward the
 * smaller second pixel, repeating the first pixel at the end). */
#define RSB_ROAD_MAX_SIZE 4096
#define RSB_ROAD_MAX_WORDS 16384
int rsb_road_thin(const uint8_t* planes, int64_t image_stride, int32_t N, int32_t H, int32_t W, uint8_t* skel, int32_t* iterations, void* stream);
int rsb_road_degree(const uint8_t* skel, int32_t N, int32_t H, int32_t W, int8_t* deg, void* stream);
int rsb_road_prune(const uint8_t* skel, const int8_t* deg, int32_t N, int32_t H, int32_t W, int32_t min_length, uint8_t* out, void* stream);
int rsb_road_chain_count(const uint8_t* skel, const int8_t* deg, const int32_t* labels, int32_t* flags, int32_t N, int32_t H, int32_t W,
                         int32_t* counts, int64_t* row_offsets, int64_t* totals, void* stream);
int rsb_road_chain_write(const uint8_t* skel, const int8_t* deg, const int32_t* labels, const int32_t* flags, int32_t N, int32_t H, int32_t W,
                         const int32_t* counts, const int64_t* row_offsets, const int64_t* chain_base, const int64_t* pixel_base,
                         int64_t* chain_offsets, int32_t* pixels, void* stream);

/* `rs rasterize` polygon fill (robosat/tools/rasterize.py:64-83: rasterio.features.rasterize, all_touched=False, burn value 1,
 * merge "replace"). All arrays are DEVICE pointers. Polygons: vertices float64 [num_vertices][2] (EPSG:3857 X, Y; 16-byte aligned);
 * ring r owns vertices [ring_offsets[r], ring_offsets[r + 1]) and is closed implicitly; polygon p owns rings
 * [poly_rings[p], poly_rings[p + 1]) (outer ring and holes, filled even-odd). Tile n burns polygons
 * tile_polys[tile_poly_offsets[n] .. tile_poly_offsets[n + 1]) (ids outside [0, num_polys) are skipped) with the transform
 * tile_transforms[n] = (c0, c1, r0, r1): px = c0 + X * c1, py = r0 + Y * r1, every float64 operation rounded separately (no FMA).
 * Row r is filled on the line r + 0.5: an edge with y1 <= y2 crosses it iff y1 <= r + 0.5 < y2, at
 * x = (r + 0.5 - y1) * (x2 - x1) / (y2 - y1) + x1; sorted crossings pair into column spans [floor(a + 0.5), floor(b + 0.5)) clipped
 * to [0, size). The polygons of a tile are unioned. out uint8 {0, 1}: row y of tile n at out + n * image_stride + y * size;
 * fg_counts int32 [N] = number of 1 pixels per tile. 1 <= size <= RSB_RASTER_MAX_SIZE; tile_polys is never NULL (pass a one-element
 * array when no tile has a polygon), the polygon arrays may be NULL when num_polys = 0. Arguments are validated on the host before
 * any device call; allocates nothing and does not synchronise. */
#define RSB_RASTER_MAX_SIZE 4096
int rsb_rasterize_polygons(const double* vertices, const int64_t* ring_offsets, const int32_t* poly_rings, int32_t num_polys,
                           const int32_t* tile_poly_offsets, const int32_t* tile_polys, const double* tile_transforms, int32_t N, int32_t size,
                           uint8_t* out, int64_t image_stride, int32_t* fg_counts, void* stream);

/* `rs cover` (robosat/tools/cover.py: supermercado burntiles.burn, rasterio's rasterize with all_touched=True on each feature's
 * own tile grid; the rule is restated in DESIGN.md §8). All arrays are DEVICE pointers; the polygon arrays are those of
 * rsb_rasterize_polygons. Feature f (0 <= f < F) owns polygons [feature_polys[f], feature_polys[f + 1]) and vertex_offsets[f] is
 * the prefix of the batch's vertex counts (vertex_offsets[F] = num_vertices). transforms[f] = (c0, c1, r0, r1) maps EPSG:3857 to
 * its grid (px = c0 + X * c1, py = r0 + Y * r1, no FMA); grids[f] = int64 (xmin, ymin, W, H, row_lo, rows): the grid is W x H tiles
 * from (xmin, ymin), and rows [row_lo, row_lo + rows) of it are burned into bitmap + bitmap_offsets[f], rows of ceil(W / 32) uint32
 * words, bit c of a row = column c (bitmap_offsets[F] = bitmap_words). A cell is set when the scanline fill of
 * rsb_rasterize_polygons sets it or GDAL's all-touched line walk over an edge of a ring reaches it. The fill runs one CTA per band:
 * bands int32 [num_bands][3] = (feature, first row within the window, rows <= band_rows), covering every window row once;
 * max_words >= ceil(W / 32) for every feature, band_rows * max_words <= RSB_COVER_MAX_WIDTH / 32. status int64 [4]: [0] = set
 * cells of the batch, [1] != 0 when a walk exceeded its step bound (coordinates outside float64's resolution), [2] the key
 * cursor of rsb_cover_emit_keys, [3] unused. The bitmap and status are cleared here. Validated on the host before any device
 * call; allocates nothing and does not synchronise. */
#define RSB_COVER_MAX_WIDTH 1856000
#define RSB_COVER_MAX_ZOOM 30
int rsb_cover_polygons(const double* vertices, const int64_t* ring_offsets, const int32_t* poly_rings, int32_t num_polys,
                       const int32_t* feature_polys, const int64_t* vertex_offsets, const double* transforms, const int64_t* grids,
                       const int64_t* bitmap_offsets, int32_t F, int64_t num_vertices, const int32_t* bands, int32_t num_bands,
                       int32_t band_rows, int32_t max_words, uint32_t* bitmap, int64_t bitmap_words, int64_t* status, void* stream);
/* One key ((xmin + c) << zoom) | (ymin + row_lo + r) per set cell of the bitmap burned by rsb_cover_polygons, in no particular
 * order, into keys [capacity] (status[0] of the burn is the number written; status[2] is reset and used as the cursor). */
int rsb_cover_emit_keys(const uint32_t* bitmap, int64_t bitmap_words, const int64_t* bitmap_offsets, const int64_t* grids, int32_t F,
                        int32_t zoom, int64_t* keys, int64_t capacity, int64_t* status, void* stream);
/* Ascending sort of n non-negative int64 keys below 2^key_bits (an LSD radix sort of ceil(key_bits / 8) 8-bit passes; key_bits = 64
 * sorts the whole word as unsigned; bits at or above key_bits are not looked at, so keys that have them come out unsorted) and
 * removal of adjacent duplicates: keys[0 .. *unique_count) holds the result, in place. workspace: DEVICE bytes, at least
 * rsb_sort_unique_workspace_bytes(n). Does not synchronise. */
int64_t rsb_sort_unique_workspace_bytes(int64_t n);
int rsb_sort_unique_u64(int64_t* keys, int64_t n, int32_t key_bits, void* workspace, int64_t workspace_bytes, int64_t* unique_count, void* stream);

/* `rs dedupe` (robosat/tools/dedupe.py, robosat/spatial/core.py; the rule is DESIGN.md §8). A set of features as DEVICE arrays
 * (the struct itself is a HOST pointer): vertices double [num_vertices][2], 16-byte aligned; next int32 [num_vertices], the
 * vertex the edge from v ends at (rings close implicitly and repeat no vertex consecutively; exterior rings counter-clockwise
 * and holes clockwise in projected coordinates); feature f's edges start at vertices [feature_vertices[f], feature_vertices[f + 1]);
 * exteriors[exterior_offsets[f] .. exterior_offsets[f + 1]) are the first vertices of its components' exterior rings; boxes
 * double [num_features][4] = (xmin, ymin, xmax, ymax) of its vertices. A y-band index of the edges (read by rsb_dedupe_areas):
 * feature f has nb = feature_bands[f + 1] - feature_bands[f] bands (0: no index, its edges are scanned in full); y maps to band
 * clamp(floor((y - band_ranges[f][0]) * band_ranges[f][1]), 0, nb - 1), and band b lists in band_edges[band_offsets[fb + b] ..
 * band_offsets[fb + b + 1]) (fb = feature_bands[f]) the first vertices of the edges whose y ranges meet it. */
typedef struct RsbShapes {
    const double* vertices;
    const int32_t* next;
    const int64_t* feature_vertices;
    const int64_t* exterior_offsets;
    const int64_t* exteriors;
    const double* boxes;
    const int64_t* feature_bands;
    const double* band_ranges;
    const int64_t* band_offsets;
    const int32_t* band_edges;
    int64_t num_vertices;
    int32_t num_features;
    int32_t reserved;
} RsbShapes;
/* out[i] = 1 when predicted feature pairs[i][0] and OSM feature pairs[i][1] are not disjoint (GEOS `intersects`: some edges
 * meet, touching included, or one lies inside the other), else 0; exact orientation predicates on the lon/lat vertices. */
int rsb_dedupe_intersects(const RsbShapes* predicted, const RsbShapes* osm, const int32_t* pairs, int64_t num_pairs, uint8_t* out, void* stream);
/* For B predictions b (feature pred[b]) with the OSM features S(b) = set_ids[set_offsets[b] .. set_offsets[b + 1]) (ascending,
 * set_offsets[0] = 0): areas double [B][3] = (A(P), A(P ∩ U), A(U)) of P and U = the union of S(b), on projected vertices relative
 * to origins double [B][2]. The work items are the edges of P then those of each feature of S(b): segment b + set_offsets[b] is
 * P's, segment b + set_offsets[b] + 1 + k is S(b)[k]'s; item_offsets int64 [num_segments + 1] (item_offsets[0] = 0) gives each
 * segment's items (one per edge of its feature) and segment_pred int32 [num_segments] its b. terms: DEVICE double
 * [2 * num_items] workspace. Sums run in item order, so the result is identical from run to run and across batches. */
int rsb_dedupe_areas(const RsbShapes* predicted, const RsbShapes* osm, int32_t B, const int32_t* pred, const double* origins, const int64_t* set_offsets,
                     const int32_t* set_ids, int64_t num_segments, const int64_t* item_offsets, const int32_t* segment_pred, int64_t num_items,
                     double* terms, double* areas, void* stream);

/* `rs merge` (robosat/tools/merge.py, robosat/graph/core.py; the rule is DESIGN.md §8). All arrays are DEVICE pointers.
 * rsb_merge_near: out[i] = 1 when features pairs[i][0] and pairs[i][1] of `shapes` (RsbShapes on EPSG:3395 vertices; the band
 * index is not read) are within `threshold` of each other: some vertex of one has |p - q|^2 <= threshold^2 to the nearest point q
 * of some edge of the other, q = a + clamp(((p - a).(b - a)) / |b - a|^2, 0, 1) (b - a), every float64 operation rounded on its
 * own. */
int rsb_merge_near(const RsbShapes* shapes, const int32_t* pairs, int64_t num_pairs, double threshold, uint8_t* out, void* stream);
/* Connected components of n nodes under the pairs i with linked[i] != 0: labels int32 [n] = the smallest node of each node's
 * component, the same on every run. parent: int32 [n] workspace. */
int rsb_merge_components(const int32_t* pairs, const uint8_t* linked, int64_t num_pairs, int32_t n, int32_t* parent, int32_t* labels, void* stream);
/* Cell fill of C components on their own grids: component c fills polygons comp_polys[comp_poly_offsets[c] .. comp_poly_offsets[c + 1])
 * of the polygon arrays of rsb_rasterize_polygons (even-odd per polygon, union across polygons) with rsb_rasterize_polygons's
 * scanline rule under transforms[c] = (c0, c1, r0, r1) (px = c0 + X * c1, py = r0 + Y * r1, no FMA). grids int64 [C][2] = (W, H);
 * rows of ceil(W / 32) uint32 words at bitmap + bitmap_offsets[c], bit b of word w = column 32 w + b. One CTA per band: bands
 * int32 [num_bands][3] = (component, first row, rows <= band_rows), covering every row once; max_words >= every ceil(W / 32),
 * band_rows * max_words <= RSB_COVER_MAX_WIDTH / 32. The bitmap (bitmap_words words) is cleared here. */
int rsb_merge_fill(const double* vertices, const int64_t* ring_offsets, const int32_t* poly_rings, int32_t num_polys,
                   const int32_t* comp_poly_offsets, const int32_t* comp_polys, const double* transforms, const int64_t* grids,
                   const int64_t* bitmap_offsets, int32_t C, const int32_t* bands, int32_t num_bands, int32_t band_rows, int32_t max_words,
                   uint32_t* bitmap, int64_t bitmap_words, void* stream);
/* Closing erode(dilate(fill)) with the disk {(i, j): i^2 + j^2 <= radius^2}, cells outside a grid counting as 0, into out (same
 * layout as fill, not aliasing it); counts int64 [C] = set cells of each closed grid. One CTA per tile: tiles int32
 * [num_tiles][3] = (component, first row, first word) of 32 rows x 32 words, covering every grid. 1 <= radius <= RSB_MERGE_MAX_RADIUS. */
#define RSB_MERGE_MAX_RADIUS 16
int rsb_merge_close(const uint32_t* fill, const int64_t* grids, const int64_t* bitmap_offsets, int32_t C, const int32_t* tiles, int32_t num_tiles,
                    int32_t radius, uint32_t* out, int64_t* counts, void* stream);

/* ---------------------------------------------------------------------------------------------
 * `rs extract` (robosat/tools/extract.py, robosat/osm/{core,parking,building}.py; the rule is DESIGN.md §8): OpenStreetMap PBF files.
 * Host entry points (HOST pointers, plain C++ over zlib, csrc/rsb_pbf.cpp) frame, inflate and parse; the device entry points
 * (csrc/rsb_extract.cu) decode DenseNodes, join node locations to way refs and check ring validity.
 *
 * rsb_pbf_frames: lists the [uint32 BE length][BlobHeader][Blob] frames of file_host[0 .. n) into frames_host int64
 * [capacity][RSB_PBF_FRAME_FIELDS] = (kind, compression, data offset, data length, raw_size, frame offset); *count_host = the number of
 * frames (only the first `capacity` are written). Errors: a truncated frame, a BlobHeader of 64 KiB or more, a Blob or raw_size over
 * 32 MiB, malformed messages.
 * rsb_pbf_inflate: blob i (frames_host row i) -> out_host + out_offsets_host[i], exactly raw_size bytes, with RSB_PBF_INFLATE_PAD
 * writable bytes after each; `threads` threads. raw and zlib_data are supported; any other compression, a corrupt zlib stream or an
 * inflated size other than raw_size is an error naming the blob.
 * rsb_pbf_check_header: an OSMHeader's HeaderBlock; a required feature other than OsmSchema-V0.6 and DenseNodes is an error naming it.
 * rsb_pbf_parse: the PrimitiveBlocks blocks_host + offsets_host[i] (sizes_host[i] bytes) -> *result (free with rsb_pbf_result_free;
 * read with rsb_pbf_result_sizes / rsb_pbf_result_copy, element counts of RSB_PBF_OUT_*):
 *   RSB_PBF_WAYS: keys_host = nkeys NUL-terminated keys back to back; keys[0] is the anchor. The ways whose first keys[0] tag exists
 *     (and equals anchor_value_host, unless that is NULL or empty), in file order: WAY_IDS int64 [W], REF_OFFSETS int64 [W + 1],
 *     REFS int64 node ids (delta-decoded), TAGS int32 [W][nkeys] = index of the key's first value in STRING_OFFSETS int64 [S + 1] /
 *     STRING_BYTES, or -1. KINDS int32 [n] = RSB_PBF_HAS_* bits of each block.
 *   RSB_PBF_NODES: SEGS int64 [G][RSB_PBF_SEG_FIELDS], the node runs of the blocks in element order: kind 0 is a DenseNodes group
 *     whose packed id / lat / lon fields lie at the given offsets from its block's start (COUNT values each), kind 1 a run of COUNT
 *     nodes decoded here into HOST_IDS int64 / HOST_XY int32 [][2] from HOST_FIRST (plain Nodes, and DenseNodes with unpacked fields).
 *     Coordinates: x = (lon * granularity + lon_offset) / 100 in int64 (truncating), INT32_MIN outside +-180e7; y likewise with
 *     lat, +-90e7. */
#define RSB_PBF_FRAME_FIELDS 6
#define RSB_PBF_BLOB_HEADER 0
#define RSB_PBF_BLOB_DATA 1
#define RSB_PBF_BLOB_OTHER 2
#define RSB_PBF_RAW 0
#define RSB_PBF_ZLIB 1
#define RSB_PBF_NO_DATA 6
#define RSB_PBF_INFLATE_PAD 64
#define RSB_PBF_WAYS 0
#define RSB_PBF_NODES 1
#define RSB_PBF_MAX_KEYS 8
#define RSB_PBF_HAS_NODES 1
#define RSB_PBF_HAS_DENSE 2
#define RSB_PBF_HAS_WAYS 4
#define RSB_PBF_HAS_RELATIONS 8
#define RSB_PBF_OUT_KINDS 0
#define RSB_PBF_OUT_WAY_IDS 1
#define RSB_PBF_OUT_REF_OFFSETS 2
#define RSB_PBF_OUT_REFS 3
#define RSB_PBF_OUT_TAGS 4
#define RSB_PBF_OUT_STRING_OFFSETS 5
#define RSB_PBF_OUT_STRING_BYTES 6
#define RSB_PBF_OUT_SEGS 7
#define RSB_PBF_OUT_HOST_IDS 8
#define RSB_PBF_OUT_HOST_XY 9
#define RSB_PBF_OUT_COUNT 10
#define RSB_PBF_SEG_FIELDS 16
#define RSB_PBF_SEG_BLOCK 0
#define RSB_PBF_SEG_KIND 1
#define RSB_PBF_SEG_COUNT 2
#define RSB_PBF_SEG_ID_OFF 3
#define RSB_PBF_SEG_ID_LEN 4
#define RSB_PBF_SEG_LAT_OFF 5
#define RSB_PBF_SEG_LAT_LEN 6
#define RSB_PBF_SEG_LON_OFF 7
#define RSB_PBF_SEG_LON_LEN 8
#define RSB_PBF_SEG_GRANULARITY 9
#define RSB_PBF_SEG_LAT_OFFSET 10
#define RSB_PBF_SEG_LON_OFFSET 11
#define RSB_PBF_SEG_HOST_FIRST 12
#define RSB_PBF_SEG_OUT_FIRST 13
int rsb_pbf_frames(const uint8_t* file_host, int64_t n, int64_t* frames_host, int64_t capacity, int64_t* count_host);
int rsb_pbf_inflate(const uint8_t* file_host, const int64_t* frames_host, int32_t n, uint8_t* out_host, const int64_t* out_offsets_host, int32_t threads);
int rsb_pbf_check_header(const uint8_t* block_host, int64_t n);
int rsb_pbf_parse(const uint8_t* blocks_host, const int64_t* offsets_host, const int64_t* sizes_host, int32_t n, int32_t mode, const char* keys_host,
                  int32_t nkeys, const char* anchor_value_host, int32_t threads, void** result);
int rsb_pbf_result_sizes(const void* result, int64_t* sizes_host);
int rsb_pbf_result_copy(const void* result, int32_t what, void* dst_host, int64_t count);
void rsb_pbf_result_free(void* result);
/* Device. rsb_pbf_dense_nodes: decodes the DenseNodes segments (kind 0 rows of rsb_pbf_parse's SEGS, DEVICE int64 [G][RSB_PBF_SEG_FIELDS],
 * offsets relative to blocks + block_offsets[SEG_BLOCK], blocks padded by RSB_PBF_INFLATE_PAD readable bytes) into records
 * SEG_OUT_FIRST .. + COUNT of ids int64 [] and xy int32 [][2] (coordinates as above). Varints of up to 10 bytes; status int32 [1] is
 * cleared and then set non-zero for a varint longer than 10 bytes or a segment that does not hold COUNT values. */
int rsb_pbf_dense_nodes(const uint8_t* blocks, const int64_t* block_offsets, const int64_t* segs, int32_t G, int64_t* ids, int32_t* xy, int32_t* status,
                        void* stream);
/* rsb_extract_locate: for node records i < n (ids int64, xy int32 [n][2]) of global ordinal ordinal_base + i, whose biased id
 * (id XOR 2^63, as uint64) is found in the ascending unique keys[0 .. num_keys), best[k] = max(best[k], ordinal + 1) and then, where
 * that ordinal won, loc[k] = xy[i]: the last record of an id in file order wins. best (uint64, zero = not seen) and loc (int32 [][2])
 * persist across calls made in file order. */
int rsb_extract_locate(const int64_t* ids, const int32_t* xy, int64_t n, int64_t ordinal_base, const int64_t* keys, int64_t num_keys, int64_t* best,
                       int32_t* loc, void* stream);
/* rsb_extract_gather: for refs i < num_refs (biased ids) of way ref_way[i] < num_ways: verts int32 [num_refs][2] = the location of the ref;
 * flags int32 [num_ways] (cleared here) |= 1 for a ref not in keys or never located, 2 for an invalid location. */
int rsb_extract_gather(const int64_t* refs, const int32_t* ref_way, int64_t num_refs, int32_t num_ways, const int64_t* keys, int64_t num_keys,
                       const int64_t* best, const int32_t* loc, int32_t* verts, int32_t* flags, void* stream);
/* rsb_extract_valid: `features.polygon_is_valid([ring])` for rings r < R (verts int32 [][2] from ring_offsets[r] to ring_offsets[r + 1],
 * closed: the last vertex repeats the first) on the integer lattice, exactly: after dropping the closing vertex and consecutive
 * repeats (the compacted ring goes to scratch int32 [][2] at the same offsets, its length to lens int32 [R]), >= 3 distinct
 * positions, non-zero area, and no two edges meet except adjacent edges in their shared vertex. Rings with flags[r] != 0 are
 * skipped (valid 0). Rings of more than RSB_EXTRACT_WARP_RING vertices are checked pair tile by pair tile: long int32 [L] lists
 * them (ascending), tile_offsets int64 [L + 1] the prefix of their tile counts ceil(n / 64)^2. valid uint8 [R]. */
#define RSB_EXTRACT_WARP_RING 256
int rsb_extract_valid(const int32_t* verts, const int64_t* ring_offsets, int32_t R, const int32_t* flags, const int32_t* long_rings, int32_t L,
                      const int64_t* tile_offsets, int32_t* scratch, int32_t* lens, uint8_t* valid, void* stream);

/* `rs compare` (robosat/tools/compare.py; the rule is restated in DESIGN.md §8). Device pointers unless noted.
 * rsb_compare_count: masks uint8 [N][M] planes of hw bytes, plane (n, m) at masks + (n * M + m) * pitch; labels uint8 [N] planes at
 * labels + n * pitch, or NULL. counts int64 [N][M][4] = (tp, fp, fn, tn) of mask (n, m) against label n, where "foreground" is
 * index != 0 in both; without labels the label is taken as all background (tp = fn = 0). The mask's non-zero count, the
 * numerator of the coverage filter, is tp + fp. pitch % 16 == 0 and 16-byte aligned planes; integer sums, so the counts do not
 * depend on the launch shape. 1 <= M <= RSB_COMPARE_MAX_PLANES - 1; allocates nothing and does not synchronise. */
#define RSB_COMPARE_MAX_PLANES 32
int rsb_compare_count(const uint8_t* masks, const uint8_t* labels, int32_t N, int32_t M, int64_t hw, int64_t pitch, int64_t* counts, void* stream);
/* rsb_compare_class_counts: the per-class agreement of `rs compare --csv --dataset`, on the planes of rsb_compare_count (same
 * layout, pitch and alignment rules; labels NULL counts every label pixel as class 0). For C classes, 2 <= C <=
 * RSB_COMPARE_MAX_CLASSES, it writes int64 label_hist [N][C] (pixels of label n equal to c), mask_hist [N][M][C] (pixels of mask
 * (n, m) equal to c), both_hist [N][M][C] (pixels where label n == mask (n, m) == c) and out_of_range [N][1 + M] (pixels >= C in
 * label n, then in each mask). Then tp = both, fp = mask - both, fn = label - both, tn = hw - label - mask + both per class.
 * Integer sums, so the counts do not depend on the launch shape; allocates nothing and does not synchronise. */
#define RSB_COMPARE_MAX_CLASSES 256
int rsb_compare_class_counts(const uint8_t* masks, const uint8_t* labels, int32_t N, int32_t M, int32_t C, int64_t hw, int64_t pitch,
                             int64_t* label_hist, int64_t* mask_hist, int64_t* both_hist, int64_t* out_of_range, void* stream);
/* rsb_compare_compose: the side-by-side composite image | plane 0 | plane 1 | ... of N tiles of H x W. images uint8 [N][H][W][3]
 * (image n at images + n * H * W * 3); planes uint8 [N][P] index planes of H * W bytes at planes + (n * P + p) * pitch (plane 0 is
 * the label, planes 1.. the masks); palettes uint32 [N][P][256] (r | g << 8 | b << 16). out uint8 [N][H][(1 + P) * W][3], tile n
 * at out + n * out_stride, out_stride % 16 == 0; `out` may be pinned host memory (written through its device mapping) or device
 * memory. 1 <= P <= RSB_COMPARE_MAX_PLANES - 1; allocates nothing and does not synchronise. */
int rsb_compare_compose(const uint8_t* images, const uint8_t* planes, const uint32_t* palettes, int32_t N, int32_t P, int32_t H, int32_t W,
                        int64_t pitch, uint8_t* out, int64_t out_stride, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Host-side PNG codec for the files either side of the predict path (HOST pointers, plain C over zlib, no Python / GIL so the
 * tools' pool threads run truly in parallel). Pixel-identical to PIL; not a compute fallback -- no device work happens here.
 */
/* `Image.open(path).convert("RGB")` (robosat/tiles.py:150-159,181) for 8-bit non-interlaced PNGs (gray, RGB, palette, +alpha):
 * out_rgb_host uint8 [h][w][3]. RSB_E_UNSUPPORTED for other PNG flavours / non-PNG files (the caller then uses PIL). */
/* zlib-wrapped DEFLATE stream (RFC 1950 / 1951; what PNG IDAT chunks carry) -> exactly out_len bytes, Adler-32 verified, with the
 * library's own decoder (csrc/rsb_inflate.cpp); RSB_E_INVALID for anything it rejects (the PNG reader then asks zlib). */
int rsb_zlib_inflate(const uint8_t* stream_host, int64_t n, uint8_t* out_host, int64_t out_len);
int rsb_png_decode_rgb(const uint8_t* file_bytes_host, int64_t n, uint8_t* out_rgb_host, int32_t w_expected, int32_t h_expected);
int rsb_png_read_rgb(const char* path, uint8_t* out_rgb_host, int32_t w_expected, int32_t h_expected);
/* `Image.fromarray(q, mode="P"); putpalette(palette); save(path)` (robosat/tools/predict.py:105-113): 8-bit palette PNG,
 * palette_rgb_host uint8 [entries][3]; level = zlib level (0-9, <0 default). Noise-like rasters (a level-1 probe of 16 rows does not
 * shrink below 90 %) are coded with zlib's Z_RLE strategy: same size, a third of the time. encode returns the byte count or a
 * negative code. */
int64_t rsb_png_encode_p8(const uint8_t* pixels_host, int32_t w, int32_t h, const uint8_t* palette_rgb_host, int32_t entries, int32_t level,
                          uint8_t* out_host, int64_t capacity);
int rsb_png_write_p8(const char* path, const uint8_t* pixels_host, int32_t w, int32_t h, const uint8_t* palette_rgb_host, int32_t entries,
                     int32_t level);

/* Whole-batch variants, fanned out over `threads` threads inside the library (one call per tile batch from the tools):
 * read: rcs_host[i] receives the per-file code (RSB_E_UNSUPPORTED entries are left for another decoder); the return value is the
 * worst real error. write: image i is pixels_host + i*image_stride; make_dirs != 0 creates the parent directories (z/x/). */
int rsb_png_read_rgb_batch(const char* const* paths, int32_t n, uint8_t* const* outs_rgb_host, int32_t w_expected, int32_t h_expected,
                           int32_t threads, int32_t* rcs_host);
int rsb_png_write_p8_batch(const char* const* paths, int32_t n, const uint8_t* pixels_host, int64_t image_stride, int32_t w, int32_t h,
                           const uint8_t* palette_rgb_host, int32_t entries, int32_t level, int32_t threads, int32_t make_dirs);

/* `Image.open(path).convert("P")` of `rs compare` (robosat/tools/compare.py:31-38) for non-interlaced palette PNGs of 1, 2, 4 or 8
 * bits and 8-bit gray PNGs: out_index_host uint8 [h][w] (the index plane; gray: index = value), out_palette_rgb_host uint8 [256][3]
 * (the PLTE entries, zero past them; gray: the ramp (i, i, i)), *entries_host = the PLTE entry count (gray: 256). A tRNS chunk is
 * ignored. RSB_E_UNSUPPORTED for other PNG flavours / non-PNG files (the caller then uses PIL). */
int rsb_png_decode_indexed(const uint8_t* file_bytes_host, int64_t n, uint8_t* out_index_host, uint8_t* out_palette_rgb_host, int32_t* entries_host,
                           int32_t w_expected, int32_t h_expected);
int rsb_png_read_indexed(const char* path, uint8_t* out_index_host, uint8_t* out_palette_rgb_host, int32_t* entries_host, int32_t w_expected,
                         int32_t h_expected);
/* file i -> outs_index_host[i], palettes_rgb_host + i * 768, entries_host[i]; per-file codes in rcs_host as rsb_png_read_rgb_batch */
int rsb_png_read_indexed_batch(const char* const* paths, int32_t n, uint8_t* const* outs_index_host, uint8_t* palettes_rgb_host,
                               int32_t* entries_host, int32_t w_expected, int32_t h_expected, int32_t threads, int32_t* rcs_host);
/* `combined.save(path, optimize=True)` of `rs compare` (compare.py:66-67): 8-bit RGB PNG (colour type 2) of pixels_host uint8
 * [h][w][3], with rsb_png_encode_p8's level and Z_RLE policy; same pixels as PIL's file, different compressed bytes. */
int64_t rsb_png_encode_rgb8(const uint8_t* pixels_host, int32_t w, int32_t h, int32_t level, uint8_t* out_host, int64_t capacity);
/* image i is pixels_host + i * image_stride; make_dirs != 0 creates the parent directories (z/x/) */
int rsb_png_write_rgb8_batch(const char* const* paths, int32_t n, const uint8_t* pixels_host, int64_t image_stride, int32_t w, int32_t h,
                             int32_t level, int32_t threads, int32_t make_dirs);

/* ---------------------------------------------------------------------------------------------
 * `rs tile`: slippy-map RGB tiles from a GeoTIFF (the rule is DESIGN.md §8; robosat_b200/tile.py plans the work).
 */
/* Decode raster rows [row0, row0 + rows) x columns [col0, col0 + cols) of an 8-bit chunky (PlanarConfiguration 1) TIFF image into
 * out_host uint8 [rows][cols][spp], on `threads` threads of the library's own. file_host: the file's bytes [file_len] (e.g. a memory
 * map); chunk i (strip, or tile in row-major order) is file_host[chunk_offsets_host[i] .. + chunk_bytes_host[i]). tiled = 0: strips
 * of chunk_h rows (chunk_w = width; the last strip holds the remaining rows); tiled = 1: tiles of chunk_w x chunk_h, ragged tiles
 * stored whole. spp 1, 3 or 4; compression 1 (none), 5 (LZW), 8 or 32946 (zlib DEFLATE); predictor 1 or 2 (horizontal
 * differencing). Only the chunks the window touches are read. A chunk that cannot be decoded (outside the file, too short, truncated
 * or corrupt stream, bad LZW code) gives RSB_E_INVALID with a message naming the strip or tile and *bad_chunk_host = its index
 * (-1 otherwise; bad_chunk_host may be NULL). Host only: no device needed. */
int rsb_tiff_decode_window(const uint8_t* file_host, int64_t file_len, const int64_t* chunk_offsets_host, const int64_t* chunk_bytes_host,
                           int64_t num_chunks, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled, int32_t spp,
                           int32_t compression, int32_t predictor, int64_t row0, int64_t rows, int64_t col0, int64_t cols, uint8_t* out_host,
                           int32_t threads, int64_t* bad_chunk_host);

/* The band rule (DESIGN.md §8): decode raster rows [row0, row0 + rows) x columns [col0, col0 + cols) of an uncompressed, LZW or
 * DEFLATE TIFF of spp samples per pixel, bits 8 or 16 each, into out_host [rows][cols][k]: sample j of a pixel is band
 * select_host[j] (0-based, 1 <= k <= 4), uint8 or native-endian uint16. planar 1: chunky chunks as rsb_tiff_decode_window;
 * planar 2: num_chunks holds spp planes of chunks, band after band, and only the selected bands' chunks are read. big_endian: the
 * file's byte order. predictor 2 undoes horizontal differencing on whole samples, modulo 2^bits, after the byte-order conversion.
 * Errors as rsb_tiff_decode_window (the bad chunk's index counts the planes before it). Host only: no device needed. */
int rsb_tiff_decode_bands(const uint8_t* file_host, int64_t file_len, const int64_t* chunk_offsets_host, const int64_t* chunk_bytes_host,
                          int64_t num_chunks, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled, int32_t spp,
                          int32_t bits, int32_t planar, int32_t big_endian, int32_t compression, int32_t predictor, const int32_t* select_host,
                          int32_t k, int64_t row0, int64_t rows, int64_t col0, int64_t cols, void* out_host, int32_t threads, int64_t* bad_chunk_host);

/* JPEG (Compression 7) strips or tiles (DESIGN.md §8). Parse JPEGTables (tables_host [tables_len], tables_len 0 when absent) and
 * the headers of the chunks select_host [num_select] (NULL: all num_chunks chunks, in order) of file_host (chunk_offsets_host,
 * chunk_bytes_host, the raster and chunk sizes as rsb_tiff_decode_window; rows_per_strip is the TIFF's RowsPerStrip, at least
 * chunk_h, and bounds a strip's frame height) on `threads` of the library's threads. spp 1 with photometric 1, or spp 3 with
 * photometric 2 (RGB) or 6 (YCbCr). descs_host int64 [chunks parsed][RSB_JPEG_DESC_FIELDS], in parse order: the file offset and
 * length of the chunk's entropy-coded bytes, its table set, frame width and height, luma sampling h and v, restart interval,
 * block count, 0 (the first block, for the decoder), its index and 0. sets_host NULL: no table sets are built, the descriptors'
 * table set is -1 and *num_sets_host = 0. Otherwise the distinct table sets of the parsed chunks, in order of first use, go to
 * sets_host int32 [max_sets][RSB_JPEG_SET_WORDS] (quantisation tables in natural order, then per component libjpeg's derived DC and
 * AC Huffman tables); *num_sets_host gets their count, and when it exceeds max_sets nothing is written to sets_host (call again
 * with room). A stream outside the rule gives RSB_E_INVALID with a message starting "Compression 7 (JPEG)" that names the value
 * found and the strip or tile, *bad_chunk_host = its index (-1 otherwise; may be NULL). Host only: no device needed. */
#define RSB_JPEG_DESC_FIELDS 12
#define RSB_JPEG_SET_WORDS 3480
#define RSB_JPEG_SCRATCH_PER_BLOCK 192
int rsb_jpeg_parse_chunks(const uint8_t* file_host, int64_t file_len, const uint8_t* tables_host, int64_t tables_len, const int64_t* chunk_offsets_host,
                          const int64_t* chunk_bytes_host, int64_t num_chunks, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h,
                          int64_t rows_per_strip, int32_t tiled, int32_t spp, int32_t photometric, const int64_t* select_host, int64_t num_select,
                          int32_t threads, int64_t* descs_host, int32_t* sets_host, int32_t max_sets, int32_t* num_sets_host, int64_t* bad_chunk_host);
/* scratch bytes of rsb_jpeg_decode_window for total_blocks blocks: RSB_JPEG_SCRATCH_PER_BLOCK * total_blocks (-1 if negative) */
int64_t rsb_jpeg_scratch_bytes(int64_t total_blocks);
/* Decode raster rows [row0, row0 + rows) x columns [col0, col0 + cols) of a JPEG TIFF into out uint8 [rows][cols][spp] on `stream`
 * (device pointers). The chunks the window touches, row-major over their rectangle, are descs int64 [num_chunks][RSB_JPEG_DESC_FIELDS]
 * as rsb_jpeg_parse_chunks gives them, but with offsets into staged [staged_len] (their entropy-coded bytes) and first blocks
 * ascending, each chunk's blocks inside [0, total_blocks); sets int32 [num_sets][RSB_JPEG_SET_WORDS]. scratch: at least
 * rsb_jpeg_scratch_bytes(total_blocks) bytes, 16-byte aligned. errors int64 [num_chunks]: 0, or a data error code | MCU << 8 (1
 * invalid Huffman code, 2 AC index past 63, 3 unexpected marker or RST number, 4 extraneous bytes before a marker, 5 data ends
 * before the last MCU, 6 a descriptor outside the staged bytes, the scratch or the table sets, or inconsistent with its block
 * count); the IDCT and pixel stages skip a chunk whose error word is not 0, so its pixels are left 0. Pixels follow libjpeg-turbo's default decompression (islow IDCT, fancy upsampling, integer YCbCr -> RGB for
 * photometric 6). Arguments are validated before the device check; allocates nothing and does not synchronise. */
int rsb_jpeg_decode_window(const uint8_t* staged, int64_t staged_len, const int64_t* descs, int32_t num_chunks, const int32_t* sets,
                           int32_t num_sets, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled, int32_t spp,
                           int32_t photometric, int64_t row0, int64_t rows, int64_t col0, int64_t cols, uint8_t* out, void* scratch,
                           int64_t scratch_bytes, int64_t total_blocks, int64_t* errors, void* stream);

/* Warp N tiles of size x size of zoom z from a source window. src uint8 [win_rows][src_pitch] holds raster rows
 * [win_row0, + win_rows) x columns [win_col0, + win_cols) of a raster_w x raster_h image, spp (1, 3 or 4) samples per pixel (spp = 4:
 * 4-byte aligned rows). A pixel is valid unless alpha = 1 and its 4th sample is 0, or its colour samples (1 or 3) all equal nodata
 * (-1: none). nodes float64 [nodes_h][nodes_w][2] (16-byte aligned): the source coordinates (u, v) of global tile pixel centres
 * (kG + 1/2, lG + 1/2) for k = node_x0 + column, l = node_y0 + row, G = grid_step (a power of two <= RSB_TILE_MAX_STEP). tiles
 * int64 [N][2] = (x, y); pixel (c, r) of tile n is global pixel (x S + c, y S + r) and interpolates the four nodes of its lattice
 * cell with weights (g - kG) / G, then samples: nearest (resampling 0) or bilinear (1), per DESIGN.md §8; every float64 operation
 * rounded separately. out uint8 RGB [N][size][size][3] at out + n * image_stride; an uncovered pixel is (0, 0, 0). covered int64
 * [N] = covered pixels per tile; misses int64 [1] = samples inside the raster but outside the window, plus pixels whose lattice
 * cell lies outside `nodes` (0 unless the host planned wrongly; such pixels are left uncovered). Both are cleared by the call.
 * 1 <= N <= 65535, 1 <= size <= RSB_TILE_MAX_SIZE. Arguments are validated before the device check; allocates nothing and does
 * not synchronise. */
#define RSB_TILE_MAX_SIZE 4096
#define RSB_TILE_MAX_STEP 64
int rsb_tile_warp(const uint8_t* src, int64_t src_pitch, int64_t win_row0, int64_t win_col0, int64_t win_rows, int64_t win_cols,
                  int64_t raster_w, int64_t raster_h, int32_t spp, int32_t alpha, int32_t nodata, const double* nodes, int64_t node_x0,
                  int64_t node_y0, int32_t nodes_w, int32_t nodes_h, int32_t grid_step, const int64_t* tiles, int32_t N, int32_t size,
                  int32_t resampling, uint8_t* out, int64_t image_stride, int64_t* covered, int64_t* misses, void* stream);

/* `rs tile --resampling average` (DESIGN.md §8): the arguments of rsb_tile_warp without `resampling`, but nodes hold the source
 * coordinates (u, v) of global tile pixel corners (kG, lG). Each corner of pixel (gx, gy), the integer corners (gx, gy) to
 * (gx + 1, gy + 1), interpolates the four nodes of the lattice cell that contains it; the pixel averages the source pixels its corners'
 * axis-aligned bounding box overlaps, clipped to the raster, weighted by the overlap of each pixel's row and column with the box and
 * summed row by row over valid pixels, every float64 operation rounded separately. A pixel with a NaN corner, an empty clipped box
 * or no valid weight is uncovered (0, 0, 0). A box wider or taller than RSB_TILE_MAX_FOOTPRINT source pixels is not summed: the pixel
 * is uncovered and counted in misses (the host refuses such runs first). Arguments are validated before the device check; allocates
 * nothing and does not synchronise. */
#define RSB_TILE_MAX_FOOTPRINT 64
int rsb_tile_average(const uint8_t* src, int64_t src_pitch, int64_t win_row0, int64_t win_col0, int64_t win_rows, int64_t win_cols,
                     int64_t raster_w, int64_t raster_h, int32_t spp, int32_t alpha, int32_t nodata, const double* nodes, int64_t node_x0,
                     int64_t node_y0, int32_t nodes_w, int32_t nodes_h, int32_t grid_step, const int64_t* tiles, int32_t N, int32_t size,
                     uint8_t* out, int64_t image_stride, int64_t* covered, int64_t* misses, void* stream);

/* The band rule (DESIGN.md §8). src [rows][cols][nsel + alpha] samples of `bits` (8: uint8, 16: uint16), 16-byte aligned: nsel (1
 * or 3) selected bands, then the alpha band when alpha = 1. A pixel is invalid when its alpha sample is 0 or every selected band
 * equals nodata (-1: none; else 0 .. 2^bits - 1). rsb_tile_render writes out uint8 [rows][out_pitch] (4-byte aligned, out_pitch a
 * multiple of 4 and at least 4 cols): per pixel R, G, B, A with band b's value v = floor((510 t + d) / (2 d)), d = HI - LO,
 * t = clamp(s, LO, HI) - LO for scale_host int32 [nsel][2] = (LO, HI), 0 <= LO < HI <= 2^bits - 1 (one band: R = G = B = v), and
 * A = 0 for an invalid pixel, else 255; the input rsb_tile_warp and rsb_tile_average take with spp 4, alpha 1, nodata -1.
 * rsb_band_histogram adds the count of every value of each selected band over the valid pixels to hist int64 [nsel][2^bits], which
 * it does not clear. Arguments are validated before the device check; neither allocates nor synchronises. */
int rsb_tile_render(const void* src, int64_t rows, int64_t cols, int32_t bits, int32_t nsel, int32_t alpha, int32_t nodata, const int32_t* scale_host,
                    uint8_t* out, int64_t out_pitch, void* stream);
int rsb_band_histogram(const void* src, int64_t rows, int64_t cols, int32_t bits, int32_t nsel, int32_t alpha, int32_t nodata, int64_t* hist,
                       void* stream);

/* rs mosaic (DESIGN.md §8): deflate the chunk x chunk tiles of one row of a 1-band 8-bit raster window. window_host uint8 rows x cols
 * (row pitch `pitch`, rows <= chunk); tile k holds columns [k chunk, (k + 1) chunk) and is padded with `fill` past the window's rows
 * and columns, then zlib-compressed (compress2 at `level`) into out_host + k * chunk_cap; sizes_host int64 [ceil(cols / chunk)] gets
 * the compressed byte counts. chunk_cap >= rsb_tiff_deflate_bound(chunk * chunk). Tiles are compressed on `threads` of the library's
 * threads. Host only: no device needed. */
int64_t rsb_tiff_deflate_bound(int64_t n);
int rsb_tiff_encode_chunks(const uint8_t* window_host, int64_t pitch, int32_t rows, int32_t cols, int32_t chunk, int32_t fill, int32_t level,
                           uint8_t* out_host, int64_t chunk_cap, int64_t* sizes_host, int32_t threads);

/* rs mosaic (DESIGN.md §8): slippy-map index tiles of zoom `zoom` (size x size) sampled onto a window of an output raster. planes uint8
 * [num_planes] x plane_stride: the decoded index planes (row-major size x size). slots int32 [tiles_h][tiles_w]: the plane of tile
 * (tile_x0 + column, tile_y0 + row), -1 when it has no file. nodes float64 [nodes_h][nodes_w][2] (16-byte aligned): the global
 * pixel coordinates (gx, gy) of the centres of output pixels (kG, lG), k = node_x0 + column, l = node_y0 + row, G = grid_step (a power
 * of two <= RSB_TILE_MAX_STEP). Output pixel (out_col0 + c, out_row0 + r), 0 <= c < out_cols, 0 <= r < out_rows, interpolates the
 * four nodes of its lattice cell with weights (i - kG) / G and samples nearest (resampling 0) or bilinear (1), per DESIGN.md §8, every
 * float64 operation rounded separately; it is written to out + r * out_pitch + c, `nodata` (0..255) when uncovered. covered int64 [1]
 * = covered pixels; misses int64 [1] = samples inside the world but outside the slot table, plus pixels whose lattice cell lies
 * outside `nodes` (0 unless the host planned wrongly; such pixels are left uncovered). Both are cleared by the call. Arguments are
 * validated before the device check; allocates nothing and does not synchronise. */
int rsb_mosaic_warp(const uint8_t* planes, int64_t plane_stride, int32_t num_planes, const int32_t* slots, int64_t tile_x0, int64_t tile_y0,
                    int32_t tiles_w, int32_t tiles_h, int32_t zoom, int32_t size, const double* nodes, int64_t node_x0, int64_t node_y0,
                    int32_t nodes_w, int32_t nodes_h, int32_t grid_step, int64_t out_col0, int64_t out_row0, int32_t out_cols, int32_t out_rows,
                    int32_t resampling, int32_t nodata, uint8_t* out, int64_t out_pitch, int64_t* covered, int64_t* misses, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Losses and metrics on fp32 NCHW logits + int64 targets [N][H][W].
 */
/* CrossEntropyLoss2d.forward (losses.py:24-25): weighted NLL of log_softmax, mean over sum of target weights.
 * loss_out: fp32 scalar; grad (optional, fp32 NCHW) receives dLoss/dlogits. weight may be NULL (all ones).
 * scratch: >= 2 doubles, zeroed by the call. */
int rsb_cross_entropy(const float* logits, const int64_t* targets, const float* weight, float* loss_out, float* grad,
                      double* scratch, int32_t N, int32_t C, int32_t HW, void* stream);

/* FocalLoss2d.forward (losses.py:49-50): NLLLoss(weight)((1 - softmax)^gamma * log_softmax, targets) + gradient. scratch: 2 doubles. */
int rsb_focal(const float* logits, const int64_t* targets, const float* weight, float gamma, float* loss_out, float* grad,
              double* scratch, int32_t N, int32_t C, int32_t HW, void* stream);
/* mIoULoss2d.forward (losses.py:71-83): max(1 - mean_{c,n} soft-IoU, weighted cross entropy); the gradient is the one of
 * whichever term is larger (decided on the device, no host synchronisation). scratch: rsb_miou_scratch_doubles(N, C) doubles. */
int64_t rsb_miou_scratch_doubles(int32_t N, int32_t C);
int rsb_miou(const float* logits, const int64_t* targets, const float* weight, float* loss_out, float* grad, double* scratch,
             int32_t N, int32_t C, int32_t HW, void* stream);

/* LovaszLoss2d.forward (losses.py:96-119) and its closed-form gradient (SURVEY.md A8), per image:
 * errors e = 1 - (2*onehot-1)*x over the flattened C*H*W vector, descending sort, Jaccard gradient, dot(relu(e), J).
 * workspace: rsb_lovasz_workspace_bytes(N, C, HW) bytes. loss_out: fp32 scalar (mean over N). grad optional. */
int64_t rsb_lovasz_workspace_bytes(int32_t N, int32_t C, int32_t HW);
int rsb_lovasz(const float* logits, const int64_t* targets, float* loss_out, float* grad, void* workspace,
               int64_t workspace_bytes, int32_t N, int32_t C, int32_t HW, void* stream);

/* Metrics.add (metrics.py:27-41) for a whole batch: counts[4] += {tn, fn, fp, tp} with the reference's
 * argmax / (pred/actual in {NaN, inf, 0, 1}) semantics. counts: int64[4] on the device, accumulated. */
int rsb_metrics_count(const float* logits, const int64_t* targets, int64_t* counts, int32_t N, int32_t C, int32_t HW,
                      void* stream);

/* torch.optim.Adam.step (train.py:81,188) over one flat fp32 parameter arena:
 * betas (b1,b2), eps, no weight decay, no amsgrad; `step` is the 1-based step count for bias correction. */
int rsb_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float b1,
                  float b2, float eps, int32_t step, void* stream);

/* Same update behind an overflow guard for mixed-precision training (no host synchronisation): if `grad` holds an inf / NaN the
 * whole step is skipped on the device (parameters and moments untouched). guard_state: int32[4] on the device, zero-initialised by
 * the caller once -- [0] scratch flag, [1] steps skipped so far (bias corrections use step - skipped), [2] flag of the last
 * finished step (poll it to adapt the loss scale), [3] steps seen. With no skipped step the result equals rsb_adam_step's to the last bit
 * of each value (the two kernels' updates are contracted into fused multiply-adds differently). */
int rsb_adam_step_guarded(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float b1,
                          float b2, float eps, int32_t step, int32_t* guard_state, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training path (robosat/tools/train.py:163-201: net.train() forward, loss.backward()). Activations and activation
 * gradients are NHWC fp16 [M = N*H*W][C]; gradients carry the caller's loss scale; parameter gradients are fp32, unscaled.
 */
/* train-mode BatchNorm2d (torchvision resnet50 inside unet.py:122-130): batch statistics -> apply -> backward, each launched with
 * programmatic stream serialization so that a chain of small kernels does not pay a full launch gap per link.
 * sums: 20*C doubles of scratch (8 replicated accumulator slots, arrival counter, backward coefficients), zero-initialised ONCE by
 * the caller: the last block of each reduction leaves it zeroed again, and no call clears it with a memset. The "_chained" suffix
 * marks these semantics. */
/* batch statistics from the per-quarter-tile partial sums a convolution wrote through rsb_conv_desc.stats (partials: fp32
 * [rows][2][C], rows = spatial tiles * 4; 1/8 of the bytes of z): mean, invstd, scale = gamma*invstd, shift = beta - mean*scale,
 * and running_mean / running_var (unbiased, momentum) / num_batches_tracked updated when those pointers are non-NULL. */
int rsb_bn_partials_finalize(const float* partials, int64_t rows, double* sums, const float* gamma, const float* beta, float* running_mean,
                             float* running_var, int64_t* num_batches, float* mean, float* invstd, float* scale, float* shift, int64_t M,
                             int32_t C, float eps, float momentum, void* stream);
/* y = relu?(z*scale + shift (+ residual)) */
int rsb_bn_apply_chained(const void* z, const float* scale, const float* shift, const void* residual, void* y, int64_t M, int32_t C,
                         int32_t relu, void* stream);
/* autograd of relu(bn(z) (+ identity)): g = dy * (y > 0) (y NULL: no mask); dz = gamma*invstd*(g - mean(g) - zhat*mean(g*zhat));
 * g_out (optional) receives g = the gradient of the identity branch; dgamma/dbeta fp32 multiplied by inv_loss_scale.
 * mask_scale / mask_shift (with y NULL): the output was the plain y = half(relu(z*scale + shift)) of rsb_bn_apply_chained, so its
 * ReLU mask is re-derived from z (bit-identical: half(o) > 0 <=> o > 2^-25) and y is not read at all. */
int rsb_bn_backward_chained(const void* dy, const void* y, const void* z, const float* mean, const float* invstd, const float* gamma,
                            const float* mask_scale, const float* mask_shift, double* sums, void* dz, void* g_out, float* dgamma, float* dbeta,
                            float inv_loss_scale, int64_t M, int32_t C, void* stream);
/* out = (a (+ b)) * (y > 0): ReLU backward with optional gradient fan-in (skip connections); y NULL: plain sum */
int rsb_relu_backward(const void* a, const void* b, const void* y, void* out, int64_t n, void* stream);
/* autograd of max_pool2d (unet.py:125, :132) on NHWC fp16: first maximum of every window receives its gradient.
 * argmax_scratch: N*OH*OW*C bytes of device scratch (one window position per pooled element) -> two streaming passes;
 * NULL -> single-pass kernel that re-derives the argmax per input pixel (slower, no scratch). Same results. */
int rsb_maxpool_backward(const void* x, const void* dy, void* dx, void* argmax_scratch, int32_t N, int32_t H, int32_t W, int32_t C,
                         int32_t k, int32_t s, int32_t p, void* stream);
/* autograd's AccumulateGrad for every parameter at once (loss.backward(), train.py:186): dst_i[0:n_i] += alpha * src_i[0:n_i]
 * for `segments` rows (src pointer, dst pointer, n_i <= 2^31) of a device-resident int64 table; fp32, one block per row. */
int rsb_multi_axpy(const int64_t* table, int32_t segments, float alpha, void* stream);
/* final 1x1 conv 32 -> classes with bias (unet.py:141) as its own step in training: fp32 NCHW logits from NHWC fp16 dec5 */
int rsb_final_forward(const void* y5, const float* w, const float* b, float* logits, int32_t N, int32_t HW, int32_t classes,
                      void* stream);
/* its autograd: dy5 (fp16, times loss_scale), dW [classes][32], db [classes] (fp32, unscaled). acc: classes*32 + 8 doubles. */
int rsb_final_backward(const float* dlogits, const void* y5, const float* w, void* dy5, double* acc, float* dw, float* db,
                       float loss_scale, int32_t N, int32_t HW, int32_t classes, void* stream);
/* fp32 OIHW master weights -> fp16 packed operand matrix: dst[i] = half(sum of src[map4[4i..4i+3]] (entries < 0 skipped)) */
int rsb_pack_weights(const float* src, const int32_t* map4, void* dst, int64_t n, void* stream);
/* the same with ONE source index per packed element (map1: int32 [n], -1 = zero; n a multiple of 8, map1 and dst 16-byte
 * aligned): a quarter of the map bytes; used for every layout but the pre-summed nearest-x2 taps */
int rsb_pack_weights1(const float* src, const int32_t* map1, void* dst, int64_t n, void* stream);
/* packed fp32 gradient -> OIHW fp32 gradient, the transpose of rsb_pack_weights, without atomics (deterministic): element i of the
 * compact list writes grad[dst_idx[i]] = mul * (sum of the packed gradient elements inv4[4i..4i+3], entries < 0 skipped, added in
 * index order); inv4 is the inverse of the pack map4 (robosat_b200.train_engine.invert_unpack_map) */
int rsb_unpack_grads_gather(const float* packed_grad, const int32_t* dst_idx, const int32_t* inv4, float* grad, int64_t n, float mul,
                            void* stream);

/* Weight gradient of the convolution described by `fwd` (same sources / segments / phases / tile space), on tensor cores:
 *   dw_packed[phase*Cout + co][k] = sum_pixels dy_phase[pixel][co] * x_segment(k)[pixel + (dh,dw)][k % 64-block]   (fp32)
 * i.e. the gradient in the forward kernel's packed weight layout (rsb_unpack_grads_gather folds it back to OIHW).
 * dy is addressed like fwd->out (same pitches / phase strides). Replaces autograd's conv weight gradients (train.py:186). */
typedef struct rsb_wgrad_plan rsb_wgrad_plan;
int rsb_wgrad_plan_create(const rsb_conv_desc* fwd, const void* dy, float* dw_packed, rsb_wgrad_plan** out_plan);
/* Split-K: bytes of scratch the plan needs (0 when it has a single pixel slice), and the call that hands it over. Every slice
 * stores its partial gradient there and a second kernel adds the slices in index order (bit-identical from run to run). A plan
 * that needs a scratch must get one before rsb_wgrad_run, which otherwise returns RSB_E_INVALID and launches nothing. The scratch
 * is private to a launch and may be shared by all plans that run on one stream. */
int64_t rsb_wgrad_plan_scratch_bytes(const rsb_wgrad_plan* plan);
int rsb_wgrad_plan_set_scratch(rsb_wgrad_plan* plan, float* scratch, int64_t scratch_bytes);
void rsb_wgrad_plan_destroy(rsb_wgrad_plan* plan);
int rsb_wgrad_run(const rsb_wgrad_plan* plan, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RSB200_H */
