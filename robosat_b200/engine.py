"""Host-side plan of the U-Net forward pass on librsb200.so.

`UNetEngine` turns a reference-format `state_dict` (robosat/unet.py:94-108 key names) into
  * pre-packed fp16 weight matrices (eval BatchNorm folded, decoder taps pre-summed per output phase),
  * static NHWC fp16 activation buffers in HBM,
  * one `rsb_conv_plan` (TMA descriptors + tile schedule) per convolution,
and replays them in order on the current CUDA stream. Python only sequences ~70 C-ABI calls; every
arithmetic operation runs in the hand-written sm_90a kernels (no cuDNN / cuBLAS / torch ops on the path).

Reference call sites covered: UNet.forward robosat/unet.py:110-141 (and the torchvision resnet50
Bottleneck stack it calls), ConvRelu robosat/unet.py:44, DecoderBlock robosat/unet.py:73.
"""

import ctypes
import math
import os
from collections import OrderedDict

import torch

from robosat_b200 import _lib
from robosat_b200._lib import ConvDesc, ConvSeg, ConvSrc, RowConvDesc

RESNET50_BLOCKS = (3, 4, 6, 3)
BN_EPS = 1e-5
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


# --------------------------------------------------------------------------------------------------
# weight packing (host, fp32 -> fp16). K index of a packed row = concatenation of the segments' 64-blocks.
# --------------------------------------------------------------------------------------------------
def _strip(sd):
    if any(k.startswith("module.") for k in sd):
        return {k[len("module."):]: v for k, v in sd.items()}
    return dict(sd)


def fold_bn(sd, conv_key, bn_prefix):
    """Eval-mode BatchNorm folded into the preceding bias-free conv: w' = w*s, b' = beta - mean*s.
    Folded in float64 so that the only rounding is the one to the operand format (fp16, or the fp16 hi/lo pair)."""
    w = sd[conv_key].double()
    if bn_prefix is None:
        return w, None
    s = sd[bn_prefix + ".weight"].double() / torch.sqrt(sd[bn_prefix + ".running_var"].double() + BN_EPS)
    b = sd[bn_prefix + ".bias"].double() - sd[bn_prefix + ".running_mean"].double() * s
    return w * s.view(-1, 1, 1, 1), b


def split_fp16(w):
    """float64 -> (scaled hi, scaled lo, acc_scale): w * 2^e = hi + lo with hi = half(w * 2^e), lo = half(w * 2^e - hi).

    2^e moves the largest |w| into [2^13, 2^14) so the lo parts (2^-11 of their hi) of all but vanishing weights are normal
    fp16 numbers; the kernel multiplies the fp32 accumulator by acc_scale = 2^-e (exact)."""
    m = float(w.abs().max())
    e = 0 if m == 0.0 else 13 - int(math.floor(math.log2(m)))
    ws = w.double() * (2.0 ** e)
    hi = ws.to(torch.float16)
    lo = (ws - hi.double()).to(torch.float16)
    return hi, lo, 2.0 ** (-e)


def pack_conv(w):
    """[Cout, Cin, kh, kw] -> [Cout, kh*kw*Cin] (tap-major, channel-minor)."""
    co, ci, kh, kw = w.shape
    return w.permute(0, 2, 3, 1).reshape(co, kh * kw * ci).contiguous()


def pack_upsample_phases(w):
    """3x3 conv applied after a nearest x2 upsample == four 2x2 convs on the low-res input.

    Output pixel (2i+a, 2j+b) reads low-res rows {i-1+a, i+a}: row taps pre-summed as
    a=0: [w0 | w1+w2], a=1: [w0+w1 | w2] (same for columns). Returns [4*Cout, 4*Cin], phase p=2a+b major.
    """
    co, ci, _, _ = w.shape
    groups = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    rows = []
    for a in (0, 1):
        for b in (0, 1):
            taps = []
            for th in (0, 1):
                for tw in (0, 1):
                    acc = torch.zeros(co, ci, dtype=w.dtype, device=w.device)
                    for kh in groups[a][th]:
                        for kw in groups[b][tw]:
                            acc += w[:, :, kh, kw]
                    taps.append(acc)
            rows.append(torch.stack(taps, dim=1).reshape(co, 4 * ci))
    return torch.cat(rows, dim=0).contiguous()


def pack_stem(w):
    """7x7 stride-2 pad-3 conv on 3 channels -> 4 row-taps x (4 column-taps x 16 s2d channels) = K 256.

    Input row 2*o + kh - 3 = 2*(o + t - 2) + ph with kh + 1 = 2*t + ph; the s2d channel is (ph*2+pw)*3 + c.
    """
    co = w.shape[0]
    out = torch.zeros(co, 4, 4, 16, dtype=w.dtype, device=w.device)
    for t in range(4):
        for ph in range(2):
            kh = 2 * t + ph - 1
            if not 0 <= kh < 7:
                continue
            for u in range(4):
                for pw in range(2):
                    kw = 2 * u + pw - 1
                    if not 0 <= kw < 7:
                        continue
                    out[:, t, u, (ph * 2 + pw) * 3:(ph * 2 + pw) * 3 + 3] = w[:, :, kh, kw]
    return out.reshape(co, 256).contiguous()


def pack_window3(w):
    """3x3 conv on 32 channels read as 3 row-taps of a 4-pixel window (4th pixel weight zero): K = 3*128."""
    co, ci, _, _ = w.shape
    out = torch.zeros(co, 3, 4, ci, dtype=w.dtype, device=w.device)
    out[:, :, :3, :] = w.permute(0, 2, 3, 1)
    return out.reshape(co, 3 * 4 * ci).contiguous()


def choose_tile(Wt, Ht, Nt):
    """TW x TH x TN = 128 box with the least padded work; prefer single-image, wide tiles."""
    best = None
    for tw in (16, 8, 32, 4, 64, 2, 128, 1):
        for th in (8, 16, 4, 32, 2, 64, 1, 128):
            if 128 % (tw * th):
                continue
            tn = 128 // (tw * th)
            if tn > 256 or tw > 256 or th > 256:
                continue
            tiles = -(-Wt // tw) * -(-Ht // th) * -(-Nt // tn)
            key = (tiles, tn, abs(tw - 16) + abs(th - 8))
            if best is None or key < best[0]:
                best = (key, (tw, th, tn))
    return best[1]


# wide tiles (block_n >= 128) with long K loops are computed by CTA pairs (clusters of 2 that multicast the shared weight
# tile): each SM loads half of it from L2. Results are bit-identical; RSB_CTA_PAIR=0 keeps one CTA per tile everywhere.
CTA_PAIR = os.environ.get("RSB_CTA_PAIR", "1") == "1"


def choose_block_n(cout, m_tiles, phases, kblocks=8, sms=132, split=False):
    """N tile with the lowest modelled time for the persistent grid (ties -> the widest).

    Model (relative cycles per tile; its constants were fitted on an earlier GPU generation and have not been re-fitted on
    H100; the measured table `plan_table()` replaces it for the shapes it covers): a tile's K loop issues 4 MMAs per K block
    at max(66, N/2) cycles each (narrow tiles are bound by the shared-memory read of the A operand); the epilogue costs
    ~16 (N >= 128) or ~28 cycles per output column; the grid runs ceil(tiles / SMs) rounds of that."""
    # strict precision stops at 128 columns: on H100 (700 W) the whole strict predict step at batch 32 x 512^2 ran 1.5 % faster
    # with every 256-wide layer narrowed to 128 (24.5 vs 24.9 ms, identical logits; scripts/ab_block_n.py), while the fast step
    # ran 11 % slower (12.1 vs 10.8 ms) -- the 256-wide strict kernels spill registers
    cands = [bn for bn in ((128, 64, 32) if split else (256, 128, 64, 32)) if cout % bn == 0]
    assert cands, "Cout must be a multiple of 32"

    def cost(bn):
        tiles = m_tiles * phases * (cout // bn)
        if split:  # three MMAs per K step (two for the N-concatenated narrow tiles), always the 4-warp epilogue
            mma = 8 * 66 if bn <= 64 else 12 * max(66, bn // 2)
            per_tile = max(kblocks * mma, bn * 28) + 300
        else:
            per_tile = max(kblocks * 4 * max(66, bn // 2), bn * (16 if bn >= 128 else 28)) + 300
        return -(-tiles // sms) * per_tile

    return min(cands, key=lambda bn: (cost(bn), -bn))


# --------------------------------------------------------------------------------------------------
class ConvOp:
    """One convolution: the C descriptor, its plan handle and the tensors it must keep alive."""

    def __init__(self, name, desc, keep, create_plan=True):
        self.name = name
        self.desc = desc
        self.keep = keep
        self.plan = ctypes.c_void_p()
        if create_plan:
            lib = _lib.load()
            _lib.check(lib.rsb_conv_plan_create(ctypes.byref(desc), ctypes.byref(self.plan)), "rsb_conv_plan_create[%s]" % name)

    def run(self, stream):
        _lib.check(_lib.load().rsb_conv_run(self.plan, stream), "rsb_conv_run[%s]" % self.name)

    def info(self):
        g, t, k, s = (ctypes.c_int32() for _ in range(4))
        _lib.check(_lib.load().rsb_conv_plan_info(self.plan, ctypes.byref(g), ctypes.byref(t), ctypes.byref(k), ctypes.byref(s)), "plan_info")
        return {"grid": g.value, "tiles": t.value, "kblocks": k.value, "smem": s.value}

    def __del__(self):
        try:
            if self.plan:
                _lib.load().rsb_conv_plan_destroy(self.plan)
                self.plan = ctypes.c_void_p()
        except Exception:
            pass


class RowConvOp:
    """Line-buffer convolution plan (csrc/rsb_conv_row.cu) with the ConvOp interface."""

    def __init__(self, name, desc, keep=(), create_plan=True):
        self.name, self.desc, self.keep = name, desc, keep
        self.plan = ctypes.c_void_p()
        if create_plan:
            _lib.check(_lib.load().rsb_rowconv_plan_create(ctypes.byref(desc), ctypes.byref(self.plan)), "rsb_rowconv_plan_create[%s]" % name)

    def run(self, stream):
        _lib.check(_lib.load().rsb_rowconv_run(self.plan, stream), "rsb_rowconv_run[%s]" % self.name)

    def info(self):
        return {"grid": 0, "tiles": -(-self.desc.Wt // 128) * self.desc.Ht * self.desc.Nt * self.desc.nsub * self.desc.nphase_a, "kblocks": 0, "smem": 0}

    def __del__(self):
        try:
            if self.plan:
                _lib.load().rsb_rowconv_plan_destroy(self.plan)
                self.plan = ctypes.c_void_p()
        except Exception:
            pass


def make_rowconv_desc(src, cin, weights, bias, cout, tile_space, out, out_pitches, upsample=False, relu=True, head=None,
                      out_offset_elems=0, rows_per_unit=0, split=False, acc_scale=1.0):
    """3x3 stride-1 conv (upsample=False) or the fused nearest-x2 + 3x3 (upsample=True: 2x2 taps, 4 phases) on the
    line-buffer kernel. weights: fp16 [phases*Cout][taps*cin] in the packed layout of pack_conv / pack_upsample_phases."""
    d = RowConvDesc()
    d.src = src
    d.cin = cin
    d.taps_h = d.taps_w = 2 if upsample else 3
    d.dh0 = d.dw0 = -1
    d.nsub = d.nphase_a = 2 if upsample else 1
    phases = 4 if upsample else 1
    d.split = 1 if split else 0
    d.acc_scale = acc_scale
    wshape = (phases * cout, d.taps_h * d.taps_w * cin)
    assert weights.dtype == torch.float16 and tuple(weights.shape) == ((2,) + wshape if split else wshape), tuple(weights.shape)
    d.weights = weights.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.Cout = cout
    d.Wt, d.Ht, d.Nt = tile_space
    d.relu = 1 if relu else 0
    d.rows_per_unit = rows_per_unit
    if head is None:
        d.mode = 0
        d.out = out.data_ptr() + 2 * out_offset_elems
        d.out_pitch_w, d.out_pitch_h, d.out_pitch_n = out_pitches
        d.out_sy = d.out_sx = 2 if upsample else 1
    else:
        head_w, head_b, head_out, classes = head
        d.mode = 1
        d.head_classes = classes
        d.head_w, d.head_b, d.head_out = head_w.data_ptr(), head_b.data_ptr(), head_out.data_ptr()
    return d


def _src_dense(t, N, H, W, C, plane=0):
    return ConvSrc(t.data_ptr(), C, W * C, H * W * C, C, W, H, N, plane)


def _src_parity(t, N, H, W, C, ph, pw, plane=0):
    return ConvSrc(t.data_ptr() + 2 * (ph * W + pw) * C, 2 * C, 2 * W * C, H * W * C, C, W // 2, H // 2, N, plane)


def make_conv_desc(srcs, segs, weights, bias, cout, phases, tile_space, out, out_pitches, out_scale=(1, 1),
                   residual=None, relu=True, block_n=None, head=None, out_offset_elems=0, cta_pair=None,
                   split=False, acc_scale=1.0, out_plane=0, res_plane=0, scratch=None):
    """Fill an `rsb_conv_desc`. tile_space = (Wt, Ht, Nt); out_pitches = (pitch_w, pitch_h, pitch_n) in elements.
    split=True: strict precision -- weights fp16 [2][phases*Cout][K] (hi, lo planes), sources / out / residual carry
    plane strides, the accumulator is multiplied by acc_scale (see include/rsb200.h)."""
    d = ConvDesc()
    d.split = 1 if split else 0
    d.acc_scale = acc_scale
    d.out_plane = out_plane
    d.res_plane = res_plane
    d.nsrc = len(srcs)
    for i, s in enumerate(srcs):
        d.srcs[i] = s
    d.nseg = len(segs)
    for i, (src, dh, dw, cb) in enumerate(segs):
        d.segs[i] = ConvSeg(src, dh, dw, cb)
    K = 64 * sum(s[3] for s in segs)
    assert weights.dtype == torch.float16 and weights.is_contiguous()
    wshape = (2, phases * cout, K) if split else (phases * cout, K)
    assert tuple(weights.shape) == wshape, (tuple(weights.shape), wshape)
    d.weights = weights.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.Cout = cout
    d.phases = phases
    Wt, Ht, Nt = tile_space
    d.Wt, d.Ht, d.Nt = Wt, Ht, Nt
    d.TW, d.TH, d.TN = choose_tile(Wt, Ht, Nt)
    m_tiles = -(-Wt // d.TW) * -(-Ht // d.TH) * -(-Nt // d.TN)
    d.block_n = block_n or choose_block_n(cout, m_tiles, phases, K // 64, split=split)
    if residual is not None and block_n is None and d.block_n == 256:
        d.block_n = 128  # the residual staging slices take shared memory from the pipeline: keep it deeper with 128 columns
    d.out_sy, d.out_sx = out_scale
    d.relu = 1 if relu else 0
    if head is None:
        d.mode = 0
        d.out = out.data_ptr() + 2 * out_offset_elems
        d.out_pitch_w, d.out_pitch_h, d.out_pitch_n = out_pitches
        d.residual = residual.data_ptr() if residual is not None else None
        if cta_pair is None:
            # pairs pay once the K loop is long enough for the weight traffic to matter; short, epilogue-bound K loops keep one CTA.
            # The K-length thresholds were tuned on an earlier GPU generation, not re-tuned on H100 (scripts/tune_plans.py, RSB_CTA_PAIR=0)
            kblocks = K // 64
            if split:
                # the weight tile is the larger half of a split stage (2 planes): sharing it between two SMs pays as soon as
                # the K loop is long enough to amortise the cluster synchronisation
                cta_pair = CTA_PAIR and m_tiles >= 2 and d.block_n >= 128 and kblocks >= 4
            else:
                cta_pair = CTA_PAIR and m_tiles >= 2 and ((d.block_n == 256 and kblocks >= 6) or (d.block_n == 128 and kblocks >= 18))
        d.cta_pair = 1 if cta_pair else 0
        if split and scratch is not None:
            # long K loops are accumulated in chunks that the epilogue adds in round-to-nearest fp32 (the tensor core's fp32
            # accumulation is not round-to-nearest, so its error grows with the length of a chain of MMAs). Wide tiles chain 12 MMAs per K block on the
            # main accumulator, the N-concatenated narrow tiles 4; chunks keep a chain at <= MAX_MMA_CHAIN MMAs.
            kblocks = K // 64
            per_kb = 12 if d.block_n >= 128 else 4
            if MAX_MMA_CHAIN > 0 and kblocks * per_kb > 2 * MAX_MMA_CHAIN - MAX_MMA_CHAIN // 2:
                nchunks = -(-kblocks * per_kb // MAX_MMA_CHAIN)
                d.kchunk = -(-kblocks // nchunks)
                d.scratch = scratch.data_ptr()
                d.scratch_bytes = scratch.numel() * scratch.element_size()
    else:
        head_w, head_b, head_out, classes = head
        d.mode = 1
        d.head_classes = classes
        d.head_w = head_w.data_ptr()
        d.head_b = head_b.data_ptr()
        d.head_out = head_out.data_ptr()
    return d


PRECISIONS = ("strict", "fast")
# every chunk boundary moves one 128 x block_n fp32 tile through L2 in each direction: fewer, longer chains cost less time.
# 400 was chosen on an earlier GPU generation and has not been re-tuned on H100.
MAX_MMA_CHAIN = int(os.environ.get("RSB_MAX_MMA_CHAIN", "400"))  # 0 disables K chunking (A/B measurements)


def default_precision():
    """`strict` (hi/lo fp16 operand pairs, fp32-class results: the parity contract) unless RSB_PRECISION=fast."""
    p = os.environ.get("RSB_PRECISION", "strict").lower()
    if p not in PRECISIONS:
        raise ValueError("RSB_PRECISION must be one of %s" % (PRECISIONS,))
    return p


_PLAN_TABLE = None


def plan_table():
    """Measured tile choices per (precision, batch, height, width): `robosat_b200/plans_h100.json`, written by
    scripts/tune_plans.py on an H100 (every layer timed alone for each (block_n, CTA pair) candidate; a table is kept for a shape
    only where the whole step confirmed it). RSB_PLAN_TABLE=<path> reads another file, RSB_PLAN_TABLE=0 disables it."""
    global _PLAN_TABLE
    if _PLAN_TABLE is None:
        path = os.environ.get("RSB_PLAN_TABLE", os.path.join(os.path.dirname(os.path.abspath(__file__)), "plans_h100.json"))
        table = {}
        if path not in ("0", "") and os.path.exists(path):
            import json

            with open(path) as fp:
                table = json.load(fp).get("plans", {})
        _PLAN_TABLE = table
    return _PLAN_TABLE


def _override_valid(ov, cout, tile_space, split, has_res):
    """what rsb_conv_plan_create would accept (include/rsb200.h), checked here so that the GPU-less plan_only mode agrees"""
    bn, pair = int(ov.get("block_n", 0)), bool(ov.get("cta_pair", 0))
    if bn not in (32, 64, 128, 256) or cout % bn:
        return False
    Wt, Ht, Nt = tile_space
    TW, TH, TN = choose_tile(Wt, Ht, Nt)
    m_tiles = -(-Wt // TW) * -(-Ht // TH) * -(-Nt // TN)
    if pair and (bn < 128 or m_tiles < 2 or not CTA_PAIR):
        return False
    if split and bn == 256:  # strict plans use <= 128 columns (choose_block_n); K chunking needs <= 128
        return False
    return True


class UNetEngine:
    """Static-shape inference plan for `UNet(num_classes)` on one GPU.

    precision="strict" (default): every activation / weight is an fp16 (hi, lo) pair and every K step runs three MMAs
    (hi*lo + lo*hi + hi*hi, fp32 accumulate) -- logits agree with the fp32 reference to ~1e-5 relative, argmax up to
    the fp32 noise floor. precision="fast": single fp16 operands (one MMA per K step, ~3x the throughput, logits ~2e-3)."""

    def __init__(self, state_dict, num_classes, batch, height, width, device="cuda", plan_only=False, use_row=True, precision=None,
                 plan_overrides=None):
        """plan_only=True builds buffers and descriptors on `device` without touching the GPU library
        (used by the CPU tests, which execute the descriptors with tests/emulate.py).
        plan_overrides: {layer name: {"block_n": int, "cta_pair": 0|1}} replacing the modelled tile choice of those layers
        (None: the measured table `plan_table()` has for this precision and shape, if any; {}: the model only)."""
        assert height % 32 == 0 and width % 32 == 0, "image resolution has to be divisible by 32 for resnet"
        # the reference's torch.cat([enc4, center]) (unet.py:134) only works when enc4's extent is even
        assert height % 64 == 0 and width % 64 == 0, "enc4 must have even extents (input divisible by 64), as in the reference"
        self.plan_only = plan_only
        self.precision = precision or default_precision()
        assert self.precision in PRECISIONS, self.precision
        self.strict = self.precision == "strict"
        self._overrides = plan_overrides if plan_overrides is not None else plan_table().get(
            "%s:%dx%dx%d" % (self.precision, batch, height, width), {})
        # line-buffer kernel for the >= 128-pixel-wide, small-Cout layers (layer1 3x3, dec4, dec5 + final). In strict precision
        # only dec5 + final has one (resident weights + a 2-plane row ring must fit in shared memory)
        self.use_row_head = use_row
        self.use_row = use_row and not self.strict
        if not plan_only:
            _lib.require_device()
        self.device = torch.device(device)
        self.N, self.H, self.W, self.C = batch, height, width, num_classes
        self.ops = []  # ("conv", ConvOp) | ("prepass",) | ("maxpool", src, dst, N, H, W, C, k, s, p)
        self.feats = OrderedDict()  # name -> (tensor, (N, H, W, C) logical view) for layer-wise checks
        self._keep = []
        # Weight preparation (BN folding in float64, tap pre-summing, hi/lo split, packing) is a one-off setup step made of a few
        # hundred small tensor ops over 39 M weights: it runs on the plan's device (under torchrun the host has
        # OMP_NUM_THREADS=1, where the same ops took 17 s per plan), on the host only for the GPU-less plan_only mode.
        # state_dicts may live on any device (e.g. straight out of the NCCL broadcast).
        where = torch.device("cpu") if plan_only else self.device
        self._build({k: v.detach().to(where) for k, v in _strip(state_dict).items()})

    # ---------------------------------------------------------------- helpers
    def _buf(self, *shape, dtype=torch.float16):
        t = torch.zeros(shape, dtype=dtype, device=self.device)
        self._keep.append(t)
        return t

    def _act(self, *shape):
        """activation buffer: NHWC fp16, with a leading (hi, lo) plane axis in strict mode"""
        return self._buf(*((2,) + shape if self.strict else shape))

    def _plane(self, t):
        return t.numel() // 2 if self.strict else 0

    def _dev(self, t, dtype):
        t = t.to(dtype).contiguous().to(self.device)
        self._keep.append(t)
        return t

    def _wts(self, w):
        """packed float64 weight matrix -> (device fp16 operand, acc_scale)"""
        if not self.strict:
            return self._dev(w, torch.float16), 1.0
        hi, lo, scale = split_fp16(w)
        return self._dev(torch.stack([hi, lo]), torch.float16), scale

    def _scratch(self):
        """one fp32 scratch tile per SM for the K-chunked accumulation, shared by all layers (launches are stream ordered)"""
        if getattr(self, "_scratch_buf", None) is None:
            n = 132 * 128 * 256 if self.plan_only else int(_lib.load().rsb_conv_scratch_bytes(256)) // 4
            self._scratch_buf = self._buf(n, dtype=torch.float32)
        return self._scratch_buf

    def _dense(self, t, N, H, W, C):
        return _src_dense(t, N, H, W, C, self._plane(t))

    def _parity(self, t, N, H, W, C, ph, pw):
        return _src_parity(t, N, H, W, C, ph, pw, self._plane(t))

    def _conv(self, name, srcs, segs, w, b, cout, phases, tile_space, out, out_pitches, residual=None, **kw):
        wd, scale = self._wts(w)
        bd = self._dev(b, torch.float32) if b is not None else None

        def build(extra):
            desc = make_conv_desc(srcs, segs, wd, bd, cout, phases, tile_space, out, out_pitches, residual=residual,
                                  split=self.strict, acc_scale=scale, out_plane=self._plane(out) if out is not None else 0,
                                  res_plane=self._plane(residual) if residual is not None else 0,
                                  scratch=self._scratch() if self.strict else None, **dict(kw, **extra))
            return ConvOp(name, desc, (wd, bd), create_plan=not self.plan_only)

        op = None
        ov = self._overrides.get(name)
        if ov and "block_n" not in kw and "cta_pair" not in kw and "head" not in kw and _override_valid(ov, cout, tile_space, self.strict, residual is not None):
            try:
                op = build({"block_n": int(ov["block_n"]), "cta_pair": bool(ov["cta_pair"])})
            except _lib.RsbError:  # e.g. no shared memory for this tile on this device: the modelled choice always fits
                op = None
        if op is None:
            op = build({})
        self.ops.append(("conv", op))
        return op

    def _add_row(self, name, desc):
        op = RowConvOp(name, desc, (), create_plan=not self.plan_only)
        self.ops.append(("conv", op))
        return op

    # ---------------------------------------------------------------- graph
    def _build(self, sd):
        N, H, W = self.N, self.H, self.W
        H2, W2 = H // 2, W // 2
        dev = self._dev

        # input pre-pass: fp32 NCHW (or u8 NHWC) -> space-to-depth fp16 [N, H2, W2+4, 16]
        self.s2d = self._act(N, H2, W2 + 4, 16)
        self.ops.append(("prepass",))

        # stem: conv1 7x7/2 + bn1 + relu (unet.py:122-124) on tensor cores via the overlapped window view
        w, b = fold_bn(sd, "resnet.conv1.weight", "resnet.bn1")
        stem = self._act(N, H2, W2, 64)
        Wp = W2 + 4
        src = ConvSrc(self.s2d.data_ptr(), 16, Wp * 16, H2 * Wp * 16, 64, W2, H2, N, self._plane(self.s2d))
        segs = [(0, t - 2, 0, 1) for t in range(4)]
        self._conv("stem", [src], segs, pack_stem(w), b, 64, 1, (W2, H2, N), stem, (64, W2 * 64, H2 * W2 * 64))
        self.feats["stem"] = (stem, (N, H2, W2, 64))

        # maxpool 3x3/2 pad 1 (unet.py:125)
        H4, W4 = H // 4, W // 4
        enc0 = self._act(N, H4, W4, 64)
        self.ops.append(("maxpool", stem, enc0, N, H2, W2, 64, 3, 2, 1))
        self.feats["enc0"] = (enc0, (N, H4, W4, 64))

        # resnet layer1..4 (unet.py:127-130)
        cur, curC, curH, curW = enc0, 64, H4, W4
        encs = []
        for li, blocks in enumerate(RESNET50_BLOCKS, start=1):
            planes = 64 * 2 ** (li - 1)
            for bi in range(blocks):
                p = "resnet.layer%d.%d" % (li, bi)
                stride = 2 if (bi == 0 and li > 1) else 1
                oH, oW = curH // stride, curW // stride
                # conv1 1x1 + bn1 + relu
                w, b = fold_bn(sd, p + ".conv1.weight", p + ".bn1")
                t1 = self._act(N, curH, curW, planes)
                self._conv(p + ".conv1", [self._dense(cur, N, curH, curW, curC)], [(0, 0, 0, curC // 64)], pack_conv(w), b,
                           planes, 1, (curW, curH, N), t1, (planes, curW * planes, curH * curW * planes))
                # conv2 3x3 (stride) + bn2 + relu
                w, b = fold_bn(sd, p + ".conv2.weight", p + ".bn2")
                t2 = self._act(N, oH, oW, planes)
                if stride == 1 and planes == 64 and self.use_row and curW >= 128:
                    self._add_row(p + ".conv2", make_rowconv_desc(_src_dense(t1, N, curH, curW, planes), planes, dev(pack_conv(w), torch.float16),
                                                                  dev(b, torch.float32), planes, (oW, oH, N), t2, (planes, oW * planes, oH * oW * planes)))
                    srcs = None
                elif stride == 1:
                    srcs = [self._dense(t1, N, curH, curW, planes)]
                    segs = [(0, kh - 1, kw - 1, planes // 64) for kh in range(3) for kw in range(3)]
                else:
                    srcs = [self._parity(t1, N, curH, curW, planes, ph, pw) for ph in range(2) for pw in range(2)]
                    segs = []
                    for kh in range(3):
                        for kw in range(3):
                            ph, dh = (kh - 1) % 2, (kh - 1) // 2
                            pw, dw = (kw - 1) % 2, (kw - 1) // 2
                            segs.append((ph * 2 + pw, dh, dw, planes // 64))
                if srcs is not None:
                    self._conv(p + ".conv2", srcs, segs, pack_conv(w), b, planes, 1, (oW, oH, N), t2, (planes, oW * planes, oH * oW * planes))
                outC = planes * 4
                w3, b3 = fold_bn(sd, p + ".conv3.weight", p + ".bn3")
                out = self._act(N, oH, oW, outC)
                t2src = self._dense(t2, N, oH, oW, planes)
                if (p + ".downsample.0.weight") in sd:
                    # block 0: relu(bn3(conv3(t2)) + bn_d(downsample(x))) is ONE contraction over [t2 | x]:
                    # two 1x1 convs into the same output = two segments with concatenated weights and summed biases.
                    # The identity branch is never written to / re-read from HBM.
                    wd, bd = fold_bn(sd, p + ".downsample.0.weight", p + ".downsample.1")
                    xsrc = self._dense(cur, N, curH, curW, curC) if stride == 1 else self._parity(cur, N, curH, curW, curC, 0, 0)
                    wcat = torch.cat([pack_conv(w3), pack_conv(wd)], dim=1)
                    self._conv(p + ".conv3+downsample", [t2src, xsrc], [(0, 0, 0, planes // 64), (1, 0, 0, curC // 64)], wcat, b3 + bd,
                               outC, 1, (oW, oH, N), out, (outC, oW * outC, oH * oW * outC))
                else:
                    # conv3 1x1 + bn3 + identity + relu
                    self._conv(p + ".conv3", [t2src], [(0, 0, 0, planes // 64)], pack_conv(w3), b3, outC, 1,
                               (oW, oH, N), out, (outC, oW * outC, oH * oW * outC), residual=cur)
                self.feats[p] = (out, (N, oH, oW, outC))
                cur, curC, curH, curW = out, outC, oH, oW
            encs.append((cur, curC, curH, curW))
            self.feats["enc%d" % li] = (cur, (N, curH, curW, curC))
        (enc1, c1, h1, w1), (enc2, c2, h2, w2), (enc3, c3, h3, w3), (enc4, c4, h4, w4) = encs

        # max_pool2d(enc4, 2, 2) (unet.py:132)
        hp, wpx = h4 // 2, w4 // 2
        pool4 = self._act(N, hp, wpx, c4)
        self.ops.append(("maxpool", enc4, pool4, N, h4, w4, c4, 2, 2, 0))
        self.feats["pool4"] = (pool4, (N, hp, wpx, c4))

        def decoder(name, sources, lh, lw, cout, out, out_pitches, out_offset=0):
            # DecoderBlock: nearest x2 + 3x3 conv + relu (unet.py:73, :44) as 4 phases of 2x2 taps on the low-res inputs
            w = sd[name + ".block.block.weight"].double()
            srcs = [self._dense(t, N, lh, lw, c) for t, c in sources]
            segs = [(si, th - 1, tw - 1, c // 64) for th in range(2) for tw in range(2) for si, (_, c) in enumerate(sources)]
            self._conv(name, srcs, segs, pack_upsample_phases(w), None, cout, 4, (lw, lh, N), out, out_pitches,
                       out_scale=(2, 2), out_offset_elems=out_offset)

        def dense_pitches(h, w, c):
            return (c, w * c, h * w * c)

        center = self._act(N, h4, w4, 256)
        decoder("center", [(pool4, c4)], hp, wpx, 256, center, dense_pitches(h4, w4, 256))
        self.feats["center"] = (center, (N, h4, w4, 256))
        dec0 = self._act(N, h3, w3, 256)
        decoder("dec0", [(enc4, c4), (center, 256)], h4, w4, 256, dec0, dense_pitches(h3, w3, 256))
        self.feats["dec0"] = (dec0, (N, h3, w3, 256))
        dec1 = self._act(N, h2, w2, 256)
        decoder("dec1", [(enc3, c3), (dec0, 256)], h3, w3, 256, dec1, dense_pitches(h2, w2, 256))
        self.feats["dec1"] = (dec1, (N, h2, w2, 256))
        dec2 = self._act(N, h1, w1, 64)
        decoder("dec2", [(enc2, c2), (dec1, 256)], h2, w2, 64, dec2, dense_pitches(h1, w1, 64))
        self.feats["dec2"] = (dec2, (N, h1, w1, 64))
        dec3 = self._act(N, H2, W2, 128)
        decoder("dec3", [(enc1, c1), (dec2, 64)], h1, w1, 128, dec3, dense_pitches(H2, W2, 128))
        self.feats["dec3"] = (dec3, (N, H2, W2, 128))

        # dec4 writes into a W-padded buffer [N, H, W+4, 32] (pixel w at column w+1) so dec5 can read 4-pixel windows
        Wq = W + 4
        self.dec4 = self._act(N, H, Wq, 32)
        if self.use_row and W2 >= 128:
            w4 = sd["dec4.block.block.weight"].double()
            self._add_row("dec4", make_rowconv_desc(_src_dense(dec3, N, H2, W2, 128), 128, dev(pack_upsample_phases(w4), torch.float16), None, 32,
                                                    (W2, H2, N), self.dec4, (32, Wq * 32, H * Wq * 32), upsample=True, out_offset_elems=32))
        else:
            decoder("dec4", [(dec3, 128)], H2, W2, 32, self.dec4, (32, Wq * 32, H * Wq * 32), out_offset=32)
        self.feats["dec4"] = (self.dec4, (N, H, Wq, 32))

        # dec5 (3x3 32->32 + relu, unet.py:139) fused with final (1x1 32->C + bias, unet.py:141) -> fp32 NCHW logits
        w5 = sd["dec5.block.weight"].double()
        self.logits = self._buf(N, self.C, H, W, dtype=torch.float32)
        head_w = dev(sd["final.weight"].float().reshape(self.C, 32), torch.float32)
        head_b = dev(sd["final.bias"].float(), torch.float32)
        if self.use_row_head and W >= 128:
            # the real pixels of the W-padded dec4 buffer as a dense view: column -1 / W are outside the view (zero fill)
            src = ConvSrc(self.dec4.data_ptr() + 2 * 32, 32, Wq * 32, H * Wq * 32, 32, W, H, N, self._plane(self.dec4))
            w5p, w5scale = self._wts(pack_conv(w5))
            self._add_row("dec5+final", make_rowconv_desc(src, 32, w5p, None, 32, (W, H, N), None, None,
                                                          head=(head_w, head_b, self.logits, self.C), split=self.strict, acc_scale=w5scale))
        else:
            src = ConvSrc(self.dec4.data_ptr(), 32, Wq * 32, H * Wq * 32, 128, W, H, N, self._plane(self.dec4))
            segs = [(0, kh - 1, 0, 2) for kh in range(3)]
            self._conv("dec5+final", [src], segs, pack_window3(w5), None, 32, 1, (W, H, N), None, None,
                       head=(head_w, head_b, self.logits, self.C))

        self._mean = (ctypes.c_float * 3)(*IMAGENET_MEAN)
        self._std = (ctypes.c_float * 3)(*IMAGENET_STD)

    # ---------------------------------------------------------------- execution
    def conv_ops(self):
        return [op[1] for op in self.ops if op[0] == "conv"]

    def num_launches(self):
        return len(self.ops)

    def forward(self, x):
        """x: fp32 NCHW normalised (reference API) or uint8 NHWC raw RGB, on this engine's device.
        Returns the engine-owned fp32 NCHW logits buffer (valid until the next call)."""
        if self.plan_only:
            raise _lib.RsbError("UNetEngine was built with plan_only=True; there is no CPU execution path")
        N, H, W = self.N, self.H, self.W
        if x.dtype == torch.float32:
            assert tuple(x.shape) == (N, 3, H, W) and x.is_contiguous() and x.is_cuda, "expected contiguous cuda fp32 [N,3,H,W]"
        elif x.dtype == torch.uint8:
            assert tuple(x.shape) == (N, H, W, 3) and x.is_contiguous() and x.is_cuda, "expected contiguous cuda uint8 [N,H,W,3]"
        else:
            raise TypeError("unsupported input dtype %s" % x.dtype)
        self.run_ops(self.ops, x)
        return self.logits

    def run_ops(self, ops, x):
        """Launch `ops` (entries of self.ops, in order) on the current stream; `x` is forward's validated input, read by the
        pre-pass. forward() is run_ops(self.ops, x); a sub-list runs single launches (tests/predict_lockstep.py)."""
        lib = _lib.load()
        N, H, W = self.N, self.H, self.W
        kind = 1 if x.dtype == torch.uint8 else 0
        stream = _lib.current_stream_ptr()
        for op in ops:
            if op[0] == "conv":
                op[1].run(stream)
            elif op[0] == "prepass":
                if self.strict:
                    _lib.check(lib.rsb_prepass_s2d_split(x.data_ptr(), kind, self.s2d.data_ptr(), self._plane(self.s2d), N, H, W,
                                                         self._mean, self._std, stream), "rsb_prepass_s2d_split")
                else:
                    _lib.check(lib.rsb_prepass_s2d(x.data_ptr(), kind, self.s2d.data_ptr(), N, H, W, self._mean, self._std, stream), "rsb_prepass_s2d")
            else:
                _, src, dst, n, h, w, c, k, s, p = op
                if self.strict:
                    _lib.check(lib.rsb_maxpool_nhwc_split(src.data_ptr(), self._plane(src), dst.data_ptr(), self._plane(dst), n, h, w, c, k, s, p, stream),
                               "rsb_maxpool_nhwc_split")
                else:
                    _lib.check(lib.rsb_maxpool_nhwc(src.data_ptr(), dst.data_ptr(), n, h, w, c, k, s, p, stream), "rsb_maxpool_nhwc")

    def feature_nchw(self, name):
        """Debug/parity view of an intermediate as fp32 NCHW on the CPU (strict mode: hi + lo)."""
        t, (n, h, w, c) = self.feats[name]
        t = t.detach().cpu()
        if self.strict:
            t = (t[0].double() + t[1].double()).float()
        t = t.float().reshape(n, h, w, c)
        if name == "dec4":
            t = t[:, :, 1:w - 3, :]
        return t.permute(0, 3, 1, 2).contiguous()
