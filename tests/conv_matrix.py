"""The case matrix of the two convolution kernels: every compiled instance at every tile box, ragged edges, multi-wave
schedules, K chunking and offset, padded output placement.

Test infrastructure only. `compiled_instances()` reads the instance list from the dispatch code in the checkout
(`conv_act<...>` in conv_dispatch / conv_dispatch_stats of csrc/rsb_conv.cu, `launch_row<...>` in rsb_rowconv_run of
csrc/rsb_conv_row.cu); `instance_of(desc)` restates which of them a descriptor selects, and which descriptors the plan
rejects. `matrix(device)` lists the cases; the CPU test asserts that they reach exactly the compiled set, the GPU test
(test_conv_matrix_gpu.py) runs each against a float64 replay.

Every case is built deterministically from its seed, so `case.build("cpu")` and `case.build("cuda")` hold the same values:
the float64 reference is taken from the host copy (tests/emulate.py reads host pointers), the kernel runs on the device
copy. Placement, the same in both copies:
  * sources carry 8 padding channels per pixel (NaN: a read past the view's C shows), dense or stride-2 parity views;
  * the output (both planes in strict precision) and the residual sit at an element offset inside a larger buffer with
    pitches wider than Cout; everything outside the view is a sentinel (NaN bits) that must survive bit for bit;
  * head logits sit at an offset inside a larger fp32 sentinel buffer;
  * the K-chunk scratch and the statistics partials have a sentinel tail past their stated sizes.
"""

import ctypes
import itertools
import os
import re

import torch

from conv_cases import _rand
from robosat_b200 import engine as E
from robosat_b200._lib import ConvDesc, ConvSrc, RowConvDesc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "robosat_b200", "csrc")

SMS = 132                     # H100 SXM; the scratch buffers are sized for this many CTAs
SMEM_OPTIN = 232448           # 227 KB: the per-block opt-in shared-memory limit of sm_90
SENTINEL16 = 0x7E5A           # fp16 quiet NaN with a payload no kernel computes
SENTINEL32 = 0x7FA5A5A5       # fp32 NaN, same purpose
PAD_C = 8                     # padding channels per pixel (16 bytes) of every source / output / residual view

# every TW x TH x TN = 128 box
BOXES = [(1 << a, 1 << b, 1 << (7 - a - b)) for a in range(8) for b in range(8 - a)]


class Rejected(ValueError):
    """instance_of: the plan refuses this descriptor"""


# ----------------------------------------------------------------------------------------------------------------------
# the compiled instances, read from the dispatch code
# ----------------------------------------------------------------------------------------------------------------------
def _function_body(text, signature):
    i = text.index(signature)
    j = text.index("{", i)
    depth = 0
    for k in range(j, len(text)):
        depth += {"{": 1, "}": -1}.get(text[k], 0)
        if depth == 0:
            return text[j:k + 1]
    raise ValueError("unbalanced braces after %r" % signature)


def _int(tok, env):
    tok = tok.strip()
    if tok in env:
        return env[tok]
    return {"true": 1, "false": 0}[tok] if tok in ("true", "false") else int(tok)


def compiled_instances():
    """{("conv", BLOCK_N, MODE, HAS_RES, TWO, SPLIT, STATS)} | {("row", CBLK, BLOCK_N, MODE, TAPS, CBLOCKS, NSUB, SPLIT)}"""
    text = open(os.path.join(CSRC, "rsb_conv.cu")).read()
    out = set()
    sel = _function_body(text, "static int conv_select(")
    splits = [int(s) for s in re.findall(r"conv_dispatch<(\d)>", sel)]
    assert sorted(splits) == [0, 1], splits
    body = _function_body(text, "static int conv_dispatch(")
    narrow = re.search(r"constexpr int NARROW = SPLIT \? (\d) : (\d);", body)
    for split in splits:
        env = {"SPLIT": split, "NARROW": int(narrow.group(1)) if split else int(narrow.group(2))}
        for line in body.splitlines():
            for m in re.finditer(r"conv_act<([^>]*)>", line):
                if split and re.search(r"if constexpr \(!SPLIT\)", line[:m.start()]):
                    continue  # discarded statement of conv_dispatch<1>
                args = [_int(a, env) for a in m.group(1).split(",")]
                out.add(("conv",) + tuple(args + [0] * (6 - len(args))))
    for m in re.finditer(r"conv_act<([^>]*)>", _function_body(text, "static int conv_dispatch_stats(")):
        args = [_int(a, {}) for a in m.group(1).split(",")]
        out.add(("conv",) + tuple(args + [0] * (6 - len(args))))
    text = open(os.path.join(CSRC, "rsb_conv_row.cu")).read()
    for m in re.finditer(r"launch_row<([^>]*)>\(plan", _function_body(text, 'extern "C" int rsb_rowconv_run(')):
        args = [_int(a, {}) for a in m.group(1).split(",")]
        out.add(("row",) + tuple(args + [0] * (7 - len(args))))
    return out


# ----------------------------------------------------------------------------------------------------------------------
# conv_select / rsb_rowconv_run restated
# ----------------------------------------------------------------------------------------------------------------------
def _conv_instance(d):
    """validate_desc + the checks of rsb_conv_plan_create, then the instance conv_select picks"""
    bn, res, split, pair = d.block_n, bool(d.residual), bool(d.split), bool(d.cta_pair)
    if bn not in (32, 64, 128, 256):
        raise Rejected("block_n must be 32/64/128/256")
    if d.Cout <= 0 or d.Cout % bn:
        raise Rejected("Cout not a multiple of block_n")
    if d.phases not in (1, 4):
        raise Rejected("phases must be 1 or 4")
    if d.TW * d.TH * d.TN != 128:
        raise Rejected("TW*TH*TN must be 128")
    if d.split not in (0, 1):
        raise Rejected("split must be 0 or 1")
    if d.mode == 0:
        if split and res and bn == 256:
            raise Rejected("split + residual supports block_n <= 128")
    elif d.mode == 1:
        if bn != 32 or d.Cout != 32 or d.phases != 1:
            raise Rejected("head mode needs Cout == block_n == 32, phases == 1")
        if not 1 <= d.head_classes <= 8:
            raise Rejected("bad head arguments")
    else:
        raise Rejected("unknown mode")
    if pair and (d.mode != 0 or bn < 128):
        raise Rejected("cta_pair needs mode 0 and block_n >= 128")
    if d.kchunk > 0 and bn > 128:
        raise Rejected("kchunk supports block_n <= 128")
    if d.stats and (d.mode != 0 or split or res or d.phases != 1):
        raise Rejected("stats needs mode 0, fast precision, no residual, phases == 1")
    # rsb_conv_plan_create, after the device check
    if d.mode == 0 and 64 % d.TW and d.TW % 64:
        raise Rejected("TW must divide or be a multiple of 64")
    if d.mode == 0 and res and d.phases != 1:
        raise Rejected("residual needs phases == 1")
    kblocks = sum(d.segs[i].cblocks for i in range(d.nseg))
    if 0 < d.kchunk < kblocks and d.mode != 0:
        raise Rejected("kchunk needs mode 0")
    if d.stats:
        return ("conv", bn, 0, 0, int(pair), 0, 1)
    narrow = 2 if split else 0
    if d.mode == 1:
        return ("conv", 32, 1, 0, 0, narrow, 0)
    if pair:
        return ("conv", bn, 0, int(res), 1, int(split), 0)
    return ("conv", bn, 0, int(res), 0, narrow if bn <= 64 else int(split), 0)


def _row_instance(d):
    """rsb_rowconv_plan_create's checks, then the key rsb_rowconv_run switches on"""
    if d.cin not in (32, 64, 128):
        raise Rejected("cin must be 32, 64 or 128")
    if d.Cout not in (32, 64):
        raise Rejected("Cout must be 32 or 64")
    if d.taps_h != d.taps_w or d.taps_h not in (2, 3):
        raise Rejected("taps must be 3x3 or 2x2")
    if d.nsub not in (1, 2) or d.nphase_a not in (1, 2):
        raise Rejected("nsub / nphase_a must be 1 or 2")
    cblk = 32 if d.cin == 32 else 64
    cblocks = d.cin // cblk
    if d.nsub * d.taps_h * d.taps_w * cblocks > 16:
        raise Rejected("too many weight blocks")
    if d.mode == 1 and (d.Cout != 32 or d.nsub != 1 or d.nphase_a != 1 or not 1 <= d.head_classes <= 8):
        raise Rejected("bad head arguments")
    if d.split and not (d.mode == 1 and d.cin == 32 and d.taps_h == 3 and d.src.plane > 0):
        raise Rejected("the strict-precision line buffer exists for the 3x3 32 -> 32 head layer only")
    # shared memory: resident weights + epilogue staging + a ring of at least taps_h + 1 input rows
    planes = 2 if d.split else 1
    slot = -(-(128 + d.taps_w + d.nsub - 2) * cblk * 2 // 1024) * 1024
    stage = 2 * 2 * 64 * (64 if d.Cout >= 64 else 32) * 2 if d.mode == 0 else 0
    fixed = d.nsub * d.taps_h * d.taps_w * cblocks * planes * d.Cout * cblk * 2 + stage + 512 + 1088 + 1024
    if (SMEM_OPTIN - 1024 - fixed) // (slot * cblocks * planes) < d.taps_h + 1:
        raise Rejected("not enough shared memory for the row ring")
    key = ("row", cblk, d.Cout, d.mode, d.taps_h, cblocks, d.nsub, int(bool(d.split)))
    if key not in _ROW_KEYS:
        raise Rejected("no kernel instance for this layer")
    return key


_ROW_KEYS = {k for k in compiled_instances() if k[0] == "row"}


def instance_of(desc):
    """the compiled instance the plan of `desc` launches (an rsb_conv_desc or an rsb_rowconv_desc); Rejected if none"""
    return _row_instance(desc) if isinstance(desc, RowConvDesc) else _conv_instance(desc)


# ----------------------------------------------------------------------------------------------------------------------
# operand buffers
# ----------------------------------------------------------------------------------------------------------------------
def _nan16(n):
    return torch.full((n,), SENTINEL16, dtype=torch.int16).view(torch.float16)


def _planes(v, split):
    """float64 [...] -> fp16 planes [P, ...]: (hi, lo) in strict precision, one fp16 plane otherwise"""
    hi = v.to(torch.float16)
    if not split:
        return hi[None]
    return torch.stack([hi, (v - hi.double()).to(torch.float16)])


class _Act:
    """an NHWC activation with PAD_C sentinel channels per pixel, planes `plane` elements apart"""

    def __init__(self, v, split, pad=PAD_C, fill=None):
        N, H, W, C = v.shape
        self.N, self.H, self.W, self.C, self.pc = N, H, W, C, C + pad
        self.plane = N * H * W * self.pc + 64
        self.buf = _nan16(self.plane * (2 if split else 1)) if fill is None else torch.full((self.plane * (2 if split else 1),), fill, dtype=torch.float16)
        p = _planes(v, split)
        for i in range(p.shape[0]):
            self.buf[i * self.plane:i * self.plane + N * H * W * self.pc].view(N, H, W, self.pc)[..., :C] = p[i]
        self.split = split

    def dense(self, buf):
        return ConvSrc(buf.data_ptr(), self.pc, self.W * self.pc, self.H * self.W * self.pc, self.C, self.W, self.H, self.N,
                       self.plane if self.split else 0)

    def parity(self, buf, ph, pw):
        return ConvSrc(buf.data_ptr() + 2 * (ph * self.W * self.pc + pw * self.pc), 2 * self.pc, 2 * self.W * self.pc, self.H * self.W * self.pc,
                       self.C, self.W // 2, self.H // 2, self.N, self.plane if self.split else 0)


class _Out:
    """an output view [N, oH, oW, Cout] at element offset `off` of a sentinel buffer, pitches wider than Cout"""

    def __init__(self, N, oH, oW, C, split):
        self.pw = C + PAD_C
        self.ph = oW * self.pw + 8
        self.pn = oH * self.ph + 16
        self.off = 24
        self.plane = self.off + N * self.pn + 40
        self.size = self.plane * (2 if split else 1)
        self.split = split

    def pitches(self):
        return (self.pw, self.ph, self.pn)

    def fill(self, v):
        """a buffer holding v [N, oH, oW, C] (float64, planes as the split) in the view and the sentinel elsewhere"""
        buf = _nan16(self.size)
        N, oH, oW, C = v.shape
        p = _planes(v, self.split)
        for i in range(p.shape[0]):
            torch.as_strided(buf, (N, oH, oW, C), (self.pn, self.ph, self.pw, 1), i * self.plane + self.off).copy_(p[i])
        return buf


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
class Built:
    """one case's tensors (`t`, by name) on one device, its descriptor, and what the checks need to know about them"""

    def __init__(self, case, t, desc, meta):
        self.case, self.t, self.desc, self.meta = case, t, desc, meta

    def to(self, device):
        t = {k: (v.to(device) if v is not None else None) for k, v in self.t.items()}
        return Built(self.case, t, self.case._desc(t, self.meta), self.meta)


class TcCase:
    """One launch of the tensor-core kernel (csrc/rsb_conv.cu).

    kind: '3x3' (dense source, 9 taps), '3x3s2' (four parity sources), 'cat1x1' (two sources, one 1x1 contraction over
    both: the conv3 + downsample segment pair), 'dec' (nearest x2 + 3x3 over two concatenated sources: 4 output phases of
    2x2 taps, out_scale 2), 'head' (dec5 + final: the 4-pixel window view of a W-padded 32-channel buffer, fused 1x1 head).
    tile = (Wt, Ht, Nt): the tile space (the low-resolution grid of 'dec')."""

    kernel = "conv"

    def __init__(self, name, kind, tile, cout=64, block_n=64, split=False, residual=False, pair=False, stats=False, box=None,
                 kchunk=0, classes=2, relu=True, bias=True, cin=64, seed=0):
        self.name, self.kind, self.tile, self.cout, self.block_n = name, kind, tile, cout, block_n
        self.split, self.residual, self.pair, self.stats, self.box = split, residual, pair, stats, box
        self.kchunk, self.classes, self.relu, self.bias, self.cin, self.seed = kchunk, classes, relu, bias, cin, seed

    def __repr__(self):
        return self.name

    @property
    def desc(self):
        """the host descriptor (for instance_of); it keeps its tensors alive"""
        b = self.build("cpu")
        b.desc._keep = b
        return b.desc

    def build(self, device="cpu"):
        g = torch.Generator().manual_seed(self.seed)
        Wt, Ht, Nt = self.tile
        split, cout, cin = self.split, self.cout, self.cin
        t, meta = {}, {}
        if self.kind == "head":
            cout = 32
            x = _rand((Nt, Ht, Wt, 32), g).double()
            # W-padded buffer [N, H, W + 4, 32] (pixel w at column w + 1), zero padding: the window view reads it
            xb = torch.zeros(Nt, Ht, Wt + 4, 32, dtype=torch.float64)
            xb[:, :, 1:Wt + 1] = x
            a = _Act(xb, split, pad=0, fill=0.0)
            t["src0"] = a.buf
            meta["acts"] = [a]
            w = E.pack_window3(_rand((32, 32, 3, 3), g, (2.0 / 288) ** 0.5).double())
            meta["segs"] = [(0, kh - 1, 0, 2) for kh in range(3)]
            phases, oshape = 1, (Nt, Ht, Wt)
        elif self.kind == "dec":
            cins = (cin, cin)
            acts = [_Act(_rand((Nt, Ht, Wt, c), g).double(), split) for c in cins]
            w = E.pack_upsample_phases(_rand((cout, sum(cins), 3, 3), g, (2.0 / (9 * sum(cins))) ** 0.5).double())
            meta["segs"] = [(si, th - 1, tw - 1, c // 64) for th in range(2) for tw in range(2) for si, c in enumerate(cins)]
            phases, oshape = 4, (Nt, 2 * Ht, 2 * Wt)
        elif self.kind == "cat1x1":
            cins = (cin, 2 * cin)
            acts = [_Act(_rand((Nt, Ht, Wt, c), g).double(), split) for c in cins]
            w = E.pack_conv(_rand((cout, sum(cins), 1, 1), g, (2.0 / sum(cins)) ** 0.5).double())
            meta["segs"] = [(0, 0, 0, cins[0] // 64), (1, 0, 0, cins[1] // 64)]
            phases, oshape = 1, (Nt, Ht, Wt)
        elif self.kind == "3x3s2":
            acts = [_Act(_rand((Nt, 2 * Ht, 2 * Wt, cin), g).double(), split)]
            w = E.pack_conv(_rand((cout, cin, 3, 3), g, (2.0 / (9 * cin)) ** 0.5).double())
            segs = []
            for kh in range(3):
                for kw in range(3):
                    segs.append((((kh - 1) % 2) * 2 + (kw - 1) % 2, (kh - 1) // 2, (kw - 1) // 2, cin // 64))
            meta["segs"] = segs
            phases, oshape = 1, (Nt, Ht, Wt)
        else:
            acts = [_Act(_rand((Nt, Ht, Wt, cin), g).double(), split)]
            w = E.pack_conv(_rand((cout, cin, 3, 3), g, (2.0 / (9 * cin)) ** 0.5).double())
            meta["segs"] = [(0, kh - 1, kw - 1, cin // 64) for kh in range(3) for kw in range(3)]
            phases, oshape = 1, (Nt, Ht, Wt)
        if self.kind != "head":
            meta["acts"] = acts
            for i, a in enumerate(acts):
                t["src%d" % i] = a.buf
        if split:
            hi, lo, scale = E.split_fp16(w)
            t["weights"] = torch.stack([hi, lo]).contiguous()
        else:
            t["weights"], scale = w.to(torch.float16).contiguous(), 1.0
        meta["scale"], meta["phases"], meta["cout"] = scale, phases, cout
        t["bias"] = (_rand((cout,), g, 0.1).float() if self.bias else None)
        if self.kind == "head":
            t["head_w"] = _rand((self.classes, 32), g, 0.3).float().contiguous()
            t["head_b"] = _rand((self.classes,), g, 0.1).float()
            meta["lsize"] = Nt * self.classes * Ht * Wt
            meta["loff"] = 5
            t["out"] = torch.full((meta["loff"] + meta["lsize"] + 27,), SENTINEL32, dtype=torch.int32).view(torch.float32)
        else:
            o = _Out(oshape[0], oshape[1], oshape[2], cout, split)
            meta["o"] = o
            t["out"] = _nan16(o.size)
            if self.residual:
                t["residual"] = o.fill(_rand((oshape[0], oshape[1], oshape[2], cout), g).double())
        if self.kchunk:
            bn = self.block_n
            meta["scratch_bytes"] = SMS * 128 * bn * 4
            t["scratch"] = torch.full((SMS * 128 * bn + 256,), SENTINEL32, dtype=torch.int32).view(torch.float32)
        if self.stats:
            TW, TH, TN = self.box or E.choose_tile(Wt, Ht, Nt)
            rows = 4 * -(-Wt // TW) * -(-Ht // TH) * -(-Nt // TN)
            meta["stats_rows"] = rows
            t["stats"] = torch.full((rows * 2 * cout + 64,), SENTINEL32, dtype=torch.int32).view(torch.float32)
        b = Built(self, t, None, meta)
        return b.to(device) if torch.device(device).type != "cpu" else Built(self, t, self._desc(t, meta), meta)

    def _desc(self, t, meta):
        Wt, Ht, Nt = self.tile
        split = self.split
        acts = meta["acts"]
        if self.kind == "3x3s2":
            srcs = [acts[0].parity(t["src0"], ph, pw) for ph in range(2) for pw in range(2)]
        elif self.kind == "head":
            a = acts[0]
            # the 4-pixel window over the W-padded buffer: C = 128 channels at a 32-channel pixel pitch
            srcs = [ConvSrc(t["src0"].data_ptr(), 32, a.W * 32, a.H * a.W * 32, 128, Wt, Ht, Nt, a.plane if split else 0)]
        else:
            srcs = [a.dense(t["src%d" % i]) for i, a in enumerate(acts)]
        common = dict(relu=self.relu, block_n=self.block_n, split=split, acc_scale=meta["scale"], cta_pair=self.pair)
        if self.kind == "head":
            loff = meta["loff"]
            logits = t["out"][loff:loff + meta["lsize"]]
            d = E.make_conv_desc(srcs, meta["segs"], t["weights"], t["bias"], 32, 1, self.tile, None, None,
                                 head=(t["head_w"], t["head_b"], logits, self.classes), **common)
        else:
            o = meta["o"]
            d = E.make_conv_desc(srcs, meta["segs"], t["weights"], t["bias"], meta["cout"], meta["phases"], self.tile, t["out"], o.pitches(),
                                 out_scale=(2, 2) if self.kind == "dec" else (1, 1), residual=t.get("residual"), out_offset_elems=o.off,
                                 out_plane=o.plane if split else 0, res_plane=o.plane if split and self.residual else 0, **common)
            if self.residual:
                d.residual = t["residual"].data_ptr() + 2 * o.off
        if self.box:
            d.TW, d.TH, d.TN = self.box
        if self.kchunk:
            d.kchunk = self.kchunk
            d.scratch, d.scratch_bytes = t["scratch"].data_ptr(), meta["scratch_bytes"]
        if self.stats:
            d.stats, d.stats_bytes = t["stats"].data_ptr(), meta["stats_rows"] * 2 * meta["cout"] * 4
        return d

    def readonly(self):
        """tensors the launch must not modify"""
        return ["src0", "src1", "weights", "bias", "residual", "head_w", "head_b"]


class RowCase:
    """One launch of the line-buffer kernel (csrc/rsb_conv_row.cu). kind: 'row3x3' (3x3 stride 1), 'rowup' (nearest x2 + 3x3:
    2 row phases x 2 column sub-tiles), 'rowhead' (3x3 + ReLU + the fused 1x1 head). tile = (Wt, Ht, Nt) of the input grid."""

    kernel = "row"

    def __init__(self, name, kind, tile, cin, cout, rows_per_unit=0, split=False, classes=2, relu=True, bias=True, seed=0):
        self.name, self.kind, self.tile, self.cin, self.cout = name, kind, tile, cin, cout
        self.rows_per_unit, self.split, self.classes, self.relu, self.bias, self.seed = rows_per_unit, split, classes, relu, bias, seed

    def __repr__(self):
        return self.name

    desc = TcCase.desc

    def build(self, device="cpu"):
        g = torch.Generator().manual_seed(self.seed)
        Wt, Ht, Nt = self.tile
        split, cin = self.split, self.cin
        cout = 32 if self.kind == "rowhead" else self.cout
        t, meta = {}, {}
        a = _Act(_rand((Nt, Ht, Wt, cin), g).double(), split)
        t["src0"], meta["acts"] = a.buf, [a]
        w = _rand((cout, cin, 3, 3), g, (2.0 / (9 * cin)) ** 0.5).double()
        w = E.pack_upsample_phases(w) if self.kind == "rowup" else E.pack_conv(w)
        if split:
            hi, lo, scale = E.split_fp16(w)
            t["weights"] = torch.stack([hi, lo]).contiguous()
        else:
            t["weights"], scale = w.to(torch.float16).contiguous(), 1.0
        meta["scale"], meta["cout"] = scale, cout
        # the kernel's head adds no conv bias (the engine's dec5 has none); mode 0 adds it
        t["bias"] = _rand((cout,), g, 0.1).float() if self.bias and self.kind != "rowhead" else None
        if self.kind == "rowhead":
            t["head_w"] = _rand((self.classes, 32), g, 0.3).float().contiguous()
            t["head_b"] = _rand((self.classes,), g, 0.1).float()
            meta["lsize"] = Nt * self.classes * Ht * Wt
            meta["loff"] = 7
            t["out"] = torch.full((meta["loff"] + meta["lsize"] + 29,), SENTINEL32, dtype=torch.int32).view(torch.float32)
        else:
            up = 2 if self.kind == "rowup" else 1
            o = _Out(Nt, up * Ht, up * Wt, cout, False)
            meta["o"] = o
            t["out"] = _nan16(o.size)
        b = Built(self, t, None, meta)
        return b.to(device) if torch.device(device).type != "cpu" else Built(self, t, self._desc(t, meta), meta)

    def _desc(self, t, meta):
        a = meta["acts"][0]
        src = a.dense(t["src0"])
        kw = dict(rows_per_unit=self.rows_per_unit, relu=self.relu, split=self.split, acc_scale=meta["scale"])
        if self.kind == "rowhead":
            loff = meta["loff"]
            return E.make_rowconv_desc(src, self.cin, t["weights"], None, 32, self.tile, None, None,
                                       head=(t["head_w"], t["head_b"], t["out"][loff:loff + meta["lsize"]], self.classes), **kw)
        o = meta["o"]
        return E.make_rowconv_desc(src, self.cin, t["weights"], t["bias"], meta["cout"], self.tile, t["out"], o.pitches(),
                                   upsample=self.kind == "rowup", out_offset_elems=o.off, **kw)

    def readonly(self):
        return ["src0", "weights", "bias", "head_w", "head_b"]


# ----------------------------------------------------------------------------------------------------------------------
# the matrix
# ----------------------------------------------------------------------------------------------------------------------
def _ragged(box):
    """a tile space that is not a multiple of the box along any axis that can be ragged (two tiles along each)"""
    return tuple(b + max(1, b // 2) if b > 1 else 3 for b in box)


def _tc_instances():
    return sorted(k[1:] for k in compiled_instances() if k[0] == "conv")


def _tag(inst):
    bn, mode, res, two, split, stats = inst
    return "%s%s_bn%d%s%s%s" % ("strict" if split else "fast", "_head" if mode else "", bn, "_res" if res else "",
                                 "_pair" if two else "", "_stats" if stats else "")


def _tc_kwargs(inst):
    bn, mode, res, two, split, stats = inst
    return dict(block_n=bn, split=bool(split), residual=bool(res), pair=bool(two), stats=bool(stats),
                cout=32 if mode else (bn if bn == 256 else 2 * bn))


def _tc_cases():
    cases = []
    seed = itertools.count(100)
    for inst in _tc_instances():
        mode, res, two, stats = inst[1], inst[2], inst[3], inst[5]
        tag, kw = _tag(inst), _tc_kwargs(inst)
        # every box, ragged along every axis that can be; the operation rotates over the layer kinds the instance serves
        kinds = ["head"] if mode else (["3x3", "cat1x1", "3x3s2"] if (res or stats) else ["3x3", "cat1x1", "3x3s2", "dec"])
        for i, box in enumerate(BOXES):
            kind = kinds[i % len(kinds)]
            if mode == 0 and 64 % box[0] and box[0] % 64:
                continue
            extra = dict(classes=(1, 8)[i % 2]) if mode else dict(relu=bool(i % 3), bias=bool(i % 4))
            cases.append(TcCase("%s_%s_box%dx%dx%d" % (tag, kind, *box), kind, _ragged(box), box=box, seed=next(seed), **kw, **extra))
        # more tiles than SMs; an odd number of spatial tiles under a CTA pair (the last pair's second CTA has no tile)
        if mode:
            cases.append(TcCase("%s_multiwave" % tag, "head", (45, 61, 7), classes=8, seed=next(seed), **kw))  # 3 x 8 x 7 tiles of 16x8x1
        else:
            nb = kw["cout"] // inst[0]
            m = 133 // nb + 1
            m += 1 - m % 2 if two else 0
            cases.append(TcCase("%s_multiwave_%dtiles" % (tag, m * nb), "cat1x1", (16 * m - 5, 5, 1), box=(16, 8, 1), seed=next(seed), **kw))
    # K chunking: narrow and wide, paired and single, with and without a residual; kchunk 1, K - 1 and one that does not
    # divide K (the 3x3 on 64 channels has 9 K blocks: chunks 1 x 9, 8 + 1, 4 + 4 + 1)
    for inst in _tc_instances():
        bn, mode, res, two, split, stats = inst
        if mode or stats or bn > 128 or not split:
            continue
        for kc in (1, 8, 4):
            cases.append(TcCase("%s_kchunk%d" % (_tag(inst), kc), "3x3", (21, 11, 3), kchunk=kc, seed=next(seed), **_tc_kwargs(inst)))
    # ... in fast precision too (the ABI accepts it; every instance of <= 128 columns has the fold)
    for bn, res in ((32, True), (128, False)):
        inst = (bn, 0, int(res), 0, 0, 0)
        cases.append(TcCase("%s_kchunk4" % _tag(inst), "3x3", (21, 11, 3), kchunk=4, seed=next(seed), **_tc_kwargs(inst)))
    # long K (a decoder over 2 x 1024 channels: 4 taps x 32 = 128 K blocks), chunks that do not divide it
    cases.append(TcCase("strict_bn128_pair_dec_longK_kchunk34", "dec", (4, 4, 2), cin=1024, cout=256, block_n=128, split=True, pair=True,
                        kchunk=34, seed=next(seed)))
    cases.append(TcCase("strict_bn64_dec_longK_kchunk100", "dec", (4, 4, 2), cin=1024, cout=64, block_n=64, split=True,
                        kchunk=100, seed=next(seed)))
    return cases


def _row_cases():
    cases = []
    seed = itertools.count(900)
    for key in sorted(k for k in compiled_instances() if k[0] == "row"):
        _, cblk, cout, mode, taps, cblocks, nsub, split = key
        cin = cblk * cblocks
        kind = "rowhead" if mode else ("rowup" if taps == 2 else "row3x3")
        tag = "%s_%s_%d-%d" % ("strict" if split else "fast", kind, cin, cout)
        kw = dict(split=bool(split))
        # ragged: W not a multiple of 128 (partial last strip), H not a multiple of rows_per_unit (short last unit)
        cases.append(RowCase(tag + "_ragged", kind, (200, 13, 2), cin, cout, rows_per_unit=4, classes=8, seed=next(seed), **kw))
        # units of more rows than the ring holds (at most 16 slots): the ring wraps inside a unit
        cases.append(RowCase(tag + "_ringwrap", kind, (130, 45, 1), cin, cout, rows_per_unit=20, classes=1, relu=False, seed=next(seed), **kw))
        # more units than SMs; for the upsample (2 row phases) an odd number of units per phase, so that the units past the
        # first wave land on CTAs whose resident weights are the same row phase (the grid is even: units are an even count)
        tile = (100, 67, 1) if kind == "rowup" else (140, 36, 4)
        cases.append(RowCase(tag + "_multiwave", kind, tile, cin, cout, rows_per_unit=1 if kind == "rowup" else 2, classes=2, bias=False,
                             seed=next(seed), **kw))
        # the plan's own rows_per_unit
        cases.append(RowCase(tag + "_auto", kind, (256, 20, 2), cin, cout, classes=3, seed=next(seed), **kw))
    return cases


_MATRIX = None


def matrix(device=None):
    """every case (specs: `case.build(device)` makes the tensors; `case.desc` is a host descriptor). `device` is accepted for
    symmetry with the other case builders: the specs do not depend on it."""
    global _MATRIX
    if _MATRIX is None:
        _MATRIX = _tc_cases() + _row_cases()
    return list(_MATRIX)


def plan_create_code(lib, desc):
    """return code of the plan constructor (a created plan is destroyed)"""
    plan = ctypes.c_void_p()
    create = lib.rsb_rowconv_plan_create if isinstance(desc, RowConvDesc) else lib.rsb_conv_plan_create
    rc = create(ctypes.byref(desc), ctypes.byref(plan))
    if rc == 0:
        (lib.rsb_rowconv_plan_destroy if isinstance(desc, RowConvDesc) else lib.rsb_conv_plan_destroy)(plan)
    return rc


__all__ = ["BOXES", "Built", "ConvDesc", "Rejected", "RowCase", "TcCase", "compiled_instances", "instance_of", "matrix", "plan_create_code"]
