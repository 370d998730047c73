"""CPU emulation of the semantics of `rsb_conv_run` for descriptors whose pointers are HOST memory.

Test infrastructure only. It reads the raw pointers of an `rsb_conv_desc` exactly the way the kernel's TMA
boxes do (views with arbitrary -- possibly overlapping -- pitches, zero fill outside the view extents) so the
host-side logic (weight packing, parity views, upsample phases, window views, output addressing) can be
verified without a GPU.
"""

import concurrent.futures
import ctypes
import os

import numpy as np

WORKERS = max(1, min(16, len(os.sched_getaffinity(0))))


def pmap(fn, items):
    """[fn(x) for x in items] on a thread pool: the float64 references are numpy work on large arrays, which runs outside the
    interpreter lock, so independent chunks use the host's cores"""
    items = list(items)
    if len(items) < 2:
        return [fn(x) for x in items]
    with concurrent.futures.ThreadPoolExecutor(min(len(items), WORKERS)) as ex:
        return list(ex.map(fn, items))


def _view(ptr, shape, strides_elems, dtype=np.float16, writable=False):
    item = np.dtype(dtype).itemsize
    span = 1 + sum((s - 1) * abs(st) for s, st in zip(shape, strides_elems))
    raw = (ctypes.c_uint8 * (span * item)).from_address(ptr)
    base = np.frombuffer(raw, dtype=dtype)
    v = np.lib.stride_tricks.as_strided(base, shape=shape, strides=[st * item for st in strides_elems], writeable=writable)
    return v


def prepass_s2d_cpu(x):
    """torch fp32 NCHW -> fp16 [N, H/2, W/2+4, 16] (what rsb_prepass_s2d writes)"""
    import torch

    N, C, H, W = x.shape
    out = torch.zeros(N, H // 2, W // 2 + 4, 16, dtype=torch.float16)
    for ph in range(2):
        for pw in range(2):
            out[:, :, 2:2 + W // 2, (ph * 2 + pw) * 3:(ph * 2 + pw) * 3 + 3] = x[:, :, ph::2, pw::2].permute(0, 2, 3, 1).half()
    return out


def prepass_s2d_split_cpu(x):
    """rsb_prepass_s2d_split: [2, N, H/2, W/2+4, 16], plane 0 = half(x), plane 1 = half(x - float(half(x)))"""
    import torch

    hi = prepass_s2d_cpu(x)
    N, C, H, W = x.shape
    xs = torch.zeros(N, H // 2, W // 2 + 4, 16, dtype=torch.float32)
    for ph in range(2):
        for pw in range(2):
            xs[:, :, 2:2 + W // 2, (ph * 2 + pw) * 3:(ph * 2 + pw) * 3 + 3] = x[:, :, ph::2, pw::2].permute(0, 2, 3, 1)
    return torch.stack([hi, (xs - hi.float()).half()])


def split_pair(v32):
    """fp32 array -> (hi, lo) fp16 arrays the way the kernels' epilogues do it (residue exact in fp32)"""
    hi = v32.astype(np.float16)
    lo = (v32 - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def _pair(ptr, plane, shape, strides):
    """value of an operand view: fast mode = the fp16 plane; split mode = hi + lo (exact in fp32), as float64"""
    v = _view(ptr, shape, strides).astype(np.float64)
    if plane:
        v = v + _view(ptr + 2 * plane, shape, strides).astype(np.float64)
    return v


def _operand(ptr, plane, shape, strides):
    """float64 (hi, lo) planes of an operand view; lo is None for a single fp16 operand (plane 0)"""
    hi = _view(ptr, shape, strides).astype(np.float64)
    return hi, (_view(ptr + 2 * plane, shape, strides).astype(np.float64) if plane else None)


class _F64Acc:
    """float64 replay of one output phase, added up term by term (a: (hi, lo) [..., k], w: (hi, lo) [Cout, k]):
      val   the contraction of the operands' values (hi + lo in split mode);
      dot   sum (|a_hi| + |a_lo|)(|w_hi| + |w_lo|) >= sum |a||w| (fast mode: sum |a||w|), the magnitude that scales the
            kernel's accumulation error;
      split mode only: lolo = sum |a_lo||w_lo| (the product the kernel omits) and hihi = sum |a_hi||w_hi| (the main chain of
            the N-concatenated schedule; dot - hihi - lolo is its cross chain)."""

    def __init__(self, split):
        self.split = split
        self.val = self.dot = self.lolo = self.hihi = 0.0

    def add(self, a, w):
        (ah, al), (wh, wl) = a, w

        def td(x, y):
            return np.tensordot(x, y, axes=([x.ndim - 1], [1]))

        if not self.split:
            self.val = self.val + td(ah, wh)
            self.dot = self.dot + td(np.abs(ah), np.abs(wh))
            return
        aa, wa, la, lw = np.abs(ah), np.abs(wh), np.abs(al), np.abs(wl)
        self.val = self.val + td(ah + al, wh + wl)
        self.dot = self.dot + td(aa + la, wa + lw)
        self.lolo = self.lolo + td(la, lw)
        self.hihi = self.hihi + td(aa, wa)


def _f64_emit(d, acc, scale, out, shape, strides, res, out_plane, res_plane, sink):
    """the float64 epilogue of one output phase: * acc_scale, + bias, (mode 0) + residual, ReLU; mode 1 contracts ReLU(conv),
    kept in float64, with `final`'s fp32 weights. sink(ptr, shape, strides, value, mag, parts, plane):
      mode 0: value [Nt, Ht, Wt, Cout] at `out` (and its lo plane `plane` elements further in split mode), mag = dot + |bias|
              + |residual|, parts = the magnitudes of _F64Acc times acc_scale;
      mode 1: the logits [Nt, classes, Ht, Wt] at head_out, mag = sum_c |w_c y_c| + |b|, parts = sum_c |w_c| part_c, the
              conv's magnitudes carried through the 1x1 head (ReLU is 1-Lipschitz), with |bias| added to dot."""
    parts = {"dot": acc.dot * scale}
    if acc.split:
        parts.update(lolo=acc.lolo * scale, hihi=acc.hihi * scale)
    v = acc.val * scale
    mag = parts["dot"]
    if d.bias:
        b = _view(d.bias, (d.Cout,), (1,), np.float32).astype(np.float64)
        v, mag = v + b, mag + np.abs(b)
    if d.mode == 0:
        if res:
            r = _pair(res, res_plane, shape, strides)
            v, mag = v + r, mag + np.abs(r)
        sink(out, shape, strides, np.maximum(v, 0) if d.relu else v, mag, parts, out_plane)
        return
    parts["dot"] = mag
    y = np.maximum(v, 0) if d.relu else v
    hw = _view(d.head_w, (d.head_classes, 32), (32, 1), np.float32).astype(np.float64)
    hb = _view(d.head_b, (d.head_classes,), (1,), np.float32).astype(np.float64)

    def head(t, w):
        return np.transpose(np.tensordot(t, w, axes=([3], [1])), (0, 3, 1, 2))

    logits = head(y, hw) + hb[None, :, None, None]
    lmag = head(np.abs(y), np.abs(hw)) + np.abs(hb)[None, :, None, None]
    Nt, Ht, Wt = shape[:3]
    sink(d.head_out, (Nt, d.head_classes, Ht, Wt), (d.head_classes * Ht * Wt, Ht * Wt, Wt, 1), logits, lmag,
         {k: head(p, np.abs(hw)) for k, p in parts.items()}, 0)


def _run_desc_f64(d, sink):
    split = bool(d.split)
    K = 64 * sum(d.segs[i].cblocks for i in range(d.nseg))
    rows = d.phases * d.Cout
    w = _operand(d.weights, rows * K if split else 0, (rows, K), (K, 1))
    srcs = [_operand(s.ptr, s.plane if split else 0, (s.N, s.H, s.W, s.C), (s.pitch_n, s.pitch_h, s.pitch_w, 1))
            for s in (d.srcs[i] for i in range(d.nsrc))]
    for phase in range(d.phases):
        pa, pb = phase >> 1, phase & 1
        acc = _F64Acc(split)
        k0 = 0
        for si in range(d.nseg):
            seg = d.segs[si]
            width = seg.cblocks * 64
            a = tuple(None if p is None else _gather(p, d.srcs[seg.src], seg.dh + pa, seg.dw + pb, d.Nt, d.Ht, d.Wt, width) for p in srcs[seg.src])
            acc.add(a, tuple(None if p is None else p[phase * d.Cout:(phase + 1) * d.Cout, k0:k0 + width] for p in w))
            k0 += width
        off = 2 * (pa * d.out_pitch_h + pb * d.out_pitch_w)
        strides = (d.out_pitch_n, d.out_sy * d.out_pitch_h, d.out_sx * d.out_pitch_w, 1)
        _f64_emit(d, acc, float(d.acc_scale) if d.acc_scale != 0 else 1.0, (d.out or 0) + off, (d.Nt, d.Ht, d.Wt, d.Cout), strides,
                  (d.residual + off) if d.residual else None, d.out_plane if split else 0, d.res_plane if split else 0, sink)


def _gather(sv, src, dh, dw, Nt, Ht, Wt, width):
    """A operand of one tap: [Nt, Ht, Wt, width] of the view `sv` [N, H, W, C] shifted by (dh, dw), zero outside the view"""
    hh = np.arange(Ht)[:, None] + dh
    ww = np.arange(Wt)[None, :] + dw
    inb = (hh >= 0) & (hh < src.H) & (ww >= 0) & (ww < src.W)
    g = sv[:, np.clip(hh, 0, src.H - 1), np.clip(ww, 0, src.W - 1), :min(width, sv.shape[-1])] * inb[None, :, :, None]
    a = np.zeros((Nt, Ht, Wt, width), dtype=sv.dtype)
    nn = min(Nt, src.N)
    a[:nn, :, :, :g.shape[-1]] = g[:nn]
    return a


def _gather_at(sv, src, dh, dw, n, y, x, width):
    """A operand rows of one tap at output pixels (n, y, x) (int64 arrays): [S, width] of the view `sv` [N, H, W, C] at
    (n, y + dh, x + dw), zero outside the view (as _gather)"""
    hh, ww = y + dh, x + dw
    inb = (hh >= 0) & (hh < src.H) & (ww >= 0) & (ww < src.W) & (n < src.N)
    c = min(width, sv.shape[-1])
    g = sv[np.minimum(n, src.N - 1), np.clip(hh, 0, src.H - 1), np.clip(ww, 0, src.W - 1), :c] * inb[:, None]
    if c == width:
        return g
    a = np.zeros((len(n), width), dtype=g.dtype)
    a[:, :c] = g
    return a


def conv_out_views(d):
    """(phase, byte address, shape, element strides) of every output phase of a mode-0 descriptor, as the kernel addresses them"""
    strides = (d.out_pitch_n, d.out_sy * d.out_pitch_h, d.out_sx * d.out_pitch_w, 1)
    return [(ph, d.out + 2 * ((ph >> 1) * d.out_pitch_h + (ph & 1) * d.out_pitch_w), (d.Nt, d.Ht, d.Wt, d.Cout), strides)
            for ph in range(d.phases)]


def conv_f64_at(d, pix):
    """The float64 reference of mode-0 descriptor `d` (what run_desc(d, sink) gives) at sampled output pixels only.
    pix: int64 [S, 3] (n, y, x) in the tile space, or [S, 4] with the output phase (2 pa + pb) of a 4-phase decoder last.
    Returns (value, mag, addr): value and mag [S, Cout] as the sink receives them (mag = sum |a||w| (+ |bias| + |residual|),
    with the (hi, lo) pair magnitudes in split mode) and addr [S], the byte address of channel 0 of each pixel's output (the
    lo plane of a split output lies d.out_plane elements further)."""
    assert d.mode == 0, "conv_f64_at: head descriptors are checked whole"
    pix = np.asarray(pix, dtype=np.int64)
    if pix.shape[1] == 3:
        assert d.phases == 1
        pix = np.concatenate([pix, np.zeros((len(pix), 1), np.int64)], axis=1)
    split = bool(d.split)
    K = 64 * sum(d.segs[i].cblocks for i in range(d.nseg))
    rows = d.phases * d.Cout
    w = _operand(d.weights, rows * K if split else 0, (rows, K), (K, 1))
    # fp16 views of the sources (and their lo planes): only the gathered rows are converted to float64
    srcs = [tuple(None if pl is None else _view(s.ptr + 2 * pl, (s.N, s.H, s.W, s.C), (s.pitch_n, s.pitch_h, s.pitch_w, 1))
                  for pl in (0, s.plane if split else None))
            for s in (d.srcs[i] for i in range(d.nsrc))]
    scale = float(d.acc_scale) if d.acc_scale != 0 else 1.0
    S = len(pix)
    val, mag, addr = np.zeros((S, d.Cout)), np.zeros((S, d.Cout)), np.zeros(S, dtype=np.int64)
    for phase, base, _, strides in conv_out_views(d):
        sel = np.nonzero(pix[:, 3] == phase)[0]
        if not sel.size:
            continue
        n, y, x = pix[sel, 0], pix[sel, 1], pix[sel, 2]
        assert (n >= 0).all() and (n < d.Nt).all() and (y >= 0).all() and (y < d.Ht).all() and (x >= 0).all() and (x < d.Wt).all()
        pa, pb = phase >> 1, phase & 1
        acc = _F64Acc(split)
        k0 = 0
        for si in range(d.nseg):
            seg = d.segs[si]
            width = seg.cblocks * 64
            a = tuple(None if p is None else _gather_at(p, d.srcs[seg.src], seg.dh + pa, seg.dw + pb, n, y, x, width).astype(np.float64)
                      for p in srcs[seg.src])
            acc.add(a, tuple(None if p is None else p[phase * d.Cout:(phase + 1) * d.Cout, k0:k0 + width] for p in w))
            k0 += width
        v, m = acc.val * scale, acc.dot * scale
        if d.bias:
            b = _view(d.bias, (d.Cout,), (1,), np.float32).astype(np.float64)
            v, m = v + b, m + np.abs(b)
        eoff = n * strides[0] + y * strides[1] + x * strides[2]
        if d.residual:
            rbase = d.residual + (base - d.out)
            r = _pair(rbase, d.res_plane if split else 0, (d.Nt, d.Ht, d.Wt, d.Cout), strides)[n, y, x]
            v, m = v + r, m + np.abs(r)
        val[sel] = np.maximum(v, 0) if d.relu else v
        mag[sel] = m
        addr[sel] = base + 2 * eoff
    return val, mag, addr


def run_desc(d, sink=None):
    """Execute descriptor `d` (host pointers) and write its outputs like the device kernel would.
    Split descriptors: operands are hi + lo pairs; the contraction is done in float64 (the kernel's fp32 accumulation of
    hi*hi + hi*lo + lo*hi differs from it by ~1e-7 relative), the epilogue in fp32 exactly like the kernel.
    sink: float64 reference mode, both precisions and both modes. Nothing is written; for every output phase
    sink(ptr, shape, strides, value, mag, parts, plane) receives the exact float64 result of the operands' values and the
    magnitudes that scale the kernel's error (see _F64Acc and _f64_emit)."""
    if sink is not None:
        return _run_desc_f64(d, sink)
    split = bool(d.split)
    K = 64 * sum(d.segs[i].cblocks for i in range(d.nseg))
    rows = d.phases * d.Cout
    wts = _pair(d.weights, rows * K if split else 0, (rows, K), (K, 1))
    if not split:
        wts = wts.astype(np.float32)
    scale = np.float32(d.acc_scale if d.acc_scale != 0 else 1.0)
    bias = _view(d.bias, (d.Cout,), (1,), np.float32) if d.bias else None
    Nt, Ht, Wt = d.Nt, d.Ht, d.Wt
    acc_t = np.float64 if split else np.float32
    for phase in range(d.phases):
        pa, pb = phase >> 1, phase & 1
        acc = np.zeros((Nt, Ht, Wt, d.Cout), dtype=acc_t)
        k0 = 0
        for si in range(d.nseg):
            seg = d.segs[si]
            src = d.srcs[seg.src]
            width = seg.cblocks * 64
            sv = _pair(src.ptr, src.plane if split else 0, (src.N, src.H, src.W, min(width, src.C)), (src.pitch_n, src.pitch_h, src.pitch_w, 1))
            a = _gather(sv.astype(acc_t), src, seg.dh + pa, seg.dw + pb, Nt, Ht, Wt, width)
            acc += np.tensordot(a, wts[phase * d.Cout:(phase + 1) * d.Cout, k0:k0 + width], axes=([3], [1]))
            k0 += width
        acc = acc.astype(np.float32) * scale
        if bias is not None:
            acc += bias
        if d.mode == 0:
            base = d.out + 2 * (pa * d.out_pitch_h + pb * d.out_pitch_w)
            strides = (d.out_pitch_n, d.out_sy * d.out_pitch_h, d.out_sx * d.out_pitch_w, 1)
            if d.residual:
                rbase = d.residual + 2 * (pa * d.out_pitch_h + pb * d.out_pitch_w)
                acc += _pair(rbase, d.res_plane if split else 0, (Nt, Ht, Wt, d.Cout), strides).astype(np.float32)
            if d.relu:
                acc = np.maximum(acc, 0)
            ov = _view(base, (Nt, Ht, Wt, d.Cout), strides, writable=True)
            if split:
                hi, lo = split_pair(acc)
                ov[...] = hi
                _view(base + 2 * d.out_plane, (Nt, Ht, Wt, d.Cout), strides, writable=True)[...] = lo
            else:
                ov[...] = acc.astype(np.float16)
        else:
            if d.relu:
                acc = np.maximum(acc, 0)
            hw = _view(d.head_w, (d.head_classes, 32), (32, 1), np.float32)
            hb = _view(d.head_b, (d.head_classes,), (1,), np.float32)
            logits = np.tensordot(acc, hw, axes=([3], [1])) + hb  # [N, H, W, classes]
            ov = _view(d.head_out, (Nt, d.head_classes, Ht, Wt), (d.head_classes * Ht * Wt, Ht * Wt, Wt, 1), np.float32, writable=True)
            ov[...] = np.transpose(logits, (0, 3, 1, 2))


def run_rowdesc(d, sink=None):
    """CPU semantics of rsb_rowconv_run (line-buffer kernel): same arithmetic as run_desc, described by taps instead of segments.
    sink: the float64 reference mode of run_desc."""
    nph = d.nphase_a * d.nsub
    K = d.taps_h * d.taps_w * d.cin
    split = bool(getattr(d, "split", 0))
    if sink is not None:
        w = _operand(d.weights, nph * d.Cout * K if split else 0, (nph * d.Cout, K), (K, 1))
        s = d.src
        sv = _operand(s.ptr, s.plane if split else 0, (s.N, s.H, s.W, d.cin), (s.pitch_n, s.pitch_h, s.pitch_w, 1))
        strides = (d.out_pitch_n, d.out_sy * d.out_pitch_h, d.out_sx * d.out_pitch_w, 1)
        for a in range(d.nphase_a):
            for s_ in range(d.nsub):
                acc = _F64Acc(split)
                r0 = (a * d.nsub + s_) * d.Cout
                for th in range(d.taps_h):
                    for tw in range(d.taps_w):
                        k0 = (th * d.taps_w + tw) * d.cin
                        acc.add(tuple(None if p is None else _gather(p, s, d.dh0 + a + th, d.dw0 + s_ + tw, d.Nt, d.Ht, d.Wt, d.cin) for p in sv),
                                tuple(None if p is None else p[r0:r0 + d.Cout, k0:k0 + d.cin] for p in w))
                _f64_emit(d, acc, float(d.acc_scale) if split and d.acc_scale != 0 else 1.0,
                          (d.out or 0) + 2 * (a * d.out_pitch_h + s_ * d.out_pitch_w), (d.Nt, d.Ht, d.Wt, d.Cout), strides, None, 0, 0, sink)
        return
    wts = _pair(d.weights, nph * d.Cout * K if split else 0, (nph * d.Cout, K), (K, 1))
    if not split:
        wts = wts.astype(np.float32)
    scale = np.float32(d.acc_scale if split and d.acc_scale != 0 else 1.0)
    bias = _view(d.bias, (d.Cout,), (1,), np.float32) if d.bias else None
    src = d.src
    sv = _pair(src.ptr, src.plane if split else 0, (src.N, src.H, src.W, d.cin), (src.pitch_n, src.pitch_h, src.pitch_w, 1))
    if not split:
        sv = sv.astype(np.float32)
    for a in range(d.nphase_a):
        for s_ in range(d.nsub):
            acc = np.zeros((d.Nt, d.Ht, d.Wt, d.Cout), dtype=np.float64 if split else np.float32)
            for th in range(d.taps_h):
                for tw in range(d.taps_w):
                    hh = np.arange(d.Ht)[:, None] + d.dh0 + a + th
                    ww = np.arange(d.Wt)[None, :] + d.dw0 + s_ + tw
                    inb = (hh >= 0) & (hh < src.H) & (ww >= 0) & (ww < src.W)
                    g = sv[:, np.clip(hh, 0, src.H - 1), np.clip(ww, 0, src.W - 1), :] * inb[None, :, :, None]
                    k0 = (th * d.taps_w + tw) * d.cin
                    wseg = wts[(a * d.nsub + s_) * d.Cout:(a * d.nsub + s_ + 1) * d.Cout, k0:k0 + d.cin]
                    acc += np.tensordot(g[:d.Nt], wseg, axes=([3], [1]))
            acc = acc.astype(np.float32) * scale
            if bias is not None:
                acc += bias
            if d.relu:
                acc = np.maximum(acc, 0)
            if d.mode == 0:
                base = d.out + 2 * (a * d.out_pitch_h + s_ * d.out_pitch_w)
                ov = _view(base, (d.Nt, d.Ht, d.Wt, d.Cout), (d.out_pitch_n, d.out_sy * d.out_pitch_h, d.out_sx * d.out_pitch_w, 1), writable=True)
                ov[...] = acc.astype(np.float16)
            else:
                hw = _view(d.head_w, (d.head_classes, 32), (32, 1), np.float32)
                hb = _view(d.head_b, (d.head_classes,), (1,), np.float32)
                logits = np.tensordot(acc, hw, axes=([3], [1])) + hb
                ov = _view(d.head_out, (d.Nt, d.head_classes, d.Ht, d.Wt), (d.head_classes * d.Ht * d.Wt, d.Ht * d.Wt, d.Wt, 1), np.float32, writable=True)
                ov[...] = np.transpose(logits, (0, 3, 1, 2))


def run_engine(engine, x):
    """Execute a plan_only UNetEngine (CPU buffers) op by op; returns fp32 NCHW logits (torch)."""
    run_engine_ops(engine, engine.ops, x)
    return engine.logits.clone()


def run_engine_ops(engine, ops, x):
    """Execute `ops` (entries of engine.ops) of a plan_only UNetEngine; x: fp32 NCHW normalised input (CPU), read by the pre-pass."""
    import torch
    import torch.nn.functional as F

    assert engine.plan_only and engine.device.type == "cpu"
    strict = getattr(engine, "strict", False)
    for op in ops:
        if op[0] == "prepass":
            engine.s2d.copy_(prepass_s2d_split_cpu(x) if strict else prepass_s2d_cpu(x))
        elif op[0] == "maxpool":
            _, src, dst, n, h, w, c, k, s, p = op
            if strict:
                v = (src[0].float() + src[1].float()).reshape(n, h, w, c).permute(0, 3, 1, 2)
                y = F.max_pool2d(v, kernel_size=k, stride=s, padding=p).permute(0, 2, 3, 1)
                hi = y.half()
                dst.copy_(torch.stack([hi, (y - hi.float()).half()]).reshape(dst.shape))
            else:
                y = F.max_pool2d(src.float().reshape(n, h, w, c).permute(0, 3, 1, 2), kernel_size=k, stride=s, padding=p)
                dst.copy_(y.permute(0, 2, 3, 1).half())
        elif hasattr(op[1].desc, "taps_h"):
            run_rowdesc(op[1].desc)
        else:
            run_desc(op[1].desc)


# --------------------------------------------------------------------------------------------------
# training plan emulation (robosat_b200/train_engine.py op lists on CPU buffers)
# --------------------------------------------------------------------------------------------------
def _gather_segment(d, seg, phase, dtype=np.float32):
    """A operand of one segment for all tile-space pixels: [Nt, Ht, Wt, 64*cblocks] of `dtype` (zero outside the view)"""
    pa, pb = phase >> 1, phase & 1
    src = d.srcs[seg.src]
    width = seg.cblocks * 64
    sv = _view(src.ptr, (src.N, src.H, src.W, min(width, src.C)), (src.pitch_n, src.pitch_h, src.pitch_w, 1))
    return _gather(sv, src, seg.dh + pa, seg.dw + pb, d.Nt, d.Ht, d.Wt, width).astype(dtype)


def run_wgrad(d, dy_ptr, dw, f64=False):
    """dw[phase*Cout + co][k] = sum_pixels dy_phase[p][co] * A_segment(k)[p]  (what rsb_wgrad_run accumulates); dw: torch fp32.
    f64=True: nothing is written; returns float64 (gradient, same contraction over |dy|*|A|), both [phases*Cout, K]."""
    K = 64 * sum(d.segs[i].cblocks for i in range(d.nseg))
    dt = np.float64 if f64 else np.float32
    if f64:
        out, mag = np.zeros((d.phases * d.Cout, K)), np.zeros((d.phases * d.Cout, K))
    else:
        out = dw.numpy().reshape(d.phases * d.Cout, K)
        out[...] = 0
    for phase in range(d.phases):
        pa, pb = phase >> 1, phase & 1
        base = dy_ptr + 2 * (pa * d.out_pitch_h + pb * d.out_pitch_w)
        dyv = _view(base, (d.Nt, d.Ht, d.Wt, d.Cout), (d.out_pitch_n, d.out_sy * d.out_pitch_h, d.out_sx * d.out_pitch_w, 1)).astype(dt)
        k0 = 0
        for si in range(d.nseg):
            a = _gather_segment(d, d.segs[si], phase, dt)
            rows = slice(phase * d.Cout, (phase + 1) * d.Cout)
            out[rows, k0:k0 + a.shape[-1]] = np.tensordot(dyv, a, axes=([0, 1, 2], [0, 1, 2]))
            if f64:
                mag[rows, k0:k0 + a.shape[-1]] = np.tensordot(np.abs(dyv), np.abs(a), axes=([0, 1, 2], [0, 1, 2]))
            k0 += a.shape[-1]
    if f64:
        return out, mag


def _band(sv, src, dh, dw, n, h0, h1, Wt, width):
    """A operand of one tap for output rows h0:h1 of image n: [h1 - h0, Wt, width] float64 of the view `sv` [N, H, W, C] shifted
    by (dh, dw), zero outside the view (as _gather)"""
    a = np.zeros((h1 - h0, Wt, width))
    ya, yb = max(h0, -dh), min(h1, src.H - dh)
    xa, xb = max(0, -dw), min(Wt, src.W - dw)
    if n < src.N and ya < yb and xa < xb:
        c = min(width, sv.shape[-1])
        a[ya - h0:yb - h0, xa:xb, :c] = sv[n, ya + dh:yb + dh, xa + dw:xb + dw, :c]
    return a


def run_wgrad_rows(d, dy_ptr, rows, chunk_bytes=64 << 20):
    """rows `rows` (indices into the phases*Cout rows of the packed gradient) of run_wgrad(d, dy_ptr, None, f64=True), all K
    columns, in float64 over all pixels. The A operand is gathered in bands of output rows of at most `chunk_bytes` of float64
    per segment, the bands in parallel. Returns (gradient, magnitude), both [len(rows), K]."""
    rows = np.asarray(rows, dtype=np.int64)
    K = 64 * sum(d.segs[i].cblocks for i in range(d.nseg))
    out, mag = np.zeros((len(rows), K)), np.zeros((len(rows), K))
    band = max(1, min(d.Ht, chunk_bytes // (8 * K * d.Wt)))
    svs = [_view(s.ptr, (s.N, s.H, s.W, s.C), (s.pitch_n, s.pitch_h, s.pitch_w, 1)) for s in (d.srcs[i] for i in range(d.nsrc))]
    for phase in range(d.phases):
        sel = np.nonzero(rows // d.Cout == phase)[0]
        if not sel.size:
            continue
        co = rows[sel] % d.Cout
        pa, pb = phase >> 1, phase & 1
        base = dy_ptr + 2 * (pa * d.out_pitch_h + pb * d.out_pitch_w)
        dyv = _view(base, (d.Nt, d.Ht, d.Wt, d.Cout), (d.out_pitch_n, d.out_sy * d.out_pitch_h, d.out_sx * d.out_pitch_w, 1))

        def part(task):
            n, h0 = task
            h1 = min(d.Ht, h0 + band)
            g = dyv[n, h0:h1][..., co].astype(np.float64).reshape(-1, len(co))  # [pixels, rows]
            ga = np.abs(g)
            o, m = np.zeros((len(co), K)), np.zeros((len(co), K))
            k0 = 0
            for si in range(d.nseg):
                seg = d.segs[si]
                width = seg.cblocks * 64
                a = _band(svs[seg.src], d.srcs[seg.src], seg.dh + pa, seg.dw + pb, n, h0, h1, d.Wt, width).reshape(-1, width)
                o[:, k0:k0 + width] = g.T @ a
                m[:, k0:k0 + width] = ga.T @ np.abs(a)
                k0 += width
            return o, m

        for o, m in pmap(part, [(n, h0) for n in range(d.Nt) for h0 in range(0, d.Ht, band)]):
            out[sel] += o
            mag[sel] += m
    return out, mag


def run_train_ops(eng, ops, x=None, dlogits=None):
    """Replay a UNetTrainEngine op list (plan_only, CPU buffers) with torch / numpy semantics of the C ABI entry points."""
    import torch
    import torch.nn.functional as F

    P = eng.params
    for op in ops:
        k = op[0]
        if k == "conv":
            run_desc(op[1].desc)
        elif k == "pack_all":
            for wname, m, dst, _c, _o in eng.pack_list:
                src = P[wname].reshape(-1)
                mm = m.long()
                vals = torch.where(mm >= 0, src[mm.clamp_min(0)], torch.zeros(()))
                dst.copy_(vals.sum(1).half())
        elif k == "unpack_all":
            for dwp, m, wname, _c, _o in eng.unpack_list:
                flat = eng._grad(wname).reshape(-1)
                mm = m.long()
                for j in range(4):
                    sel = mm[:, j] >= 0
                    flat.index_add_(0, mm[sel, j], dwp[sel] / eng.loss_scale)
        elif k == "bn_stats":
            b = op[1]
            z = b.z.reshape(b.M, b.C).double()
            b.sums[:b.C] = z.sum(0)
            b.sums[b.C:2 * b.C] = (z * z).sum(0)
        elif k == "bn_finalize":
            b = op[1]
            pf = b.prefix
            mean = b.sums[:b.C] / b.M
            var = (b.sums[b.C:2 * b.C] / b.M - mean * mean).clamp_min(0)
            invstd = (1.0 / torch.sqrt(var + eng_eps())).float()
            b.mean.copy_(mean.float())
            b.invstd.copy_(invstd)
            b.scale.copy_(P[pf + ".weight"] * invstd)
            b.shift.copy_(P[pf + ".bias"] - mean.float() * b.scale)
            P[pf + ".running_mean"].mul_(0.9).add_(0.1 * mean.float())
            P[pf + ".running_var"].mul_(0.9).add_(0.1 * (var * b.M / (b.M - 1)).float())
            P[pf + ".num_batches_tracked"].add_(1)
            b.sums.zero_()  # the chained kernels leave their accumulators cleared for the next call
        elif k == "bn_apply":
            _, b, res, y, relu = op
            o = b.z.reshape(b.M, b.C).float() * b.scale + b.shift
            if res is not None:
                o = o + res.reshape(b.M, b.C).float()
            y.copy_((F.relu(o) if relu else o).half().reshape(y.shape))
        elif k == "bn_bwd":
            _, b, dy, y, dz, g_out = op
            pf = b.prefix
            g = dy.reshape(b.M, b.C).float()
            if y is not None:
                g = g * (y.reshape(b.M, b.C).float() > 0)
            zhat = (b.z.reshape(b.M, b.C).float() - b.mean) * b.invstd
            s0 = g.double().sum(0)
            s1 = (g * zhat).double().sum(0)
            if g_out is not None:
                g_out.copy_(g.half().reshape(g_out.shape))
            o = P[pf + ".weight"] * b.invstd * (g - (s0 / b.M).float() - zhat * (s1 / b.M).float())
            dz.copy_(o.half().reshape(dz.shape))
            eng._grad(pf + ".weight").copy_((s1 / eng.loss_scale).float())
            eng._grad(pf + ".bias").copy_((s0 / eng.loss_scale).float())
        elif k == "relu_bwd":
            _, a, b2, y, out = op
            g = a.float()
            if b2 is not None:
                g = g + b2.float()
            if y is not None:
                g = g * (y.float() > 0)
            out.copy_(g.half())
        elif k == "maxpool":
            _, src, dst, n, h, w, c, kk, s, p = op
            yy = F.max_pool2d(src.float().reshape(n, h, w, c).permute(0, 3, 1, 2), kk, s, p)
            dst.copy_(yy.permute(0, 2, 3, 1).half())
        elif k == "maxpool_bwd":
            _, xx, dy, dx, n, h, w, c, kk, s, p = op
            xin = xx.float().reshape(n, h, w, c).permute(0, 3, 1, 2).clone().requires_grad_(True)
            yy = F.max_pool2d(xin, kk, s, p)
            yy.backward(dy.float().reshape(n, yy.shape[2], yy.shape[3], c).permute(0, 3, 1, 2))
            dx.copy_(xin.grad.permute(0, 2, 3, 1).half())
        elif k == "wgrad":
            _, u, dy = op
            run_wgrad(u.desc, dy.data_ptr() + 2 * u.out_offset, u.dw_packed)
        elif k == "prepass":
            eng.s2d.copy_(prepass_s2d_cpu(x))
        elif k == "final_fwd":
            _, y5, logits = op
            yv = y5.float().permute(0, 3, 1, 2)
            logits.copy_(F.conv2d(yv, P["final.weight"], P["final.bias"]))
        elif k == "final_bwd":
            _, y5, d_y5 = op
            w = P["final.weight"].reshape(eng.C, 32)
            d = torch.einsum("nkhw,kc->nhwc", dlogits, w) * eng.loss_scale
            d_y5.copy_(d.half())
            eng._grad("final.weight").copy_(torch.einsum("nkhw,nhwc->kc", dlogits, y5.float()).reshape(eng.C, 32, 1, 1))
            eng._grad("final.bias").copy_(dlogits.sum((0, 2, 3)))
        elif k == "zero_grads":
            eng._grad("final.bias")
            eng._grads_flat.zero_()
        else:
            raise AssertionError(k)


def eng_eps():
    return 1e-5


def stitch_halo_cpu(store, table, size, overlap):
    """numpy restatement of csrc/rsb_elementwise.cu:stitch_halo_kernel (same index arithmetic), for the CPU suite."""
    import numpy as np

    B = table.shape[0]
    F = size + 2 * overlap
    out = np.zeros((B, F, F, 3), dtype=np.uint8)
    for b in range(B):
        for Y in range(F):
            dy = -1 if Y < overlap else (0 if Y < overlap + size else 1)
            sy = Y - overlap - dy * size
            for dx, (x0, x1) in ((-1, (0, overlap)), (0, (overlap, overlap + size)), (1, (overlap + size, F))):
                if x1 <= x0:
                    continue
                slot = int(table[b, (dy + 1) * 3 + (dx + 1)])
                if slot < 0:
                    continue
                out[b, Y, x0:x1] = store[slot, sy, x0 - overlap - dx * size:x1 - overlap - dx * size]
    return out
