"""Lockstep check of the inference plan (robosat_b200/engine.py `UNetEngine`): every launch of `eng.ops` against a float64
replay of that one op, computed from exactly the inputs the executor under test had.

Test infrastructure only; the machinery (buffer pairing, stray-write check, comparison, teacher forcing, report) is
tests/lockstep.py's `Harness`. The executor under test (`dut`: a GPU engine, or a plan_only CPU engine driven by the
emulator) and a plan_only CPU `twin` of the same precision, H, W and classes build their buffers (`_keep`) and `ops` in the
same order: buffers pair by position, ops pair by position. The shared K-chunk scratch (`_scratch_buf`) is not paired: its
size differs between the two modes and its layout is the kernel's business. Per op:

  1. the float64 reference is computed from the twin's buffers (tests/emulate.py, `sink` mode);
  2. the executor runs the op (`UNetEngine.run_ops`, the loop body of `forward`);
  3. no stray writes: every paired buffer of the executor is bit-compared, on its device, with a snapshot taken after the
     previous op; only the elements the op is meant to write may differ (this includes the zero pad columns of `s2d` and
     of the W-padded `dec4`, which later convolutions read as padding);
  4. the outputs are compared elementwise (strict precision: the value hi + lo of each fp16 pair), then copied into the twin.

Batch subset: a batch-32 plan is replayed on a few of its images (`images`: e.g. the first, one in the middle, and the last,
where a ragged TN tile ends) by a twin built at that batch. A buffer whose shape differs only on the batch axis (axis 0, or
axis 1 behind the strict (hi, lo) plane axis; logits [N, C, H, W]) pairs by those images; same-shape buffers (weights,
biases, the head) pair whole. The stray-write check still covers the executor's whole buffers: an op may write the
positions its twin writes, in every image. The twin's plan (tile widths, K chunks) may differ from the executor's, which
does not change a float64 reference; the bounds below take the chain lengths from the EXECUTOR's descriptor.

Weights: the twin takes the executor's packed weights and acc_scale. Whether its own packing (host float64 -> fp32 -> fp16
in torch, where the executor's was prepared on its device) was bit-identical is counted and reported, not required.

Tolerances, elementwise. u = 2^-24; a tensor-core adder is not guaranteed to round to nearest, so every fp32 accumulator
addition is charged 2u = 2^-23 of the running magnitude, and a chain of m MMAs (each adds 16 exact fp16 products, aligned to
the largest and truncated) errs by at most 2^-23 (m + 17) times the sum of the magnitudes of its terms (tests/lockstep.py,
wgrad). The float64 replay (emulate._F64Acc) gives, all times acc_scale (a power of two: exact):
  A    = sum (|a_hi| + |a_lo|)(|w_hi| + |w_lo|), at least the magnitude of the three products the kernel accumulates;
  A_ll = sum |a_lo||w_lo|, the product it omits (an error of at most A_ll, exactly);
  A_hh = sum |a_hi||w_hi| (main chain of the N-concatenated schedule), A_x = A - A_hh - A_ll (its cross chain);
  M    = A + |bias| + |residual|.
kc = K blocks per chunk (the executor's `kchunk`, else all K blocks), n = number of chunks (DESIGN.md 3.1, strict precision).

  strict conv, SPLIT = 1   e = 2^-23 (12 kc + 17) A + n u A + A_ll + 2u M
  (block_n >= 128)         three MMAs per k16 step (A_hi W_lo, A_lo W_hi, A_hi W_hi) = 12 per K block on one accumulator;
                           chunk results are added with round-to-nearest fp32 adds (<= one per chunk, each <= u A);
                           fma(acc, 2^-e, bias) and + residual (hi + lo is exact in fp32) round once each: 2u M.
  strict conv, SPLIT = 2   e = 2^-23 (4 kc + 17) A_hh + 2^-23 (8 kc + 17) A_x + 2 n u A + A_ll + 2u M
  (block_n <= 64)          main chain A_hi W_hi (4 MMAs per K block), cross chain A_hi W_lo + A_lo W_hi (8), bounded
                           separately; main + cross and the chunk sum are two round-to-nearest fp32 adds per chunk.
  fp16 pair store          tol = e + 2^-22 (|ref| + e) + 2^-25: hi = half(v) and v - hi are exact, lo = half(v - hi) rounds
                           by half an fp16 ulp of |v - hi| <= 2^-11 |v|, i.e. <= 2^-22 |v|, or 2^-25 below the normal range.
  strict line-buffer head  the SPLIT = 2 form with the line-buffer schedule: K = 9 taps x 32 channels = 18 k16 steps, main chain
                           18 MMAs, cross chain 36, one chunk.
  fast conv, line buffer   ulp16(ref) + K 2^-24 M, as in training: (K/16 + 17) 2^-23 A + 2u M <= K 2^-24 M for K >= 64, and the
                           fp16 rounding of the result (half an ulp, with room for values next to a rounding boundary).
  head mode (dec5 + final) the conv's error e_c (the forms above without the pair store; the bias add is covered by the
                           2 n u A term, |bias| being added to A) reaches the logits through ReLU (1-Lipschitz) and the fp32
                           weights of `final`: sum_c |w_c| e_c, plus 34 u (sum_c |w_c y_c| + |b|) for the 32 fp32 fmas, the two
                           shuffle adds and the bias (no fp16 rounding of the intermediate). Fast: e_c = K 2^-24 A_c.
  prepass (u8 or fp32 input, both precisions), max pools (split: max of the exact pair values): exact.
"""

import numpy as np
import torch
import torch.nn.functional as F

import emulate
import lockstep
from lockstep import U, _Write, _bits, _view, ulp16

P22, P23, P25 = 2.0 ** -22, 2.0 ** -23, 2.0 ** -25


class EmulatorExecutor:
    """Runs ops with the CPU emulator on a plan_only engine."""

    def __init__(self, eng):
        assert eng.plan_only
        self.eng = eng

    def run(self, op, x):
        emulate.run_engine_ops(self.eng, [op], x)

    def sync(self):
        pass


class GpuExecutor:
    """Runs ops launch by launch through UNetEngine.run_ops (forward() is run_ops over the whole list)."""

    def __init__(self, eng):
        self.eng = eng

    def run(self, op, x):
        self.eng.run_ops([op], x)

    def sync(self):
        torch.cuda.synchronize()


def schedule(dd):
    """(main chain MMAs, cross chain MMAs (0: a single chain), chunks) of the executor's strict descriptor `dd`"""
    if hasattr(dd, "taps_h"):  # line buffer: one chain per output over taps x channels, N-concatenated
        steps = dd.taps_h * dd.taps_w * dd.cin // 16
        return steps, 2 * steps, 1
    kb = sum(dd.segs[j].cblocks for j in range(dd.nseg))
    kc = dd.kchunk if 0 < dd.kchunk < kb else kb
    n = -(-kb // kc)
    if dd.mode == 1 or dd.block_n <= 64:
        return 4 * kc, 8 * kc, n
    return 12 * kc, 0, n


def strict_acc_bound(dd, parts):
    """e of the module docstring without the 2u M epilogue term (parts: magnitudes of emulate._F64Acc, possibly carried
    through the head)"""
    m_main, m_cross, n = schedule(dd)
    A, ll = parts["dot"], parts["lolo"]
    if m_cross:
        hh = parts["hihi"]
        x = np.maximum(A - hh - ll, 0.0)
        return P23 * (m_main + 17) * hh + P23 * (m_cross + 17) * x + 2 * n * U * A + ll
    return P23 * (m_main + 17) * A + n * U * A + ll


def conv_tol(dd, strict, val, mag, parts):
    """elementwise tolerance of one convolution's outputs (the forms of the module docstring) from the float64 replay's
    value, magnitude and parts (emulate.run_desc / run_rowdesc `sink`); the chain lengths come from descriptor `dd`"""
    row = hasattr(dd, "taps_h")
    K = dd.taps_h * dd.taps_w * dd.cin if row else 64 * sum(dd.segs[j].cblocks for j in range(dd.nseg))
    if strict:
        e = strict_acc_bound(dd, parts)
        if dd.mode == 0:
            e = e + 2 * U * mag
            return e + P22 * (np.abs(val) + e) + P25
        return e + 34 * U * mag
    return ulp16(val) + K * U * mag if dd.mode == 0 else K * U * parts["dot"] + 34 * U * mag


def op_kind(dd, strict):
    """report tag of a convolution from the executor's descriptor"""
    if hasattr(dd, "taps_h"):
        return "line-buffer head" if dd.mode == 1 else "line buffer"
    if dd.mode == 1:
        return "conv head"
    if not strict:
        return "conv"
    m_main, m_cross, n = schedule(dd)
    return "conv split=%d%s" % (2 if m_cross else 1, " K-chunked" if n > 1 else "")


class PredictLockstep(lockstep.Harness):
    def __init__(self, executor, twin, images=None):
        """executor: EmulatorExecutor / GpuExecutor of the engine under test; twin: plan_only CPU UNetEngine of the same
        precision, H, W and classes, built at batch len(images); images: the executor's images the twin replays (all by default)"""
        E, T = executor.eng, twin
        self.dut, self.tw = executor, twin
        assert T.plan_only and T.device.type == "cpu"
        assert (T.precision, T.H, T.W, T.C) == (E.precision, E.H, E.W, E.C), "the twin must share precision, H, W and classes"
        self.strict = T.strict
        self.sel = list(range(E.N)) if images is None else [int(i) for i in images]
        assert len(self.sel) == T.N and all(0 <= i < E.N for i in self.sel)
        assert [o[0] for o in E.ops] == [o[0] for o in T.ops], "the two engines built different op lists"
        assert [o[1].name for o in E.ops if o[0] == "conv"] == [o[1].name for o in T.ops if o[0] == "conv"]
        self.db, self.tb = list(E._keep), list(T._keep)
        assert len(self.db) == len(self.tb), "the two engines built different buffer lists"
        skip = {i for i, t in enumerate(self.tb) if t is getattr(T, "_scratch_buf", None)}
        assert skip == {i for i, t in enumerate(self.db) if t is getattr(E, "_scratch_buf", None)}
        self.bmap = {}
        for i, (a, b) in enumerate(zip(self.db, self.tb)):
            if i in skip:
                continue
            assert a.dtype == b.dtype and a.dim() == b.dim(), "buffer %d pairs %s with %s" % (i, a.dtype, b.dtype)
            if a.shape == b.shape:
                continue
            axes = [k for k in range(a.dim()) if a.shape[k] != b.shape[k]]
            ax = axes[0]
            assert axes == [ax] and (ax == 0 or (ax == 1 and self.strict and a.shape[0] == 2)) and a.shape[ax] == E.N and b.shape[ax] == T.N, \
                "buffer %d pairs %s with %s: not a batch subset" % (i, tuple(a.shape), tuple(b.shape))
            self.bmap[i] = (ax, int(np.prod(b.shape[ax + 1:])))
        self._index()
        self.labels = {}
        for name, (t, _) in T.feats.items():
            self._label(t, name)
        for name in ("s2d", "logits"):
            self._label(getattr(T, name), name)
        # the twin computes with the executor's weights (and acc_scale); count whether its own packing was the same
        wts = set()
        for (_, od), (_, ot) in ((o, p) for o, p in zip(E.ops, T.ops) if o[0] == "conv"):
            ot.desc.acc_scale = od.desc.acc_scale
            for f in ("weights", "bias", "head_w", "head_b"):
                if getattr(ot.desc, f, None):
                    wts.add(self._locate(getattr(ot.desc, f))[0])
        self.weights_identical = (sum(bool(torch.equal(_bits(self.tb[i]), _bits(self.db[i].cpu()))) for i in wts), len(wts))
        self.tracked = [i for i in range(len(self.tb)) if i not in skip and self.tb[i].numel()]
        self._sel_dev = torch.tensor(self.sel, dtype=torch.long, device=E.device)
        for i in self.tracked:
            self.tb[i].copy_(self._pull(i))
        self.snap = {i: self.db[i].clone() for i in self.tracked}
        self.stats = {}
        self.failures = []
        self.checked = set()

    # ------------------------------------------------------------------ batch subset
    def _remap(self, b, off):
        """element offset in twin buffer b -> the same position of the executor's buffer, image sel[0] -> image 0 base"""
        _, inner = self.bmap[b]
        outer, rem = divmod(off, inner * self.tw.N)
        img, rest = divmod(rem, inner)
        assert img == 0, "an output view must start at the first image"
        return outer * inner * self.dut.eng.N + rest

    def _batch_dim(self, b, shape, strides):
        _, inner = self.bmap[b]
        dims = [k for k in range(len(shape)) if strides[k] == inner and shape[k] == self.tw.N]
        assert dims, "output view without a batch axis"
        return dims[0]

    def _full(self, b, off, shape, strides):
        d = self._batch_dim(b, shape, strides)
        full = list(shape)
        full[d] = self.dut.eng.N
        return d, self._remap(b, off), full

    def _dut_view(self, b, off, shape, strides):
        if b not in self.bmap:
            return super()._dut_view(b, off, shape, strides)
        d, doff, full = self._full(b, off, shape, strides)
        return _view(self.db[b], doff, full, strides).index_select(d, self._sel_dev)

    def _dut_mark(self, mask, b, off, shape, strides):
        if b not in self.bmap:
            return super()._dut_mark(mask, b, off, shape, strides)
        _, doff, full = self._full(b, off, shape, strides)
        torch.as_strided(mask, full, strides, doff).fill_(True)

    def _pull(self, b):
        if b not in self.bmap:
            return self.db[b].cpu()
        return self.db[b].index_select(self.bmap[b][0], self._sel_dev).cpu()

    # ------------------------------------------------------------------ driver
    def run(self, x, dut_x=None, raise_on_fail=True):
        """x: fp32 NCHW normalised input of the twin's images (CPU); dut_x: the executor's whole input (fp32 NCHW or uint8
        NHWC, on its device), by default x"""
        self.raise_on_fail = raise_on_fail
        dx = x if dut_x is None else dut_x
        for i, (od, ot) in enumerate(zip(self.dut.eng.ops, self.tw.ops)):
            writes = self._reference(od, ot, x)
            self.dut.run(od, dx)
            self.dut.sync()
            self._check_stray("predict", i, ot, writes)
            for w in writes:
                self._compare("predict", i, ot, w)
            self.checked.add(i)
        assert len(self.checked) == len(self.tw.ops)
        return self.failures

    def _name(self, ot):
        if ot[0] == "conv":
            return ot[1].name
        if ot[0] == "maxpool":
            return self._blabel(self._locate(ot[2].data_ptr())[0])
        return ot[0]

    def _table_extra(self):
        n, m = self.weights_identical
        return ["twin's own packed weights bit-identical to the executor's: %d of %d buffers" % (n, m),
                "ops checked: %d of %d" % (len(self.checked), len(self.tw.ops))]

    # ------------------------------------------------------------------ float64 references of single ops
    def _pair_write(self, label, t, ref, tag):
        """an exact output covering the whole of twin activation `t` (both planes in strict precision)"""
        if not self.strict:
            return self._write_t(label, t, ref, 0.0, tag)
        hi = t[0]
        i, off = self._locate(hi.data_ptr())
        return _Write(label, i, off, hi.shape, hi.stride(), np.asarray(ref).reshape(hi.shape), 0.0, tag, hi.numel())

    def _value(self, t):
        """float64 value of a twin activation (hi + lo in strict precision)"""
        return (t[0].double() + t[1].double()) if self.strict else t.double()

    def _reference(self, od, ot, x):
        if ot[0] == "prepass":
            s2d = emulate.prepass_s2d_split_cpu(x) if self.strict else emulate.prepass_s2d_cpu(x)
            return [self._pair_write("s2d", self.tw.s2d, self._value(s2d).numpy(), "prepass")]
        if ot[0] == "maxpool":
            _, src, dst, n, h, w, c, k, s, p = ot
            v = self._value(src).reshape(n, h, w, c).permute(0, 3, 1, 2)
            y = F.max_pool2d(v, k, s, p).permute(0, 2, 3, 1)
            return [self._pair_write("maxpool out", dst, y.numpy(), "maxpool")]
        return self._ref_conv(od[1].desc, ot[1])

    def _ref_conv(self, dd, op):
        td = op.desc
        row = hasattr(td, "taps_h")
        tag = op_kind(dd, self.strict)
        writes = []

        def sink(ptr, shape, strides, val, mag, parts, plane):
            idx, off = self._locate(ptr)
            tol = conv_tol(dd, self.strict, val, mag, parts)
            writes.append(_Write("%s out (%s)" % (op.name, self._blabel(idx)), idx, off, shape, strides, val, tol, tag, plane))

        (emulate.run_rowdesc if row else emulate.run_desc)(td, sink=sink)
        return writes


def make_pair(sd, C, N, H, W, precision, device, images=None, plan_overrides=None):
    """(dut engine, plan_only CPU twin at batch len(images)) from one state dict"""
    from robosat_b200.engine import UNetEngine

    cpu = torch.device(device).type == "cpu"
    dut = UNetEngine(sd, C, N, H, W, device=device, plan_only=cpu, precision=precision, plan_overrides=plan_overrides)
    k = N if images is None else len(images)
    twin = UNetEngine(sd, C, k, H, W, device="cpu", plan_only=True, precision=precision)
    return dut, twin
