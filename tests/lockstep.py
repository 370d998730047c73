"""Lockstep check of the training plan (robosat_b200/train_engine.py): every op of `fwd_ops` / `bwd_ops` against a float64
reference of that one op, computed from exactly the inputs the executor under test had.

Test infrastructure only. Two engines with the same configuration build their buffers and op lists in the same order:
the one under test (`dut`: the GPU engine, or a plan_only CPU engine driven by the emulator) and a plan_only CPU `twin`.
Buffers pair by position (`_keep`, then the parameters, then the flat gradient buffer), ops pair by position. Per op:

  1. the float64 reference of the op is computed from the twin's buffers, which hold the executor's current state;
  2. the executor runs the op (bn_stats together with its bn_finalize: the GPU folds the finalize into the stats launch);
  3. no stray writes: every tracked buffer is bit-compared, on the executor's device, with a snapshot taken after the
     previous op; only the elements the op is meant to write may differ (this includes the zero pad columns of `s2d`
     and of the W-padded `dec4` / `d_dec4`, which later convolutions read as padding);
  4. the op's outputs are compared elementwise with the reference, then copied into the twin (teacher forcing), so the
     next op starts from identical inputs on both sides and a ReLU mask or max-pool argmax can never differ between them.

Not compared (per-op scratch whose layout is the executor's business): BatchNorm accumulators `Unit.sums` (except that
the BatchNorm ops must leave their slots and arrival counter zero), the conv-statistics partials (their column sums are
checked against the convolution's own output instead), `final_acc`, and the int32 weight-packing maps (constants).

Tolerances, elementwise. u = 2^-24 is the fp32 unit roundoff; a tensor-core adder is not guaranteed to round to nearest,
so every fp32 accumulator addition is charged 2u = 2^-23 of the running magnitude. ulp16(r) is the fp16 spacing at |r|
(2^-24 below the normal range), which bounds the final fp16 rounding (half an ulp) with room for the fp32 error of values
that sit next to a rounding boundary. A is the float64 sum of the magnitudes of the terms of the same expression.

  conv        fp16 out     ulp16(ref) + K * 2^-24 * A, A = sum_k |x_k| |w_k| (+ |residual|). The wgmma chain adds K/16
                           partial products of 16 terms each into an fp32 accumulator (bound as for wgrad below):
                           (K/16 + 17) * 2^-23 * A <= K * 2^-24 * A for K >= 64.
  conv stats  partials     sum of the partial rows vs float64 column sums / sums of squares of the kernel's own fp16 z:
                           gamma_31 of sum |z| / sum z^2 (each partial adds 32 rows in fp32: 31 roundings).
  wgrad       fp32 dw      2^-23 * (P/16 + P/64 + 17) * A, A = sum_p |dy_p| |x_p|: P/16 accumulator additions of 16-pixel MMAs,
                           at most P/64 slice partials added afterwards (a slice holds at least one 64-pixel tile), and the
                           sum inside each MMA: its 16 products are aligned to the largest one and truncated, so each can lose
                           2^-23 of that block maximum, at most 16 * 2^-23 * A over all blocks (+1 for the normalisation).
                           Layers with fewer than 16 pixels per phase (center, dec0) need that term: measured errors there
                           reach 2-4 fp32 ulps of a result made of a handful of same-sign products.
  bn_stats    mean etc.    from the sums' error e_s = e_sum(partial_reduce launch) relative to sum |z| (tests/train_launch.py derives
                           it from the launch geometry: the 32-row conv-stats partials, the rows each thread folds, the shared-
                           memory fold, then fp64): d_mean = e_s E|z| + u |mean|, d_var = e_s E[z^2] + 2 |mean| d_mean,
                           d_invstd = invstd (d_var / 2 (var + eps) + 2u), d_scale = |gamma| d_invstd + u |scale|,
                           d_shift = |mean| d_scale + |scale| d_mean + 2u (|beta| + |mean scale|); running stats: momentum
                           times those plus 4u of their magnitudes; num_batches_tracked exact.
  bn_apply    fp16 y       ulp16(ref) + 2^-23 (|z scale| + |shift| + |res|): one fma and one add in fp32, then fp16.
  bn_bwd      dz           ulp16(ref) + 2^-22 (|A g| + |B z| + |D|) + |A| (d_s0 + |zhat| d_s1) / M, with dz = A g + B z + D the
                           kernel's fp32 form, d_s0 = e_s sum |g| and d_s1 = e_s invstd (sum |g z| + |mean| sum |g|),
                           e_s = e_sum(channel_reduce launch)
                           (the kernel forms sum g zhat as (sum g z - mean sum g) invstd);
              g_out        exact (a masked copy);
              dgamma/dbeta d_s1 / loss_scale + 2u |ref|, d_s0 / loss_scale + 2u |ref|.
  relu_bwd, maxpool, prepass, zero_grads: exact (one fp32 add of two fp16 values rounded once, a max, a copy, zeros).
  maxpool_bwd fp16 dx      ulp16(ref): at most ceil(k/s)^2 exact fp16 values summed in fp32, rounded once.
  pack_all    fp16 packed  exact for single-source layouts (one rounding of the fp32 weight); ulp16(ref) + 2^-22 A for the
                           pre-summed upsample taps (<= 3 fp32 additions, then fp16).
  final_fwd   fp32 logits  34 u A (32 fmas + the bias, A = sum |w y| + |b|).
  final_bwd   fp16 dy5     ulp16(ref) + (C + 2) u A; dW, db: e_s A + 2u |ref|, e_s = e_sum(final_bwd_dw launch) (fp32
                           per-thread partials and a warp shuffle tree, fp64 totals).
  unpack_all  fp32 grads   2^-22 A + 2u |ref| (<= 4 fp32 additions and the 1/loss_scale product).

Sampled mode (Lockstep(..., sample_above=n), for the shapes the benchmark trains at): a convolution (forward or .dgrad) with more
than n output pixels is compared at sampled pixels only -- for every image the whole first, last (ragged) and one seeded random
tile box of the kernel's own tiling (TW x TH x TN from the descriptor), the four corners and 256 seeded random pixels, all Cout
channels, every phase -- with emulate.conv_f64_at; a weight gradient of such a layer at rows 0, 63, 64, 127, 128, the last and
4 seeded random rows, all K columns, with emulate.run_wgrad_rows. The stray-write check and the teacher forcing still cover
the op's whole output, and every other op is checked element by element in chunks of at most `chunk` elements, so the host
memory of the references stays bounded. The chunks run on a thread pool (emulate.pmap).

The stray-write snapshot lives on the executor's device, or, with snapshot="host", one host copy per buffer: each op then
pulls every tracked buffer back to compare it, slower but without a second copy of the engine on the device.
"""

import bisect

import numpy as np
import torch
import torch.nn.functional as F

import emulate
import train_launch

U = 2.0 ** -24
E_CONV_STATS = train_launch.conv_stats_partial()  # the conv epilogue's 32-row fp32 partial sums
BN_EPS = 1e-5
BN_MOMENTUM = 0.1


class LockstepError(AssertionError):
    def __init__(self, msg, index, which, kind, name, buffer):
        super().__init__(msg)
        self.index, self.which, self.kind, self.name, self.buffer = index, which, kind, name, buffer


def ulp16(x):
    """spacing of fp16 numbers at |x| (the subnormal spacing 2^-24 below 2^-14)"""
    m = np.maximum(np.abs(np.asarray(x, dtype=np.float64)), 2.0 ** -14)
    p2 = (m.view(np.int64) & np.int64(0x7FF0000000000000)).view(np.float64)  # 2^floor(log2 m), exactly
    return np.where(np.isnan(m), np.nan, p2 * 2.0 ** -10)


def _f64(t):
    return t.detach().cpu().double().numpy()


class EmulatorExecutor:
    """Runs ops with the CPU emulator on a plan_only engine. Its BatchNorm ops clear their accumulators like the kernels,
    and it is deterministic, but running a weight gradient twice would only repeat the same numpy call."""

    repeat_wgrad = False
    conv_stats = False  # the emulated convolution does not write the BatchNorm partials (its bn_stats reads z)

    def __init__(self, eng):
        assert eng.plan_only
        self.eng = eng

    def run(self, op, x=None, dlogits=None):
        if op[0] == "wgrad":
            # float64 sums rounded once: numpy's float32 GEMM adds a layer4 tile's pixels with more error than the kernel bound allows
            _, u, dy = op
            ref, _ = emulate.run_wgrad(u.desc, dy.data_ptr() + 2 * u.out_offset, None, f64=True)
            u.dw_packed.copy_(torch.from_numpy(ref.reshape(-1)))
            return
        emulate.run_train_ops(self.eng, [op], x=x, dlogits=dlogits)

    def sync(self):
        pass


class GpuExecutor:
    """Runs ops kernel by kernel through UNetTrainEngine._run (graph replay is checked bit-identical elsewhere)."""

    repeat_wgrad = True  # the split-K weight gradient must give the same bits when run twice
    conv_stats = True

    def __init__(self, eng):
        self.eng = eng

    def run(self, op, x=None, dlogits=None):
        self.eng._run([op], x=x, dlogits=dlogits)

    def sync(self):
        torch.cuda.synchronize()


class _Write:
    """an output view (base buffer index, element offset, shape, element strides) with its reference and tolerance.
    plane > 0: the output is an fp16 (hi, lo) pair whose lo plane lies `plane` elements behind the hi plane; the value
    compared with the reference is hi + lo.
    sample: the reference covers only these elements (absolute element offsets into the base buffer, ref's shape).
    fn: the reference is computed lazily, fn(a, b) -> (ref, tol) for rows a:b of the view's first axis, chunk by chunk; fn reads
    the twin before the chunk's outputs are copied into it (an op that writes in place reads only the chunk it writes)."""

    __slots__ = ("label", "idx", "off", "shape", "strides", "ref", "tol", "tag", "plane", "sample", "fn")

    def __init__(self, label, idx, off, shape, strides, ref, tol, tag, plane=0, sample=None, fn=None):
        self.label, self.idx, self.off, self.shape, self.strides = label, idx, off, tuple(shape), tuple(strides)
        self.ref, self.tol, self.tag, self.plane, self.sample, self.fn = ref, tol, tag, plane, sample, fn

    def offsets(self):
        return (self.off, self.off + self.plane) if self.plane else (self.off,)


def _bases(eng):
    return list(eng._keep) + list(eng.params.values()) + [eng._grads_flat]


def _view(base, off, shape, strides):
    flat = base.reshape(-1)
    return torch.as_strided(flat, shape, strides, flat.storage_offset() + off)


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()]) if t.dtype.is_floating_point else t


def _same(a, b):
    """bit equality of two tensors of one shape and dtype (on the CPU as 8-byte words: torch.equal there is ~10x slower)"""
    if a.device.type != "cpu":
        return torch.equal(_bits(a), _bits(b))
    x, y = a.reshape(-1).view(torch.uint8).numpy(), b.reshape(-1).view(torch.uint8).numpy()
    n = x.size - x.size % 8
    return np.array_equal(x[:n].view(np.int64), y[:n].view(np.int64)) and np.array_equal(x[n:], y[n:])


def _judge(tag, got, ref, tol, where):
    """elementwise check of one piece of an output. Returns (worst err/tol, or the worst |err| of an exact check; exact?;
    elements out of tolerance; (err/tol, position, got, ref, tol) of the worst of them or None; bn_apply outputs one fp16 ulp
    from the correctly rounded value; bn_apply elements)"""
    tol = np.broadcast_to(np.asarray(tol, dtype=np.float64), ref.shape)
    err = np.abs(got - ref)
    nan = np.isnan(err)
    if nan.any():  # NaN where both are NaN is a match, any other NaN an unbounded error
        err = np.where(nan, np.where(np.isnan(got) & np.isnan(ref), 0.0, np.inf), err)
    exact = not np.any(tol)
    if exact:
        ratio = float(err.max()) if err.size else 0.0
        bad = err > 0
    else:
        q = np.divide(err, tol, out=np.where(err > 0, np.inf, 0.0), where=tol > 0)
        ratio = float(q.max()) if q.size else 0.0
        bad = err > tol
    flips = elems = 0
    if tag == "bn_apply":
        elems = got.size
        flips = int(np.count_nonzero(got != ref.astype(np.float16).astype(np.float64)))
    nbad, worst = int(np.count_nonzero(bad)), None
    if nbad:
        score = np.where(bad, err / np.maximum(tol, 1e-300), -1)
        k = int(np.argmax(score))
        worst = (float(score.reshape(-1)[k]), where(k), float(got.reshape(-1)[k]), float(ref.reshape(-1)[k]), float(tol.reshape(-1)[k]))
    return ratio, exact, nbad, worst, flips, elems


class Harness:
    """What the training and the inference lockstep checks share: buffers of the executor under test (`db`) and of the CPU
    twin (`tb`) paired by position, pointer -> (buffer, offset) lookup in the twin, the stray-write check on the executor's
    device, the elementwise comparison with teacher forcing, and the report. The twin's elements map to the executor's
    one to one here; a subclass that replays a subset of the executor's batch overrides _dut_view / _dut_mark / _pull."""

    def _index(self):
        self._order = sorted((t.data_ptr(), i) for i, t in enumerate(self.tb) if t.numel())
        self._starts = [p for p, _ in self._order]

    # ------------------------------------------------------------------ addressing
    def _locate(self, ptr):
        k = bisect.bisect_right(self._starts, ptr) - 1
        assert k >= 0, "pointer outside every buffer"
        p, i = self._order[k]
        t = self.tb[i]
        assert ptr < p + t.numel() * t.element_size(), "pointer outside every buffer"
        assert (ptr - p) % t.element_size() == 0
        return i, (ptr - p) // t.element_size()

    def _label(self, t, name):
        i, off = self._locate(t.data_ptr())
        if off == 0 and t.numel() == self.tb[i].numel():
            self.labels.setdefault(i, name)

    def _blabel(self, i):
        return self.labels.get(i, "buffer#%d %s%s" % (i, self.tb[i].dtype, tuple(self.tb[i].shape)))

    def _write_t(self, label, t, ref, tol, tag):
        """output = the whole of (twin) tensor `t`"""
        i, off = self._locate(t.data_ptr())
        tol = np.asarray(tol)
        return _Write(label, i, off, t.shape, t.stride(), np.asarray(ref).reshape(t.shape), tol.reshape(t.shape) if tol.ndim else tol, tag)

    def _dut_view(self, b, off, shape, strides):
        """the executor's elements that twin view (buffer b, off, shape, strides) stands for, same shape"""
        return _view(self.db[b], off, shape, strides)

    def _dut_mark(self, mask, b, off, shape, strides):
        """mark in `mask` (flat bool, executor buffer b's size and device) every element the op may write for that twin view"""
        torch.as_strided(mask, shape, strides, off).fill_(True)

    def _pull(self, b):
        """executor buffer b as the twin holds it, on the CPU"""
        return self.db[b].cpu()

    def _fail(self, which, i, ot, buffer, msg):
        text = "%s op %d (%s %s), buffer %s: %s" % (which, i, ot[0], self._name(ot), buffer, msg)
        err = LockstepError(text, i, which, ot[0], self._name(ot), buffer)
        if self.raise_on_fail:
            raise err
        self.failures.append(err)

    def _check_stray(self, which, i, ot, writes):
        by_base = {}
        for w in writes:
            by_base.setdefault(w.idx, []).append(w)
        for b in self.tracked:
            cur, snap = self.db[b], self.snap[b]
            if cur.device != snap.device:  # host snapshot: a buffer the op does not write is compared through a device staging
                if b not in by_base and self._same_as_host(cur, snap):
                    continue
                cur = cur.cpu()
            if b not in by_base:
                if _same(cur, snap):
                    continue
                changed = (_bits(cur) != _bits(snap)).reshape(-1)
            else:
                mask = torch.zeros(cur.numel(), dtype=torch.bool, device=cur.device)
                for w in by_base[b]:
                    for off in w.offsets():
                        self._dut_mark(mask, b, off, w.shape, w.strides)
                changed = (_bits(cur) != _bits(snap)).reshape(-1) & ~mask
                if not bool(changed.any()):
                    snap.copy_(cur)
                    continue
            first = int(torch.nonzero(changed)[0])
            n = int(changed.sum())
            pos = np.unravel_index(first, tuple(cur.shape)) if cur.dim() else ()
            self._fail(which, i, ot, self._blabel(b), "%d stray write(s) outside the op's outputs, first at %s" % (n, tuple(int(v) for v in pos)))
            snap.copy_(cur)
            self.tb[b].copy_(self._pull(b))  # the twin follows, so later ops are checked on what the executor really holds

    def _same_as_host(self, cur, snap):
        """bit equality of device buffer cur and its pinned host snapshot, uploaded in pieces through one staging buffer"""
        c, h = cur.reshape(-1).view(torch.uint8), snap.reshape(-1).view(torch.uint8)
        if self._stage is None or self._stage.device != cur.device:
            self._stage = torch.empty(256 << 20, dtype=torch.uint8, device=cur.device)
        n = self._stage.numel()
        for a in range(0, c.numel(), n):
            m = min(n, c.numel() - a)
            self._stage[:m].copy_(h[a:a + m], non_blocking=True)
            if not torch.equal(self._stage[:m], c[a:a + m]):
                return False
        return True

    def _compare(self, which, i, ot, w):
        st = self.stats.setdefault(w.tag, [0, 0.0, True])
        st[0] += 1
        if w.sample is not None:
            flat = self.db[w.idx].reshape(-1)
            got = sum(flat[torch.from_numpy(w.sample.reshape(-1) + (off - w.off)).to(flat.device)].double().cpu()
                      for off in w.offsets()).numpy().reshape(w.sample.shape)
            res = [_judge(w.tag, got, w.ref, w.tol, lambda k: np.unravel_index(int(w.sample.reshape(-1)[k]), tuple(self.tb[w.idx].shape)))]
            for off in w.offsets():
                _view(self.tb[w.idx], off, w.shape, w.strides).copy_(self._dut_view(w.idx, off, w.shape, w.strides).cpu())
        elif w.fn is None:
            got_t = [self._dut_view(w.idx, off, w.shape, w.strides).cpu() for off in w.offsets()]
            got = sum(t.double() for t in got_t).numpy()
            ref = np.asarray(w.ref, dtype=np.float64)
            res = [_judge(w.tag, got, ref, w.tol, lambda k: np.unravel_index(k, ref.shape))]
            for off, t in zip(w.offsets(), got_t):
                _view(self.tb[w.idx], off, w.shape, w.strides).copy_(t)
        else:
            lead, inner = w.shape[0], int(np.prod(w.shape[1:]))
            step = max(1, self.chunk // max(inner, 1))

            def piece(a):
                # one chunk: its reference (read from the twin before the chunk's outputs are copied into it), the check, the copy
                b = min(lead, a + step)
                shape = (b - a,) + w.shape[1:]
                offs = [off + a * w.strides[0] for off in w.offsets()]
                got_t = [self._dut_view(w.idx, off, shape, w.strides).cpu() for off in offs]
                got = sum(t.double() for t in got_t).numpy()
                ref, tol = w.fn(a, b)
                r = _judge(w.tag, got, np.asarray(ref, dtype=np.float64).reshape(shape), tol,
                           lambda k: (lambda p: (p[0] + a,) + p[1:])(np.unravel_index(k, shape)))
                for off, t in zip(offs, got_t):
                    _view(self.tb[w.idx], off, shape, w.strides).copy_(t)
                return r

            res = emulate.pmap(piece, range(0, lead, step))
        nbad, worst = 0, None
        for ratio, exact, bad, wst, flips, elems in res:
            st[1] = max(st[1], ratio)
            st[2] = st[2] and exact
            if elems:
                self.ulp_flips += flips
                self.bn_apply_elems += elems
            nbad += bad
            if wst is not None and (worst is None or wst[0] > worst[0]):
                worst = wst
        if nbad:
            _, pos, g, r, t = worst
            self._fail(which, i, ot, w.label, "%d element(s) out of tolerance; worst at %s: got %r, float64 reference %r, tolerance %r" % (
                nbad, tuple(int(v) for v in pos), g, r, t))

    def table(self):
        lines = ["%-22s %7s  %s" % ("kind", "checks", "worst err/tol (exact kinds: worst |err|)")]
        for tag in sorted(self.stats):
            n, worst, exact = self.stats[tag]
            lines.append("%-22s %7d  %s" % (tag, n, ("exact, max |err| %g" % worst) if exact else "%.3g" % worst))
        return "\n".join(lines + self._table_extra())


class Lockstep(Harness):
    """the training plan: fwd_ops then bwd_ops of a UNetTrainEngine"""

    def __init__(self, dut, twin, sample_above=None, chunk=1 << 22, sms=train_launch.SMS, seed=0, snapshot="device"):
        """sample_above: sampled mode for convolutions with more output pixels and their weight gradients (see above);
        chunk: elements per piece of the chunked elementwise checks; sms: the device's SM count (the bn_stats grid reads it);
        snapshot: "device" or "host", where the stray-write check keeps its copy of the executor's buffers"""
        self.dut, self.tw = dut, twin
        self.sample_above, self.chunk, self.seed = sample_above, chunk, seed
        self.launches = train_launch.plan_launches(twin, sms=sms)
        self.launch = train_launch.by_op(self.launches)
        E, T = dut.eng, twin
        assert T.plan_only and T.device.type == "cpu"
        self.db, self.tb = _bases(E), _bases(T)
        assert len(self.db) == len(self.tb), "the two engines built different buffer lists"
        for i, (a, b) in enumerate(zip(self.db, self.tb)):
            assert a.shape == b.shape and a.dtype == b.dtype, ("buffer %d pairs %s %s with %s %s" % (i, tuple(a.shape), a.dtype, tuple(b.shape), b.dtype))
        for which in ("fwd_ops", "bwd_ops"):
            a, b = getattr(E, which), getattr(T, which)
            assert [o[0] for o in a] == [o[0] for o in b], "the two engines built different %s" % which
        self._index()
        # labels of the base buffers, for messages
        self.labels = {}
        for name, t in list(T.params.items()):
            self._label(t, name)
        self._label(T._grads_flat, "grads")
        for d in (T.feats, T.relu_outs):
            for name, (t, _) in d.items():
                self._label(t, name)
        for u in T.units.values():
            self._label(u.out, u.name + ".out")
        scratch = set()
        self.bn_units = []
        for op in T.fwd_ops:
            if op[0] == "bn_stats":
                b = op[1]
                self.bn_units.append(b)
                scratch.add(self._locate(b.sums.data_ptr())[0])
                for nm in ("z", "mean", "invstd", "scale", "shift"):
                    self._label(getattr(b, nm), b.prefix + "." + nm)
        for t in T._stats_buf.values():
            scratch.add(self._locate(t.data_ptr())[0])
        scratch.add(self._locate(T.final_acc.data_ptr())[0])
        for i, t in enumerate(self.tb):
            if t.dtype == torch.int32:
                scratch.add(i)
        for name in ("s2d", "logits"):
            self._label(getattr(T, name), name)
        self.tracked = [i for i in range(len(self.tb)) if i not in scratch and self.tb[i].numel()]
        # the executor's state is the starting point: copy it into the twin once, snapshot it on the executor's device
        for i in self.tracked:
            self.tb[i].copy_(self.db[i].cpu())
        if snapshot == "host" and self.db[0].device.type != "cpu":
            self.snap = {i: self.db[i].cpu().pin_memory() for i in self.tracked}
        else:
            self.snap = {i: self.db[i].clone() for i in self.tracked}
        self._stage = None
        self.units_by_conv = {id(u.fwd): u for u in T.units.values()}
        self.d_units_by_conv = {id(u.fwd): u for u in E.units.values()}
        self.stats = {}       # tag -> [checks, worst err/tol (or worst error of exact checks), exact?]
        self.ulp_flips = 0    # bn_apply outputs one fp16 ulp away from the correctly rounded reference
        self.bn_apply_elems = 0
        self.failures = []
        self.checked = {"fwd": set(), "bwd": set()}

    def _table_extra(self):
        lines = []
        if self.bn_apply_elems:
            lines.append("bn_apply outputs one fp16 ulp from the correctly rounded value: %d of %d" % (self.ulp_flips, self.bn_apply_elems))
        lines.append("ops checked: %d forward, %d backward" % (len(self.checked["fwd"]), len(self.checked["bwd"])))
        for fam in ("partial_reduce", "channel_reduce", "final_bwd_dw"):
            ls_ = [la for la in self.launches if la.family == fam]
            if ls_:
                la = max(ls_, key=lambda la: la.chain)
                lines.append("derived sum bound %-15s longest fp32 chain %4d (%s), e_sum %.3g; %d of %d launches capped" % (
                    fam, la.chain, la.name, la.e_sum(), sum(x.capped for x in ls_), len(ls_)))
        lines.append("conv.stats bound gamma_31 = %.3g" % E_CONV_STATS)
        return lines

    # ------------------------------------------------------------------ driver
    def run(self, x, dlogits, raise_on_fail=True, dut_x=None, dut_dlogits=None, log=None):
        """x: fp32 NCHW input (CPU), dlogits: fp32 NCHW logit gradient (CPU); dut_*: the same on the executor's device;
        log: called with a line per op (its time) when given"""
        import time

        self.raise_on_fail = raise_on_fail
        dx = x if dut_x is None else dut_x
        ddl = dlogits if dut_dlogits is None else dut_dlogits
        for which, lst_d, lst_t in (("fwd", self.dut.eng.fwd_ops, self.tw.fwd_ops), ("bwd", self.dut.eng.bwd_ops, self.tw.bwd_ops)):
            for i, (od, ot) in enumerate(zip(lst_d, lst_t)):
                if ot[0] == "bn_finalize":
                    assert i - 1 in self.checked[which] and lst_t[i - 1][0] == "bn_stats" and lst_t[i - 1][1] is ot[1]
                    self.checked[which].add(i)
                    continue
                fin = (lst_d[i + 1], lst_t[i + 1]) if ot[0] == "bn_stats" else None
                t0 = time.time()
                self._step(which, i, od, ot, fin, x, dlogits, dx, ddl)
                self.checked[which].add(i)
                if log is not None:
                    log("%s %3d %-12s %-36s %6.2f s" % (which, i, ot[0], self._name(ot), time.time() - t0))
        assert len(self.checked["fwd"]) == len(self.tw.fwd_ops) and len(self.checked["bwd"]) == len(self.tw.bwd_ops)
        return self.failures

    def _name(self, ot):
        k = ot[0]
        if k == "conv":
            return ot[1].name
        if k in ("bn_stats", "bn_finalize", "bn_apply", "bn_bwd"):
            return ot[1].prefix
        if k == "wgrad":
            return ot[1].name
        return k

    def _step(self, which, i, od, ot, fin, x, dlogits, dx, ddl):
        self._cur = (which, i)
        writes = self._reference(ot, x, dlogits)
        self.dut.run(od, x=dx, dlogits=ddl)
        if fin is not None:
            self.dut.run(fin[0], x=dx, dlogits=ddl)
        self.dut.sync()
        if ot[0] == "wgrad" and self.dut.repeat_wgrad:
            w = writes[0]
            first = _view(self.db[w.idx], w.off, w.shape, w.strides).clone()
            self.dut.run(od, x=dx, dlogits=ddl)
            self.dut.sync()
            if not torch.equal(_bits(first), _bits(_view(self.db[w.idx], w.off, w.shape, w.strides))):
                self._fail(which, i, ot, w.label, "a second run of the weight gradient is not bit-identical")
        self._check_stray(which, i, ot, writes)
        for w in writes:
            self._compare(which, i, ot, w)
        self._extra(which, i, ot)

    # ------------------------------------------------------------------ invariants
    def _extra(self, which, i, ot):
        k = ot[0]
        if k == "conv":
            u = self.units_by_conv.get(id(ot[1]))
            if u is not None and u.stats is not None and self.dut.conv_stats:
                du = self.d_units_by_conv[id(self._dut_op(which, i)[1])]
                rows, C = u.stats_rows, u.desc.Cout
                part = du.stats[:rows * 2 * C].double().cpu().reshape(rows, 2, C).sum(0).numpy()
                z = self._colsums(u.out, C, lambda z: (z, np.abs(z), z * z))  # the kernel's own output, already copied into the twin
                e = E_CONV_STATS + rows * 2.0 ** -53
                for j, (ref, mag) in enumerate(((z[0], z[1]), (z[2], z[2]))):
                    err, tol = np.abs(part[j] - ref), e * mag + 1e-30
                    st = self.stats.setdefault("conv.stats", [0, 0.0, False])
                    st[0] += 1
                    st[1] = max(st[1], float((err / tol).max()))
                    if (err > tol).any():
                        c = int(np.argmax(err / tol))
                        self._fail(which, i, ot, u.name + ".stats", "%s of channel %d: partials give %r, float64 %r" % (
                            ("column sum", "sum of squares")[j], c, float(part[j][c]), float(ref[c])))
        if k in ("bn_stats", "bn_bwd"):
            b = ot[1]
            idx, _ = self._locate(b.sums.data_ptr())
            acc = self.db[idx][:16 * b.C + 1]
            if bool((acc != 0).any()):
                first = int(torch.nonzero(acc != 0)[0])
                self._fail(which, i, ot, b.prefix + ".sums", "accumulator slots / arrival counter not cleared (first nonzero double %d)" % first)
            self.tb[idx].copy_(self.db[idx].cpu())

    def _colsums(self, t, C, terms):
        """column sums over the rows of (twin) tensor t viewed [M, C] as float64, of each array terms(rows) returns, in chunks"""
        v = t.reshape(-1, C)
        step = max(1, self.chunk // C)
        parts = emulate.pmap(lambda a: [p.sum(0) for p in terms(v[a:a + step].double().numpy())], range(0, v.shape[0], step))
        return [sum(col) for col in zip(*parts)]

    def _write_lazy(self, label, t, shape, fn, tag):
        """output = the whole of contiguous (twin) tensor t viewed as `shape`, reference fn(a, b) over rows a:b of it"""
        i, off = self._locate(t.data_ptr())
        assert t.is_contiguous() and int(np.prod(shape)) == t.numel()
        strides = tuple(int(np.prod(shape[k + 1:])) for k in range(len(shape)))
        return _Write(label, i, off, shape, strides, None, None, tag, fn=fn)

    def _e_sum(self, family):
        return self.launch[self._cur][family].e_sum()

    def _dut_op(self, which, i):
        return (self.dut.eng.fwd_ops if which == "fwd" else self.dut.eng.bwd_ops)[i]

    # ------------------------------------------------------------------ float64 references of single ops
    def _reference(self, op, x, dlogits):
        return getattr(self, "_ref_" + op[0])(op, x, dlogits)

    def _ref_conv(self, op, x, dlogits):
        d = op[1].desc
        K = 64 * sum(d.segs[j].cblocks for j in range(d.nseg))
        tag = "conv.dgrad" if ".dgrad" in op[1].name else "conv"
        writes = []
        if self.sample_above is not None and d.mode == 0 and d.phases * d.Nt * d.Ht * d.Wt > self.sample_above:
            pix = self._conv_sample(d)
            val, mag, addr = emulate.conv_f64_at(d, pix)
            tol = ulp16(val) + K * U * mag
            for phase, base, shape, strides in emulate.conv_out_views(d):
                sel = pix[:, 3] == phase
                idx, off = self._locate(base)
                sample = ((addr[sel] - self.tb[idx].data_ptr()) // 2)[:, None] + np.arange(d.Cout)[None, :]
                writes.append(_Write("%s out (%s, sampled)" % (op[1].name, self._blabel(idx)), idx, off, shape, strides, val[sel], tol[sel], tag,
                                     d.out_plane if d.split else 0, sample=sample))
            return writes

        def sink(ptr, shape, strides, val, mag, parts, plane):
            idx, off = self._locate(ptr)
            writes.append(_Write("%s out (%s)" % (op[1].name, self._blabel(idx)), idx, off, shape, strides, val, ulp16(val) + K * U * mag, tag))

        emulate.run_desc(d, sink=sink)
        return writes

    def _rng(self):
        which, i = self._cur
        return np.random.default_rng([self.seed, 0 if which == "fwd" else 1, i])

    def _conv_sample(self, d):
        """sampled output pixels of descriptor d, [S, 4] (n, y, x, phase): for every image the whole first, last and one seeded
        random tile box of the kernel's TW x TH x TN tiling (the random box is shared by the TN images of a box), the four
        corners and 256 seeded random pixels; every phase of each"""
        rng = self._rng()
        nbw, nbh, nbn = -(-d.Wt // d.TW), -(-d.Ht // d.TH), -(-d.Nt // d.TN)
        rand_box = [(int(rng.integers(nbw)), int(rng.integers(nbh))) for _ in range(nbn)]
        pts = []
        for n in range(d.Nt):
            for bx, by in ((0, 0), (nbw - 1, nbh - 1), rand_box[n // d.TN]):
                yy, xx = np.meshgrid(np.arange(by * d.TH, min(d.Ht, (by + 1) * d.TH)), np.arange(bx * d.TW, min(d.Wt, (bx + 1) * d.TW)), indexing="ij")
                pts.append(np.stack([np.full(yy.size, n), yy.reshape(-1), xx.reshape(-1)], 1))
            pts.append(np.array([[n, 0, 0], [n, 0, d.Wt - 1], [n, d.Ht - 1, 0], [n, d.Ht - 1, d.Wt - 1]]))
            pts.append(np.stack([np.full(256, n), rng.integers(d.Ht, size=256), rng.integers(d.Wt, size=256)], 1))
        pix = np.unique(np.concatenate(pts).astype(np.int64), axis=0)
        return np.concatenate([np.concatenate([pix, np.full((len(pix), 1), ph, np.int64)], 1) for ph in range(d.phases)])

    def _ref_wgrad(self, op, x, dlogits):
        _, u, dy = op
        d = u.desc
        P = d.Nt * d.Ht * d.Wt
        ptr = dy.data_ptr() + 2 * u.out_offset
        if self.sample_above is not None and d.phases * P > self.sample_above:
            R = d.phases * d.Cout
            K = 64 * sum(d.segs[j].cblocks for j in range(d.nseg))
            rows = {r for r in (0, 63, 64, 127, 128, R - 1) if r < R} | {int(r) for r in self._rng().choice(R, min(4, R), replace=False)}
            rows = np.array(sorted(rows), dtype=np.int64)
            ref, mag = emulate.run_wgrad_rows(d, ptr, rows)
            idx, off = self._locate(u.dw_packed.data_ptr())
            sample = off + rows[:, None] * K + np.arange(K)[None, :]
            return [_Write(u.name + ".dw_packed (sampled rows)", idx, off, u.dw_packed.shape, u.dw_packed.stride(), ref,
                           2.0 ** -23 * (P / 16 + P / 64 + 17) * mag, "wgrad", sample=sample)]
        ref, mag = emulate.run_wgrad(d, ptr, None, f64=True)
        tol = 2.0 ** -23 * (P / 16 + P / 64 + 17) * mag
        return [self._write_t(u.name + ".dw_packed", u.dw_packed, ref, tol, "wgrad")]

    def _bn_params(self, b):
        P = self.tw.params
        return (_f64(P[b.prefix + ".weight"]), _f64(P[b.prefix + ".bias"]))

    def _ref_bn_stats(self, op, x, dlogits):
        b = op[1]
        P = self.tw.params
        s1, sa, s2 = self._colsums(b.z, b.C, lambda z: (z, np.abs(z), z * z))
        M = float(b.M)
        mean = s1 / M
        ez2 = s2 / M
        var = np.maximum(ez2 - mean * mean, 0)
        invstd = 1.0 / np.sqrt(var + BN_EPS)
        gamma, beta = self._bn_params(b)
        scale = gamma * invstd
        shift = beta - mean * scale
        rm, rv = _f64(P[b.prefix + ".running_mean"]), _f64(P[b.prefix + ".running_var"])
        unb = var * M / (M - 1) if M > 1 else var
        e_s = self._e_sum("partial_reduce")
        d_mean = e_s * sa / M + U * np.abs(mean)
        d_var = e_s * ez2 + 2 * np.abs(mean) * d_mean
        d_inv = invstd * (d_var / (2 * (var + BN_EPS)) + 2 * U)
        d_scale = np.abs(gamma) * d_inv + U * np.abs(scale)
        d_shift = np.abs(mean) * d_scale + np.abs(scale) * d_mean + 2 * U * (np.abs(beta) + np.abs(mean * scale))
        new_rm = (1 - BN_MOMENTUM) * rm + BN_MOMENTUM * mean
        new_rv = (1 - BN_MOMENTUM) * rv + BN_MOMENTUM * unb
        nbt = P[b.prefix + ".num_batches_tracked"]
        return [self._write_t(b.prefix + ".mean", b.mean, mean, d_mean, "bn_stats"),
                self._write_t(b.prefix + ".invstd", b.invstd, invstd, d_inv, "bn_stats"),
                self._write_t(b.prefix + ".scale", b.scale, scale, d_scale, "bn_stats"),
                self._write_t(b.prefix + ".shift", b.shift, shift, d_shift, "bn_stats"),
                self._write_t(b.prefix + ".running_mean", P[b.prefix + ".running_mean"], new_rm,
                              BN_MOMENTUM * d_mean + 4 * U * (np.abs(rm) + np.abs(mean)), "bn_stats.running"),
                self._write_t(b.prefix + ".running_var", P[b.prefix + ".running_var"], new_rv,
                              BN_MOMENTUM * d_var * M / max(M - 1, 1) + 4 * U * (np.abs(rv) + np.abs(unb)), "bn_stats.running"),
                self._write_t(b.prefix + ".num_batches_tracked", nbt, _f64(nbt) + 1, 0.0, "bn_stats.counter")]

    def _ref_bn_apply(self, op, x, dlogits):
        _, b, res, y, relu = op
        C = b.C
        sc, sh = _f64(b.scale), _f64(b.shift)
        zv = b.z.reshape(-1, C)
        rv = res.reshape(-1, C) if res is not None else None

        def fn(a, e):
            z = zv[a:e].double().numpy()
            o = z * sc + sh
            mag = np.abs(z * sc) + np.abs(sh)
            if rv is not None:
                r = rv[a:e].double().numpy()
                o = o + r
                mag = mag + np.abs(r)
            if relu:
                o = np.maximum(o, 0)
            return o, ulp16(o) + 2.0 ** -23 * mag

        return [self._write_lazy(b.prefix + " y", y, (b.M, C), fn, "bn_apply")]

    def _ref_bn_bwd(self, op, x, dlogits):
        _, b, dy, y, dz, g_out = op
        M, C = b.M, b.C
        mu, inv = _f64(b.mean), _f64(b.invstd)
        dyv, yv, zv = dy.reshape(M, C), (y.reshape(M, C) if y is not None else None), b.z.reshape(M, C)

        def g_of(a, e):
            g = dyv[a:e].double().numpy()
            return g * (yv[a:e].double().numpy() > 0) if yv is not None else g

        def part(a):
            g, z = g_of(a, a + step), zv[a:a + step].double().numpy()
            return [p.sum(0) for p in (g, g * ((z - mu) * inv), np.abs(g), np.abs(g * z))]

        step = max(1, self.chunk // C)
        s0, s1, sg, sgz = [sum(col) for col in zip(*emulate.pmap(part, range(0, M, step)))]
        gamma, _ = self._bn_params(b)
        A = gamma * inv
        Bc = -gamma * inv * inv * s1 / M
        D = -gamma * inv * s0 / M + gamma * inv * inv * mu * s1 / M
        e_s = self._e_sum("channel_reduce")
        d_s0 = e_s * sg
        d_s1 = e_s * inv * (sgz + np.abs(mu) * sg)

        def fn_dz(a, e):
            g, z = g_of(a, e), zv[a:e].double().numpy()
            zh = (z - mu) * inv
            ref = A * g + Bc * z + D
            return ref, ulp16(ref) + 2.0 ** -22 * (np.abs(A * g) + np.abs(Bc * z) + np.abs(D)) + np.abs(A) * (d_s0 + np.abs(zh) * d_s1) / M

        ls = float(self.tw.loss_scale)
        out = [self._write_lazy(b.prefix + " dz", dz, (M, C), fn_dz, "bn_bwd.dz")]
        if g_out is not None:
            out.append(self._write_lazy(b.prefix + " g_out", g_out, (M, C), lambda a, e: (g_of(a, e), 0.0), "bn_bwd.g_out"))
        out.append(self._write_t(b.prefix + ".weight grad", self.tw.grads[b.prefix + ".weight"], s1 / ls, d_s1 / ls + 2 * U * np.abs(s1 / ls), "bn_bwd.dgamma_dbeta"))
        out.append(self._write_t(b.prefix + ".bias grad", self.tw.grads[b.prefix + ".bias"], s0 / ls, d_s0 / ls + 2 * U * np.abs(s0 / ls), "bn_bwd.dgamma_dbeta"))
        return out

    def _ref_relu_bwd(self, op, x, dlogits):
        _, a_, b2, y, out = op
        C = out.shape[-1]
        av, bv, yv = a_.reshape(-1, C), (b2.reshape(-1, C) if b2 is not None else None), (y.reshape(-1, C) if y is not None else None)

        def fn(a, e):
            s = av[a:e].float()
            if bv is not None:
                s = s + bv[a:e].float()
            if yv is not None:
                s = s * (yv[a:e].float() > 0)
            return _f64(s.half()), 0.0

        return [self._write_lazy("relu_bwd out", out, (out.numel() // C, C), fn, "relu_bwd")]

    def _ref_maxpool(self, op, x, dlogits):
        _, src, dst, n, h, w, c, kk, s, p = op
        sv = src.reshape(n, h, w, c)

        def fn(a, e):
            return F.max_pool2d(sv[a:e].double().permute(0, 3, 1, 2), kk, s, p).permute(0, 2, 3, 1).numpy(), 0.0

        return [self._write_lazy("maxpool out", dst, tuple(dst.shape), fn, "maxpool")]

    def _ref_maxpool_bwd(self, op, x, dlogits):
        _, xx, dy, dx, n, h, w, c, kk, s, p = op
        xv = xx.reshape(n, h, w, c)
        oh, ow = (h + 2 * p - kk) // s + 1, (w + 2 * p - kk) // s + 1
        dyv = dy.reshape(n, oh, ow, c)

        def fn(a, e):
            xin = xv[a:e].double().permute(0, 3, 1, 2).clone().requires_grad_(True)
            yy = F.max_pool2d(xin, kk, s, p)
            yy.backward(dyv[a:e].double().permute(0, 3, 1, 2))
            ref = xin.grad.permute(0, 2, 3, 1).numpy()
            return ref, ulp16(ref)

        return [self._write_lazy("maxpool_bwd dx", dx, (n, h, w, c), fn, "maxpool_bwd")]

    def _ref_prepass(self, op, x, dlogits):
        return [self._write_t("s2d", self.tw.s2d, _f64(emulate.prepass_s2d_cpu(x)), 0.0, "prepass")]

    def _ref_zero_grads(self, op, x, dlogits):
        return [self._write_t("grads", self.tw._grads_flat, np.zeros(self.tw._grads_flat.numel()), 0.0, "zero_grads")]

    def _ref_pack_all(self, op, x, dlogits):
        P = self.tw.params
        out = []
        for wname, m, dst, _c, _o in self.tw.pack_list:
            src = P[wname].reshape(-1)
            mm = m.long()
            if bool((mm[:, 1:] < 0).all()):
                ref = torch.where(mm[:, 0] >= 0, src[mm[:, 0].clamp_min(0)], torch.zeros(())).half().numpy()
                out.append(self._write_t(wname + " packed", dst, ref, 0.0, "pack_all.single"))
            else:
                vals = torch.where(mm >= 0, src.double()[mm.clamp_min(0)], torch.zeros((), dtype=torch.float64))
                ref = vals.sum(1).numpy()
                out.append(self._write_t(wname + " packed (summed taps)", dst, ref, ulp16(ref) + 2.0 ** -22 * vals.abs().sum(1).numpy(), "pack_all.summed"))
        return out

    def _ref_unpack_all(self, op, x, dlogits):
        T = self.tw
        flat_ref = T._grads_flat.double().clone()
        flat_mag = torch.zeros_like(flat_ref)
        touched = {}
        for dwp, m, wname, _c, _o in T.unpack_list:
            off = T._grad_offset[wname]
            mm = m.long()
            v = dwp.double() / T.loss_scale
            for j in range(4):
                sel = mm[:, j] >= 0
                flat_ref.index_add_(0, mm[sel, j] + off, v[sel])
                flat_mag.index_add_(0, mm[sel, j] + off, v[sel].abs())
            touched[wname] = off
        out = []
        for wname, off in touched.items():
            g = T.grads[wname]
            n = g.numel()
            r, a = flat_ref[off:off + n].numpy(), flat_mag[off:off + n].numpy()
            out.append(self._write_t(wname + " grad", g, r, 2.0 ** -22 * a + 2 * U * np.abs(r), "unpack_all"))
        return out

    def _ref_final_fwd(self, op, x, dlogits):
        _, y5, logits = op
        P = self.tw.params
        w = _f64(P["final.weight"]).reshape(self.tw.C, 32)
        b = _f64(P["final.bias"])

        def fn(a, e):
            y = y5[a:e].double().numpy()  # [n, H, W, 32]
            ref = np.einsum("nhwc,kc->nkhw", y, w) + b[None, :, None, None]
            mag = np.einsum("nhwc,kc->nkhw", np.abs(y), np.abs(w)) + np.abs(b)[None, :, None, None]
            return ref, 34 * U * mag

        return [self._write_lazy("logits", logits, tuple(logits.shape), fn, "final_fwd")]

    def _ref_final_bwd(self, op, x, dlogits):
        _, y5, d_y5 = op
        T = self.tw
        w = _f64(T.params["final.weight"]).reshape(T.C, 32)
        ls = float(T.loss_scale)
        def part(n):  # one image: [classes, HW] x [HW, 32]
            dl, y = dlogits[n].double().numpy().reshape(T.C, -1), y5[n].double().numpy().reshape(-1, 32)
            return dl @ y, np.abs(dl) @ np.abs(y), dl.sum(1), np.abs(dl).sum(1)

        dw, dwm, db, dbm = [sum(col) for col in zip(*emulate.pmap(part, range(y5.shape[0])))]

        def fn(a, e):
            dl = dlogits[a:e].double().numpy()
            d = np.einsum("nkhw,kc->nhwc", dl, w) * ls
            dmag = np.einsum("nkhw,kc->nhwc", np.abs(dl), np.abs(w)) * ls
            return d, ulp16(d) + (T.C + 2) * U * dmag

        e_s = self._e_sum("final_bwd_dw")
        return [self._write_lazy("d_y5", d_y5, tuple(d_y5.shape), fn, "final_bwd.dy5"),
                self._write_t("final.weight grad", T.grads["final.weight"], dw, e_s * dwm + 2 * U * np.abs(dw), "final_bwd.dw_db"),
                self._write_t("final.bias grad", T.grads["final.bias"], db, e_s * dbm + 2 * U * np.abs(db), "final_bwd.dw_db")]


def make_pair(C, B, H, W, loss_scale, device, seed=0):
    """(state dict, dut engine, plan_only CPU twin) with identical parameters"""
    from robosat_b200 import synth
    from robosat_b200.train_engine import UNetTrainEngine

    sd0 = {k[7:]: v.clone() for k, v in synth.make_state_dict(C, seed=seed).items()}
    dut = UNetTrainEngine({k: v.clone().to(device) for k, v in sd0.items()}, C, B, H, W, device=device, loss_scale=loss_scale,
                          plan_only=(torch.device(device).type == "cpu"))
    twin = UNetTrainEngine({k: v.clone() for k, v in sd0.items()}, C, B, H, W, device="cpu", loss_scale=loss_scale, plan_only=True)
    return sd0, dut, twin


def n_ops(eng):
    return len(eng.fwd_ops) + len(eng.bwd_ops)

