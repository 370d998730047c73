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
chained kernels must leave their slots and arrival counter zero), the conv-statistics partials (their column sums are
checked against the convolution's own output instead), `final_acc`, and the int32 weight-packing maps (constants).

Tolerances, elementwise. u = 2^-24 is the fp32 unit roundoff; a tensor-core adder is not guaranteed to round to nearest,
so every fp32 accumulator addition is charged 2u = 2^-23 of the running magnitude. ulp16(r) is the fp16 spacing at |r|
(2^-24 below the normal range), which bounds the final fp16 rounding (half an ulp) with room for the fp32 error of values
that sit next to a rounding boundary. A is the float64 sum of the magnitudes of the terms of the same expression.

  conv        fp16 out     ulp16(ref) + K * 2^-24 * A, A = sum_k |x_k| |w_k| (+ |residual|). The wgmma chain adds K/16
                           partial products of 16 terms each into an fp32 accumulator (bound as for wgrad below):
                           (K/16 + 17) * 2^-23 * A <= K * 2^-24 * A for K >= 64.
  conv stats  partials     sum of the partial rows vs float64 column sums / sums of squares of the kernel's own fp16 z:
                           rel 1e-5 of sum |z| / sum z^2 (each partial adds 32 rows in fp32, 32 u = 1.9e-6).
  wgrad       fp32 dw      2^-23 * (P/16 + P/64 + 17) * A, A = sum_p |dy_p| |x_p|: P/16 accumulator additions of 16-pixel MMAs,
                           at most P/64 slice partials added afterwards (a slice holds at least one 64-pixel tile), and the
                           sum inside each MMA: its 16 products are aligned to the largest one and truncated, so each can lose
                           2^-23 of that block maximum, at most 16 * 2^-23 * A over all blocks (+1 for the normalisation).
                           Layers with fewer than 16 pixels per phase (center, dec0) need that term: measured errors there
                           reach 2-4 fp32 ulps of a result made of a handful of same-sign products.
  bn_stats    mean etc.    from the sums' error e_s = 1e-5 relative to sum |z| (<= ~160 fp32 additions per partial before the
                           fp64 accumulation: 160 u < 1e-5): d_mean = e_s E|z| + u |mean|, d_var = e_s E[z^2] + 2 |mean| d_mean,
                           d_invstd = invstd (d_var / 2 (var + eps) + 2u), d_scale = |gamma| d_invstd + u |scale|,
                           d_shift = |mean| d_scale + |scale| d_mean + 2u (|beta| + |mean scale|); running stats: momentum
                           times those plus 4u of their magnitudes; num_batches_tracked exact.
  bn_apply    fp16 y       ulp16(ref) + 2^-23 (|z scale| + |shift| + |res|): one fma and one add in fp32, then fp16.
  bn_bwd      dz           ulp16(ref) + 2^-22 (|A g| + |B z| + |D|) + |A| (d_s0 + |zhat| d_s1) / M, with dz = A g + B z + D the
                           kernel's fp32 form, d_s0 = e_s sum |g| and d_s1 = e_s invstd (sum |g z| + |mean| sum |g|)
                           (the kernel forms sum g zhat as (sum g z - mean sum g) invstd);
              g_out        exact (a masked copy);
              dgamma/dbeta d_s1 / loss_scale + 2u |ref|, d_s0 / loss_scale + 2u |ref|.
  relu_bwd, maxpool, prepass, zero_grads: exact (one fp32 add of two fp16 values rounded once, a max, a copy, zeros).
  maxpool_bwd fp16 dx      ulp16(ref): at most ceil(k/s)^2 exact fp16 values summed in fp32, rounded once.
  pack_all    fp16 packed  exact for single-source layouts (one rounding of the fp32 weight); ulp16(ref) + 2^-22 A for the
                           pre-summed upsample taps (<= 3 fp32 additions, then fp16).
  final_fwd   fp32 logits  34 u A (32 fmas + the bias, A = sum |w y| + |b|).
  final_bwd   fp16 dy5     ulp16(ref) + (C + 2) u A; dW, db: e_s A + 2u |ref| (fp32 per-thread partials, fp64 totals).
  unpack_all  fp32 grads   2^-22 A + 2u |ref| (<= 4 fp32 additions and the 1/loss_scale product).
"""

import bisect

import numpy as np
import torch
import torch.nn.functional as F

import emulate

U = 2.0 ** -24
E_SUM = 1e-5
BN_EPS = 1e-5
BN_MOMENTUM = 0.1


class LockstepError(AssertionError):
    def __init__(self, msg, index, which, kind, name, buffer):
        super().__init__(msg)
        self.index, self.which, self.kind, self.name, self.buffer = index, which, kind, name, buffer


def ulp16(x):
    """spacing of fp16 numbers at |x| (the subnormal spacing 2^-24 below 2^-14)"""
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -14)))
    return np.exp2(e - 10)


def _f64(t):
    return t.detach().cpu().double().numpy()


class EmulatorExecutor:
    """Runs ops with the CPU emulator on a plan_only engine. Its BatchNorm ops clear their accumulators like the chained
    kernels, and it is deterministic, but running a weight gradient twice would only repeat the same numpy call."""

    chained_bn = True
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

    conv_stats = True

    def __init__(self, eng, chained_bn, repeat_wgrad):
        self.eng, self.chained_bn, self.repeat_wgrad = eng, chained_bn, repeat_wgrad

    def run(self, op, x=None, dlogits=None):
        self.eng._run([op], x=x, dlogits=dlogits)

    def sync(self):
        torch.cuda.synchronize()


class _Write:
    """an output view (base buffer index, element offset, shape, element strides) with its reference and tolerance"""

    __slots__ = ("label", "idx", "off", "shape", "strides", "ref", "tol", "tag")

    def __init__(self, label, idx, off, shape, strides, ref, tol, tag):
        self.label, self.idx, self.off, self.shape, self.strides = label, idx, off, tuple(shape), tuple(strides)
        self.ref, self.tol, self.tag = ref, tol, tag


def _bases(eng):
    return list(eng._keep) + list(eng.params.values()) + [eng._grads_flat]


def _view(base, off, shape, strides):
    flat = base.reshape(-1)
    return torch.as_strided(flat, shape, strides, flat.storage_offset() + off)


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()]) if t.dtype.is_floating_point else t


class Lockstep:
    def __init__(self, dut, twin):
        self.dut, self.tw = dut, twin
        E, T = dut.eng, twin
        assert T.plan_only and T.device.type == "cpu"
        self.db, self.tb = _bases(E), _bases(T)
        assert len(self.db) == len(self.tb), "the two engines built different buffer lists"
        for i, (a, b) in enumerate(zip(self.db, self.tb)):
            assert a.shape == b.shape and a.dtype == b.dtype, ("buffer %d pairs %s %s with %s %s" % (i, tuple(a.shape), a.dtype, tuple(b.shape), b.dtype))
        for which in ("fwd_ops", "bwd_ops"):
            a, b = getattr(E, which), getattr(T, which)
            assert [o[0] for o in a] == [o[0] for o in b], "the two engines built different %s" % which
        self._order = sorted((t.data_ptr(), i) for i, t in enumerate(self.tb) if t.numel())
        self._starts = [p for p, _ in self._order]
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
        self.snap = {i: self.db[i].clone() for i in self.tracked}
        self.units_by_conv = {id(u.fwd): u for u in T.units.values()}
        self.d_units_by_conv = {id(u.fwd): u for u in E.units.values()}
        self.stats = {}       # tag -> [checks, worst err/tol (or worst error of exact checks), exact?]
        self.ulp_flips = 0    # bn_apply outputs one fp16 ulp away from the correctly rounded reference
        self.bn_apply_elems = 0
        self.failures = []
        self.checked = {"fwd": set(), "bwd": set()}

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

    # ------------------------------------------------------------------ driver
    def run(self, x, dlogits, raise_on_fail=True, dut_x=None, dut_dlogits=None):
        """x: fp32 NCHW input (CPU), dlogits: fp32 NCHW logit gradient (CPU); dut_*: the same on the executor's device"""
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
                self._step(which, i, od, ot, fin, x, dlogits, dx, ddl)
                self.checked[which].add(i)
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

    def _fail(self, which, i, ot, buffer, msg):
        text = "%s op %d (%s %s), buffer %s: %s" % (which, i, ot[0], self._name(ot), buffer, msg)
        err = LockstepError(text, i, which, ot[0], self._name(ot), buffer)
        if self.raise_on_fail:
            raise err
        self.failures.append(err)

    def _step(self, which, i, od, ot, fin, x, dlogits, dx, ddl):
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
    def _check_stray(self, which, i, ot, writes):
        by_base = {}
        for w in writes:
            by_base.setdefault(w.idx, []).append(w)
        for b in self.tracked:
            cur, snap = self.db[b], self.snap[b]
            if b not in by_base:
                if torch.equal(_bits(cur), _bits(snap)):
                    continue
                changed = (_bits(cur) != _bits(snap)).reshape(-1)
            else:
                mask = torch.zeros(cur.numel(), dtype=torch.bool, device=cur.device)
                for w in by_base[b]:
                    torch.as_strided(mask, w.shape, w.strides, w.off).fill_(True)
                changed = (_bits(cur) != _bits(snap)).reshape(-1) & ~mask
                if not bool(changed.any()):
                    snap.copy_(cur)
                    continue
            first = int(torch.nonzero(changed)[0])
            n = int(changed.sum())
            pos = np.unravel_index(first, tuple(cur.shape)) if cur.dim() else ()
            self._fail(which, i, ot, self._blabel(b), "%d stray write(s) outside the op's outputs, first at %s" % (n, tuple(int(v) for v in pos)))
            snap.copy_(cur)
            self.tb[b].copy_(cur.cpu())  # the twin follows, so later ops are checked on what the executor really holds

    def _compare(self, which, i, ot, w):
        got_t = _view(self.db[w.idx], w.off, w.shape, w.strides).cpu()
        got = got_t.double().numpy()
        ref = np.asarray(w.ref, dtype=np.float64)
        tol = np.broadcast_to(np.asarray(w.tol, dtype=np.float64), ref.shape)
        err = np.abs(got - ref)
        err = np.where(np.isnan(err) & ~(np.isnan(got) & np.isnan(ref)), np.inf, err)
        err = np.where(np.isnan(err), 0.0, err)
        exact = not np.any(tol)
        st = self.stats.setdefault(w.tag, [0, 0.0, exact])
        st[0] += 1
        st[2] = st[2] and exact
        if exact:
            worst = float(err.max()) if err.size else 0.0
            st[1] = max(st[1], worst)
            bad = err > 0
        else:
            ratio = np.divide(err, tol, out=np.where(err > 0, np.inf, 0.0), where=tol > 0)
            st[1] = max(st[1], float(ratio.max()) if ratio.size else 0.0)
            bad = err > tol
        if w.tag == "bn_apply":
            self.bn_apply_elems += got.size
            self.ulp_flips += int((got != ref.astype(np.float16).astype(np.float64)).sum())
        if bad.any():
            k = int(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), -1)))
            pos = np.unravel_index(k, ref.shape)
            self._fail(which, i, ot, w.label, "%d element(s) out of tolerance; worst at %s: got %r, float64 reference %r, tolerance %r" % (
                int(bad.sum()), tuple(int(v) for v in pos), float(got.reshape(-1)[k]), float(ref.reshape(-1)[k]), float(tol.reshape(-1)[k])))
        _view(self.tb[w.idx], w.off, w.shape, w.strides).copy_(got_t)

    def _extra(self, which, i, ot):
        k = ot[0]
        if k == "conv":
            u = self.units_by_conv.get(id(ot[1]))
            if u is not None and u.stats is not None and self.dut.conv_stats:
                du = self.d_units_by_conv[id(self._dut_op(which, i)[1])]
                rows, C = u.stats_rows, u.desc.Cout
                part = du.stats[:rows * 2 * C].double().cpu().reshape(rows, 2, C).sum(0).numpy()
                z = _f64(u.out).reshape(-1, C)  # the kernel's own output, already copied into the twin
                for j, (ref, mag) in enumerate(((z.sum(0), np.abs(z).sum(0)), ((z * z).sum(0), (z * z).sum(0)))):
                    err, tol = np.abs(part[j] - ref), E_SUM * mag + 1e-30
                    st = self.stats.setdefault("conv.stats", [0, 0.0, False])
                    st[0] += 1
                    st[1] = max(st[1], float((err / tol).max()))
                    if (err > tol).any():
                        c = int(np.argmax(err / tol))
                        self._fail(which, i, ot, u.name + ".stats", "%s of channel %d: partials give %r, float64 %r" % (
                            ("column sum", "sum of squares")[j], c, float(part[j][c]), float(ref[c])))
        if k in ("bn_stats", "bn_bwd") and self.dut.chained_bn:
            b = ot[1]
            idx, _ = self._locate(b.sums.data_ptr())
            acc = self.db[idx][:16 * b.C + 1]
            if bool((acc != 0).any()):
                first = int(torch.nonzero(acc != 0)[0])
                self._fail(which, i, ot, b.prefix + ".sums", "accumulator slots / arrival counter not cleared (first nonzero double %d)" % first)
            self.tb[idx].copy_(self.db[idx].cpu())

    def _dut_op(self, which, i):
        return (self.dut.eng.fwd_ops if which == "fwd" else self.dut.eng.bwd_ops)[i]

    # ------------------------------------------------------------------ float64 references of single ops
    def _reference(self, op, x, dlogits):
        return getattr(self, "_ref_" + op[0])(op, x, dlogits)

    def _ref_conv(self, op, x, dlogits):
        d = op[1].desc
        K = 64 * sum(d.segs[j].cblocks for j in range(d.nseg))
        writes = []

        def sink(ptr, shape, strides, val, mag):
            idx, off = self._locate(ptr)
            tag = "conv.dgrad" if ".dgrad" in op[1].name else "conv"
            writes.append(_Write("%s out (%s)" % (op[1].name, self._blabel(idx)), idx, off, shape, strides, val, ulp16(val) + K * U * mag, tag))

        emulate.run_desc(d, sink=sink)
        return writes

    def _ref_wgrad(self, op, x, dlogits):
        _, u, dy = op
        d = u.desc
        ref, mag = emulate.run_wgrad(d, dy.data_ptr() + 2 * u.out_offset, None, f64=True)
        P = d.Nt * d.Ht * d.Wt
        tol = 2.0 ** -23 * (P / 16 + P / 64 + 17) * mag
        return [self._write_t(u.name + ".dw_packed", u.dw_packed, ref, tol, "wgrad")]

    def _bn_params(self, b):
        P = self.tw.params
        return (_f64(P[b.prefix + ".weight"]), _f64(P[b.prefix + ".bias"]))

    def _ref_bn_stats(self, op, x, dlogits):
        b = op[1]
        P = self.tw.params
        z = _f64(b.z).reshape(b.M, b.C)
        M = float(b.M)
        mean = z.sum(0) / M
        ez2 = (z * z).sum(0) / M
        var = np.maximum(ez2 - mean * mean, 0)
        invstd = 1.0 / np.sqrt(var + BN_EPS)
        gamma, beta = self._bn_params(b)
        scale = gamma * invstd
        shift = beta - mean * scale
        rm, rv = _f64(P[b.prefix + ".running_mean"]), _f64(P[b.prefix + ".running_var"])
        unb = var * M / (M - 1) if M > 1 else var
        d_mean = E_SUM * np.abs(z).sum(0) / M + U * np.abs(mean)
        d_var = E_SUM * ez2 + 2 * np.abs(mean) * d_mean
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
        z = _f64(b.z).reshape(b.M, b.C)
        sc, sh = _f64(b.scale), _f64(b.shift)
        o = z * sc + sh
        mag = np.abs(z * sc) + np.abs(sh)
        if res is not None:
            r = _f64(res).reshape(b.M, b.C)
            o = o + r
            mag = mag + np.abs(r)
        if relu:
            o = np.maximum(o, 0)
        return [self._write_t(b.prefix + " y", y, o, ulp16(o) + 2.0 ** -23 * mag, "bn_apply")]

    def _ref_bn_bwd(self, op, x, dlogits):
        _, b, dy, y, dz, g_out = op
        M, C = b.M, b.C
        g = _f64(dy).reshape(M, C)
        if y is not None:
            g = g * (_f64(y).reshape(M, C) > 0)
        z = _f64(b.z).reshape(M, C)
        mu, inv = _f64(b.mean), _f64(b.invstd)
        gamma, _ = self._bn_params(b)
        zh = (z - mu) * inv
        s0, s1 = g.sum(0), (g * zh).sum(0)
        A = gamma * inv
        Bc = -gamma * inv * inv * s1 / M
        D = -gamma * inv * s0 / M + gamma * inv * inv * mu * s1 / M
        ref = A * g + Bc * z + D
        d_s0 = E_SUM * np.abs(g).sum(0)
        d_s1 = E_SUM * inv * (np.abs(g * z).sum(0) + np.abs(mu) * np.abs(g).sum(0))
        tol = ulp16(ref) + 2.0 ** -22 * (np.abs(A * g) + np.abs(Bc * z) + np.abs(D)) + np.abs(A) * (d_s0 + np.abs(zh) * d_s1) / M
        ls = float(self.tw.loss_scale)
        out = [self._write_t(b.prefix + " dz", dz, ref, tol, "bn_bwd.dz")]
        if g_out is not None:
            out.append(self._write_t(b.prefix + " g_out", g_out, g, 0.0, "bn_bwd.g_out"))
        out.append(self._write_t(b.prefix + ".weight grad", self.tw.grads[b.prefix + ".weight"], s1 / ls, d_s1 / ls + 2 * U * np.abs(s1 / ls), "bn_bwd.dgamma_dbeta"))
        out.append(self._write_t(b.prefix + ".bias grad", self.tw.grads[b.prefix + ".bias"], s0 / ls, d_s0 / ls + 2 * U * np.abs(s0 / ls), "bn_bwd.dgamma_dbeta"))
        return out

    def _ref_relu_bwd(self, op, x, dlogits):
        _, a, b2, y, out = op
        s = a.float()
        if b2 is not None:
            s = s + b2.float()
        if y is not None:
            s = s * (y.float() > 0)
        return [self._write_t("relu_bwd out", out, _f64(s.half()), 0.0, "relu_bwd")]

    def _ref_maxpool(self, op, x, dlogits):
        _, src, dst, n, h, w, c, kk, s, p = op
        yy = F.max_pool2d(src.double().reshape(n, h, w, c).permute(0, 3, 1, 2), kk, s, p).permute(0, 2, 3, 1)
        return [self._write_t("maxpool out", dst, yy.numpy(), 0.0, "maxpool")]

    def _ref_maxpool_bwd(self, op, x, dlogits):
        _, xx, dy, dx, n, h, w, c, kk, s, p = op
        xin = xx.double().reshape(n, h, w, c).permute(0, 3, 1, 2).clone().requires_grad_(True)
        yy = F.max_pool2d(xin, kk, s, p)
        yy.backward(dy.double().reshape(n, yy.shape[2], yy.shape[3], c).permute(0, 3, 1, 2))
        ref = xin.grad.permute(0, 2, 3, 1).numpy()
        return [self._write_t("maxpool_bwd dx", dx, ref, ulp16(ref), "maxpool_bwd")]

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
        y = _f64(y5)  # [N, H, W, 32]
        w = _f64(P["final.weight"]).reshape(self.tw.C, 32)
        b = _f64(P["final.bias"])
        ref = np.einsum("nhwc,kc->nkhw", y, w) + b[None, :, None, None]
        mag = np.einsum("nhwc,kc->nkhw", np.abs(y), np.abs(w)) + np.abs(b)[None, :, None, None]
        return [self._write_t("logits", logits, ref, 34 * U * mag, "final_fwd")]

    def _ref_final_bwd(self, op, x, dlogits):
        _, y5, d_y5 = op
        T = self.tw
        w = _f64(T.params["final.weight"]).reshape(T.C, 32)
        dl = dlogits.double().numpy()
        y = _f64(y5)
        ls = float(T.loss_scale)
        d = np.einsum("nkhw,kc->nhwc", dl, w) * ls
        dmag = np.einsum("nkhw,kc->nhwc", np.abs(dl), np.abs(w)) * ls
        dw = np.einsum("nkhw,nhwc->kc", dl, y)
        dwm = np.einsum("nkhw,nhwc->kc", np.abs(dl), np.abs(y))
        db, dbm = dl.sum((0, 2, 3)), np.abs(dl).sum((0, 2, 3))
        return [self._write_t("d_y5", d_y5, d, ulp16(d) + (T.C + 2) * U * dmag, "final_bwd.dy5"),
                self._write_t("final.weight grad", T.grads["final.weight"], dw, E_SUM * dwm + 2 * U * np.abs(dw), "final_bwd.dw_db"),
                self._write_t("final.bias grad", T.grads["final.bias"], db, E_SUM * dbm + 2 * U * np.abs(db), "final_bwd.dw_db")]

    # ------------------------------------------------------------------ report
    def table(self):
        lines = ["%-22s %7s  %s" % ("kind", "checks", "worst err/tol (exact kinds: worst |err|)")]
        for tag in sorted(self.stats):
            n, worst, exact = self.stats[tag]
            lines.append("%-22s %7d  %s" % (tag, n, ("exact, max |err| %g" % worst) if exact else "%.3g" % worst))
        if self.bn_apply_elems:
            lines.append("bn_apply outputs one fp16 ulp from the correctly rounded value: %d of %d" % (self.ulp_flips, self.bn_apply_elems))
        lines.append("ops checked: %d forward, %d backward" % (len(self.checked["fwd"]), len(self.checked["bwd"])))
        return "\n".join(lines)


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

