"""Every case of the convolution matrix (tests/conv_matrix.py) on the GPU, element by element against a float64 replay.

Per case:
  * reference: tests/emulate.py's float64 mode on the host copy of the same operands (the values the fp16 planes represent:
    hi + lo times acc_scale, plus bias, residual, ReLU; the head's fp32 1x1 on top), and the elementwise bound of
    tests/predict_lockstep.py (`conv_tol`) from the float64 sums of |x w|; the worst err/tol is printed;
  * placement: every element of the output buffer outside the view (both planes in strict precision; the logits buffer
    of a head) still holds the sentinel bit for bit; sources, weights, bias, residual and head parameters are unchanged;
    the K-chunk scratch and the statistics partials are untouched past their stated sizes;
  * repeats: two runs of one plan give the same bits; where both schedules are valid (mode 0, >= 128 columns) the CTA-pair
    and the one-CTA schedules give the same bits too;
  * rsb_conv_plan_info: tiles, K blocks, grid and shared memory as the descriptor implies;
  * statistics instances: every per-quarter-tile partial equals the float64 sums of the stored fp16 outputs of its 32 rows
    (ragged rows excluded) within lockstep.py's E_CONV_STATS (31 fp32 roundings).
"""

import ctypes

import numpy as np
import pytest
import torch

import conv_matrix as CM
import emulate
from lockstep import E_CONV_STATS
from predict_lockstep import conv_tol
from robosat_b200 import _lib
from robosat_b200._lib import RowConvDesc

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _reference(host):
    """[(offset, shape, strides, plane, value, tol)] of every output view, offsets in elements of host.t['out']"""
    d = host.desc
    base = host.t["out"]
    item = base.element_size()
    strict = bool(d.split)
    writes = []

    def sink(ptr, shape, strides, val, mag, parts, plane):
        off = (ptr - base.data_ptr()) // item
        writes.append((off, tuple(shape), tuple(strides), plane, np.asarray(val), np.broadcast_to(conv_tol(d, strict, val, mag, parts), np.shape(val))))

    (emulate.run_rowdesc if isinstance(d, RowConvDesc) else emulate.run_desc)(d, sink=sink)
    return writes


class _Plan:
    def __init__(self, lib, desc):
        self.lib, self.row = lib, isinstance(desc, RowConvDesc)
        self.h = ctypes.c_void_p()
        create = lib.rsb_rowconv_plan_create if self.row else lib.rsb_conv_plan_create
        _lib.check(create(ctypes.byref(desc), ctypes.byref(self.h)), "plan_create")

    def run(self):
        _lib.check((self.lib.rsb_rowconv_run if self.row else self.lib.rsb_conv_run)(self.h, _lib.current_stream_ptr()), "run")
        torch.cuda.synchronize()

    def info(self):
        v = [ctypes.c_int32() for _ in range(4)]
        _lib.check(self.lib.rsb_conv_plan_info(self.h, *[ctypes.byref(x) for x in v]), "plan_info")
        return [x.value for x in v]

    def close(self):
        (self.lib.rsb_rowconv_plan_destroy if self.row else self.lib.rsb_conv_plan_destroy)(self.h)


def _launch(plan, dev, init):
    """reset the written buffers to their sentinels, run, return host copies of them"""
    for k, v in init.items():
        dev.t[k].copy_(v)
    plan.run()
    return {k: dev.t[k].cpu() for k in init}


def _check_plan_info(plan, d, device):
    grid, tiles, kblocks, smem = plan.info()
    sp = [-(-n // b) for n, b in zip((d.Wt, d.Ht, d.Nt), (d.TW, d.TH, d.TN))]
    assert tiles == sp[0] * sp[1] * sp[2] * d.phases * (d.Cout // d.block_n)
    assert kblocks == sum(d.segs[i].cblocks for i in range(d.nseg))
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    assert 0 < grid <= sms and grid <= (tiles if not d.cta_pair else 2 * tiles)
    if d.cta_pair:
        assert grid % 2 == 0, grid
    assert 0 < smem <= CM.SMEM_OPTIN


def _check_stats(case, d, got_out, got_stats, meta):
    """per-quarter partials of the stored fp16 outputs (tile rows in the kernel's order: w fastest, then h, then n)"""
    o, C = meta["o"], d.Cout
    z = torch.as_strided(got_out, (d.Nt, d.Ht, d.Wt, C), (o.pn, o.ph, o.pw, 1), o.off).double()
    tw, th = -(-d.Wt // d.TW), -(-d.Ht // d.TH)
    n, h, w = torch.meshgrid(torch.arange(d.Nt), torch.arange(d.Ht), torch.arange(d.Wt), indexing="ij")
    spatial = (w // d.TW) + tw * ((h // d.TH) + th * (n // d.TN))
    row = (w % d.TW) + d.TW * ((h % d.TH) + d.TH * (n % d.TN))
    q = (spatial * 4 + row // 32).reshape(-1)
    rows = meta["stats_rows"]
    zf = z.reshape(-1, C)
    ref = torch.zeros(2, rows, C, dtype=torch.float64)
    ref[0].index_add_(0, q, zf)
    ref[1].index_add_(0, q, zf * zf)
    mag = torch.stack([torch.zeros(rows, C, dtype=torch.float64).index_add_(0, q, zf.abs()), ref[1]])
    part = got_stats[:rows * 2 * C].double().reshape(rows, 2, C).permute(1, 0, 2)
    err = (part - ref).abs()
    tol = E_CONV_STATS * mag + 1e-30
    bad = ~(err <= tol)
    assert not bad.any(), "%s: %d statistics partial(s) off, first at (sum|sq, quarter row, channel) %s: %r vs %r" % (
        case.name, int(bad.sum()), tuple(torch.nonzero(bad)[0].tolist()), float(part[bad][0]), float(ref[bad][0]))
    bits = _bits(got_stats[rows * 2 * C:])
    assert bool((bits == CM.SENTINEL32).all()), "%s: statistics written past the stated size" % case.name


@pytest.mark.parametrize("case", CM.matrix(), ids=str)
def test_conv_matrix_case(case, cuda_device):
    lib = _lib.load()
    host = case.build("cpu")
    writes = _reference(host)
    dev = host.to(cuda_device)
    d = dev.desc
    ro = {k: dev.t[k].clone() for k in case.readonly() if dev.t.get(k) is not None}
    init = {k: dev.t[k].clone() for k in ("out", "scratch", "stats") if dev.t.get(k) is not None}
    plan = _Plan(lib, d)
    try:
        if not plan.row:
            _check_plan_info(plan, d, cuda_device)
        runs = [_launch(plan, dev, init) for _ in range(2)]
    finally:
        plan.close()
    for k in runs[0]:
        assert torch.equal(_bits(runs[0][k]), _bits(runs[1][k])), "%s: %s differs between two runs of one plan" % (case.name, k)
    got = runs[0]["out"]

    # placement: the views and nothing else
    inview = torch.zeros(got.numel(), dtype=torch.bool)
    for off, shape, strides, plane, _, _ in writes:
        for o in ((off, off + plane) if plane else (off,)):
            torch.as_strided(inview, shape, strides, o).fill_(True)
    sentinel = CM.SENTINEL16 if got.element_size() == 2 else CM.SENTINEL32
    stray = (_bits(got) != sentinel) & ~inview
    assert not stray.any(), "%s: %d element(s) written outside the output view, first at element %d" % (
        case.name, int(stray.sum()), int(torch.nonzero(stray)[0]))
    for k, v in ro.items():
        assert torch.equal(_bits(dev.t[k]), _bits(v)), "%s: the launch modified %s" % (case.name, k)
    if "scratch" in dev.t:
        tail = _bits(runs[0]["scratch"][host.meta["scratch_bytes"] // 4:])
        assert bool((tail == CM.SENTINEL32).all()), "%s: K-chunk scratch written past its stated size" % case.name

    # values, elementwise
    worst = 0.0
    for off, shape, strides, plane, val, tol in writes:
        v = torch.as_strided(got, shape, strides, off).double()
        if plane:
            v = v + torch.as_strided(got, shape, strides, off + plane).double()
        err = np.abs(v.numpy() - val)
        ok = err <= tol
        ratio = np.where(tol > 0, err / np.maximum(tol, 1e-300), np.where(err > 0, np.inf, 0.0))
        worst = max(worst, float(np.max(np.where(ok, ratio, np.inf))))
        if not ok.all():
            i = np.unravel_index(int(np.argmax(np.where(ok, -1.0, ratio))), ok.shape)
            pytest.fail("%s: %d of %d element(s) out of bound; worst at %s: got %r, float64 %r, bound %r" % (
                case.name, int((~ok).sum()), ok.size, tuple(int(x) for x in i), float(v.numpy()[i]), float(val[i]), float(tol[i])))
    print("\n%-48s worst err/tol %.4f" % (case.name, worst))

    if case.kernel == "conv" and d.stats:
        _check_stats(case, d, got, runs[0]["stats"], host.meta)

    # the other schedule, where the descriptor allows it: the same bits
    if case.kernel == "conv" and d.mode == 0 and d.block_n >= 128 and not (d.split and d.residual and d.block_n == 256):
        alt = case._desc(dev.t, dev.meta)
        alt.cta_pair = 0 if d.cta_pair else 1
        assert CM.instance_of(alt) != CM.instance_of(d)
        plan = _Plan(lib, alt)
        try:
            _check_plan_info(plan, alt, cuda_device)
            other = _launch(plan, dev, init)
        finally:
            plan.close()
        for k in ("out", "stats"):
            if k in other:
                assert torch.equal(_bits(other[k]), _bits(runs[0][k])), "%s: %s differs between the CTA-pair and the one-CTA schedule" % (case.name, k)
