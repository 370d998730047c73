"""The inference lockstep harness (tests/predict_lockstep.py) run on the CPU: the emulator passes every op of small plans in
both precisions against the float64 replay, and a copy of the emulator with injected faults is reported at exactly the
faulty op and buffer. Three of the faults are subtle enough that the whole-network check of tests/test_unet_gpu.py
(`_check`: strict rel-L2, rel-max and argmax-flip limits against the fp32 oracle) passes with them in place."""

import ctypes

import pytest
import torch

import emulate
import predict_lockstep as pl
from oracle import unet_oracle
from robosat_b200 import synth
from robosat_b200._lib import ConvSrc
from test_unet_gpu import _check


def _input(N, H, W):
    return synth.normalize_tiles(synth.make_tiles_u8(N, max(H, W), seed=1))[:, :, :H, :W].contiguous()


class FaultyEmulator(pl.EmulatorExecutor):
    def __init__(self, eng, faults):
        super().__init__(eng)
        self.faults = faults  # id(op) -> fn(executor, op, run)

    def run(self, op, x):
        fault = self.faults.get(id(op))
        if fault is None:
            return super().run(op, x)
        fault(self, op, lambda: super(FaultyEmulator, self).run(op, x))


def _op(eng, kind, name):
    hits = [op for op in eng.ops if op[0] == kind and (kind != "conv" or op[1].name == name)]
    hits = hits if kind == "conv" else [h for h in hits if h[2] is eng.feats[name][0]]  # a max pool by its output
    assert len(hits) == 1, (kind, name)
    return hits[0]


# ------------------------------------------------------------------ faults
def _drop_a_lo_cross_term(ex, op, run):
    """the layer computes without A_lo W_hi: its source's lo plane reads as zero"""
    d = op[1].desc
    src = next(t for t in ex.eng._keep if t.data_ptr() == d.srcs[0].ptr)
    saved = src[1].clone()
    src[1].zero_()
    run()
    src[1].copy_(saved)


def _last_tile_lo_left_zero(ex, op, run):
    """the lo plane of the layer's last (ragged: its TN box reaches past the batch) tile is never stored"""
    run()
    d = op[1].desc
    tw, th, tn = -(-d.Wt // d.TW), -(-d.Ht // d.TH), -(-d.Nt // d.TN)
    assert tw * th * tn > 1 and d.Nt % d.TN, "the fault wants a ragged last tile among several"
    out = next(t for t in ex.eng._keep if t.data_ptr() == d.out)
    out[1, (tn - 1) * d.TN:, (th - 1) * d.TH:, (tw - 1) * d.TW:, :] = 0


def _dec4_writes_its_pad_column(ex, op, run):
    run()
    ex.eng.dec4[0, 1, 5, 0, 7] = 1.0  # column 0 of the W-padded buffer: dec5 reads it as zero padding


def _bottom_border_reads_last_row(ex, op, run):
    """image 0 reads its last input row again below the bottom border, where the kernel must see zero fill"""
    d = op[1].desc
    s = d.src
    src = next(t for t in ex.eng._keep if t.data_ptr() == s.ptr).reshape(s.N, s.H, s.W, -1)
    ext = torch.zeros((s.N, s.H + 1, s.W, src.shape[-1]), dtype=src.dtype)
    ext[:, :s.H] = src
    ext[0, s.H] = src[0, s.H - 1]
    saved = ConvSrc.from_buffer_copy(s)
    d.src = ConvSrc(ext.data_ptr(), s.pitch_w, s.pitch_h, (s.H + 1) * s.pitch_h, s.C, s.W, s.H + 1, s.N, s.plane)
    run()
    d.src = saved


def _maxpool_max_of_hi(ex, op, run):
    """the split max pool compares hi alone, so where two hi values tie it may keep the smaller pair"""
    _, src, dst, n, h, w, c, k, s, p = op
    hi = src[0].float().reshape(n, h, w, c).permute(0, 3, 1, 2)
    lo = src[1].float().reshape(n, h, w, c).permute(0, 3, 1, 2)
    m, idx = torch.nn.functional.max_pool2d(hi, k, s, p, return_indices=True)
    y = (m.double() + lo.flatten(2).gather(2, idx.flatten(2)).reshape(m.shape).double()).float().permute(0, 2, 3, 1)
    yh = y.half()
    dst.copy_(torch.stack([yh, (y - yh.float()).half()]).reshape(dst.shape))


# (kind, op name (a max pool: its output), fault, substring of the reported buffer, invisible to the whole-network check)
STRICT_FAULTS = [("conv", "resnet.layer1.0.conv1", _drop_a_lo_cross_term, "resnet.layer1.0.conv1 out", True),
                 ("conv", "resnet.layer2.1.conv1", _last_tile_lo_left_zero, "resnet.layer2.1.conv1 out", True),
                 ("conv", "dec4", _dec4_writes_its_pad_column, "dec4", False),
                 ("maxpool", "enc0", _maxpool_max_of_hi, "maxpool out", True)]
FAST_FAULTS = [("conv", "dec4", _bottom_border_reads_last_row, "dec4 out", False)]


def _lockstep(C, N, H, W, precision, faults=()):
    sd = synth.make_state_dict(C, seed=0)
    dut, twin = pl.make_pair(sd, C, N, H, W, precision, "cpu")
    targets = {}
    table = {}
    for kind, name, fn, buf, _ in faults:
        op = _op(dut, kind, name)
        table[id(op)] = fn
        targets[dut.ops.index(op)] = (kind, name, buf)
    ls = pl.PredictLockstep(FaultyEmulator(dut, table), twin)
    failures = ls.run(_input(N, H, W), raise_on_fail=False)
    print(ls.table())
    for f in failures:
        print(f)
    assert len(ls.checked) == len(dut.ops)
    return sd, dut, ls, failures, targets


@pytest.mark.parametrize("precision", ["strict", "fast"])
@pytest.mark.parametrize("C,N,H,W", [(2, 1, 64, 512), (6, 2, 64, 64)])
def test_predict_lockstep_clean_emulator_passes_every_op(C, N, H, W, precision):
    _, dut, ls, failures, _ = _lockstep(C, N, H, W, precision)
    assert not failures, "\n".join(str(f) for f in failures[:10])
    assert ls.weights_identical[0] == ls.weights_identical[1] > 0
    kinds = {"prepass", "maxpool"} | ({"conv split=2"} if precision == "strict" else {"conv"})
    if W >= 128:
        kinds |= {"line-buffer head"} | (set() if precision == "strict" else {"line buffer"})
    else:
        kinds |= {"conv head"}
    assert kinds <= set(ls.stats), sorted(ls.stats)


@pytest.mark.parametrize("precision,shape,faults", [("strict", (6, 3, 64, 64), STRICT_FAULTS), ("fast", (2, 1, 64, 512), FAST_FAULTS)])
def test_predict_lockstep_reports_each_injected_fault_at_its_op(precision, shape, faults):
    sd, dut, ls, failures, targets = _lockstep(*shape, precision, faults)
    got = {}
    for f in failures:
        got.setdefault(f.index, []).append(f)
    assert set(got) == set(targets), (sorted(got), sorted(targets))
    for i, (kind, name, buf) in targets.items():
        for f in got[i]:  # one report per output view (an upsample op writes four phases)
            assert f.kind == kind and buf in f.buffer, str(f)
            if kind == "conv":
                assert f.name == name, str(f)
    pad = [i for i, t in targets.items() if t[2] == "dec4"]
    assert all("stray" in str(got[i][0]) for i in pad)


def test_whole_network_check_misses_the_subtle_faults():
    """faults (cross term, ragged tile's lo plane, max pool tie) each pass the strict whole-network limits of
    tests/test_unet_gpu.py on the emulated plan: only the per-op check sees them"""
    C, N, H, W = 6, 3, 64, 64
    sd = synth.make_state_dict(C, seed=0)
    x = _input(N, H, W)
    with torch.no_grad():
        ref = unet_oracle.unet_forward(sd, x)
    for kind, name, fn, _, subtle in [(None, None, None, None, True)] + STRICT_FAULTS:
        if not subtle:
            continue
        eng, _ = pl.make_pair(sd, C, N, H, W, "strict", "cpu")
        ex = FaultyEmulator(eng, {} if fn is None else {id(_op(eng, kind, name)): fn})
        for op in eng.ops:
            ex.run(op, x)
        _check(eng.logits.clone(), ref, "emulated strict plan, fault %s" % (fn.__name__ if fn else "none"), "strict")
