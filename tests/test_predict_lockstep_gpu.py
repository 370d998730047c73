"""Every launch of the inference plan against a float64 replay of the same op on the kernel's own inputs
(tests/predict_lockstep.py; bounds derived in its docstring), at the plans the tools run -- the measured table entries of
`rs serve` (strict 1 x 512^2) and `rs predict` (batch 32 at 512^2 and at the 576^2 of a 512 tile with its 32-pixel
overlap, both precisions) -- and at plans that reach kernel configurations those do not: the model's own plan (CTA pairs),
K-chunked narrow tiles, 6 classes at a rectangular shape, and folded weights spanning many binades."""

import time

import pytest
import torch

import predict_lockstep
from robosat_b200 import engine, synth

pytestmark = pytest.mark.gpu

SUBSET = (0, 16, 31)  # first, middle and last image of a batch-32 plan: the last ends a ragged TN tile


def _lockstep(cuda_device, C, N, H, W, precision, images=None, sd=None, u8=True, plan_overrides=None, what=""):
    sd = synth.make_state_dict(C, seed=0) if sd is None else sd
    dut, twin = predict_lockstep.make_pair(sd, C, N, H, W, precision, cuda_device, images=images, plan_overrides=plan_overrides)
    tiles = synth.make_tiles_u8(N, max(H, W), seed=1)[:, :H, :W].contiguous()
    sel = list(range(N)) if images is None else list(images)
    x = synth.normalize_tiles(tiles[sel])
    dut_x = tiles.to(cuda_device) if u8 else synth.normalize_tiles(tiles).to(cuda_device)
    t0 = time.time()
    ls = predict_lockstep.PredictLockstep(predict_lockstep.GpuExecutor(dut), twin, images)
    ls.run(x, dut_x=dut_x)
    print("\n%s %s %d x 3 x %d x %d, %d classes, %s input, images %s (%.0f s):\n%s" % (
        what, precision, N, H, W, C, "uint8" if u8 else "fp32", sel, time.time() - t0, ls.table()))
    assert len(ls.checked) == len(dut.ops)
    return dut, ls


def _descs(dut):
    return [op.desc for op in dut.conv_ops() if not hasattr(op.desc, "taps_h")]


def _table(key):
    assert key in engine.plan_table(), "the measured plan %s is gone from plans_h100.json" % key
    return engine.plan_table()[key]


def test_serve_plan_strict_1x512(cuda_device):
    """`rs serve` / SegmentEngine: the measured strict batch-1 plan, every image"""
    _table("strict:1x512x512")
    dut, ls = _lockstep(cuda_device, 2, 1, 512, 512, "strict", what="table plan")
    assert {d.block_n for d in _descs(dut)} >= {32, 128}
    assert "conv split=2" in ls.stats and "line-buffer head" in ls.stats


@pytest.mark.parametrize("precision", ["strict", "fast"])
@pytest.mark.parametrize("size", [576, 512])
def test_predict_plans_batch32(size, precision, cuda_device):
    """`rs predict --tile_size 512` at batch 32 (576 = 512 + 2 x 32 overlap) and the 512^2 bench plan, on three images"""
    _table("%s:32x%dx%d" % (precision, size, size))
    _lockstep(cuda_device, 2, 32, size, size, precision, images=SUBSET, what="table plan")


def test_model_plan_with_cta_pairs_strict(cuda_device):
    """the modelled plan (no table) at 2 x 256^2, where wide strict tiles run as CTA pairs"""
    dut, _ = _lockstep(cuda_device, 2, 2, 256, 256, "strict", plan_overrides={}, what="model plan")
    assert any(d.cta_pair for d in _descs(dut)), "no CTA pair in the plan: the paired kernels would go unchecked"


def test_k_chunked_narrow_and_wide_tiles_strict(cuda_device, monkeypatch):
    """chains cut at 24 MMAs, so that 32- and 64-wide (N-concatenated) tiles are K-chunked as well as 128-wide ones"""
    monkeypatch.setattr(engine, "MAX_MMA_CHAIN", 24)
    dut, ls = _lockstep(cuda_device, 2, 1, 256, 256, "strict", plan_overrides=_table("strict:1x512x512"), what="MAX_MMA_CHAIN 24")
    chunked = {d.block_n for d in _descs(dut) if 0 < d.kchunk < sum(d.segs[j].cblocks for j in range(d.nseg))}
    assert 32 in chunked and 128 in chunked, chunked
    assert "conv split=2 K-chunked" in ls.stats and "conv split=1 K-chunked" in ls.stats


def test_six_classes_rectangular_fp32_input(cuda_device):
    _lockstep(cuda_device, 6, 2, 192, 320, "strict", u8=False, what="6 classes")


def test_folded_weights_spanning_many_binades(cuda_device):
    """a few channels of one BatchNorm with running_var = 1e-6: their folded weights are ~300x the others', so after the
    hi/lo split the small weights' lo parts are subnormal fp16 numbers"""
    sd = synth.make_state_dict(2, seed=0)
    sd["module.resnet.layer2.1.bn2.running_var"][:4] = 1e-6
    sd["module.resnet.layer3.0.bn1.running_var"][5:7] = 1e-6
    dut, _ = _lockstep(cuda_device, 2, 1, 256, 256, "strict", sd=sd, what="running_var 1e-6")
    w = next(op.keep[0] for op in dut.conv_ops() if op.name == "resnet.layer2.1.conv2").float()
    lo = w[1][w[1] != 0].abs()
    assert bool((lo < 2.0 ** -14).any()), "no subnormal lo part: the case does not reach what it is for"
