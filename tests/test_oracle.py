"""Pin the oracle restatements against fixtures produced by the REAL reference (tests/golden/make_golden.py)."""

import os

import numpy as np
import torch

from oracle import losses_oracle, unet_oracle
from robosat_b200 import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_unet_oracle_matches_reference_logits_bit_exact():
    gold = np.load(os.path.join(GOLD, "unet_64.npz"))
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 64, seed=1))
    for C in (2, 6):
        sd = synth.make_state_dict(C, seed=0)
        with torch.no_grad():
            got = unet_oracle.unet_forward(sd, x).numpy()
        ref = gold["logits_c%d" % C]
        assert got.shape == ref.shape == (2, C, 64, 64)
        # same torch build, same op sequence: bit-identical in the build container; on another host oneDNN may pick a
        # different blocking for its fp32 kernels, which moves results by a few 1e-5 (summation order), never more
        assert np.abs(got - ref).max() <= 2e-4, "max abs diff %g" % np.abs(got - ref).max()


def test_unet_oracle_matches_reference_checksums_256():
    gold = np.load(os.path.join(GOLD, "unet_stats.npz"))
    sd = synth.make_state_dict(2, seed=0)
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 256, seed=1))
    with torch.no_grad():
        lo = unet_oracle.unet_forward(sd, x)
    assert np.abs(lo[:, :, ::16, ::16].numpy() - gold["sample"]).max() <= 2e-4
    ref_argmax = np.unpackbits(gold["argmax_packed"])[: lo[:, 0].numel()].reshape(lo[:, 0].shape)
    assert int((lo.argmax(1).numpy() != ref_argmax).sum()) <= 8  # only exact near-ties may flip with summation order
    assert abs(lo.double().sum().item() - float(gold["sum"])) <= 1e-6 * float(gold["abs_sum"])
    # both classes are present so argmax parity tests are not vacuous
    frac = float(gold["fg_pixels"]) / lo[:, 0].numel()
    assert 0.05 < frac < 0.95, frac


def test_state_dict_layout_matches_reference_checkpoint_contract():
    sd = synth.make_state_dict(2, seed=0)
    keys = list(sd.keys())
    assert len(keys) == 329 and all(k.startswith("module.") for k in keys)  # SURVEY.md F9
    assert keys[0] == "module.resnet.conv1.weight" and keys[-2:] == ["module.final.weight", "module.final.bias"]
    assert sum(v.dtype == torch.int64 for v in sd.values()) == 53
    assert sum(v.numel() * v.element_size() for v in sd.values()) == 157774160


def test_lovasz_oracle_matches_reference():
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    for tag in "abc":
        logits = torch.from_numpy(gold["lovasz_%s_logits" % tag])
        targets = torch.from_numpy(gold["lovasz_%s_targets" % tag])
        loss, grad = losses_oracle.lovasz_loss(logits, targets, with_grad=True)
        assert abs(float(loss) - float(gold["lovasz_%s_loss" % tag])) <= 2e-6 * abs(float(gold["lovasz_%s_loss" % tag]))
        # closed-form gradient == autograd of the reference (ties do not occur in random fp32 logits)
        np.testing.assert_allclose(grad.numpy(), gold["lovasz_%s_grad" % tag], rtol=0, atol=1e-9)


def test_lovasz_oracle_gradient_is_bit_identical_to_the_reference_also_at_n_3():
    """The GPU tests compare the kernel's gradient with this oracle bit for bit, so the oracle itself has to be bit-identical to the
    reference. Fixture b has N = 3, where scaling by fp32(1 / N) (autograd of `loss / N`) and dividing by N differ in the last bit."""
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    for tag in "abc":
        logits = torch.from_numpy(gold["lovasz_%s_logits" % tag])
        targets = torch.from_numpy(gold["lovasz_%s_targets" % tag])
        grad = losses_oracle.lovasz_loss(logits, targets, with_grad=True)[1].numpy()
        ref = gold["lovasz_%s_grad" % tag]
        # every non-zero element has the same bits; where the error is <= 0 autograd leaves -0.0 or +0.0, which compare equal
        assert np.array_equal(grad, ref) and np.array_equal(grad.view(np.int32)[ref != 0], ref.view(np.int32)[ref != 0]), tag
    assert gold["lovasz_b_logits"].shape[0] == 3


def test_cross_entropy_oracle_matches_reference():
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    for tag in "abc":
        logits = torch.from_numpy(gold["lovasz_%s_logits" % tag])
        targets = torch.from_numpy(gold["lovasz_%s_targets" % tag])
        w = torch.from_numpy(gold["ce_%s_weight" % tag])
        loss, grad = losses_oracle.cross_entropy_loss(logits, targets, w, with_grad=True)
        assert abs(float(loss) - float(gold["ce_%s_loss" % tag])) <= 2e-6 * abs(float(gold["ce_%s_loss" % tag]))
        np.testing.assert_allclose(grad.numpy(), gold["ce_%s_grad" % tag], rtol=1e-4, atol=1e-9)


def test_metrics_oracle_matches_reference():
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    for tag in "abc":
        logits = torch.from_numpy(gold["lovasz_%s_logits" % tag])
        targets = torch.from_numpy(gold["lovasz_%s_targets" % tag])
        assert list(losses_oracle.metrics_counts(logits, targets)) == gold["metrics_%s" % tag].tolist()


def test_adam_oracle_matches_reference():
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    p = gold["adam_p0"]
    m = np.zeros_like(p)
    v = np.zeros_like(p)
    for s in range(3):
        p, m, v = losses_oracle.adam_step(p, gold["adam_grads"][s], m, v, lr=1e-4, step=s + 1)
        np.testing.assert_allclose(p, gold["adam_p%d" % (s + 1)], rtol=2e-7, atol=1e-9)


def test_focal_and_miou_oracles_match_reference():
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    for tag in "abc":
        logits = torch.from_numpy(gold["lovasz_%s_logits" % tag])
        targets = torch.from_numpy(gold["lovasz_%s_targets" % tag])
        w = torch.from_numpy(gold["ce_%s_weight" % tag])
        loss, grad = losses_oracle.focal_loss(logits, targets, w, gamma=2, with_grad=True)
        assert abs(float(loss) - float(gold["focal_%s_loss" % tag])) <= 5e-6 * abs(float(gold["focal_%s_loss" % tag]))
        np.testing.assert_allclose(grad.numpy(), gold["focal_%s_grad" % tag], rtol=2e-4, atol=1e-9)
        for sub, scale in (("", 1.0), ("_sharp", 4.0), ("_aligned", None)):
            lg = logits * scale if scale is not None else torch.from_numpy(gold["miou_aligned_%s_logits" % tag])
            loss, grad = losses_oracle.miou_loss(lg, targets, w, with_grad=True)
            ref = float(gold["miou%s_%s_loss" % (sub, tag)])
            assert abs(float(loss) - ref) <= 5e-6 * abs(ref)
            np.testing.assert_allclose(grad.numpy(), gold["miou%s_%s_grad" % (sub, tag)], rtol=5e-4, atol=1e-9)


def test_predict_pipeline_restatement_matches_the_reference_tools_files(tmp_path):
    """tests/golden/predict_bins.npz holds the probability bins the UNMODIFIED robosat.tools.predict.main wrote for the five-tile
    synthetic directory (make_golden_predict.py). The pipeline restated from oracle pieces -- buffered tile, ToTensor / Normalize,
    oracle forward, softmax, unbuffer, np.digitize -- reproduces them (identically on the build host; a few bin-edge pixels may move
    with another oneDNN build), so the GPU test that uses this restatement is pinned to the reference tool itself."""
    from PIL import Image

    from robosat_b200.datasets import BufferedSlippyMapDirectory
    from robosat_b200.transforms import ImageToUint8Tensor

    gold = np.load(os.path.join(GOLD, "predict_bins.npz"))
    coords = [(100, 200), (101, 200), (100, 201), (101, 201), (103, 205)]
    u8 = synth.make_tiles_u8(5, 256, seed=9).numpy()
    for (x, y), arr in zip(coords, u8):
        os.makedirs(tmp_path / "17" / str(x), exist_ok=True)
        Image.fromarray(arr).save(tmp_path / "17" / str(x) / ("%d.png" % y))
    directory = BufferedSlippyMapDirectory(str(tmp_path), transform=ImageToUint8Tensor(), size=256, overlap=32)
    sd = synth.make_state_dict(2, seed=0)
    differing = 0
    for i in range(len(directory)):
        image, xyz = directory[i]
        x, y, _ = (int(v) for v in xyz)
        probs = unet_oracle.predict_probs(sd, synth.normalize_tiles(image.unsqueeze(0))).numpy()[0]
        bins = np.digitize(directory.unbuffer(probs)[1], np.linspace(0, 1, 256)).astype(np.uint8)
        d = np.abs(bins.astype(np.int32) - gold["bins_%d_%d" % (x, y)].astype(np.int32))
        assert d.max() <= 1
        differing += int((d > 0).sum())
    assert differing <= 64, differing
