"""Test-time augmentation on the host: the `--tta` flags, the view sets and pass rule of robosat_b200/tta.py, and the numpy
restatement of the head (tests/tta_reference.py) that the GPU tests compare the device against."""

import argparse

import numpy as np
import pytest

import tta_reference as ref
from robosat_b200 import tta
from robosat_b200.tools import predict, serve

REQUIRED = {
    "predict": ["--checkpoint", "c.pth", "--tile_size", "256", "--model", "m.toml", "--dataset", "d.toml", "tiles", "probs"],
    "serve": ["--checkpoint", "c.pth", "--model", "m.toml", "--dataset", "d.toml"],
}


def _parser():
    parser = argparse.ArgumentParser(prog="rs")
    sub = parser.add_subparsers()
    predict.add_parser(sub)
    serve.add_parser(sub)
    return parser


@pytest.mark.parametrize("tool", ["predict", "serve"])
def test_tta_flag_defaults_to_none_and_rejects_unknown_modes(tool):
    parser = _parser()
    assert parser.parse_args([tool] + REQUIRED[tool]).tta == "none"
    for mode in ("none", "flip", "d4"):
        assert parser.parse_args([tool] + REQUIRED[tool] + ["--tta", mode]).tta == mode
    for bad in ("D4", "rot90", "8", ""):
        with pytest.raises(SystemExit):
            parser.parse_args([tool] + REQUIRED[tool] + ["--tta", bad])


def test_view_sets():
    assert tta.views("none") == (0,)
    assert tta.views("flip") == (0, 1)
    assert tta.views("d4") == tuple(range(8))
    with pytest.raises(ValueError):
        tta.views("d8")
    # the eight d4 ops are eight different transforms
    probe = np.arange(12).reshape(3, 4)[:, :3]
    assert len({ref.view(probe, op).tobytes() for op in tta.views("d4")}) == 8


@pytest.mark.parametrize("batch,mode,passes,engine", [
    (1, "d4", 1, 8), (2, "d4", 1, 16), (8, "d4", 2, 32), (32, "d4", 8, 32),
    (1, "flip", 1, 2), (2, "flip", 1, 4), (8, "flip", 1, 16), (32, "flip", 2, 32),
])
def test_pass_rule(batch, mode, passes, engine):
    V = len(tta.views(mode))
    assert tta.num_passes(batch, V) == passes
    assert tta.TtaChain.engine_batch(mode, batch) == engine
    assert engine <= max(batch, tta.ENGINE_CAP) and engine * passes == batch * V


def test_pass_rule_follows_the_cap():
    assert tta.num_passes(2, 8, cap=4) == 4
    assert tta.num_passes(2, 8, cap=1) == 8  # never fewer tiles per pass than the batch itself: one view per pass
    assert tta.num_passes(3, 8, cap=5) == 8


def test_square_check():
    tta.check_shape("d4", 128, 128)
    tta.check_shape("flip", 128, 192)
    tta.check_shape("none", 128, 192)
    with pytest.raises(ValueError):
        tta.check_shape("d4", 128, 192)


@pytest.mark.parametrize("op", range(8))
def test_augment_model_is_flip_then_quarter_turns(op):
    img = np.random.default_rng(op).integers(0, 256, (7, 7, 3), dtype=np.uint8)
    assert np.array_equal(ref.augment_forward(img, op), ref.view(img, op))
    assert np.array_equal(ref.unview(ref.view(img, op), op), img)


@pytest.mark.parametrize("op", range(8))
@pytest.mark.parametrize("S,o", [(9, 0), (11, 2), (13, 3)])
def test_head_map_inverts_the_augmentation(op, S, o):
    """augment_dihedral's forward map, then the head's read of the view at forward_map, is the identity on the crop"""
    tile = np.arange(S * S).reshape(S, S)
    v = ref.augment_forward(tile, op)
    OS = S - 2 * o
    y, x = np.meshgrid(np.arange(OS), np.arange(OS), indexing="ij")
    vy, vx = ref.forward_map(op, OS, OS, y, x)
    assert np.array_equal(v[vy + o, vx + o], tile[o:S - o, o:S - o])


def test_head_map_flip_on_a_rectangle():
    tile = np.arange(5 * 8).reshape(5, 8)
    y, x = np.meshgrid(np.arange(5), np.arange(8), indexing="ij")
    vy, vx = ref.forward_map(1, 5, 8, y, x)
    assert np.array_equal(tile[:, ::-1][vy, vx], tile)


def test_restated_head_of_equivariant_views_is_the_single_view():
    """views that are exact transforms of one probability map average back to that map, bit for bit after the fixed point"""
    rng = np.random.default_rng(0)
    S, o, B = 13, 2, 2
    logits = rng.normal(0, 3, (B, 2, S, S)).astype(np.float32)
    probs = ref.softmax(logits)
    ops = tta.views("d4")
    views = np.stack([np.moveaxis(ref.augment_forward(np.moveaxis(probs[b], 0, -1), op), -1, 0) for op in ops for b in range(B)])
    acc = ref.accumulate(views, ops, B, o)
    single = ref.accumulate(probs, (0,), B, o)
    assert np.array_equal(acc, 8 * single)
    crop = probs[:, :, o:S - o, o:S - o]
    assert np.array_equal(ref.mean(single, 1), crop)  # p * 2^59 is exact for p >= 2^-35
    assert np.array_equal(ref.quantize(acc, 8), np.digitize(crop[:, 1], np.linspace(0, 1, 256)).astype(np.uint8))
    assert np.array_equal(ref.argmax(acc), crop.argmax(axis=1).astype(np.uint8))


def test_restated_softmax():
    rng = np.random.default_rng(1)
    for C in (2, 3, 5):
        l = rng.normal(0, 10, (2, C, 4, 6)).astype(np.float32)
        l[0, :, 0, 0] = 80.0
        l[1, 0, 0, 0] = -80.0
        p = ref.softmax(l)
        e = np.exp(l.astype(np.float64) - l.max(axis=1, keepdims=True))
        assert np.abs(p - e / e.sum(axis=1, keepdims=True)).max() < 1e-6
        assert p.dtype == np.float32


def test_fixed_point_sum_is_order_free_and_bounded():
    rng = np.random.default_rng(2)
    probs = ref.softmax(rng.normal(0, 4, (16, 3, 9, 9)).astype(np.float32))
    ops = tuple(range(8))
    acc = ref.accumulate(probs, ops, 2, 1)
    perm = rng.permutation(8)
    shuffled = np.concatenate([probs[2 * v:2 * v + 2] for v in perm])
    assert np.array_equal(ref.accumulate(shuffled, tuple(int(v) for v in perm), 2, 1), acc)
    assert acc.max() <= 8 * ref.ONE < 2 ** 63


def test_compose_matches_views():
    img = np.arange(25).reshape(5, 5)
    for a in range(8):
        for b in range(8):
            assert np.array_equal(ref.view(ref.view(img, b), a), ref.view(img, ref.compose(a, b)))
        assert sorted(ref.compose(a, b) for b in range(8)) == list(range(8))
