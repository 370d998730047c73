"""`rs predict` / `rs masks --dataset` for models of more than two classes, on the host: the numpy restatement's agreement with the
binary definition, its tie rule, the class-name check and the `rs masks` flag."""

import argparse

import numpy as np
import pytest

import multiclass_reference as ref
from robosat_b200.tools import masks, predict


def test_two_class_restatement_plane_one_is_the_binary_bins():
    rng = np.random.RandomState(0)
    logits = (rng.randn(3, 2, 40, 36) * 4).astype(np.float32)
    logits[0, 1, 10, 10], logits[0, 0, 10, 10] = 80.0, -80.0  # saturated: p = 1 -> bin 256 wraps to 0
    for overlap in (0, 4, 8):
        both = ref.predict_bins(logits, overlap)
        assert both.shape == (3, 2, 40 - 2 * overlap, 36 - 2 * overlap)
        assert np.array_equal(both[:, 1], ref.predict_bins_binary(logits, overlap)), overlap
    assert ref.predict_bins(logits, 0)[0, 1, 10, 10] == 0


def _hand_ties():
    """K = 2 models, C = 3 classes, 4 pixels: exact ties between classes (0, 1), (1, 2), (0, 1, 2) and no tie"""
    q = np.zeros((2, 3, 4), dtype=np.uint8)
    q[0, :, 0], q[1, :, 0] = (100, 155, 0), (155, 100, 0)    # class 0 == class 1 > class 2 -> 0
    q[0, :, 1], q[1, :, 1] = (0, 100, 155), (10, 155, 100)   # class 1 == class 2 > class 0 -> 1
    q[0, :, 2], q[1, :, 2] = (85, 85, 85), (85, 85, 85)      # all equal -> 0
    q[0, :, 3], q[1, :, 3] = (0, 0, 255), (0, 0, 255)        # class 2
    return q


@pytest.mark.parametrize("weights", [None, [0.5, 0.5], [1.0, 1.0]])
def test_softvote_ties_pick_the_first_class(weights):
    q = _hand_ties()
    got = ref.softvote(q, weights)
    assert got.tolist() == [0, 1, 0, 2]
    direct = np.argmax(np.average(np.linspace(0, 1, 256)[q], axis=0, weights=weights), axis=0)
    assert np.array_equal(got, direct)


def test_softvote_agrees_with_numpy_on_random_planes():
    rng = np.random.RandomState(1)
    for K, C, w in [(1, 3, None), (3, 6, [0.2, 0.3, 0.5]), (2, 4, None)]:
        q = rng.randint(0, 256, size=(K, C, 16, 12)).astype(np.uint8)
        want = np.average(np.linspace(0, 1, 256)[q], axis=0, weights=w).argmax(axis=0)
        assert np.array_equal(ref.softvote(q, w), want)


def test_class_names_are_checked():
    assert predict.check_class_names(["background", "parking", "building"]) == ["background", "parking", "building"]
    assert predict.check_class_names(["a.b", "road-1", "x y"]) == ["a.b", "road-1", "x y"]
    bad = [
        (["background", ""], "non-empty"),
        (["background", "parking", "parking"], "'parking' appears more than once"),
        (["background", "a/b", "c"], "'a/b' must not contain a path separator"),
        (["background", "a\\b", "c"], "path separator"),
        (["background", "a\0b", "c"], "NUL"),
        (["background", "..", "c"], "'..'"),
        (["background", ".", "c"], "'.'"),
        (["background", "18", "c"], "'18' is an integer"),
        (["background", "-3", "c"], "integer"),
        (["background", 7, "c"], "non-empty string"),
    ]
    for names, message in bad:
        with pytest.raises(ValueError, match=message.replace(".", r"\.").replace("(", r"\(")):
            predict.check_class_names(names)


def test_predict_main_rejects_bad_names_before_any_work(tmp_path):
    (tmp_path / "dataset.toml").write_text("[common]\ndataset = 'x'\nclasses = ['background', 'parking', '17']\ncolors = ['denim', 'orange', 'red']\n")
    args = argparse.Namespace(dataset=str(tmp_path / "dataset.toml"), model=str(tmp_path / "missing.toml"))
    with pytest.raises(SystemExit, match="'17' is an integer"):
        predict.main(args)


def test_masks_parser_dataset_flag():
    parser = argparse.ArgumentParser()
    masks.add_parser(parser.add_subparsers())
    a = parser.parse_args(["masks", "out", "p1", "p2", "--weights", "0.25", "0.75"])
    assert vars(a) == {"masks": "out", "probs": ["p1", "p2"], "weights": [0.25, 0.75], "dataset": None, "func": masks.main}
    b = parser.parse_args(["masks", "out", "p1", "--dataset", "d.toml"])
    assert b.dataset == "d.toml" and b.probs == ["p1"] and b.weights is None
