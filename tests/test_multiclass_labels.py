"""Multi-class labels on the CPU: `rs rasterize --class` and `rs compare --dataset` flag parsing, their validation before the
device check, the per-class CSV rows, and the restatement (tests/multiclass_labels_reference.py) on hand grids with the max
rule's order independence and idempotence."""

import argparse
import itertools
import os

import numpy as np
import pytest
from PIL import Image

import multiclass_labels_reference as mr
from robosat_b200 import compare as C
from robosat_b200.colors import make_palette
from robosat_b200.tiles import Tile


def _parsers():
    from robosat_b200.tools import compare, rasterize

    p = argparse.ArgumentParser()
    sub = p.add_subparsers()
    rasterize.add_parser(sub)
    compare.add_parser(sub)
    return p


def test_flags_parse():
    p = _parsers()
    args = p.parse_args(["rasterize", "f.geojson", "t.csv", "out", "--dataset", "d.toml", "--zoom", "18", "--class", "building"])
    assert args.class_name == "building"
    assert p.parse_args(["rasterize", "f.geojson", "t.csv", "out", "--dataset", "d.toml", "--zoom", "18"]).class_name is None
    args = p.parse_args(["compare", "out", "images", "labels", "m0", "m1", "--csv", "rows.csv", "--dataset", "d.toml"])
    assert (args.masks, args.csv, args.dataset) == (["m0", "m1"], "rows.csv", "d.toml")
    assert p.parse_args(["compare", "out", "images", "labels", "m0"]).dataset is None


def _dataset(tmp_path, classes, colors=None):
    colors = colors if colors is not None else (["denim", "orange", "dark", "red", "pink"] * 60)[:len(classes)]
    path = tmp_path / "dataset.toml"
    path.write_text("[common]\nclasses = [%s]\ncolors = [%s]\n" % (", ".join("'%s'" % c for c in classes), ", ".join("'%s'" % c for c in colors)))
    return str(path)


def _rasterize_args(tmp_path, ds, name, zoom=18, size=64):
    csv = tmp_path / "tiles.csv"
    csv.write_text("1,2,18\n3,4,18\n1,2,18\n")
    (tmp_path / "f.geojson").write_text('{"type": "FeatureCollection", "features": []}')
    return argparse.Namespace(features=str(tmp_path / "f.geojson"), tiles=str(csv), out=str(tmp_path / "out"), dataset=ds, zoom=zoom,
                              size=size, class_name=name)


def _run_rasterize(args):
    from robosat_b200.tools import rasterize as tool

    tool.main(args)


@pytest.mark.parametrize("classes,colors,name,match", [
    (["background", "parking", "building"], None, "road", "not one of the dataset's classes"),
    (["background", "parking", "building"], None, "background", "background class"),
    (["background", "parking", "building"], ["denim", "orange"], "parking", "3 classes and 2 colors"),
    (["background"], None, "background", "1 classes"),
    (["c%d" % i for i in range(257)], None, "c5", "257 classes"),
])
def test_rasterize_class_validation(tmp_path, classes, colors, name, match):
    with pytest.raises(SystemExit, match=match):
        _run_rasterize(_rasterize_args(tmp_path, _dataset(tmp_path, classes, colors), name))
    assert not (tmp_path / "out").exists()


def test_rasterize_class_keeps_the_zoom_and_size_checks(tmp_path):
    ds = _dataset(tmp_path, ["background", "parking", "building"])
    with pytest.raises(AssertionError):
        _run_rasterize(_rasterize_args(tmp_path, ds, "building", zoom=17))
    with pytest.raises(SystemExit, match="--size"):
        _run_rasterize(_rasterize_args(tmp_path, ds, "building", size=4097))


def _save(path, array, mode, bits=None, palette=True):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    im = Image.fromarray(array, mode=mode) if mode in ("P", "L") else Image.fromarray(array)
    if mode == "P" and palette:
        im.putpalette(make_palette("denim", "orange", "dark"))
    im.save(path, **({"bits": bits} if bits else {}))


def _label(tmp_path, x, y):
    return str(tmp_path / "out" / "18" / str(x) / ("%d.png" % y))


@pytest.mark.parametrize("kind,match", [
    ("rgb", "colour type 2"),
    ("gray16", "colour type 0, 16 bits"),
    ("size", "is 32x64, --size is 64"),
    ("jpeg", "not a PNG"),
])
def test_rasterize_class_refuses_existing_labels_before_writing(tmp_path, kind, match):
    ds = _dataset(tmp_path, ["background", "parking", "building"])
    good = _label(tmp_path, 1, 2)
    _save(good, np.zeros((64, 64), np.uint8), "P")
    bad = _label(tmp_path, 3, 4)
    if kind == "rgb":
        _save(bad, np.zeros((64, 64, 3), np.uint8), "RGB")
    elif kind == "gray16":
        _save(bad, np.zeros((64, 64), np.uint16), None)
    elif kind == "size":
        _save(bad, np.zeros((64, 32), np.uint8), "P")
    else:
        os.makedirs(os.path.dirname(bad), exist_ok=True)
        Image.fromarray(np.zeros((64, 64), np.uint8)).save(bad, format="JPEG")
    before = {p: os.stat(p).st_mtime_ns for p in (good, bad)}
    with pytest.raises(SystemExit, match=match) as e:
        _run_rasterize(_rasterize_args(tmp_path, ds, "building"))
    assert bad in str(e.value)
    assert {p: os.stat(p).st_mtime_ns for p in (good, bad)} == before
    assert sorted(os.listdir(tmp_path / "out" / "18")) == ["1", "3"]


def test_rasterize_accepts_every_palette_depth_and_gray_in_the_header_check(tmp_path):
    from robosat_b200.tools.rasterize import check_existing_labels

    tiles = [Tile(i, 0, 18) for i in range(6)]
    for i, (mode, bits) in enumerate([("P", 1), ("P", 2), ("P", 4), ("P", 8), ("L", None)]):
        _save(_label(tmp_path, i, 0), np.zeros((16, 16), np.uint8), mode, bits)
    assert check_existing_labels(str(tmp_path / "out"), tiles, 16) == [True] * 5 + [False]
    depths = [open(_label(tmp_path, i, 0), "rb").read(29)[24:26] for i in range(5)]
    assert depths == [bytes([1, 3]), bytes([2, 3]), bytes([4, 3]), bytes([8, 3]), bytes([8, 0])]  # (bit depth, colour type)


def test_compare_dataset_validation(tmp_path):
    from robosat_b200.tools import compare as tool

    def run(ds, csv="rows.csv"):
        tool.main(argparse.Namespace(out=str(tmp_path / "o"), images="i", labels="l", masks=["m"], minimum=0.0, maximum=1.0, csv=csv, dataset=ds))

    with pytest.raises(SystemExit, match="--dataset needs --csv"):
        run(_dataset(tmp_path, ["background", "parking"]), csv=None)
    for classes, match in ((["background", "17"], "integer"), (["background", "a/b"], "path separator"), (["background", "x", "x"], "more than once"),
                           (["background"], "1 classes"), (["c%d" % i for i in range(257)], "257 classes")):
        with pytest.raises(SystemExit, match=match):
            run(_dataset(tmp_path, classes))
    assert not (tmp_path / "o").exists()
    with pytest.raises(C.CompareError, match="csv"):
        C.compare_device("i", "l", ["m"], str(tmp_path / "o"), classes=["background", "parking"])


def test_class_csv_rows_and_the_out_of_range_message():
    job = C.Job(Tile(5, 6, 18), "i.png", "labels/18/5/6.png", ["m0/18/5/6.png", "m1/18/5/6.png"], (4, 2))
    label = np.array([0, 0, 1, 2, 2, 2, 0, 1], np.uint8)
    masks = np.array([[0, 1, 1, 2, 2, 0, 0, 0], [0, 0, 0, 0, 0, 0, 0, 0]], np.uint8)
    lh, mh, bh, oor = mr.class_counts(label, masks, 4)
    cov = np.array([[0.5, 0.0]])
    rows = C.class_csv_rows([job], lh[None], mh[None], bh[None], cov, ["background", "parking", "building", "road"], 8)
    assert rows[:4] == [
        [18, 5, 6, 0, "background", "0.5", 2, 2, 1, 3, repr(2 / 5)],
        [18, 5, 6, 0, "parking", "0.5", 1, 1, 1, 5, repr(1 / 3)],
        [18, 5, 6, 0, "building", "0.5", 2, 0, 1, 5, repr(2 / 3)],
        [18, 5, 6, 0, "road", "0.5", 0, 0, 0, 8, ""],
    ]
    assert [r[4] for r in rows[4:]] == ["background", "parking", "building", "road"] and rows[4][6:] == [3, 5, 0, 0, repr(3 / 8)]
    want = mr.class_rows(lh, mh, bh, 8)
    assert [[r[3]] + r[6:10] for r in rows] == [[m, tp, fp, fn, tn] for m, _, tp, fp, fn, tn, _ in want]
    assert C.out_of_range_error([job], oor[None], 4) is None
    err = C.out_of_range_error([job], np.array([[0, 0, 3]]), 3)
    assert "tile 18/5/6" in str(err) and "m1/18/5/6.png" in str(err) and "3 pixels" in str(err)
    assert "labels/18/5/6.png" in str(C.out_of_range_error([job], np.array([[1, 0, 0]]), 3))


def test_tile_bytes_add_the_class_counts_only_with_classes():
    base = C.tile_bytes((512, 512), 3, True)
    assert C.tile_bytes((512, 512), 3, True, 0) == base
    assert C.tile_bytes((512, 512), 3, True, 17) == base + 3 * 3 * 17 * 8


def test_class_counts_on_a_hand_grid():
    label = np.array([[0, 1, 2], [2, 2, 7]], np.uint8)
    masks = np.array([[[0, 1, 1], [2, 9, 7]], [[0, 0, 0], [0, 0, 0]]], np.uint8)
    lh, mh, bh, oor = mr.class_counts(label, masks, 3)
    assert lh.tolist() == [1, 1, 3] and mh.tolist() == [[1, 2, 1], [6, 0, 0]] and bh.tolist() == [[1, 1, 1], [1, 0, 0]]
    assert oor.tolist() == [1, 2, 0]


def _square(x0, y0, x1, y1):
    return [np.array([(x0, y0), (x1, y0), (x1, y1), (x0, y1)], np.float64)]


def test_max_rule_on_hand_grids_is_order_independent_and_idempotent():
    ident = (0.0, 1.0, 0.0, 1.0)  # pixel coordinates
    size = 8
    burns = {1: [_square(0, 0, 5, 5)], 2: [_square(3, 3, 8, 6)], 3: [_square(1, 4, 2, 8)]}
    layers = {c: mr.burn_class(ident, p, size, c) for c, p in burns.items()}
    assert layers[1][0, 0] == 1 and layers[1][5, 5] == 0 and layers[2][3, 3] == 2 and layers[2].max() == 2
    results = set()
    for order in itertools.permutations(layers):
        out = np.zeros((size, size), np.uint8)
        for c in order:
            out = np.maximum(out, layers[c])
            assert np.array_equal(np.maximum(out, layers[c]), out)  # repeating a run changes nothing
        results.add(out.tobytes())
    assert len(results) == 1
    out = np.frombuffer(results.pop(), np.uint8).reshape(size, size)
    assert out[4, 4] == 2 and out[4, 1] == 3 and out[1, 1] == 1 and out[7, 7] == 0  # the higher index wins where they overlap
    assert out[6, 1] == 3 and out[0, 6] == 0
