"""Multi-class labels on the H100: `rs rasterize --class` against the restatement (tests/multiclass_labels_reference.py) and the
default run, its merge with every accepted label flavour and its refusals, rsb_compare_class_counts against np.bincount,
`rs compare --csv --dataset` end to end, and the chain rasterize -> weights -> train -> compare on a three-class dataset."""

import argparse
import csv
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import multiclass_labels_reference as mr
import rasterize_reference as rr
from robosat_b200 import compare as C
from robosat_b200 import rasterize as RZ
from robosat_b200.colors import make_palette
from robosat_b200.tiles import Tile

pytestmark = pytest.mark.gpu

CLASSES = ["background", "parking", "building"]
COLORS = ["denim", "orange", "dark"]


def _dataset(path, classes=CLASSES, colors=COLORS, root=None, weights=None):
    text = "[common]\nclasses = [%s]\ncolors = [%s]\n" % (", ".join("'%s'" % c for c in classes), ", ".join("'%s'" % c for c in colors))
    if root is not None:
        text += "dataset = '%s'\n" % root
    if weights is not None:
        text += "[weights]\nvalues = [%s]\n" % ", ".join(repr(float(w)) for w in weights)
    path.write_text(text)
    return str(path)


def _rasterize(features, tiles_csv, out, ds, size, name=None, batch=64):
    from robosat_b200.tools import rasterize as tool

    ns = argparse.Namespace(features=features, tiles=tiles_csv, out=str(out), dataset=ds, zoom=18, size=size)
    if name is not None:
        ns.class_name = name
    tool.main(ns, batch=batch)


def _files(root):
    root = str(root)
    return {os.path.relpath(os.path.join(d, f), root): open(os.path.join(d, f), "rb").read() for d, _, fs in os.walk(root) for f in fs}


def _write_tiles(path, tiles):
    path.write_text("".join("%d,%d,%d\n" % tuple(t) for t in tiles))
    return str(path)


def test_class_run_on_two_classes_is_the_default_run(cuda_device, tmp_path):
    g = rr.load_golden()
    features = tmp_path / "f.geojson"
    features.write_text(json.dumps(g["features"]))
    tiles_csv = _write_tiles(tmp_path / "tiles.csv", g["tiles"])
    ds = _dataset(tmp_path / "d.toml", ["background", "parking"], ["denim", "orange"])
    _rasterize(str(features), tiles_csv, tmp_path / "default", ds, 512)
    _rasterize(str(features), tiles_csv, tmp_path / "class", ds, 512, name="parking")
    default, klass = _files(tmp_path / "default"), _files(tmp_path / "class")
    assert len(default) == 4 and default == klass
    for t, mask in g["masks"].items():
        assert np.array_equal(np.array(Image.open(str(tmp_path / "class" / str(t[2]) / str(t[0]) / ("%d.png" % t[1])))), mask)


def _lonlat(X, Y):
    return [float(np.degrees(X / RZ.R)), float(np.degrees(2 * np.arctan(np.exp(Y / RZ.R)) - np.pi / 2))]


def _features(rng, base, n, block):
    """n seeded polygons over a block x block area from `base`, as GeoJSON features and as the Mercator rings the tool burns"""
    left, bottom, right, top = RZ.xy_bounds(base)
    side = right - left
    feats = []
    for _ in range(n):
        cu, cv, r = rng.uniform(-0.2, block + 0.2, 2).tolist() + [rng.uniform(0.05, 0.5)]
        a = np.sort(rng.uniform(0, 2 * np.pi, rng.randint(3, 10)))
        ring = [_lonlat(left + (cu + r * np.cos(t)) * side, top - (cv + r * np.sin(t)) * side) for t in a]
        feats.append({"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [ring + [ring[0]]]}})
    polygons, warnings = RZ.polygons_from_features(feats)
    assert not warnings
    return {"type": "FeatureCollection", "features": feats}, polygons


def _two_class_inputs(tmp_path, size):
    rng = np.random.RandomState(11)
    base = Tile(70500, 104100, 18)
    tiles = [Tile(base.x + dx, base.y + dy, 18) for dy in range(3) for dx in range(3)]
    inputs = {}
    for name, n in (("parking", 25), ("building", 60)):
        fc, polygons = _features(rng, base, n, 3)
        path = tmp_path / ("%s.geojson" % name)
        path.write_text(json.dumps(fc))
        inputs[name] = (str(path), polygons)
    return tiles, _write_tiles(tmp_path / "tiles.csv", tiles + [tiles[4]]), inputs


def _want(tiles, inputs, size):
    want = {}
    for t in tiles:
        out = None
        for name, (_, polygons) in inputs.items():
            out = mr.rasterize_class(t, polygons, size, CLASSES.index(name), out)
        want[t] = out
    return want


def test_overlapping_classes_in_either_order(cuda_device, tmp_path):
    size = 96
    tiles, tiles_csv, inputs = _two_class_inputs(tmp_path, size)
    ds = _dataset(tmp_path / "d.toml")
    for order, batch in ((("parking", "building"), 64), (("building", "parking"), 4)):
        for name in order:
            _rasterize(inputs[name][0], tiles_csv, tmp_path / "-".join(order), ds, size, name=name, batch=batch)
    a, b = _files(tmp_path / "parking-building"), _files(tmp_path / "building-parking")
    assert len(a) == len(tiles) and a == b
    want = _want(tiles, inputs, size)
    overlap = 0
    for t in tiles:
        im = Image.open(str(tmp_path / "parking-building" / "18" / str(t.x) / ("%d.png" % t.y)))
        assert im.mode == "P" and im.getpalette()[:9] == make_palette(*COLORS)
        got = np.array(im)
        assert np.array_equal(got, want[t]), t
        overlap += int((mr.burn_class(rr.transform(t, size), inputs["parking"][1], size, 1) & (got == 2)).sum())
    assert overlap > 0  # building won over parking somewhere
    _rasterize(inputs["building"][0], tiles_csv, tmp_path / "parking-building", ds, size, name="building")
    assert _files(tmp_path / "parking-building") == a


def _save_label(path, array, mode, bits=None):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    im = Image.fromarray(array, mode=mode)
    if mode == "P":
        im.putpalette(make_palette(*COLORS, "blue"))
    im.save(path, **({"bits": bits} if bits else {}))


def test_existing_labels_of_every_flavour_merge_as_the_reference(cuda_device, tmp_path):
    size = 64
    tiles, tiles_csv, inputs = _two_class_inputs(tmp_path, size)
    ds = _dataset(tmp_path / "d.toml", CLASSES + ["water"], COLORS + ["blue"])
    out = tmp_path / "out"
    rng = np.random.RandomState(3)
    prev = {}
    for t, (mode, bits) in zip(tiles, [("P", 1), ("P", 2), ("P", 4), ("P", 8), ("L", None)]):
        hi = 2 if bits == 1 else 4
        arr = rng.randint(0, hi, size=(size, size)).astype(np.uint8)
        path = str(out / "18" / str(t.x) / ("%d.png" % t.y))
        _save_label(path, arr, mode, bits)
        read = np.array(Image.open(path))
        assert np.array_equal(read, arr)
        prev[t] = read
    _rasterize(inputs["parking"][0], tiles_csv, out, ds, size, name="parking", batch=3)
    _, polygons = inputs["parking"]
    for t in tiles:
        want = mr.burn_class(rr.transform(t, size), polygons, size, 1)
        if t in prev:
            want = np.maximum(want, prev[t])
        got = np.array(Image.open(str(out / "18" / str(t.x) / ("%d.png" % t.y))))
        assert np.array_equal(got, want), t


def test_refused_existing_labels_name_the_file(cuda_device, tmp_path):
    size = 64
    tiles, tiles_csv, inputs = _two_class_inputs(tmp_path, size)
    ds = _dataset(tmp_path / "d.toml")
    for kind in ("rgb", "size", "value"):
        out = tmp_path / kind
        bad = str(out / "18" / str(tiles[5].x) / ("%d.png" % tiles[5].y))
        if kind == "rgb":
            _save_label(bad, np.zeros((size, size, 3), np.uint8), "RGB")
        elif kind == "size":
            _save_label(bad, np.zeros((size, size + 1), np.uint8), "P")
        else:
            arr = np.zeros((size, size), np.uint8)
            arr[7, 9] = 3
            _save_label(bad, arr, "P")
        with pytest.raises(SystemExit) as e:
            _rasterize(inputs["building"][0], tiles_csv, out, ds, size, name="building", batch=4)
        assert bad in str(e.value), kind
        written = sorted(_files(out))
        if kind == "value":
            assert "value 3" in str(e.value) and len(written) == 1 + 4  # the first batch of 4 tiles was written, then it stopped
        else:
            assert written == [os.path.relpath(bad, str(out))]


def _seeded_planes(rng, N, M, hw, C):
    """label and masks with runs of classes, noise, values >= C, and empty planes"""
    planes = np.zeros((N, 1 + M, hw), np.uint8)
    for n in range(N):
        for p in range(1 + M):
            kind = rng.randint(4)
            if kind == 0:
                continue
            if kind == 1:
                planes[n, p] = rng.randint(0, 256, hw)
            else:
                runs = np.repeat(rng.randint(0, C, hw // 37 + 1), 37)[:hw]
                planes[n, p] = np.where(rng.rand(hw) < 0.01, rng.randint(0, 256, hw), runs)
    return planes


def _run_class_counts(planes, C_):
    N, P, hw = planes.shape
    pitch = C.pitch_of(hw)
    padded = np.full((N, P, pitch), 0xEE, np.uint8)  # padding past hw must not count
    padded[..., :hw] = planes
    d = torch.from_numpy(padded).cuda()
    out = C.class_counts_device(d[:, 1:].contiguous(), d[:, 0].contiguous(), hw, C_)
    return [t.cpu().numpy() for t in out]


@pytest.mark.parametrize("w,h", [(512, 512), (509, 131), (1, 1)])
@pytest.mark.parametrize("C_", [2, 3, 17, 256])
def test_class_counts_match_numpy(cuda_device, w, h, C_):
    rng = np.random.RandomState(w + h + C_)
    for M in (1, 2, 3, 4):
        N = 3
        planes = _seeded_planes(rng, N, M, w * h, C_)
        if C_ < 256 and w * h > 1:
            planes[0, 0, 5] = C_  # a value >= C in the label and in a mask
            planes[1, M, 7] = 255
        lh, mh, bh, oor = _run_class_counts(planes, C_)
        assert lh.shape == (N, C_) and mh.shape == (N, M, C_) and bh.shape == (N, M, C_) and oor.shape == (N, 1 + M)
        for n in range(N):
            want = mr.class_counts(planes[n, 0], planes[n, 1:], C_)
            for got, exp in zip((lh[n], mh[n], bh[n], oor[n]), want):
                assert np.array_equal(got, exp), (w, h, C_, M, n)
        if C_ < 256 and w * h > 1:
            assert oor[0, 0] >= 1 and oor[1, M] >= 1


def test_class_counts_do_not_depend_on_the_batch_split(cuda_device):
    rng = np.random.RandomState(5)
    planes = _seeded_planes(rng, 7, 3, 509 * 509, 5)
    whole = _run_class_counts(planes, 5)
    for split in (((0, 2), (2, 7)), ((0, 1), (1, 4), (4, 7))):
        parts = [_run_class_counts(planes[a:b], 5) for a, b in split]
        for k in range(4):
            assert np.array_equal(whole[k], np.concatenate([p[k] for p in parts])), (split, k)
    d = torch.from_numpy(np.zeros((1, 2, 16), np.uint8)).cuda()
    with pytest.raises(Exception, match="bad arguments"):
        C.class_counts_device(d[:, 1:], d[:, 0], 16, 257)
    hw = 509 * 509
    padded = np.zeros((2, 3, C.pitch_of(hw)), np.uint8)
    padded[..., :hw] = planes[:2, 1:]
    no_label = [t.cpu().numpy() for t in C.class_counts_device(torch.from_numpy(padded).cuda(), None, hw, 5)]
    for n in range(2):  # without labels every label pixel is class 0
        want = mr.class_counts(np.zeros(hw, np.uint8), planes[n, 1:], 5)
        assert all(np.array_equal(g[n], w) for g, w in zip(no_label, want)), n


def _write_planes(root, sub, tiles, planes, palette_colors=COLORS):
    for t, arr in zip(tiles, planes):
        path = os.path.join(root, sub, "18", str(t.x), "%d.png" % t.y)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        im = Image.fromarray(arr, mode="P")
        im.putpalette(make_palette(*palette_colors))
        im.save(path)


def _check_class_csv(path, tiles, labels, masks, classes, size):
    rows = list(csv.reader(open(path)))
    assert rows[0] == C.CLASS_CSV_COLUMNS
    hw = size * size
    expect = []
    for i, t in enumerate(tiles):
        lh, mh, bh, _ = mr.class_counts(labels[i], masks[:, i], len(classes))
        for m, c, tp, fp, fn, tn, iou in mr.class_rows(lh, mh, bh, hw):
            cov = float((masks[m, i] != 0).sum()) / hw
            expect.append([str(t.z), str(t.x), str(t.y), str(m), classes[c], repr(cov), str(tp), str(fp), str(fn), str(tn),
                           repr(iou) if iou is not None else ""])
    assert rows[1:] == expect
    return rows[1:]


def test_compare_csv_dataset_end_to_end(cuda_device, tmp_path):
    from robosat_b200.tools import compare as tool

    rng = np.random.RandomState(9)
    size, M = 64, 2
    tiles = sorted([Tile(100 + i % 3, 200 + i // 3, 18) for i in range(7)], key=lambda t: (t.z, t.x, t.y))
    root = str(tmp_path)
    labels = np.repeat(rng.randint(0, 3, (7, size, size // 8)), 8, axis=2).astype(np.uint8)
    masks = np.where(rng.rand(M, 7, size, size) < 0.2, rng.randint(0, 3, (M, 7, size, size)), labels[None]).astype(np.uint8)
    masks[1, 2] = 0  # a mask without foreground: iou of the absent classes is empty
    for i, t in enumerate(tiles):
        path = os.path.join(root, "images", "18", str(t.x), "%d.png" % t.y)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        Image.fromarray(rng.randint(0, 256, (size, size, 3)).astype(np.uint8)).save(path)
    _write_planes(root, "labels", tiles, labels)
    for m in range(M):
        _write_planes(root, "m%d" % m, tiles, masks[m])
    ds = _dataset(tmp_path / "d.toml")
    ns = lambda out, rows, dataset: argparse.Namespace(out=os.path.join(root, out), images=os.path.join(root, "images"),  # noqa: E731
                                                       labels=os.path.join(root, "labels"), masks=[os.path.join(root, "m%d" % m) for m in range(M)],
                                                       minimum=0.0, maximum=1.0, csv=os.path.join(root, rows), dataset=dataset)
    tool.main(ns("out", "rows.csv", ds))
    got = _check_class_csv(os.path.join(root, "rows.csv"), tiles, labels, masks, CLASSES, size)
    assert len(got) == 7 * M * 3
    # the composites are the ones written without --dataset
    tool.main(ns("out_plain", "plain.csv", None))
    assert _files(os.path.join(root, "out")) == _files(os.path.join(root, "out_plain"))
    assert list(csv.reader(open(os.path.join(root, "plain.csv"))))[0] == C.CSV_COLUMNS
    # small batches: the same rows
    C.compare_device(os.path.join(root, "images"), os.path.join(root, "labels"), [os.path.join(root, "m0"), os.path.join(root, "m1")],
                     os.path.join(root, "out_small"), csv=os.path.join(root, "small.csv"), classes=CLASSES,
                     budget=2 * C.tile_bytes((size, size), M, True, 3))
    assert open(os.path.join(root, "small.csv")).read() == open(os.path.join(root, "rows.csv")).read()
    # a mask value outside the classes names the tile and the file
    bad = masks[1].copy()
    bad[4, 3, 3] = 3
    _write_planes(root, "m1", tiles, bad, COLORS + ["blue"])
    with pytest.raises(SystemExit) as e:
        tool.main(ns("out_bad", "bad.csv", ds))
    assert "tile 18/%d/%d" % (tiles[4].x, tiles[4].y) in str(e.value) and os.path.join(root, "m1", "18", str(tiles[4].x)) in str(e.value)


def test_chain_rasterize_weights_train_compare(cuda_device, tmp_path, capsys, monkeypatch):
    from robosat_b200.tools import compare as compare_tool
    from robosat_b200.tools import train as train_tool
    from robosat_b200.tools import weights as weights_tool
    from robosat_b200.tools.train import check_mask_range
    from robosat_b200.tools.weights import weights_from_counts
    from robosat_b200 import synth

    size = 128
    tiles, tiles_csv, inputs = _two_class_inputs(tmp_path, size)
    ds_root = tmp_path / "ds"
    ds = _dataset(tmp_path / "d.toml", root=str(ds_root))
    labels_dir = ds_root / "training" / "labels"
    for name in ("building", "parking"):
        _rasterize(inputs[name][0], tiles_csv, labels_dir, ds, size, name=name)
    capsys.readouterr()
    labels = np.stack([np.array(Image.open(str(labels_dir / "18" / str(t.x) / ("%d.png" % t.y)))) for t in tiles])
    assert np.array_equal(labels, np.stack([_want(tiles, inputs, size)[t] for t in tiles]))
    counts = np.bincount(labels.ravel(), minlength=3)
    assert len(counts) == 3 and (counts > 0).all()

    weights_tool.main(argparse.Namespace(dataset=ds))
    printed = capsys.readouterr().out.strip()
    weights = weights_from_counts(counts, labels.size)
    assert printed == str(weights)
    check_mask_range(torch.from_numpy(labels), None, 3)

    # one epoch of rs train on the labels, with the weights just computed
    images = synth.make_tiles_u8(len(tiles), size, seed=4).numpy()
    for split in ("training", "validation"):
        for t, img, lab in zip(tiles, images, labels):
            for sub, arr in (("images", img), ("labels", lab)):
                path = ds_root / split / sub / "18" / str(t.x) / ("%d.png" % t.y)
                path.parent.mkdir(parents=True, exist_ok=True)
                if split == "training" and sub == "labels":
                    continue
                im = Image.fromarray(arr, mode="P" if sub == "labels" else None)
                if sub == "labels":
                    im.putpalette(make_palette(*COLORS))
                im.save(str(path))
    ds = _dataset(tmp_path / "d.toml", root=str(ds_root), weights=weights)
    ck = tmp_path / "ck"
    (tmp_path / "model.toml").write_text("[common]\ncuda = true\nbatch_size = 3\nimage_size = %d\ncheckpoint = '%s'\n[opt]\nepochs = 1\nlr = 0.0001\n"
                                         "loss = 'CrossEntropy'\n" % (size, ck))
    monkeypatch.setenv("RSB_GPUS", "1")
    train_tool.main(argparse.Namespace(model=str(tmp_path / "model.toml"), dataset=ds, checkpoint=None, resume=False, workers=0))
    log = open(ck / "log").read()
    assert "Epoch: 1/1" in log and os.path.exists(ck / "checkpoint-00001-of-00001.pth")

    # the labels as their own mask: iou 1.0 for every class present in a tile, empty for the absent ones
    rows_path = str(tmp_path / "rows.csv")
    compare_tool.main(argparse.Namespace(out=str(tmp_path / "cmp"), images=str(ds_root / "training" / "images"), labels=str(labels_dir),
                                         masks=[str(labels_dir)], minimum=0.0, maximum=1.0, csv=rows_path, dataset=ds))
    rows = list(csv.reader(open(rows_path)))[1:]
    assert len(rows) == len(tiles) * 3
    order = sorted(range(len(tiles)), key=lambda i: (tiles[i].z, tiles[i].x, tiles[i].y))
    for k, i in enumerate(order):
        present = np.bincount(labels[i].ravel(), minlength=3) > 0
        for c in range(3):
            row = rows[3 * k + c]
            assert row[4] == CLASSES[c] and int(row[7]) == int(row[8]) == 0
            assert row[10] == ("1.0" if present[c] else ""), (tiles[i], c)
