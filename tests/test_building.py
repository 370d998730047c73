"""`rs features --type building` on the CPU: the numpy / scipy restatement against OpenCV, the host polygon step on hand masks,
the command line, the dataset check and the C entry points' validation."""

import argparse
import ctypes

import numpy as np
import pytest

import building_reference as br
from robosat_b200 import _lib
from robosat_b200 import features as F
from robosat_b200.tiles import Tile

cv2 = pytest.importorskip("cv2")

TILE = Tile(70100, 104000, 18)


def _canonical(cv_labels):
    """OpenCV component labels -> (smallest pixel index of each pixel's component or -1, its area): OpenCV's numbering is not
    always in raster order, so only the relabelled form is comparable"""
    flat = cv_labels.ravel()
    ids, first, area = np.unique(flat, return_index=True, return_counts=True)
    root = np.full(ids.max() + 1, -1, np.int64)
    size = np.zeros(ids.max() + 1, np.int64)
    root[ids], size[ids] = first, area
    root[0], size[0] = -1, 0
    return root[cv_labels], size[cv_labels]


def _noise(seed, shape, density):
    return (np.random.RandomState(seed).rand(*shape) < density).astype(np.uint8)


@pytest.mark.parametrize("connectivity", [4, 8])
@pytest.mark.parametrize("density", [0.3, 0.5, 0.6])
@pytest.mark.parametrize("shape", [(512, 512), (509, 131), (1, 77), (77, 1)])
def test_components_match_opencv(connectivity, density, shape):
    m = _noise(int(density * 10) + shape[1], shape, density)
    for value in (0, 1):
        plane = (m == value).astype(np.uint8)
        _, cv_labels = cv2.connectedComponents(plane, connectivity=connectivity)
        want_root, want_area = _canonical(cv_labels)
        root, area, _ = br.components(m, value, connectivity)
        assert np.array_equal(root, want_root) and np.array_equal(area, want_area), value


def test_border_flags():
    m = np.zeros((9, 9), np.uint8)
    m[0, 3] = m[4, 4] = m[8, 8] = m[3:6, 0] = 1
    root, area, touches = br.components(m, 1, 8)
    assert touches[0, 3] and touches[8, 8] and touches[4, 0] and not touches[4, 4]
    assert area[4, 0] == 3 and root[5, 0] == 3 * 9
    _, _, bg = br.components(m, 0, 4)
    assert bg[4, 5]  # the background is one component that touches the border


@pytest.mark.parametrize("seed", range(3))
def test_opening_matches_opencv(seed):
    labels = np.random.RandomState(seed).randint(0, 3, size=(200, 150)).astype(np.uint8)
    labels[20:90, 30:100] = 2
    el = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (5, 5))
    want = cv2.morphologyEx((labels == 2).astype(np.uint8), cv2.MORPH_OPEN, el)
    assert np.array_equal(br.opened(labels, 2), want)


def _cleaned(mask):
    """steps 3-4 on a hand mask that the opening leaves as it is"""
    return br.fill(br.drop(mask, F.BuildingHandler.min_area), F.BuildingHandler.min_hole_area)


def _features(mask):
    return F.polygons_from_filled(TILE, _cleaned(mask), F.BuildingHandler.simplify_epsilon)


def _pixel_rings(feature, shape=(64, 64)):
    """lon/lat rings back to pixel coordinates"""
    west, south, east, north = F.bounds(TILE)
    return [[(round((lon - west) / (east - west) * shape[1]), round((north - lat) / (north - south) * shape[0])) for lon, lat in ring[:-1]]
            for ring in feature["geometry"]["coordinates"]]


def test_two_houses():
    m = np.zeros((64, 64), np.uint8)
    m[5:20, 5:25] = 1
    m[30:50, 35:60] = 1
    feats, warnings = _features(m)
    assert warnings == [] and len(feats) == 2
    assert sorted(sorted(_pixel_rings(f)[0]) for f in feats) == [[(5, 5), (5, 19), (24, 5), (24, 19)],
                                                              [(35, 30), (35, 49), (59, 30), (59, 49)]]
    assert all(f["properties"] == {} and f["geometry"]["type"] == "Polygon" for f in feats)


def test_diagonal_touch_is_one_component():
    m = np.zeros((64, 64), np.uint8)
    m[10:16, 10:16] = 1  # 36 px each: alone, both would be specks
    m[16:22, 16:22] = 1
    assert np.array_equal(_cleaned(m), m)
    # the traced ring passes the touching corner twice, which no valid polygon does; the simplified ring cuts across it
    (feat,), warnings = _features(m)
    assert warnings == [] and len(feat["geometry"]["coordinates"]) == 1


@pytest.mark.parametrize("hw, kept", [((7, 9), False), ((8, 8), True)])
def test_speck_threshold(hw, kept):
    m = np.zeros((40, 40), np.uint8)
    m[10:10 + hw[0], 12:12 + hw[1]] = 1
    assert np.array_equal(_cleaned(m), m if kept else np.zeros_like(m))
    assert len(_features(m)[0]) == int(kept)


@pytest.mark.parametrize("hw, filled", [((7, 9), True), ((8, 8), False)])
def test_courtyard_threshold(hw, filled):
    m = np.zeros((64, 64), np.uint8)
    m[10:40, 10:40] = 1
    m[20:20 + hw[0], 20:20 + hw[1]] = 0
    got = _cleaned(m)
    assert got[20:20 + hw[0], 20:20 + hw[1]].all() == filled
    (feat,), warnings = _features(m)
    assert warnings == [] and len(feat["geometry"]["coordinates"]) == (1 if filled else 2)


def test_hole_touching_the_tile_border_is_never_filled():
    m = np.zeros((64, 64), np.uint8)
    m[0:30, 10:40] = 1
    m[0:3, 20:23] = 0  # a 9 px notch open to the top edge: background that touches the border, not a hole
    assert np.array_equal(_cleaned(m), m)
    (feat,), _ = _features(m)
    assert len(feat["geometry"]["coordinates"]) == 1


def test_building_cut_by_the_tile_edge():
    m = np.zeros((64, 64), np.uint8)
    m[40:64, 50:64] = 1
    (feat,), warnings = _features(m)
    assert warnings == []
    (ring,) = _pixel_rings(feat)
    assert sorted(ring) == [(50, 40), (50, 63), (63, 40), (63, 63)]


def test_empty_tile():
    assert _features(np.zeros((64, 64), np.uint8)) == ([], [])


def test_simplification_falls_back_to_the_traced_rings(monkeypatch):
    m = np.zeros((64, 64), np.uint8)
    m[10:40, 10:40] = 1
    calls = []

    def valid(rings):
        calls.append(rings)
        return len(calls) > 1  # the simplified polygon is rejected, the traced one accepted

    monkeypatch.setattr(F, "polygon_is_valid", valid)
    (feat,), warnings = _features(m)
    assert warnings == [] and len(calls) == 2
    monkeypatch.setattr(F, "polygon_is_valid", lambda rings: False)
    assert _features(m) == ([], [F.W_INVALID])


def test_restatement_path_on_a_three_class_mask():
    labels = np.zeros((128, 128), np.uint8)
    labels[10:60, 10:60] = 2
    labels[30:35, 30:36] = 0       # 30 px courtyard: filled
    labels[70:120, 70:120] = 2
    labels[85:100, 85:100] = 1     # 225 px courtyard of another class: kept
    labels[5:9, 100:104] = 2       # 16 px speck: the opening removes most of it, the drop the rest
    labels[100:120, 5:40] = 1      # parking
    feats, warnings = br.cpu_features(TILE, labels, 2)
    assert warnings == [] and sorted(len(f["geometry"]["coordinates"]) for f in feats) == [1, 2]


def _parser():
    from robosat_b200.tools import features as tool

    p = argparse.ArgumentParser()
    tool.add_parser(p.add_subparsers())
    return p, tool


def test_parser_takes_building():
    p, tool = _parser()
    args = p.parse_args(["features", "masks/", "--type", "building", "--dataset", "dataset.toml", "out.geojson"])
    assert (args.type, args.func) == ("building", tool.main)
    assert tool.handlers["building"] is F.BuildingHandler


def test_dataset_without_the_class_exits_naming_it(tmp_path):
    _, tool = _parser()
    ds = tmp_path / "dataset.toml"
    ds.write_text("[common]\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n")
    masks = tmp_path / "masks"
    masks.mkdir()
    with pytest.raises(SystemExit) as e:
        tool.main(argparse.Namespace(masks=str(masks), type="building", dataset=str(ds), out=str(tmp_path / "out.geojson")))
    assert "building" in str(e.value)


def test_zoom_other_than_18_raises():
    h = F.BuildingHandler()
    with pytest.raises(NotImplementedError, match="Building"):
        h.apply(Tile(1, 2, 17), np.zeros((8, 8), np.uint8))
    with pytest.raises(NotImplementedError, match="Building"):
        h.apply_batch([Tile(1, 2, 18), Tile(1, 2, 19)], None, 1)


def test_handler_defaults():
    H = F.BuildingHandler
    assert (H.kernel_size_denoise, H.min_area, H.min_hole_area, H.simplify_epsilon) == (5, 64, 64, 1.0)


def test_label_validation_runs_before_the_device_check():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 64)()
    lab = (ctypes.c_int32 * 64)()
    area = (ctypes.c_int32 * 64)()
    cnt = (ctypes.c_int32 * 4)()

    def comp(N=1, H=4, W=4, stride=16, value=1, conn=8, planes=buf, labels=lab, areas=area):
        return lib.rsb_label_components(planes, stride, N, H, W, value, conn, labels, areas, None)

    assert comp() == -3                                             # valid, but no sm_90 device
    assert comp(conn=4, value=0) == -3
    assert comp(planes=None) == -1
    assert comp(areas=None) == -1
    assert comp(areas=lab) == -1 and "alias" in _lib.last_error()
    assert comp(stride=15) == -1 and "image_stride" in _lib.last_error()
    assert comp(H=8193, stride=8193 * 4) == -4
    assert comp(W=0) == -4
    assert comp(N=0) == -4
    assert comp(value=256) == -1
    assert comp(conn=6) == -1 and "connectivity" in _lib.last_error()

    def clean(min_area=64, min_hole=64, stride=16, out=buf, stats=area, counts=cnt):
        return lib.rsb_building_clean(buf, stride, 1, 4, 4, min_area, min_hole, lab, stats, out, counts, None)

    assert clean() == -3
    assert clean(counts=None) == -1
    assert clean(out=None) == -1
    assert clean(stats=lab) == -1 and "alias" in _lib.last_error()
    assert clean(min_area=-1) == -1
    assert clean(min_hole=-1) == -1
    assert clean(stride=3) == -1
