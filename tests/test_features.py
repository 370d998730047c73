"""`rs features` on the CPU: structuring elements, the numpy restatement of the morphology against OpenCV, the host geometry
against the reference's golden output, tile bounds, polygon validity, the command line and the C entry point's validation."""

import argparse
import ctypes
import math

import numpy as np
import pytest

import features_reference as fr
from robosat_b200 import _lib
from robosat_b200 import features as F
from robosat_b200.tiles import Tile

cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("k", range(1, 65))
def test_ellipse_spans_match_opencv(k):
    want = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (k, k))
    assert np.array_equal(fr.element(F.ellipse_op(k, False)), want)


def test_rect_and_cross_spans_match_opencv():
    for kh, kw in ((1, 1), (3, 5), (4, 4), (7, 2)):
        assert np.array_equal(fr.element(F.MorphOp(0, fr.rect_spans(kh, kw), kw, (0, 0))), cv2.getStructuringElement(cv2.MORPH_RECT, (kw, kh)))
        assert np.array_equal(fr.element(F.MorphOp(0, fr.cross_spans(kh, kw), kw, (0, 0))), cv2.getStructuringElement(cv2.MORPH_CROSS, (kw, kh)))


@pytest.mark.parametrize("shape", ["rect", "ellipse", "cross"])
@pytest.mark.parametrize("k", [1, 2, 3, 5, 8, 20, 21])
@pytest.mark.parametrize("hw", [(1, 1), (7, 33), (33, 7), (64, 70)])
def test_numpy_restatement_matches_opencv(shape, k, hw):
    rng = np.random.RandomState(k * 7 + hw[1])
    m = (rng.rand(*hw) < 0.6).astype(np.uint8)
    el = fr.element(fr.op(shape, k, False))
    for dilate, fn in ((False, cv2.erode), (True, cv2.dilate)):
        assert np.array_equal(fr.morph_ref(m, [fr.op(shape, k, dilate)]), fn(m, el)), dilate
    opened = [fr.op(shape, k, False), fr.op(shape, k, True)]
    assert np.array_equal(fr.morph_ref(m, opened), cv2.morphologyEx(m, cv2.MORPH_OPEN, el))
    assert np.array_equal(fr.morph_ref(m, opened[::-1]), cv2.morphologyEx(m, cv2.MORPH_CLOSE, el))


def test_numpy_restatement_with_off_centre_anchor():
    rng = np.random.RandomState(1)
    m = (rng.rand(40, 45) < 0.5).astype(np.uint8)
    ops = [fr.op("ellipse", 9, False, anchor=(1, 7)), fr.op("rect", 4, True, anchor=(3, 0)), fr.op("cross", 5, True, anchor=(2, 2))]
    assert np.array_equal(fr.morph_ref(m, ops), fr.cv_ref(m, ops))


@pytest.fixture(scope="module")
def golden():
    return fr.load_golden()


def test_numpy_restatement_matches_golden_grown_masks(golden):
    for case in golden:
        if case["labels"].size > 512 * 512:
            continue  # the 1024^2 cases are checked against OpenCV below; the restatement is slow there
        mask = (case["labels"] == case["class"]).astype(np.uint8)
        assert np.array_equal(fr.morph_ref(mask, F.parking_chain()), case["grown"]), case["name"]
    for case in golden:
        mask = (case["labels"] == case["class"]).astype(np.uint8)
        assert np.array_equal(fr.cpu_grow(mask), case["grown"]), case["name"]


def test_golden_cases_cover_the_issue_paths(golden):
    byname = {c["name"]: c for c in golden}
    assert max(len(f) for f in byname["twelve_holes"]["rings"]) >= 11
    assert F.W_TOO_DEEP in byname["nesting_depth_3"]["warnings"]
    assert F.W_SIMPLIFIED in byname["sliver"]["warnings"]
    assert sum(c["grown"].sum() == 0 for c in golden) >= 2


def test_handler_reproduces_the_reference_on_golden_masks(golden, monkeypatch):
    """bounds = unit box and every polygon valid, as the stubs the golden was made with: rings and warnings must be identical"""
    monkeypatch.setattr(F, "bounds", lambda tile: (0.0, 0.0, 1.0, 1.0))
    monkeypatch.setattr(F, "polygon_is_valid", lambda rings: True)
    for case in golden:
        feats, warnings = F.polygons_from_grown(Tile(*case["tile"]), case["grown"])
        rings = [[[list(pt) for pt in ring] for ring in f["geometry"]["coordinates"]] for f in feats]
        assert rings == case["rings"], case["name"]
        assert warnings == case["warnings"], case["name"]


def test_golden_polygons_are_valid(golden, monkeypatch):
    """Every polygon the reference extracts from these masks passes the validity check (none is a GEOS-invalid shape)."""
    monkeypatch.setattr(F, "bounds", lambda tile: (0.0, 0.0, 1.0, 1.0))
    for case in golden:
        feats, warnings = F.polygons_from_grown(Tile(*case["tile"]), case["grown"])
        assert F.W_INVALID not in warnings, case["name"]
        assert len(feats) == len(case["rings"])


def test_bounds_match_mercantile():
    lat = 85.0511287798066
    b = F.bounds(Tile(0, 0, 0))
    assert b[0] == -180.0 and b[2] == 180.0
    assert math.isclose(b[1], -lat, abs_tol=1e-12) and math.isclose(b[3], lat, abs_tol=1e-12)
    quads = {(0, 0): (-180.0, 0.0, 0.0, lat), (1, 0): (0.0, 0.0, 180.0, lat), (0, 1): (-180.0, -lat, 0.0, 0.0), (1, 1): (0.0, -lat, 180.0, 0.0)}
    for (x, y), want in quads.items():
        got = F.bounds(Tile(x, y, 1))
        assert all(math.isclose(g, w, abs_tol=1e-9) for g, w in zip(got, want)), (x, y, got)


def test_featurize_keeps_the_reference_axis_order():
    t = Tile(3, 5, 4)
    west, south, east, north = F.bounds(t)
    ring = F.featurize(t, [(0, 0), (100, 0), (100, 50)], (200, 100))  # (rows, cols): px scales by 200, py by 100
    assert ring[0] == ring[-1] and len(ring) == 4
    assert math.isclose(ring[0][0], west) and math.isclose(ring[0][1], north)
    assert math.isclose(ring[1][0], west + 0.5 * (east - west))
    assert math.isclose(ring[2][1], south + 0.5 * (north - south))


SQUARE = [(0, 0), (10, 0), (10, 10), (0, 10)]


@pytest.mark.parametrize("rings, valid", [
    ([SQUARE], True),
    ([SQUARE[::-1]], True),
    ([[(0, 0), (10, 10), (10, 0), (0, 10)]], False),                                 # bow-tie
    ([[(0, 0), (10, 0), (10, 10), (5, 0), (0, 10)]], False),                         # ring touching itself at (5, 0)
    ([[(0, 0), (10, 0), (20, 0)]], False),                                           # zero area
    ([[(0, 0), (10, 0)]], False),                                                    # too few points
    ([[(0, 0), (10, 0), (10, 10), (10, 5), (0, 10)]], False),                        # spike doubling back
    ([[(0, 0), (5, 0), (10, 0), (10, 10), (0, 10)]], True),                          # collinear vertex
    ([SQUARE, [(2, 2), (4, 2), (4, 4), (2, 4)]], True),                              # hole
    ([SQUARE, [(20, 2), (24, 2), (24, 4), (20, 4)]], False),                         # hole outside the shell
    ([SQUARE, [(0, 5), (3, 3), (3, 7)]], True),                                      # hole touching the shell at one point
    ([SQUARE, [(0, 3), (3, 5), (0, 7)]], False),                                     # ... and at two points
    ([SQUARE, [(0, 3), (3, 5), (0, 7), (0, 5)]], False),                             # ... along an edge
    ([SQUARE, [(1, 1), (9, 1), (9, 9), (1, 9)], [(3, 3), (5, 3), (5, 5), (3, 5)]], False),  # nested holes
    ([SQUARE, [(1, 1), (5, 1), (5, 5), (1, 5)], [(3, 3), (7, 3), (7, 7), (3, 7)]], False),  # crossing holes
    ([SQUARE, [(1, 1), (4, 1), (4, 4), (1, 4)], [(4, 4), (7, 4), (7, 7), (4, 7)]], True),   # holes touching at one point
    ([SQUARE, [(0, 5), (5, 2), (5, 8)], [(5, 8), (10, 5), (5, 5)]], False),        # touch chain shell-hole-hole-shell disconnects
    ([SQUARE, [(2, 2), (8, 2), (8, 8), (2, 8)], [(2, 2), (8, 2), (8, 8), (2, 8)]], False),  # duplicate holes share edges
    ([SQUARE, [(1, 1), (9, 1), (9, 9), (1, 9)], [(5, 0), (6, 2), (4, 2)]], False),  # hole crossing another hole and touching the shell
])
def test_polygon_validity(rings, valid):
    assert F.polygon_is_valid(rings) is valid


def _parser():
    from robosat_b200.tools import features as tool

    p = argparse.ArgumentParser()
    tool.add_parser(p.add_subparsers())
    return p, tool


def test_parser_takes_the_reference_flags():
    p, tool = _parser()
    args = p.parse_args(["features", "masks/", "--type", "parking", "--dataset", "dataset.toml", "out.geojson"])
    assert (args.masks, args.type, args.dataset, args.out, args.func) == ("masks/", "parking", "dataset.toml", "out.geojson", tool.main)
    with pytest.raises(SystemExit):
        p.parse_args(["features", "masks/", "--type", "roads", "--dataset", "d.toml", "out.geojson"])


def test_zoom_other_than_18_raises():
    h = F.ParkingHandler()
    with pytest.raises(NotImplementedError):
        h.apply(Tile(1, 2, 17), np.zeros((8, 8), np.uint8))
    with pytest.raises(NotImplementedError):
        h.apply_batch([Tile(1, 2, 18), Tile(1, 2, 19)], None, 1)


def test_handler_defaults_match_the_reference():
    assert (F.ParkingHandler.kernel_size_denoise, F.ParkingHandler.kernel_size_grow, F.ParkingHandler.simplify_threshold) == (20, 20, 0.01)


def test_morph_validation_runs_before_the_device_check():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 64)()
    cnt = (ctypes.c_int32 * 4)()

    def call(ops, N=1, H=4, W=4, stride=16, cls=1, labels=buf, out=buf, counts=cnt):
        arr = (_lib.MorphOp * len(ops))(*[F._op_struct(o) for o in ops])
        return lib.rsb_morph_binary(labels, stride, N, H, W, cls, arr, len(ops), out, counts, None)

    good = fr.op("ellipse", 3, False)
    assert call([good]) == -3                                      # valid, but no sm_90 device
    assert call([good], labels=None) == -1
    assert call([good], counts=None) == -1
    assert call([good], stride=15) == -1 and "image_stride" in _lib.last_error()
    assert call([good], H=1025, stride=1025 * 4) == -4
    assert call([good], W=0) == -4
    assert call([good], cls=256) == -1
    assert call([good] * 5) == -4
    assert call([fr.op("rect", 65, True)], H=4, W=4) == -4
    assert call([F.MorphOp(0, [(0, 3)] * 3, 3, (3, 1))]) == -1 and "anchor" in _lib.last_error()
    assert call([F.MorphOp(0, [(0, 4)] * 3, 3, (1, 1))]) == -1 and "span" in _lib.last_error()
    assert call([F.MorphOp(0, [(2, 2)] * 3, 3, (1, 1))]) == -1 and "no set cell" in _lib.last_error()
    assert call([F.MorphOp(1, [(1, 0), (0, 3), (2, 1)], 3, (1, 1))]) == -3  # empty rows are allowed
    arr = (_lib.MorphOp * 1)(F._op_struct(good))
    assert lib.rsb_morph_binary(buf, 16, 1, 4, 4, 1, arr, 0, buf, cnt, None) == -4


def test_library_struct_matches_header():
    assert ctypes.sizeof(_lib.MorphOp) == 5 * 4 + 64 * 2 * 2
