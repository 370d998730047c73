"""`rs rasterize` on the CPU: the numpy restatement of GDAL's fill against the reference's golden parking masks, the reference's own
assertions, projection and tile bounds, binning against a brute-force cover, the fill bands of `rs cover` and `rs merge`, feature
filtering, the command line and the C entry point's validation."""

import argparse
import ctypes
import math

import numpy as np
import pytest

import rasterize_reference as rr
from robosat_b200 import _lib
from robosat_b200 import rasterize as RZ
from robosat_b200.tiles import Tile


@pytest.fixture(scope="module")
def golden():
    return rr.load_golden()


def test_restatement_reproduces_the_golden_masks(golden):
    assert len(golden["masks"]) == 4
    for tile, mask in golden["masks"].items():
        got = rr.burn(tile, golden["features"]["features"], 512)
        assert got.dtype == np.uint8 and got.shape == (512, 512)
        assert np.array_equal(got, mask), tile
    assert sorted(int(m.sum()) for m in golden["masks"].values()) == [0, 10654, 56756, 63185]


def test_reference_assertions(golden):
    features = golden["features"]["features"]
    assert len(features) == 2
    assert rr.burn((70762, 104119, 18), features, 512).sum() != 0
    assert rr.burn((69623, 104946, 18), features, 512).sum() == 0
    mercator = next(RZ.feature_to_mercator(features[0]))
    assert mercator["type"] == "Polygon"
    assert int(mercator["coordinates"][0][0][0]) == -9219757


def test_host_module_matches_the_restatement(golden):
    for tile in golden["tiles"]:
        assert RZ.xy_bounds(tile) == rr.xy_bounds(*tile)
        for size in (1, 33, 512, 4096):
            assert RZ.tile_transform(tile, size) == rr.transform(tile, size)
    ring = golden["features"]["features"][1]["geometry"]["coordinates"][0]
    assert np.array_equal(RZ.project(ring), rr.project(ring))
    assert np.array_equal(RZ.project([p + [12.5] for p in ring]), rr.project(ring))  # altitude ignored


def test_xy_bounds_match_mercantile():
    assert RZ.xy_bounds(Tile(0, 0, 0)) == (-20037508.342789244, -20037508.342789244, 20037508.342789244, 20037508.342789244)
    left, bottom, right, top = RZ.xy_bounds(Tile(1, 0, 1))
    assert (left, top) == (0.0, 20037508.342789244) and math.isclose(right, 20037508.342789244) and bottom == 0.0


def _merc_polygon(tile, rings_uv):
    """rings in tile units (u right, v down, the tile is [0, 1]^2) -> Mercator rings"""
    left, bottom, right, top = RZ.xy_bounds(tile)
    return [np.array([(left + u * (right - left), top - v * (top - bottom)) for u, v in ring]) for ring in rings_uv]


def _random_polygons(rng, base, n, spread):
    polys = []
    for _ in range(n):
        cu, cv = rng.uniform(-1, spread + 1, 2)
        r = 10 ** rng.uniform(-3, 0.3)
        k = rng.randint(3, 12)
        ang = np.sort(rng.uniform(0, 2 * np.pi, k))
        rad = r * rng.uniform(0.3, 1, k)
        polys.append(_merc_polygon(base, [list(zip(cu + rad * np.cos(ang), cv + rad * np.sin(ang)))]))
    return polys


def test_binning_is_a_superset_of_the_brute_force_cover():
    rng = np.random.RandomState(0)
    base = Tile(1000, 2000, 12)
    polys = _random_polygons(rng, base, 40, 4)
    polys.append(_merc_polygon(base, [[(-30, -30), (40, -30), (40, 40), (-30, 40)]]))  # box far larger than the tile list
    near = [Tile(base.x + dx, base.y + dy, 12) for dy in range(-2, 7) for dx in range(-2, 7)]
    listed = near[::2] + near[3:5]  # a sparse list with two tiles listed twice
    ps = RZ.PolygonSet(polys)
    offsets, ids = RZ.bin_polygons(listed, ps.bboxes)
    assert len(offsets) == len(listed) + 1 and offsets[0] == 0 and (np.diff(offsets) >= 0).all()
    size = 32
    covered = 0
    for i, t in enumerate(listed):
        have = set(ids[offsets[i]:offsets[i + 1]].tolist())
        tr = rr.transform(t, size)
        for p, poly in enumerate(polys):
            if rr.burn_transform(tr, [poly], size).any():
                assert p in have, (t, p)
                covered += 1
    assert covered > len(listed)  # the cover is not trivial
    # no listed tile far from a polygon's box gets it
    far = [Tile(base.x + 500, base.y, 12)]
    o, _ = RZ.bin_polygons(far, ps.bboxes[:40])
    assert o[-1] == 0


def test_binning_of_empty_inputs():
    o, ids = RZ.bin_polygons([Tile(1, 1, 3)], np.zeros((0, 4)))
    assert o.tolist() == [0, 0] and len(ids) == 0
    o, ids = RZ.bin_polygons([], np.zeros((2, 4)))
    assert o.tolist() == [0] and len(ids) == 0
    ps = RZ.PolygonSet([[np.zeros((0, 2))], []])  # polygons without vertices meet no tile
    assert np.isnan(ps.bboxes).all()
    o, _ = RZ.bin_polygons([Tile(0, 0, 0)], ps.bboxes)
    assert o.tolist() == [0, 0]


def test_polygon_set_packing():
    a = [np.array([[0.0, 0], [1, 0], [1, 1], [0, 0]]), np.array([[0.2, 0.2], [0.4, 0.2], [0.3, 0.3], [0.2, 0.2]])]
    b = [np.array([[5.0, -1], [6, 2], [4, 3], [5, -1]])]
    ps = RZ.PolygonSet([a, [], b])
    assert len(ps) == 3
    assert ps.ring_offsets.tolist() == [0, 4, 8, 12] and ps.poly_rings.tolist() == [0, 2, 2, 3]
    assert ps.bboxes[0].tolist() == [0, 0, 1, 1] and np.isnan(ps.bboxes[1]).all() and ps.bboxes[2].tolist() == [4, -1, 6, 3]


@pytest.mark.parametrize("items", [
    [(4, 1), (0, 0), (100, 1), (300, 2)],  # narrow grids: bands of 128 rows, an empty window between them
    [(5000, 200), (1, 3)],  # 61 rows of 200 words fit in FILL_WORDS
    [(3, 20000), (7, 5)],  # one row wider than FILL_WORDS: bands of one row
    [(0, 50000), (10, 100)],  # a wide item without rows does not set the width
])
def test_fill_bands_cover_every_row_once(items):
    rows, words = np.array(items, np.int64).T
    bands, band_rows, max_words = RZ.fill_bands(rows, words)
    assert bands.dtype == np.int32 and bands.shape == (len(bands), 3)
    assert max_words == words[rows > 0].max()
    assert 1 <= band_rows <= 128 and (band_rows * max_words <= RZ.FILL_WORDS or max_words > RZ.FILL_WORDS)
    assert (bands[:, 2] >= 1).all() and (bands[:, 2] <= band_rows).all()
    assert bands[:, 2].sum() == rows.sum()
    for i, n in enumerate(rows):
        mine = bands[bands[:, 0] == i]
        assert sorted(r for _, start, count in mine for r in range(start, start + count)) == list(range(n))


def _poly(lonlat):
    return {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": lonlat}}


def test_feature_filtering_and_warnings():
    square = [[[10.0, 50.0], [10.001, 50.0], [10.001, 50.001], [10.0, 50.001], [10.0, 50.0]]]
    feats = [
        _poly(square),
        {"type": "Feature", "geometry": {"type": "Point", "coordinates": [10.0, 50.0]}},
        {"type": "Feature", "geometry": {"type": "MultiPolygon", "coordinates": [square]}},
        _poly([[[10.0, 50.0], [10.001, 50.0], [10.0, 50.0]]]),                          # 3 positions
        _poly([[[10.0, 95.0], [10.001, 95.0], [10.001, 96.0], [10.0, 95.0]]]),          # beyond the pole
        _poly([[["a", 1], [2, 3], [4, 5], ["a", 1]]]),                                 # not numbers
        _poly([]),                                                                      # no ring
        {"type": "Feature", "geometry": {"type": "LineString", "coordinates": square[0]}},
        _poly(square + [[[10.0002, 50.0002], [10.0004, 50.0002], [10.0003, 50.0004], [10.0002, 50.0002]]]),
        _poly([[p + [100.0] for p in square[0]]]),                                      # altitudes
    ]
    polygons, warnings = RZ.polygons_from_features(feats)
    assert warnings == ["Warning: invalid feature 3, skipping", "Warning: invalid feature 4, skipping",
                        "Warning: invalid feature 5, skipping", "Warning: invalid feature 6, skipping"]
    assert [len(p) for p in polygons] == [1, 2, 1]
    assert np.array_equal(polygons[0][0], rr.project(square[0]))
    assert np.array_equal(polygons[2][0], polygons[0][0])
    # the burn() drop-in takes MultiPolygon components as polygons of their own
    assert [g["type"] for f in feats[:3] for g in RZ.feature_to_mercator(f)] == ["Polygon", "Polygon"]


def _parser():
    from robosat_b200.tools import rasterize as tool

    p = argparse.ArgumentParser()
    tool.add_parser(p.add_subparsers())
    return p, tool


def test_parser_takes_the_reference_flags():
    p, tool = _parser()
    args = p.parse_args(["rasterize", "f.geojson", "tiles.csv", "out/", "--dataset", "d.toml", "--zoom", "18"])
    assert (args.features, args.tiles, args.out, args.dataset, args.zoom, args.size, args.func) == (
        "f.geojson", "tiles.csv", "out/", "d.toml", 18, 512, tool.main)
    with pytest.raises(SystemExit):
        p.parse_args(["rasterize", "f.geojson", "tiles.csv", "out/", "--dataset", "d.toml"])  # --zoom is required


def test_tool_is_registered():
    import subprocess
    import sys

    r = subprocess.run([sys.executable, "-m", "robosat_b200.tools", "rasterize", "--help"], capture_output=True, text=True,
                       cwd=rr.os.path.dirname(rr.os.path.dirname(rr.os.path.abspath(rr.__file__))))
    assert r.returncode == 0 and "--zoom" in r.stdout


def _dataset(tmp_path, colors):
    path = tmp_path / "dataset.toml"
    path.write_text("[common]\nclasses = [%s]\ncolors = [%s]\n" % (", ".join("'c%d'" % i for i in range(len(colors))),
                                                                   ", ".join("'%s'" % c for c in colors)))
    return str(path)


def test_zoom_and_colour_assertions(tmp_path):
    _, tool = _parser()
    csv = tmp_path / "tiles.csv"
    csv.write_text("1,2,18\n3,4,17\n")
    (tmp_path / "f.geojson").write_text('{"type": "FeatureCollection", "features": []}')
    ns = lambda ds, zoom: argparse.Namespace(features=str(tmp_path / "f.geojson"), tiles=str(csv), out=str(tmp_path / "out"),  # noqa: E731
                                             dataset=ds, zoom=zoom, size=64)
    with pytest.raises(AssertionError, match="binary"):
        tool.main(ns(_dataset(tmp_path, ["denim", "orange", "dark"]), 18))
    with pytest.raises(AssertionError):
        tool.main(ns(_dataset(tmp_path, ["denim", "orange"]), 18))  # a tile at z17


def test_tool_without_a_device_exits(tmp_path):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    _, tool = _parser()
    csv = tmp_path / "tiles.csv"
    csv.write_text("1,2,18\n")
    (tmp_path / "f.geojson").write_text('{"type": "FeatureCollection", "features": []}')
    with pytest.raises(SystemExit, match="CUDA"):
        tool.main(argparse.Namespace(features=str(tmp_path / "f.geojson"), tiles=str(csv), out=str(tmp_path / "out"),
                                     dataset=_dataset(tmp_path, ["denim", "orange"]), zoom=18, size=64))


def test_rasterize_validation_runs_before_the_device_check():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    verts = (ctypes.c_double * 16)()
    i64 = (ctypes.c_int64 * 4)()
    i32 = (ctypes.c_int32 * 4)()
    tr = (ctypes.c_double * 8)()
    out = (ctypes.c_uint8 * 64)()
    cnt = (ctypes.c_int32 * 2)()
    base = ctypes.addressof(verts)
    aligned = base if base % 16 == 0 else base + 8

    def call(vertices=aligned, rings=i64, polys=i32, P=1, offs=i32, ids=i32, trs=tr, N=1, size=8, o=out, stride=64, counts=cnt):
        return lib.rsb_rasterize_polygons(vertices, rings, polys, P, offs, ids, trs, N, size, o, stride, counts, None)

    assert call() == -3                                               # valid, but no sm_90 device
    assert call(vertices=None, rings=None, polys=None, P=0) == -3     # no polygons at all
    assert call(o=None) == -1
    assert call(counts=None) == -1
    assert call(offs=None) == -1
    assert call(ids=None) == -1
    assert call(trs=None) == -1
    assert call(vertices=None) == -1 and "null polygon array" in _lib.last_error()
    assert call(P=-1) == -1
    assert call(N=0) == -1
    assert call(size=0) == -1 and "size" in _lib.last_error()
    assert call(size=4097, stride=4097 * 4097) == -1
    assert call(size=4096, stride=4096 * 4096) == -3
    assert call(stride=63) == -1 and "image_stride" in _lib.last_error()
    assert call(vertices=aligned + 8) == -1 and "aligned" in _lib.last_error()
