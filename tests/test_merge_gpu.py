"""rsb_merge_near, rsb_merge_components, rsb_merge_fill / rsb_merge_close and `rs merge` on the H100, against the restatement
(tests/merge_reference.py): link flags, labels and closed bitmaps identical, `merge_device` identical to the restated
pipeline, batching and the over-budget error, the tool end to end, and the purpose: fragments of parking lots cut at z18 tile
borders by `rs rasterize` -> `rs features` come back as one feature per lot."""

import argparse
import json

import numpy as np
import pytest

import cover_reference as cr
import merge_reference as ref
import rasterize_reference as rr
from robosat_b200 import _lib
from robosat_b200 import merge as MG
from robosat_b200.tools import merge as tool

pytestmark = pytest.mark.gpu


def _metres(rings, x0=1.2e6, y0=5.6e6):
    """a Polygon feature from rings given in EPSG:3395 metres relative to (x0, y0)"""
    coords = []
    for r in rings:
        ll = MG.inverse_mercator(np.asarray(r, np.float64) + [x0, y0]).tolist()
        coords.append(ll + [ll[0]])
    return {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": coords}}


def _sq(x0, y0, x1, y1):
    return [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]


HAND = [
    _metres([_sq(0, 0, 10, 10)]),
    _metres([_sq(10, 0, 20, 10)]),                        # touches 0
    _metres([_sq(23, 2, 30, 8)]),                         # 3 m right of 1
    _metres([_sq(40, 0, 70, 30), _sq(50, 10, 60, 20)]),   # a square with a hole
    _metres([_sq(52, 12, 58, 18)]),                       # 2 m inside the hole
    _metres([_sq(43, 3, 67, 27)]),                        # overlaps the ring and its hole
    _metres([[(100, 0), (110, 0), (105, 7)]]),
    _metres([_sq(95, 9.5, 115, 20)]),                     # 2.5 m above the triangle's apex
    _metres([_sq(200, 0, 201, 1)]),                       # isolated
    _metres([_sq(0.5, 30, 0.6, 30.1)]),                   # covers no cell centre -> an empty closing
]


def _buildings(n, seed):
    return cr.buildings(n, 19, seed, span=16)


def _device_links(features, d):
    shapes, _ = MG.parse(features)
    p, q = MG.link(shapes, d)
    return sorted(zip(p.tolist(), q.tolist()))


@pytest.mark.parametrize("d", [1, 2, 3, 5])
def test_links_hand_cases(d):
    assert _device_links(HAND, d) == ref.linked(HAND, d)


def test_links_degenerate_and_buildings():
    base = _metres([_sq(0, 0, 10, 10)])
    gap = np.nextafter(13.0, 14.0)
    degenerate = [base, _metres([_sq(13, 0, 20, 10)]), _metres([_sq(gap, 20, 20, 30)]), _metres([[(0, 20), (0, 20), (5, 21), (5, 25), (0, 25)]])]
    for d in (1, 3):
        assert _device_links(degenerate, d) == ref.linked(degenerate, d)
    b = _buildings(1500, 5)
    for d in (1, 4):
        links = _device_links(b, d)
        assert links == ref.linked(b, d)
        assert len(links) > 100


def test_labels_against_host_union_find():
    n = 100000
    path = np.arange(n - 1)
    rng = np.random.default_rng(0)
    perm = rng.permutation(n)
    cases = [
        (path, path + 1),                                  # one path
        (perm[:-1], perm[1:]),                             # a path in random order
        (np.zeros(999, np.int64) + 500, np.r_[0:500, 501:1000]),  # a star around 500
        (np.zeros(0, np.int64), np.zeros(0, np.int64)),    # isolated nodes
    ]
    for p, q in cases:
        m = 1000 if len(p) == 999 else n
        want = ref.labels(m, list(zip(np.minimum(p, q).tolist(), np.maximum(p, q).tolist())))
        for _ in range(2):
            assert np.array_equal(MG.components_device(m, p, q), want)


def _closed_device(features, d, budget=MG.DEFAULT_BUDGET):
    shapes, _ = MG.parse(features)
    comps = ref.pipeline(features, d)
    dev = [MG.Component(c.members, c.grid, c.cell) for c in comps]
    for start, end in MG.plan(dev, budget):
        MG.close_device(shapes, dev[start:end], keep_fill=True)
    return comps, dev


def _assert_same_bitmaps(want, got):
    assert len(want) == len(got)
    for w, g in zip(want, got):
        assert np.array_equal(w.members, g.members) and w.grid == g.grid
        if w.grid[2] == 0:
            continue
        if getattr(g, "fill", None) is not None:
            assert np.array_equal(w.fill, g.fill)
        assert np.array_equal(w.closed, g.closed)
        assert w.count == g.count


@pytest.mark.parametrize("d", [1, 3])
def test_closed_bitmaps_hand_cases(d):
    _assert_same_bitmaps(*_closed_device(HAND, d))


def test_closed_bitmaps_golden_features():
    golden = rr.load_golden()["features"]["features"]
    want, got = _closed_device(golden, 2)
    _assert_same_bitmaps(want, got)
    assert sum(c.count for c in got) > 0


def test_closed_bitmaps_buildings_and_batches():
    b = _buildings(800, 7)
    want, got = _closed_device(b, 1)
    _assert_same_bitmaps(want, got)
    _, small = _closed_device(b, 1, budget=max(c.device_bytes() for c in got))
    _assert_same_bitmaps(want, small)


def test_closed_bitmaps_wide_grid_and_landuse():
    wide = [_metres([[(0, 0), (1000, 30), (1000, 60), (0, 8)]])]  # 4 000 cells wide at d = 1: several fill bands and closing tiles
    want, got = _closed_device(wide, 1)
    assert got[0].grid[2] > 4000 and got[0].grid[3] > MG.FILL_WORDS // ((got[0].grid[2] + 31) // 32)
    _assert_same_bitmaps(want, got)
    landuse = cr.landuse([20000], 18, 3, sizes=(3, 4))
    want, got = _closed_device(landuse, 2)
    assert got[0].grid[2] * got[0].grid[3] > 5 * 10 ** 5
    _assert_same_bitmaps(want, got)


def test_merge_device_matches_restated_pipeline():
    feats = HAND + _buildings(300, 11)
    for d in (1, 2):
        want = ref.pipeline(feats, d)
        stats = {}
        _, got = MG.merge_device(feats, d, stats=stats)
        _assert_same_bitmaps(want, got)
        assert [MG.component_feature(c) for c in got] == [MG.component_feature(c) for c in want]
        assert stats["components"] == len(want)


def test_batches_give_identical_results_and_over_budget_raises():
    feats = _buildings(400, 13)
    one, _ = MG.merge(feats, 1)
    stats = {}
    shapes, _ = MG.parse(feats)
    budget = max(c.device_bytes() for c in MG.merge_device(shapes, 1)[1])
    many, _ = MG.merge_shapes(shapes, 1, budget=budget, stats=stats)
    assert stats["batches"] > 10
    assert many == one
    with pytest.raises(_lib.RsbError, match="budget"):
        MG.merge_device(feats, 1, budget=512)


def _write_and_run(tmp_path, features, threshold):
    src = tmp_path / "in.geojson"
    src.write_text(json.dumps({"type": "FeatureCollection", "features": features}))
    out = tmp_path / "out.geojson"
    tool.main(argparse.Namespace(features=str(src), threshold=threshold, out=str(out)))
    return json.loads(out.read_text())


def test_tool_end_to_end(tmp_path, capsys):
    golden = rr.load_golden()["features"]["features"]
    feats = golden + HAND + [{"type": "Feature", "properties": {}, "geometry": {"type": "Point", "coordinates": [10.0, 45.0]}}]
    got = _write_and_run(tmp_path, feats, 2)
    want, _ = MG.merge(feats, 2)
    assert got == {"type": "FeatureCollection", "features": json.loads(json.dumps(want))}
    err = capsys.readouterr().err
    assert MG.W_GEOMETRY.format(1) in err and MG.W_NOT_POLYGON in err
    for f in got["features"]:
        assert f["geometry"]["type"] in ("Polygon", "MultiPolygon") and f["properties"]["area"] > 0


def test_fragments_at_tile_borders_merge_into_one_feature_each():
    """the purpose of `rs merge`: lots cut by tile borders come back whole"""
    source, tiles = ref.straddling(24, 17)
    frags = ref.fragments(source, tiles)
    assert len(frags) > len(source)
    merged, warnings = MG.merge(frags, 1)
    assert warnings == []
    assert len(merged) == len(source)
    want = np.array([abs(MG.ring_area(np.asarray(f["geometry"]["coordinates"][0])[:-1])) for f in source])
    got = np.array([f["properties"]["area"] for f in merged])
    # each merged feature lies over its own source polygon (they are 6 tiles apart)
    centre = np.array([np.asarray(f["geometry"]["coordinates"][0]).mean(0) for f in merged])
    source_centre = np.array([np.asarray(f["geometry"]["coordinates"][0]).mean(0) for f in source])
    match = np.argmin(np.abs(centre[:, None] - source_centre[None]).max(2), axis=1)
    assert sorted(match.tolist()) == list(range(len(source)))
    rel = np.abs(got - want[match]) / want[match]
    print("merged area / source area: max relative difference %.4f, mean %.4f" % (rel.max(), rel.mean()))
    # `rs features`' 20-pixel opening rounds the lots' corners and its polygon simplification cuts a little more, so the merged
    # lots come out slightly smaller than their sources (measured on an H100: at most 7.1 % smaller, 2.3 % on average)
    assert rel.max() < 0.1 and rel.mean() < 0.04
