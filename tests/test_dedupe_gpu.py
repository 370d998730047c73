"""rsb_dedupe_intersects, rsb_dedupe_areas and `rs dedupe` on the H100, against the exact restatement (tests/dedupe_reference.py):
intersect flags identical on the hand cases and near-degenerate ones, areas within 1e-9 relative and IoU within 1e-9, IoU
exactly 1 for identical shapes, determinism, batching, the over-budget error, seeded buildings and a landuse-sized context, and
the tool end to end on the golden parking features."""

import argparse
import json

import numpy as np
import pytest

import cover_reference as cr
import dedupe_reference as ref
import rasterize_reference as rr
import test_dedupe as cases
from robosat_b200 import _lib
from robosat_b200 import dedupe as DD

pytestmark = pytest.mark.gpu


def _flags(predicted, osm):
    """the device's intersect flag of every (prediction, OSM feature) pair"""
    import torch

    ps, _ = DD.parse(predicted, False)
    qs, _ = DD.parse(osm, True)
    dev = torch.device("cuda")
    p_ll, _ = ps.upload(dev)
    q_ll, _ = qs.upload(dev)
    p, q = np.meshgrid(np.arange(len(ps)), np.arange(len(qs)), indexing="ij")
    got = DD._intersects(_lib.load(), p_ll, q_ll, p.ravel(), q.ravel(), dev, {"intersects_ms": 0.0})
    return got.reshape(len(ps), len(qs))


def _deg(*pts):
    return {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [[list(p) for p in pts] + [list(pts[0])]]}}


Q_SQUARE = _deg((10.0, 45.0), (11.0, 45.0), (11.0, 46.0), (10.0, 46.0))
Q_DIAGONAL = _deg((10.0, 45.0), (11.0, 46.0), (10.0, 46.0))
ULP = np.nextafter(46.0, 47.0)
DEGENERATE = [
    _deg((10.5, 46.0), (10.7, 46.5), (10.3, 46.5)),          # a vertex exactly on an edge
    _deg((10.5, ULP), (10.7, 46.5), (10.3, 46.5)),            # the same vertex one ulp off it
    _deg((10.5, 46.0), (11.5, 46.0), (11.5, 47.0), (10.5, 47.0)),  # a collinear overlap along the top edge
    _deg((11.0, 46.0), (12.0, 46.0), (12.0, 47.0)),           # a corner touching a corner
    _deg((10.3, 45.3), (10.9, 45.1), (10.9, 45.2)),           # a vertex on (or next to) the diagonal y = x + 35
    _deg((10.25, 45.25), (10.9, 45.1), (10.9, 45.2)),         # a vertex exactly on the diagonal
    _deg((np.nextafter(10.25, 11.0), 45.25), (10.9, 45.1), (10.9, 45.2)),  # one ulp below it
    _deg((10.2, 45.5), (10.8, 45.5), (10.8, 45.6), (10.2, 45.6)),  # strictly inside the square, across the diagonal
    _deg((11.0, 45.2), (11.5, 45.2), (11.5, 45.4), (11.0, 45.4)),  # sharing part of the square's right edge from outside
]


def _sweep(predicted, osm, exact_ious):
    """keep decisions identical to the exact IoUs at every threshold more than 1e-9 away from each of them: 0, 1 + 1e-6 and the
    midpoints between consecutive distinct IoUs"""
    ious = np.array(sorted({float(x) for x in exact_ious.values()}))
    thresholds = [0.0, 1.0 + 1e-6] + [float(t) for t in 0.5 * (ious[1:] + ious[:-1])]
    ps, _ = DD.parse(predicted, False)
    qs, _ = DD.parse(osm, True)
    passthrough = [not DD.is_areal(f) for f in predicted]
    for t in thresholds:
        if len(ious) and np.abs(ious - t).min() <= 1e-9:
            continue
        keep, _ = DD.decide(ps, qs, t, passthrough)
        for i, iou in exact_ious.items():
            assert keep[i] == (float(iou) < t), (i, t, float(iou))


def _check_against_reference(predicted, osm, threshold=0.5, **kw):
    keep, areas = DD.dedupe_device(predicted, osm, threshold, **kw)
    want_keep, want = ref.dedupe(predicted, osm, threshold)
    assert keep.tolist() == want_keep
    _sweep(predicted, osm, {i: ref.iou(*w) for i, w in enumerate(want) if w is not None})
    for i, w in enumerate(want):
        if w is None:
            assert np.isnan(areas[i]).all(), i
            continue
        got = areas[i]
        for g, e in zip(got, w):
            assert abs(g - float(e)) <= 1e-9 * max(abs(float(e)), abs(float(w[0]))), (i, got, [float(x) for x in w])
        a_p, a_i, a_u = got
        union = a_p + a_u - a_i
        iou = 0.0 if union == 0 else a_i / union
        assert abs(iou - float(ref.iou(*w))) <= 1e-9, i
    return keep, areas


def test_intersect_flags_hand_and_degenerate(cuda_device):
    for name, (p, qs, hits, _) in cases.CASES.items():
        assert _flags([p], qs)[0].tolist() == hits, name
    got = _flags(DEGENERATE, [Q_SQUARE, Q_DIAGONAL])
    want = [[ref.intersects(p, q) for q in (Q_SQUARE, Q_DIAGONAL)] for p in DEGENERATE]
    assert got.tolist() == want
    assert want[0] == [True, True] and want[1][0] is False and want[2][0] is True and want[5][1] is True


def test_hand_case_areas(cuda_device):
    for name, (p, qs, _, _) in cases.CASES.items():
        _check_against_reference([p], qs)
    _check_against_reference(DEGENERATE, [Q_SQUARE, Q_DIAGONAL])


def test_dedupe_drop_in_matches_reference(cuda_device):
    """`dedupe` returns the reference's kept features: in order, properties dropped, rings closed, non-areal ones passed through,
    invalid ones dropped"""
    point = {"type": "Feature", "properties": {"a": 1}, "geometry": {"type": "Point", "coordinates": [10.5, 45.5]}}
    short = {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [[[10, 45], [10.1, 45], [10, 45]]]}}
    predicted = [c[0] for c in cases.CASES.values()] + DEGENERATE + [point]
    osm = [q for c in cases.CASES.values() for q in c[1]][:6] + [Q_SQUARE, Q_DIAGONAL, point]
    for t in (0.05, 0.5, 1.0):
        want_keep, _ = ref.dedupe(predicted, osm, t)
        want = [{"type": "Feature", "geometry": DD.output_geometry(f["geometry"]), "properties": {}} for f, k in zip(predicted, want_keep) if k]
        assert DD.dedupe(predicted, osm, t) == want
    assert DD.dedupe(predicted + [short], osm, 0.5) == DD.dedupe(predicted, osm, 0.5)
    assert DD.dedupe([], osm, 0.5) == [] and DD.dedupe([point], [], 0.5) == [DD.output_feature(point)]


def test_identical_shape_has_iou_exactly_one(cuda_device):
    p, qs, _, _ = cases.CASES["identical"]
    feats = rr.load_golden()["features"]["features"]
    for pred, osm in ((p, qs), (feats[0], [feats[0]]), (feats[1], [feats[1], cases.feature(cases.box(5000, 5000, 5001, 5001))])):
        keep, areas = DD.dedupe_device([pred], osm, 1.0)
        a_p, a_i, a_u = areas[0]
        assert a_p == a_i == a_u and a_p > 0
        assert a_i / (a_p + a_u - a_i) == 1.0 and not keep[0]
        keep, _ = DD.dedupe_device([pred], osm, np.nextafter(1.0, 2.0))
        assert keep[0]


def _buildings():
    predicted = cr.buildings(20_000, 19, seed=21, span=256)
    # shifted copies only: jittering the vertices of a small star can make it self-intersect, which GEOS refuses as invalid
    osm = ref.perturbed(predicted, seed=22, jitter=0.0, shift=3e-5, drop=0.3) + cr.buildings(3000, 19, seed=23, span=256)
    return predicted, osm


def test_buildings_sample_and_batching(cuda_device):
    predicted, osm = _buildings()
    stats = {}
    keep, areas = DD.dedupe_device(predicted, osm, 0.5, stats=stats)
    assert stats["intersecting"] > 10_000 and stats["batches"] == 1
    sample = np.random.default_rng(24).choice(len(predicted), 500, replace=False)
    exact_ious = {}
    qbox = np.array([[*np.concatenate(ref.rings_ll(q)).min(0), *np.concatenate(ref.rings_ll(q)).max(0)] for q in osm])
    for i in sample:
        fp = predicted[i]
        v = np.concatenate(ref.rings_ll(fp))
        lo, hi = v.min(0), v.max(0)
        cand = np.flatnonzero((qbox[:, 0] <= hi[0]) & (lo[0] <= qbox[:, 2]) & (qbox[:, 1] <= hi[1]) & (lo[1] <= qbox[:, 3]))
        s = [int(j) for j in cand if ref.intersects(fp, osm[j])]
        if not s:
            assert np.isnan(areas[i]).all(), i
            continue
        exact = ref.areas(ref.rings_xy(fp), [ref.rings_xy(osm[j]) for j in s])
        w = [float(x) for x in exact]
        assert np.all(np.abs(areas[i] - w) <= 1e-9 * np.maximum(np.abs(w), w[0])), (i, areas[i], w)
        exact_ious[int(i)] = ref.iou(*exact)
        assert keep[i] == (float(exact_ious[int(i)]) < 0.5)
    _sweep(predicted, osm, dict(list(exact_ious.items())[:40]))
    small_stats = {}
    keep2, areas2 = DD.dedupe_device(predicted, osm, 0.5, budget=1 << 16, stats=small_stats)
    assert small_stats["batches"] > 20
    assert np.array_equal(keep, keep2) and np.array_equal(areas, areas2, equal_nan=True)


def test_deterministic_and_over_budget(cuda_device):
    predicted, osm = _buildings()
    predicted = predicted[:3000]
    a = DD.dedupe_device(predicted, osm, 0.5)[1]
    b = DD.dedupe_device(predicted, osm, 0.5)[1]
    assert np.array_equal(a.view(np.int64), b.view(np.int64))
    with pytest.raises(_lib.RsbError, match="more than the budget"):
        DD.dedupe_device(predicted, osm, 0.5, budget=100)


def test_landuse_context(cuda_device):
    from robosat_b200.cover import tile

    landuse = cr.landuse([100_000], 18, seed=31)
    lu_xy = ref.rings_xy(landuse[0])
    cx, cy = tile(*np.concatenate(ref.rings_ll(landuse[0])).mean(0), 19)
    # the ring's radius is at least ~580 tiles at zoom 19, so buildings within 300 tiles of its centre lie inside it
    inside = cr.buildings(2000, 19, seed=32, origin=(cx - 300, cy - 300), span=600)
    edge = ref.boundary_squares(landuse[0], 20, 2e-4, seed=33)
    predicted = inside + edge
    stats = {}
    keep, areas = DD.dedupe_device(predicted, landuse, 0.5, stats=stats)
    a_u = abs(ref.shoelace(lu_xy))
    assert not np.isnan(areas).any() and stats["items"] > 2000 * 100_000 and stats["batches"] > 1
    assert np.all(np.abs(areas[:, 2] - a_u) <= 1e-9 * a_u)
    n = len(inside)
    assert np.all(np.abs(areas[:n, 1] - areas[:n, 0]) <= 1e-9 * areas[:n, 0]) and keep[:n].all()  # IoU = A(P) / A(U)
    for i in range(n, len(predicted)):  # boundary squares: A(P) and I against the exact slab sums over the square's x range
        p = ref.rings_xy(predicted[i])
        x0, x1 = float(np.concatenate(p)[:, 0].min()), float(np.concatenate(p)[:, 0].max())
        w = [float(x) for x in ref.areas(p, [lu_xy], window=(x0, x1))]
        assert abs(areas[i, 0] - w[0]) <= 1e-9 * w[0]
        assert abs(areas[i, 1] - w[1]) <= 1e-9 * w[0], (i, areas[i], w)
        assert 0 < areas[i, 1] < areas[i, 0]


def test_tool_end_to_end(cuda_device, tmp_path, capsys):
    from robosat_b200.tools import dedupe as tool

    feats = rr.load_golden()["features"]["features"]
    osm = ref.perturbed(feats, seed=41, jitter=2e-6, shift=2e-5, drop=0.0)[:1] + [{"type": "Feature", "geometry": {"type": "Point", "coordinates": [0, 0]}}]
    line = {"type": "Feature", "properties": {"x": 1}, "geometry": {"type": "LineString", "coordinates": [[0, 0], [1, 1]]}}
    predicted = feats + [line]
    paths = {k: tmp_path / (k + ".geojson") for k in ("osm", "predicted", "out")}
    paths["osm"].write_text(json.dumps({"type": "FeatureCollection", "features": osm}))
    paths["predicted"].write_text(json.dumps({"type": "FeatureCollection", "features": predicted}))
    want_keep, _ = ref.dedupe(predicted, osm, 0.5)
    assert want_keep == [False, True, True]
    stats = {}
    tool.main(argparse.Namespace(osm=str(paths["osm"]), predicted=str(paths["predicted"]), out=str(paths["out"]), threshold=0.5), stats=stats)
    got = json.loads(paths["out"].read_text())
    assert got == {"type": "FeatureCollection", "features": [{"type": "Feature", "geometry": DD.output_geometry(f["geometry"]), "properties": {}}
                                                             for f, k in zip(predicted, want_keep) if k]}
    assert "1 OSM features are not a Polygon or MultiPolygon" in capsys.readouterr().err
    assert stats["kept"] == 2 and stats["intersecting"] == 1


def test_huge_features_sharing_a_border(cuda_device):
    """two OSM polygons of ~5 x 10^4 vertices sharing a 2 x 10^4-edge zigzag border, both in S(P) of squares along it: the
    y-band index keeps this from costing n_k * n_l per prediction, and U is the whole disc"""
    a, b, disc, border = ref.split_disc(60_000, 20_000)
    idx = np.random.default_rng(71).choice(len(border), 200, replace=False)
    predicted = ref.squares_at(border[idx], 3e-4)
    stats = {}
    keep, areas = DD.dedupe_device(predicted, [a, b], 0.5, stats=stats)
    disc_area = abs(ref.shoelace([DD.mollweide(disc)]))
    assert stats["intersecting"] == len(predicted) and stats["items"] >= len(predicted) * 100_000
    assert np.all(np.abs(areas[:, 2] - disc_area) <= 1e-9 * disc_area)
    assert np.all(np.abs(areas[:, 1] - areas[:, 0]) <= 1e-9 * areas[:, 0]) and keep.all()
    a_xy, b_xy = ref.rings_xy(a), ref.rings_xy(b)
    for i in range(3):  # I of a square against the exact slab sums over its x range
        p = ref.rings_xy(predicted[i])
        x0, x1 = float(np.concatenate(p)[:, 0].min()), float(np.concatenate(p)[:, 0].max())
        w = [float(x) for x in ref.areas(p, [a_xy, b_xy], window=(x0, x1))]
        assert abs(areas[i, 0] - w[0]) <= 1e-9 * w[0] and abs(areas[i, 1] - w[1]) <= 1e-9 * w[0], (i, areas[i], w)
