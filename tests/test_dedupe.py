"""`rs dedupe` on the host: the exact restatement (tests/dedupe_reference.py) against hand-computed planar cases, the Mollweide
restatement, and the tool's host logic (flags, output layout, pass-through, warnings, empty collections)."""

import argparse
import json
import math
from fractions import Fraction

import numpy as np
import pytest

import dedupe_reference as ref
import rasterize_reference as rr
from robosat_b200 import dedupe as DD
from robosat_b200.tools import dedupe as tool

LON0, LAT0, UNIT = 10.0, 45.0, 1e-3  # the planar cases, in units of 0.001 degrees


def box(u0, v0, u1, v1):
    return [(u0, v0), (u1, v0), (u1, v1), (u0, v1)]


def feature(*rings, components=None):
    """a feature from rings in units (closed here); a MultiPolygon of `components` (lists of rings) when given"""
    def ring(r):
        pts = [[LON0 + UNIT * u, LAT0 + UNIT * v] for u, v in r]
        return pts + [pts[0]]

    if components is not None:
        return {"type": "Feature", "properties": {"k": 1}, "geometry": {"type": "MultiPolygon", "coordinates": [[ring(r) for r in c] for c in components]}}
    return {"type": "Feature", "properties": {"k": 1}, "geometry": {"type": "Polygon", "coordinates": [ring(r) for r in rings]}}


def planar(f):
    """the rings back in units (every case vertex is a multiple of 0.1 units)"""
    def unit(c, c0):
        return Fraction(round((c - c0) / UNIT * 10), 10)

    return [[(unit(p[0], LON0), unit(p[1], LAT0)) for p in r] for r in ref.rings_ll(f)]


# name -> (P, [Q...], intersects per Q, IoU)
CASES = {
    "overlap": (feature(box(0, 0, 2, 2)), [feature(box(1, 0, 3, 2))], [True], Fraction(1, 3)),
    "touch_edge": (feature(box(0, 0, 1, 1)), [feature(box(1, 0, 2, 1))], [True], Fraction(0)),
    "touch_point": (feature(box(0, 0, 1, 1)), [feature(box(1, 1, 2, 2))], [True], Fraction(0)),
    "disjoint": (feature(box(0, 0, 1, 1)), [feature(box(1.5, 0, 2, 1))], [False], None),
    "nested": (feature(box(1, 1, 2, 2)), [feature(box(0, 0, 4, 4))], [True], Fraction(1, 16)),
    "contains": (feature(box(0, 0, 4, 4)), [feature(box(1, 1, 2, 2))], [True], Fraction(1, 16)),
    "in_hole": (feature(box(1.5, 1.5, 2.5, 2.5)), [feature(box(0, 0, 4, 4), box(1, 1, 3, 3)[::-1])], [False], None),
    "touches_hole": (feature(box(1, 1.5, 2, 2.5)), [feature(box(0, 0, 4, 4), box(1, 1, 3, 3)[::-1])], [True], Fraction(0)),
    "adjacent_osm": (feature(box(1, 0.5, 3, 1.5)), [feature(box(0, 0, 2, 2)), feature(box(2, 0, 4, 2))], [True, True], Fraction(2, 8)),
    "same_direction_shared_edge": (feature(box(1.5, 0.5, 2.5, 1.5)), [feature(box(0, 0, 2, 2)), feature(box(1, 0, 2, 3))], [True, True], Fraction(1, 11)),
    "far_component": (feature(box(0, 0, 1, 1)), [feature(components=[[box(0, 0, 1, 1)], [box(10, 10, 11, 11)]])], [True], Fraction(1, 2)),
    "identical": (feature(box(0, 0, 3, 1), [(0.5, 0.2), (0.5, 0.8), (2.5, 0.8)]), [feature(box(0, 0, 3, 1), [(0.5, 0.2), (0.5, 0.8), (2.5, 0.8)])], [True], Fraction(1)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_hand_cases(name):
    p, qs, hits, want = CASES[name]
    assert [ref.intersects(p, q) for q in qs] == hits
    s = [q for q, h in zip(qs, hits) if h]
    if want is None:
        assert not s
        return
    a = ref.areas(planar(p), [planar(q) for q in s])
    assert ref.iou(*a) == want
    if name == "touch_edge":  # no intersection, but the union holds both squares
        assert a == (Fraction(1), Fraction(0), Fraction(1))


def test_restatement_projected_iou_is_close_to_planar():
    # the cases are 0.001 degrees across, so Mollweide is affine to ~1e-5 over them and the IoU barely moves
    for name, (p, qs, hits, want) in CASES.items():
        s = [q for q, h in zip(qs, hits) if h]
        if want is None:
            continue
        got = ref.iou(*ref.areas(ref.rings_xy(p), [ref.rings_xy(q) for q in s]))
        assert abs(float(got) - float(want)) < 1e-4, name


def test_mollweide_equator_and_poles():
    xy = DD.mollweide([[0, 0], [90, 0], [-180, 0], [0, 90], [45, -90]])
    c = 2 * math.sqrt(2) / math.pi * DD.R
    assert xy[0].tolist() == [0.0, 0.0]
    assert xy[1, 0] == pytest.approx(c * math.pi / 2, rel=1e-15) and xy[1, 1] == 0.0
    assert xy[2, 0] == pytest.approx(-c * math.pi, rel=1e-15)
    assert xy[3, 1] == pytest.approx(math.sqrt(2) * DD.R, rel=1e-15) and abs(xy[3, 0]) < 1e-6
    assert xy[4, 1] == pytest.approx(-math.sqrt(2) * DD.R, rel=1e-15)
    # theta solves 2 theta + sin 2 theta = pi sin phi
    lat = np.linspace(-89, 89, 37)
    theta = np.arcsin(DD.mollweide(np.stack([np.zeros_like(lat), lat], 1))[:, 1] / (math.sqrt(2) * DD.R))
    assert np.abs(2 * theta + np.sin(2 * theta) - np.pi * np.sin(np.radians(lat))).max() < 1e-12


@pytest.mark.parametrize("lon,lat", [(0.0, 0.0), (37.0, 52.0), (-120.0, -33.0), (170.0, 75.0)])
def test_mollweide_is_equal_area(lon, lat):
    k = 2000  # meridian sides are curved in Mollweide; densify them
    t = np.linspace(0, 1, k)
    ring = np.concatenate([np.stack([lon + t, np.full(k, lat)], 1), np.stack([np.full(k, lon + 1), lat + t], 1),
                           np.stack([lon + 1 - t, np.full(k, lat + 1)], 1), np.stack([np.full(k, lon), lat + 1 - t], 1)])
    xy = DD.mollweide(ring)
    xy -= xy.mean(0)
    area = 0.5 * np.sum(xy[:, 0] * np.roll(xy[:, 1], -1) - np.roll(xy[:, 0], -1) * xy[:, 1])
    want = DD.R ** 2 * math.radians(1.0) * (math.sin(math.radians(lat + 1)) - math.sin(math.radians(lat)))
    assert area == pytest.approx(want, rel=1e-6)


def test_shape_set_cleans_and_orients():
    cw = [[10.0, 45.0], [10.0, 45.001], [10.001, 45.001], [10.001, 45.001], [10.001, 45.0], [10.0, 45.0]]  # clockwise, a repeat
    hole_ccw = [[10.0002, 45.0002], [10.0008, 45.0002], [10.0008, 45.0008], [10.0002, 45.0008], [10.0002, 45.0002]]
    ss, warnings = DD.parse([{"geometry": {"type": "Polygon", "coordinates": [cw, hole_ccw]}}], False)
    assert warnings == [] and len(ss) == 1
    assert ss.lonlat.ring_offsets.tolist() == [0, 4, 8]  # closing repeat and the doubled vertex dropped
    xy = ss.xy.vertices
    for r, sign in ((0, 1), (1, -1)):
        v = xy[4 * r:4 * r + 4] - xy[4 * r]
        assert sign * np.sum(v[:, 0] * np.roll(v[:, 1], -1) - np.roll(v[:, 0], -1) * v[:, 1]) > 0
    assert ss.lonlat.vertices[0].tolist() == cw[0]  # reversal keeps the first vertex
    assert ss.next.tolist() == [1, 2, 3, 0, 5, 6, 7, 4]
    assert ss.exteriors.tolist() == [0] and ss.exterior_offsets.tolist() == [0, 1]
    assert np.array_equal(DD.mollweide(ss.lonlat.vertices), ss.xy.vertices)


def test_band_index_lists_each_edge_in_the_bands_it_spans():
    a, b, _, _ = ref.split_disc(6000, 2000)
    small = feature(box(0, 0, 1, 1))
    ss, _ = DD.parse([a, small, b], True)
    nb = np.diff(ss.feature_bands)
    assert nb[1] == 0 and nb[0] == ss.edges()[0] // DD.EDGES_PER_BAND and nb[2] > 0
    xy = ss.xy.vertices
    for f in (0, 2):
        y0, inv = ss.band_ranges[f]
        fb = ss.feature_bands[f]
        listed = {}
        for band in range(nb[f]):
            for v in ss.band_edges[ss.band_offsets[fb + band]:ss.band_offsets[fb + band + 1]]:
                listed.setdefault(int(v), []).append(band)
        for v in range(ss.feature_vertices[f], ss.feature_vertices[f + 1]):
            ys = sorted((xy[v, 1], xy[ss.next[v], 1]))
            lo, hi = (int(np.clip(np.floor((y - y0) * inv), 0, nb[f] - 1)) for y in ys)
            assert listed[v] == list(range(lo, hi + 1)), v


def test_candidate_pairs_match_brute_force():
    rng = np.random.default_rng(0)
    for n, m, big in ((300, 200, 0), (50, 400, 3), (1, 1, 0)):
        def boxes(k):
            lo = rng.uniform(0, 1, (k, 2))
            b = np.concatenate([lo, lo + rng.uniform(0, 0.05, (k, 2))], 1)
            b[:big, 2:] += 0.6
            return b

        p, q = boxes(n), boxes(m)
        if min(n, m) > 5:
            q[:5] = np.stack([p[:5, 2], p[:5, 1], p[:5, 2] + 0.01, p[:5, 3]], 1)  # closed boxes that only touch
            q[5, :] = np.nan
        gp, gq = DD.candidate_pairs(p, q)
        meet = (p[:, None, 0] <= q[None, :, 2]) & (q[None, :, 0] <= p[:, None, 2]) & (p[:, None, 1] <= q[None, :, 3]) & (q[None, :, 1] <= p[:, None, 3])
        wp, wq = np.nonzero(meet)
        assert np.array_equal(gp, wp) and np.array_equal(gq, wq)
    e = DD.candidate_pairs(np.zeros((0, 4)), np.zeros((3, 4)))
    assert len(e[0]) == 0


def test_parse_warnings_and_skips():
    good = feature(box(0, 0, 1, 1))
    short = {"type": "Feature", "geometry": {"type": "Polygon", "coordinates": [[[10, 45], [10.1, 45], [10, 45]]]}}
    point = {"type": "Feature", "geometry": {"type": "Point", "coordinates": [10, 45]}}
    line = {"type": "Feature", "geometry": {"type": "LineString", "coordinates": [[10, 45], [11, 46]]}}
    ps, w = DD.parse([good, short, point, good], False)
    assert ps.index.tolist() == [0, 3] and w == ["Warning: invalid feature 1, skipping"]
    qs, w = DD.parse([point, good, short, line], True)
    assert qs.index.tolist() == [1]
    assert w == ["Warning: 2 OSM features are not a Polygon or MultiPolygon, ignoring them", "Warning: invalid OSM feature 2, ignoring"]


def test_decide_without_candidates_keeps_everything_on_the_host():
    # no box meets, so no device work: areal predictions are kept with NaN areas, pass-through kept, invalid dropped
    short = {"type": "Feature", "geometry": {"type": "Polygon", "coordinates": [[[10, 45], [10.1, 45], [10, 45]]]}}
    point = {"type": "Feature", "geometry": {"type": "Point", "coordinates": [10, 45]}}
    predicted = [feature(box(0, 0, 1, 1)), point, short, feature(box(5, 5, 6, 6))]
    osm = [feature(box(20, 20, 21, 21))]
    stats = {}
    keep, areas = DD.dedupe_device(predicted, osm, 0.5, stats=stats)
    assert keep.tolist() == [True, True, False, True] and np.isnan(areas).all() and stats["pairs"] == 0
    keep, _ = DD.dedupe_device(predicted, [], 0.5)
    assert keep.tolist() == [True, True, False, True]
    keep, areas = DD.dedupe_device([], osm, 0.5)
    assert keep.shape == (0,) and areas.shape == (0, 3)


def test_budget_plan_and_over_budget():
    assert DD._plan(np.array([5, 5, 5, 0, 5]), 10) == [(0, 2), (2, 5)]
    with pytest.raises(DD._lib.RsbError, match="prediction 1 needs 11 bytes"):
        DD._plan(np.array([5, 11]), 10)


def test_tool_flags():
    parser = argparse.ArgumentParser()
    sub = parser.add_subparsers()
    tool.add_parser(sub)
    args = parser.parse_args(["dedupe", "osm.geojson", "pred.geojson", "out.geojson", "--threshold", "0.5"])
    assert (args.osm, args.predicted, args.out, args.threshold, args.func) == ("osm.geojson", "pred.geojson", "out.geojson", 0.5, tool.main)
    with pytest.raises(SystemExit):
        parser.parse_args(["dedupe", "osm.geojson", "pred.geojson", "out.geojson"])  # --threshold is required


def test_tool_output_layout(tmp_path):
    open_ring = {"type": "Feature", "properties": {"a": 1}, "geometry": {"type": "Polygon", "coordinates": [[[10, 45], [11, 45], [11, 46]]]}}
    multi = feature(components=[[box(0, 0, 1, 1)], [box(2, 2, 3, 3)]])
    point = {"type": "Feature", "properties": {"b": 2}, "geometry": {"type": "Point", "coordinates": [10, 45]}}
    out = tmp_path / "out.geojson"
    assert tool.write(str(out), [open_ring, multi, point], [True, False, True]) == 2
    got = json.loads(out.read_text())
    assert list(got) == ["type", "features"] and got["type"] == "FeatureCollection"
    f0, f1 = got["features"]
    assert list(f0) == ["type", "geometry", "properties"] and f0["properties"] == {} and f1["properties"] == {}
    assert f0["geometry"] == DD.output_geometry(open_ring["geometry"]) == {"type": "Polygon", "coordinates": [[[10.0, 45.0], [11.0, 45.0], [11.0, 46.0], [10.0, 45.0]]]}  # closed
    assert all(isinstance(c, float) for c in f0["geometry"]["coordinates"][0][0])
    assert f1["geometry"] == point["geometry"]
    assert tool.write(str(out), [], []) == 0
    assert json.loads(out.read_text()) == {"type": "FeatureCollection", "features": []}


def test_axis_order_difference_on_golden_features():
    """The reference projects (lat, lon) as if it were (lon, lat). On the golden parking features against shifted copies, the
    IoU in both orders differs by about extent / R (DESIGN.md §8 records the measured maximum)."""
    feats = rr.load_golden()["features"]["features"]
    worst = 0.0
    for f in feats:
        ring = ref.rings_ll(f)
        for du, dv in ((1e-5, 0.0), (0.0, 2e-5), (3e-5, -1e-5)):
            q = [r + [du, dv] for r in ring]
            right = ref.iou(*ref.areas([DD.mollweide(r) for r in ring], [[DD.mollweide(r) for r in q]]))
            swapped = ref.iou(*ref.areas([DD.mollweide(r[:, ::-1]) for r in ring], [[DD.mollweide(r[:, ::-1]) for r in q]]))
            worst = max(worst, abs(float(right) - float(swapped)))
    assert 1e-6 < worst < 2e-6, worst
