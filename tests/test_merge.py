"""`rs merge` on the host: the EPSG:3395 projection against mpmath, the restated distance flags against exact `Fraction`
distances, the component order, the restated closing, the tracer and its simplification, and the tool's argument errors and
warnings."""

import argparse
import json
from fractions import Fraction

import numpy as np
import pytest

import merge_reference as ref
from robosat_b200 import features as FT
from robosat_b200 import merge as MG
from robosat_b200.tools import merge as tool


# ---- projection ----

def test_mercator_against_mpmath():
    import mpmath

    mpmath.mp.dps = 40
    rng = np.random.default_rng(0)
    ll = np.stack([rng.uniform(-180, 180, 200), rng.uniform(-85, 85, 200)], axis=1)
    got = MG.mercator(ll)
    a, f = mpmath.mpf(6378137), 1 / mpmath.mpf("298.257223563")
    e = mpmath.sqrt(f * (2 - f))
    for (lon, lat), (x, y) in zip(ll.tolist(), got.tolist()):
        s = mpmath.sin(mpmath.radians(lat))
        assert abs(x - float(a * mpmath.radians(lon))) <= 1e-8
        assert abs(y - float(a * (mpmath.atanh(s) - e * mpmath.atanh(e * s)))) <= 1e-7


def test_inverse_mercator_round_trip():
    rng = np.random.default_rng(1)
    ll = np.stack([rng.uniform(-180, 180, 1000), rng.uniform(-84, 84, 1000)], axis=1)
    back = MG.inverse_mercator(MG.mercator(ll))
    assert np.abs(back - ll).max() < 1e-9


# ---- distance flags ----

def _exact_within(p, a, b, d):
    """exact: the distance from p to segment ab is at most d"""
    p, a, b = [tuple(Fraction(v) for v in x) for x in (p, a, b)]
    dx, dy = b[0] - a[0], b[1] - a[1]
    t = min(max(((p[0] - a[0]) * dx + (p[1] - a[1]) * dy) / (dx * dx + dy * dy), 0), 1)
    ex, ey = p[0] - (a[0] + t * dx), p[1] - (a[1] + t * dy)
    return ex * ex + ey * ey <= Fraction(d) ** 2


def _exact_near(ra, rb, d):
    def edges(rings):
        return [(r[i], r[(i + 1) % len(r)]) for r in rings for i in range(len(r))]

    return any(_exact_within(p, a, b, d) for p in (v for r in ra for v in r) for a, b in edges(rb)) or \
        any(_exact_within(p, a, b, d) for p in (v for r in rb for v in r) for a, b in edges(ra))


def _sq(x0, y0, x1, y1):
    return np.array([(x0, y0), (x1, y0), (x1, y1), (x0, y1)], np.float64)


NEAR_CASES = [
    ("touching", [_sq(0, 0, 10, 10)], [_sq(10, 0, 20, 10)], 1, True),
    ("gap exactly d", [_sq(0, 0, 10, 10)], [_sq(13, 2, 20, 8)], 3, True),
    ("gap just over d", [_sq(0, 0, 10, 10)], [_sq(13, 2, 20, 8)], 2, False),
    ("diagonal gap 5 = 3-4-5", [_sq(0, 0, 10, 10)], [_sq(13, 14, 20, 20)], 5, True),
    ("diagonal gap 5 at d 4", [_sq(0, 0, 10, 10)], [_sq(13, 14, 20, 20)], 4, False),
    ("inside a hole, 2 from it", [_sq(0, 0, 30, 30), _sq(10, 10, 20, 20)], [_sq(12, 12, 18, 18)], 2, True),
    ("inside a hole, 2 from it, d 1", [_sq(0, 0, 30, 30), _sq(10, 10, 20, 20)], [_sq(12, 12, 18, 18)], 1, False),
    ("nested, 5 inside", [_sq(0, 0, 30, 30)], [_sq(5, 5, 25, 25)], 4, False),
    ("vertex to edge interior", [np.array([(0, 0), (10, 0), (5, 7)], np.float64)], [_sq(-5, 10, 15, 20)], 3, True),
]


@pytest.mark.parametrize("name,ra,rb,d,want", NEAR_CASES, ids=[c[0] for c in NEAR_CASES])
def test_near_flags_against_exact_distances(name, ra, rb, d, want):
    assert _exact_near([[tuple(p) for p in r] for r in ra], [[tuple(p) for p in r] for r in rb], d) == want
    assert ref.near_rings(ra, rb, d) == want


# ---- components ----

def _graph_order(n, pairs):
    """the components in the order the reference's UndirectedGraph yields them for merge.py's add_edge calls: add_edge(i, i),
    then add_edge(i, t) for each linked t, so its dict keys (the vertices, in insertion order) are restated here"""
    adj = {i: [] for i in range(n)}
    for i, j in pairs:
        adj[i].append(j)
        adj[j].append(i)
    keys = {}
    for i in range(n):
        keys.setdefault(i, None)
        for t in sorted(adj[i]):
            keys.setdefault(t, None)
    seen, out = set(), []
    for v in keys:
        if v in seen:
            continue
        comp, stack = set(), [v]
        while stack:
            x = stack.pop()
            if x not in comp:
                comp.add(x)
                stack.extend(adj[x])
        seen |= comp
        out.append(sorted(comp))
    return out


def test_component_order_is_the_min_member_order():
    rng = np.random.default_rng(2)
    n = 300
    pairs = sorted({tuple(sorted(map(int, rng.integers(0, n, 2)))) for _ in range(200)})
    pairs = [(i, j) for i, j in pairs if i != j]
    lab = ref.labels(n, pairs)
    for i in range(n):
        assert lab[i] == np.flatnonzero(lab == lab[i]).min()
    want = [np.flatnonzero(lab == l).tolist() for l in sorted(set(lab.tolist()))]
    assert _graph_order(n, pairs) == want


def test_component_order_against_undirected_graph():
    core = pytest.importorskip("robosat.graph.core")
    rng = np.random.default_rng(3)
    n = 200
    pairs = [(int(a), int(b)) for a, b in rng.integers(0, n, (150, 2)) if a < b]
    g = core.UndirectedGraph()
    for i in range(n):
        g.add_edge(i, i)
        for a, b in pairs:
            if a == i:
                g.add_edge(a, b)
            elif b == i:
                g.add_edge(b, a)
    lab = ref.labels(n, pairs)
    got = [sorted(c) for c in g.components()]
    want = [sorted(np.flatnonzero(lab == l).tolist()) for l in sorted(set(lab.tolist()))]
    assert got == want


# ---- closing ----

def _grid(h, w, boxes):
    g = np.zeros((h, w), bool)
    for r0, c0, r1, c1 in boxes:
        g[r0:r1, c0:c1] = True
    return g


def test_closing_keeps_an_aligned_square():
    g = _grid(40, 40, [(10, 10, 30, 30)])
    assert np.array_equal(ref.close(g), g)


def test_closing_bridges_a_gap_of_two_cells():
    g = _grid(40, 60, [(10, 10, 30, 25), (10, 27, 30, 45)])
    c = ref.close(g)
    assert c[11:29, 25:27].all() and np.array_equal(c & g, g)  # bridged, except where the disk rounds the bridge's ends
    assert not c[10, 25:27].any() and not c[29, 25:27].any()
    assert not c[:10].any() and not c[30:].any()


def test_closing_gives_an_l_shape_its_fillet():
    g = _grid(50, 50, [(10, 10, 40, 20), (30, 10, 40, 40)])  # an L: vertical bar and foot
    c = ref.close(g)
    added = c & ~g
    assert np.array_equal(c & g, g) and added.any()
    r, cc = np.nonzero(added)
    assert ((r < 30) & (r >= 24) & (cc >= 20) & (cc < 26)).all()  # only in the inner corner, within K + 2 cells of it
    assert added[29, 20] and not added[24, 25]


# ---- tracing ----

def _refill(polygons, H, W):
    """the cells whose centres lie inside the traced polygons (even-odd over every ring)"""
    out = np.zeros((H, W), bool)
    for poly in polygons:
        rings = [np.stack([r[:, 0], H - r[:, 1]], axis=1).astype(np.float64) for r in poly]  # y up -> rows from the top
        out |= ref.rr.fill_polygon(rings, max(H, W))[:H, :W]
    return out


@pytest.mark.parametrize("seed", range(8))
def test_trace_random_grids(seed):
    rng = np.random.default_rng(seed)
    H, W = rng.integers(5, 40, 2)
    g = rng.random((H, W)) < rng.uniform(0.3, 0.7)
    polys = MG.trace(g)
    assert sum(MG._area2(r) for p in polys for r in p) == 2 * g.sum()
    assert np.array_equal(_refill(polys, H, W), g)
    for p in polys:
        assert FT.polygon_is_valid([[tuple(v) for v in r.tolist()] for r in p])
        for r in p:
            nxt, prv = np.roll(r, -1, axis=0), np.roll(r, 1, axis=0)
            u, v = r - prv, nxt - r
            assert (u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0] != 0).all(), "no collinear vertices"
            assert tuple(r[0]) == min(map(tuple, r.tolist())), "rings start at their smallest vertex"
    assert MG._polygons_meet_in_points(polys)


def test_trace_diagonal_contact_gives_separate_polygons():
    g = np.array([[1, 0], [0, 1]], bool)
    polys = MG.trace(g)
    assert len(polys) == 2
    assert [p[0].tolist() for p in polys] == [[[0, 1], [1, 1], [1, 2], [0, 2]], [[1, 0], [2, 0], [2, 1], [1, 1]]]


def test_trace_hole_touching_the_shell_at_a_point_is_valid():
    g = np.array([[1, 1, 1, 0, 1],
                  [1, 0, 0, 1, 1],
                  [1, 0, 0, 1, 1],
                  [1, 1, 1, 1, 1]], bool)  # the 2 x 2 hole meets the outside only at the corner under the notch
    polys = MG.trace(g)
    assert len(polys) == 1 and len(polys[0]) == 2
    shell, hole = polys[0]
    assert FT.polygon_is_valid([[tuple(v) for v in r.tolist()] for r in polys[0]])
    assert set(map(tuple, shell.tolist())) & set(map(tuple, hole.tolist())) == {(3, 3)}
    two = np.array([[1, 1, 1, 1, 1],
                    [1, 0, 1, 1, 1],
                    [1, 1, 0, 1, 1],
                    [1, 1, 1, 1, 1]], bool)  # two one-cell holes touching each other at a corner
    polys = MG.trace(two)
    assert len(polys[0]) == 3 and FT.polygon_is_valid([[tuple(v) for v in r.tolist()] for r in polys[0]])


def test_simplify_keeps_a_square_and_drops_staircase_steps():
    sq = MG.trace(np.ones((10, 10), bool))[0]
    assert MG.simplified([sq])[0][0].tolist() == sq[0].tolist()
    disc = ref.close(np.pad(ref.disk(20), 8))
    polys = MG.trace(disc)
    simple = MG.simplified(polys)
    assert len(simple[0][0]) < len(polys[0][0]) / 2
    assert FT.polygon_is_valid([[tuple(v) for v in r.tolist()] for r in simple[0]])


def test_simplify_falls_back_when_a_ring_collapses():
    g = np.array([[1, 1, 1, 1, 1],
                  [1, 0, 1, 0, 1],
                  [1, 1, 1, 1, 1]], bool)  # two one-cell holes: every vertex of a unit square is within one cell of its chord
    polys = MG.trace(g)
    assert len(polys[0]) == 3
    assert [len(MG.simplify_ring(h)) for h in polys[0][1:]] == [2, 2]
    out = MG.simplified(polys)
    assert [r.tolist() for r in out[0]] == [r.tolist() for r in polys[0]]  # so the unsimplified rings are kept
    thin = np.array([[0, 0], [9, 0], [9, 1], [0, 1]])
    assert len(MG.simplify_ring(thin)) == 2
    assert MG.simplified([[thin]])[0][0].tolist() == thin.tolist()


# ---- tool ----

def _args(tmp_path, threshold, features):
    src = tmp_path / "in.geojson"
    src.write_text(json.dumps({"type": "FeatureCollection", "features": features}))
    return argparse.Namespace(features=str(src), threshold=threshold, out=str(tmp_path / "out.geojson"))


def test_tool_rejects_non_positive_threshold(tmp_path):
    for t in (0, -3):
        with pytest.raises(SystemExit) as e:
            tool.main(_args(tmp_path, t, []))
        assert "threshold" in str(e.value)
    with pytest.raises(ValueError):
        MG._check_threshold(0)


def test_tool_parser_flags():
    p = argparse.ArgumentParser()
    sub = p.add_subparsers()
    tool.add_parser(sub)
    a = p.parse_args(["merge", "in.geojson", "--threshold", "2", "out.geojson"])
    assert (a.features, a.threshold, a.out) == ("in.geojson", 2, "out.geojson")
    with pytest.raises(SystemExit):
        p.parse_args(["merge", "in.geojson", "out.geojson"])


def test_parse_warnings():
    sq = [[10.0, 45.0], [10.001, 45.0], [10.001, 45.001], [10.0, 45.001], [10.0, 45.0]]
    feats = [{"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [sq]}},
             {"type": "Feature", "properties": {}, "geometry": {"type": "Point", "coordinates": [10.0, 45.0]}},
             {"type": "Feature", "properties": {}, "geometry": {"type": "LineString", "coordinates": sq}},
             {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [sq[:3]]}},
             {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [[[10.0, 90.0], [10.1, 90.0], [10.1, 89.0], [10.0, 90.0]]]}}]
    shapes, warnings = MG.parse(feats)
    assert list(shapes.index) == [0]
    assert warnings == [MG.W_GEOMETRY.format(2), "Warning: invalid feature 3, skipping", "Warning: invalid feature 4, skipping"]


def test_plan_raises_for_a_component_over_budget():
    c = MG.Component(np.array([0]), (0, 10, 1000, 1000), 0.25)
    with pytest.raises(MG._lib.RsbError):
        MG.plan([c], c.device_bytes() - 1)
    assert MG.plan([c, c, c], 2 * c.device_bytes()) == [(0, 2), (2, 3)]


def test_component_feature_of_an_empty_closing_warns():
    c = MG.Component(np.array([0]), (0, 10, 20, 20), 0.25)
    c.closed, c.count = np.zeros((20, 20), bool), 0
    assert MG.component_feature(c) == (None, MG.W_NOT_POLYGON)


def test_component_feature_area_and_orientation():
    c = MG.Component(np.array([0]), (400000, 2000000, 60, 60), 0.25)
    g = np.zeros((60, 60), bool)
    g[10:50, 10:50] = True
    g[20:30, 20:30] = False
    c.closed, c.count = g, int(g.sum())
    f, w = MG.component_feature(c)
    assert w is None and f["geometry"]["type"] == "Polygon"
    ext, hole = f["geometry"]["coordinates"]
    assert MG.ring_area(ext) > 0 > MG.ring_area(hole)
    assert ext[0] == ext[-1]
    # Mollweide area of (40^2 - 10^2) cells of 0.25 m in EPSG:3395 at this latitude: the Mercator scale squared shrinks it
    lat = MG.inverse_mercator([[0.0, 2000000 * 0.25]])[0, 1]
    k = 1 / np.cos(np.radians(lat))
    assert abs(f["properties"]["area"] - 1500 * 0.0625 / k ** 2) <= 1.0
