"""`rs features --type road` on the CPU: the numpy restatement (tests/road_reference.py) on hand cases, against a per-pixel
Zhang-Suen loop written from the paper and against a graph built with networkx; the crop and the host lines; the command line,
the dataset check and the C entry points' validation."""

import argparse
import ctypes

import numpy as np
import pytest

import road_reference as rr
from robosat_b200 import _lib
from robosat_b200 import features as F
from robosat_b200.tiles import Tile

L = F.RoadHandler.min_length


def zhang_suen_loop(m):
    """Zhang & Suen (1984), one pixel at a time: P2..P9 clockwise from north, each sub-iteration on the state at its start"""
    s = (np.asarray(m) != 0).astype(np.uint8)
    H, W = s.shape

    def px(a, y, x):
        return int(a[y, x]) if 0 <= y < H and 0 <= x < W else 0

    it = 0
    while True:
        it += 1
        deleted = 0
        for sub in (0, 1):
            old = s.copy()
            for y in range(H):
                for x in range(W):
                    if not old[y, x]:
                        continue
                    p = [px(old, y - 1, x), px(old, y - 1, x + 1), px(old, y, x + 1), px(old, y + 1, x + 1), px(old, y + 1, x),
                         px(old, y + 1, x - 1), px(old, y, x - 1), px(old, y - 1, x - 1)]
                    b = sum(p)
                    a = sum(1 for i in range(8) if p[i] == 0 and p[(i + 1) % 8] == 1)
                    p2, p4, p6, p8 = p[0], p[2], p[4], p[6]
                    if sub == 0:
                        ok = p2 * p4 * p6 == 0 and p4 * p6 * p8 == 0
                    else:
                        ok = p2 * p4 * p8 == 0 and p2 * p6 * p8 == 0
                    if 2 <= b <= 6 and a == 1 and ok:
                        s[y, x] = 0
                        deleted += 1
        if not deleted:
            return s, it


@pytest.mark.parametrize("seed", range(6))
def test_thinning_matches_the_per_pixel_loop(seed):
    rng = np.random.RandomState(seed)
    shape = (rng.randint(1, 40), rng.randint(1, 40))
    m = (rng.rand(*shape) < (0.3, 0.5, 0.7)[seed % 3]).astype(np.uint8)
    m[rng.randint(0, shape[0]):, :rng.randint(0, shape[1] + 1)] |= seed % 2  # some solid blocks
    want, want_it = zhang_suen_loop(m)
    got, it = rr.thin(m)
    assert np.array_equal(got, want) and it == want_it


def test_one_pixel_line_is_unchanged():
    m = np.zeros((9, 40), np.uint8)
    m[4, 3:37] = 1
    s, it = rr.thin(m)
    assert np.array_equal(s, m) and it == 1


@pytest.mark.parametrize("w", [3, 5, 8, 15])
def test_rectangle_thins_to_its_middle_line(w):
    m = np.zeros((w + 10, 80), np.uint8)
    m[5:5 + w, 5:75] = 1
    s, _ = rr.thin(m)
    ys, xs = np.nonzero(s)
    assert set(ys) <= {5 + (w - 1) // 2, 5 + w // 2}  # the middle row (one of the two middle rows for even w)
    assert xs.min() <= 5 + w and xs.max() >= 74 - w
    (chain,) = rr.chains(s)
    assert len(chain) == s.sum()


def plus(arm=30, w=1):
    m = np.zeros((2 * arm + 1 + 10, 2 * arm + 1 + 10), np.uint8)
    c = arm + 5
    m[c - w // 2:c + w // 2 + 1, 5:2 * arm + 6] = 1
    m[5:2 * arm + 6, c - w // 2:c + w // 2 + 1] = 1
    return m, c


def test_plus_sign_is_one_junction_and_four_chains():
    m, c = plus()
    s, _ = rr.thin(m)
    d = rr.degrees(s)
    assert (d >= 3).sum() == 1 and d[c, c] == 4
    ch = rr.chains(s)
    W = m.shape[1]
    assert len(ch) == 4 and all(c * W + c in (x[0], x[-1]) for x in ch)
    assert [x[:2] for x in ch] == sorted(x[:2] for x in ch)  # (first, second) order


def test_annulus_is_one_cycle():
    yy, xx = np.mgrid[:60, :60]
    r = np.hypot(yy - 29.5, xx - 29.5)
    m = ((r > 15) & (r < 22)).astype(np.uint8)
    s, _ = rr.thin(m)
    d = rr.degrees(s)
    assert (d[d >= 0] == 2).all()
    (cycle,) = rr.chains(s)
    assert cycle[0] == cycle[-1] == int(np.flatnonzero(s.ravel())[0])
    assert len(cycle) == s.sum() + 1 and cycle[1] < cycle[-2]


def test_x_crossing():
    m = np.zeros((60, 60), np.uint8)
    for i in range(60):
        m[i, max(0, i - 2):i + 3] = 1
        m[i, max(0, 57 - i):60 - i + 2] = 1
    s, _ = rr.thin(m)
    pruned = rr.prune(s, rr.degrees(s))
    ch = rr.chains(pruned)
    d = rr.degrees(pruned)
    junctions = np.argwhere(d >= 3)
    assert len(junctions) >= 1 and (np.abs(junctions - 29.5) <= 4).all()  # a crossing may thin to a small cluster of junctions
    assert sum(1 for x in ch if d.flat[x[0]] == 1 or d.flat[x[-1]] == 1) == 4


@pytest.mark.parametrize("spur, kept", [(L - 1, False), (L, True)])
def test_spur_threshold(spur, kept):
    m = np.zeros((80, 100), np.uint8)
    m[60, 5:95] = 1
    m[60 - spur:60, 50] = 1  # spur pixels, not counting the junction at (60, 50)
    d = rr.degrees(m)
    assert d[60, 50] == 3 and rr.thin(m)[0].sum() == m.sum()
    pruned = rr.prune(m, d)
    assert pruned[60 - spur:60, 50].any() == kept and pruned[60 - spur:60, 50].all() == kept
    assert pruned[60].sum() == 90
    assert len(rr.chains(pruned)) == (3 if kept else 1)


@pytest.mark.parametrize("n, kept", [(L - 1, False), (L, True)])
def test_isolated_piece_threshold(n, kept):
    m = np.zeros((10, 40), np.uint8)
    m[5, 3:3 + n] = 1
    assert rr.prune(m, rr.degrees(m)).any() == kept


def _graph(s):
    import networkx as nx

    H, W = s.shape
    g = nx.Graph()
    on = set(map(int, np.flatnonzero(s.ravel())))
    g.add_nodes_from(on)
    for p in on:
        y, x = divmod(p, W)
        for dy, dx in ((0, 1), (1, 0), (1, 1), (1, -1)):
            yy, xx = y + dy, x + dx
            if not (0 <= yy < H and 0 <= xx < W) or yy * W + xx not in on:
                continue
            if dy and dx and (s[yy, x] or s[y, xx]):
                continue
            g.add_edge(p, yy * W + xx)
    return g


@pytest.mark.parametrize("seed", range(4))
def test_degrees_and_chains_against_networkx(seed):
    rng = np.random.RandomState(seed)
    m = (rng.rand(64, 70) < 0.45).astype(np.uint8)
    s, _ = rr.thin(m)
    s = rr.prune(s, rr.degrees(s)) if seed % 2 else s
    g = _graph(s)
    d = rr.degrees(s)
    assert all(d.flat[p] == g.degree(p) for p in g.nodes)
    assert (d.ravel()[s.ravel() == 0] == -1).all()
    ch = rr.chains(s, d)
    edges = [frozenset(e) for x in ch for e in zip(x, x[1:])]
    assert sorted(map(sorted, edges)) == sorted(map(sorted, map(frozenset, g.edges)))  # every edge in exactly one chain
    for x in ch:
        assert all(g.degree(p) == 2 for p in x[1:-1])
        assert x[0] <= x[-1]
        ends_nodes = g.degree(x[0]) != 2
        if not ends_nodes:  # a node-free cycle, from its component's smallest pixel
            assert x[0] == x[-1] == min(nx_component(g, x[0]))
    assert [x[:2] for x in ch] == sorted(x[:2] for x in ch)


def nx_component(g, p):
    import networkx as nx

    return nx.node_connected_component(g, p)


def test_halo_plane_matches_the_restatement():
    rng = np.random.RandomState(2)
    masks = {(x, y): rng.randint(0, 3, size=(96, 96)).astype(np.uint8) for x in range(3) for y in range(3) if (x, y) != (2, 0)}
    h = 20
    for tile in masks:
        out = np.full((96 + 2 * h, 96 + 2 * h), 7, np.uint8)
        nb = {(dy, dx): masks.get((tile[0] + dx, tile[1] + dy)) for dy in (-1, 0, 1) for dx in (-1, 0, 1)}
        F.halo_plane(masks[tile], nb, 2, h, out)
        assert np.array_equal(out, rr.halo(masks, tile, 2, h)), tile


def test_crop_adds_midpoints_on_edges_and_corners():
    H = W = 8
    h = 2
    Wp = W + 2 * h

    def idx(y, x):  # tile coordinates -> plane index
        return (y + h) * Wp + x + h

    runs = F._runs(np.array([idx(3, -1), idx(3, 0), idx(3, 1), idx(3, 2)]), H, W, h)
    assert runs == [([(0.0, 3.5), (0.5, 3.5), (1.5, 3.5), (2.5, 3.5)], False)]
    runs = F._runs(np.array([idx(-1, -1), idx(0, 0), idx(1, 1)]), H, W, h)
    assert runs == [([(0.0, 0.0), (0.5, 0.5), (1.5, 1.5)], False)]  # a diagonal step through the corner
    runs = F._runs(np.array([idx(7, 5), idx(8, 6), idx(8, 7), idx(7, 8)]), H, W, h)
    assert runs == [([(5.5, 7.5), (6.0, 8.0)], False)]  # leaves through the bottom edge; the re-entry ends outside
    runs = F._runs(np.array([idx(2, 3), idx(2, 8), idx(2, 7)]), H, W, h)
    assert runs == [([(3.5, 2.5), (6.0, 2.5)], False), ([(8.0, 2.5), (7.5, 2.5)], False)]
    assert F._runs(np.array([idx(-2, 0), idx(-1, 0)]), H, W, h) == []
    ring = [idx(1, 1), idx(1, 2), idx(2, 2), idx(2, 1), idx(1, 1)]
    assert F._runs(np.array(ring), H, W, h) == [([(1.5, 1.5), (2.5, 1.5), (2.5, 2.5), (1.5, 2.5)], True)]


def test_lines_from_chains():
    pytest.importorskip("cv2")
    tile = Tile(70100, 104000, 18)
    H = W = 64
    h = 4
    Wp = W + 2 * h
    chain = [(10 + h) * Wp + x + h for x in range(-h, 30)]
    ring = [(40 + h) * Wp + 40 + h, (40 + h) * Wp + 41 + h, (41 + h) * Wp + 41 + h, (41 + h) * Wp + 40 + h, (40 + h) * Wp + 40 + h]
    feats = F.lines_from_chains(tile, [chain, ring], (H, W), h)
    assert len(feats) == 2 and all(f["geometry"]["type"] == "LineString" and f["properties"] == {} for f in feats)
    west, south, east, north = F.bounds(tile)
    (x0, y0), (x1, y1) = feats[0]["geometry"]["coordinates"]
    assert x0 == west and abs((north - y0) / (north - south) * H - 10.5) < 1e-9
    assert abs((x1 - west) / (east - west) * W - 29.5) < 1e-9
    closed = feats[1]["geometry"]["coordinates"]
    assert closed[0] == closed[-1] and len(closed) >= 3


def _parser():
    from robosat_b200.tools import features as tool

    p = argparse.ArgumentParser()
    tool.add_parser(p.add_subparsers())
    return p, tool


def test_parser_takes_road():
    p, tool = _parser()
    args = p.parse_args(["features", "masks/", "--type", "road", "--dataset", "dataset.toml", "out.geojson"])
    assert (args.type, args.func) == ("road", tool.main)
    assert tool.handlers["road"] is F.RoadHandler
    with pytest.raises(SystemExit):
        p.parse_args(["features", "masks/", "--type", "roads", "--dataset", "dataset.toml", "out.geojson"])


def test_dataset_without_road_exits_naming_it(tmp_path):
    _, tool = _parser()
    ds = tmp_path / "dataset.toml"
    ds.write_text("[common]\nclasses = ['background', 'building']\ncolors = ['denim', 'orange']\n")
    masks = tmp_path / "masks"
    masks.mkdir()
    with pytest.raises(SystemExit) as e:
        tool.main(argparse.Namespace(masks=str(masks), type="road", dataset=str(ds), out=str(tmp_path / "out.geojson")))
    assert "road" in str(e.value)


def test_zoom_other_than_18_raises():
    with pytest.raises(NotImplementedError, match="Road"):
        F.RoadHandler().apply_batch([Tile(1, 2, 17)], None)


def test_handler_defaults():
    H = F.RoadHandler
    assert (H.halo, H.min_area, H.min_hole_area, H.min_length, H.simplify_epsilon) == (64, 256, 256, 20, 1.0)


def test_road_validation_runs_before_the_device_check():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 64)()
    out = (ctypes.c_uint8 * 64)()
    deg = (ctypes.c_int8 * 64)()
    i32 = [(ctypes.c_int32 * 64)() for _ in range(4)]
    i64 = [(ctypes.c_int64 * 64)() for _ in range(5)]

    def thin(N=1, H=4, W=4, stride=16, planes=buf, skel=out, its=i32[0]):
        return lib.rsb_road_thin(planes, stride, N, H, W, skel, its, None)

    assert thin() == -3                                             # valid, but no sm_90 device
    assert thin(planes=None) == -1 and thin(its=None) == -1
    assert thin(stride=15) == -1 and "image_stride" in _lib.last_error()
    assert thin(N=0) == -4 and thin(W=0) == -4
    assert thin(H=4097, stride=4097 * 4) == -4
    assert thin(H=640, W=640, stride=640 * 640) == -3               # 12 800 words fit
    assert thin(H=1024, W=1024, stride=1 << 20) == -4 and "words" in _lib.last_error()
    assert lib.rsb_road_degree(buf, 1, 4, 4, deg, None) == -3
    assert lib.rsb_road_degree(buf, 1, 4, 4, None, None) == -1
    assert lib.rsb_road_prune(buf, deg, 1, 4, 4, 20, out, None) == -3
    assert lib.rsb_road_prune(buf, deg, 1, 4, 4, -1, out, None) == -1
    assert lib.rsb_road_prune(buf, deg, 1, 4, 4, 20, buf, None) == -1 and "alias" in _lib.last_error()
    assert lib.rsb_road_chain_count(buf, deg, i32[0], i32[1], 1, 4, 4, i32[2], i64[0], i64[1], None) == -3
    assert lib.rsb_road_chain_count(buf, deg, i32[0], i32[0], 1, 4, 4, i32[2], i64[0], i64[1], None) == -1
    assert lib.rsb_road_chain_count(buf, deg, i32[0], i32[1], 1, 4, 4, i32[2], i64[0], None, None) == -1
    assert lib.rsb_road_chain_write(buf, deg, i32[0], i32[1], 1, 4, 4, i32[2], i64[0], i64[1], i64[2], i64[3], i32[3], None) == -3
    assert lib.rsb_road_chain_write(buf, deg, i32[0], i32[1], 1, 4, 4, i32[2], i64[0], i64[1], i64[2], None, i32[3], None) == -1
    assert lib.rsb_road_chain_write(buf, deg, i32[0], i32[1], 0, 4, 4, i32[2], i64[0], i64[1], i64[2], i64[3], i32[3], None) == -4
