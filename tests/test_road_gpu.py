"""rsb_road_* and `rs features --type road` on the H100: skeletons, iteration counts, degrees, pruned skeletons and chain lists
bit-identical to the numpy restatement (tests/road_reference.py), repeated runs and guard bytes, the tool against the restatement
path, seeded roads burned by `rs rasterize --class road` coming back as centre lines, and the agreement of line ends at tile
borders."""

import argparse
import json
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

import road_reference as rr
from robosat_b200 import _lib
from robosat_b200 import features as F
from robosat_b200.tiles import Tile
from test_building_gpu import _device, spiral

pytestmark = pytest.mark.gpu

CLASSES = ["background", "building", "road"]
COLORS = ["denim", "dark", "orange"]
ROAD = 2


def patterns(H, W):
    yy, xx = np.mgrid[:H, :W]
    rng = np.random.RandomState(H * 5 + W)
    out = [np.zeros((H, W), np.uint8), np.ones((H, W), np.uint8), ((yy + xx) % 2).astype(np.uint8), spiral(H, W)]
    out += [(rng.rand(H, W) < p).astype(np.uint8) for p in (0.3, 0.5)]
    return out


def _chains_equal(got, want):
    return len(got) == len(want) and all(np.array_equal(np.asarray(g), np.asarray(w)) for g, w in zip(got, want))


def _check(host, planes):
    skel, its = F.road_thin_device(planes)
    deg = F.road_degree_device(skel)
    pruned = F.road_prune_device(skel, deg, F.RoadHandler.min_length)
    deg2 = F.road_degree_device(pruned)
    chains = F.road_chains_device(pruned, deg2)
    skel, its, deg, pruned, deg2 = skel.cpu().numpy(), its.cpu().numpy(), deg.cpu().numpy(), pruned.cpu().numpy(), deg2.cpu().numpy()
    for n in range(host.shape[0]):
        want, want_it = rr.thin(host[n])
        assert np.array_equal(skel[n], want) and its[n] == want_it, n
        assert np.array_equal(deg[n], rr.degrees(want)), n
        want_pruned = rr.prune(want, deg[n])
        assert np.array_equal(pruned[n], want_pruned), n
        assert np.array_equal(deg2[n], rr.degrees(want_pruned)), n
        assert _chains_equal(chains[n], rr.chains(want_pruned)), n


@pytest.mark.parametrize("shape", [(640, 640), (509, 131), (1, 1)])
def test_graph_matches_restatement(cuda_device, shape):
    H, W = shape
    base = patterns(H, W)
    _check(np.stack(base), _device(np.stack(base)))
    for p in base:
        _check(p[None], torch.from_numpy(p[None].copy()).cuda())  # N = 1


@pytest.mark.parametrize("shape", [(640, 640), (509, 131), (1, 1)])
def test_batch_of_7_and_64(cuda_device, shape):
    H, W = shape
    rng = np.random.RandomState(H + W)
    for N in (7, 64):
        if N == 64 and H == 640:
            host = np.stack([road_plane(rng, 640) for _ in range(N)])  # road-like planes keep the restatement's walks short
        else:
            host = np.stack([(rng.rand(H, W) < (0.3, 0.5)[i % 2]).astype(np.uint8) for i in range(N)])
        _check(host, _device(host, pad=0 if N == 7 else 37))


def road_plane(rng, S, roads=4):
    import cv2

    m = np.zeros((S, S), np.uint8)
    for _ in range(roads):
        pts = np.cumsum(rng.uniform(-120, 120, size=(5, 2)), axis=0) + rng.uniform(0, S, size=2)
        cv2.polylines(m, [np.round(pts).astype(np.int32)], False, 1, thickness=int(rng.randint(8, 41)))
    return m


def test_repeated_runs_and_guard_bytes(cuda_device):
    rng = np.random.RandomState(4)
    N, H, W, G = 5, 300, 257, 4096
    host = np.stack([road_plane(rng, 300)[:, :W] for _ in range(N)])
    planes = _device(host)
    a = F.road_device(planes)
    b = F.road_device(planes)
    assert all(_chains_equal(x, y) for x, y in zip(a, b))
    lib, stream = _lib.load(), _lib.current_stream_ptr()
    skel = torch.full((G + N * H * W + G,), 0xAB, dtype=torch.uint8, device=cuda_device)
    its = torch.full((N + 64,), -7, dtype=torch.int32, device=cuda_device)
    _lib.check(lib.rsb_road_thin(planes.data_ptr(), planes.stride(0), N, H, W, skel[G:].data_ptr(), its[32:].data_ptr(), stream), "rsb_road_thin")
    deg = torch.full((G + N * H * W + G,), 99, dtype=torch.int8, device=cuda_device)
    _lib.check(lib.rsb_road_degree(skel[G:].data_ptr(), N, H, W, deg[G:].data_ptr(), stream), "rsb_road_degree")
    out = torch.full((G + N * H * W + G,), 0xCD, dtype=torch.uint8, device=cuda_device)
    _lib.check(lib.rsb_road_prune(skel[G:].data_ptr(), deg[G:].data_ptr(), N, H, W, 20, out[G:].data_ptr(), stream), "rsb_road_prune")
    s, i, d, o = skel.cpu().numpy(), its.cpu().numpy(), deg.cpu().numpy(), out.cpu().numpy()
    assert (s[:G] == 0xAB).all() and (s[G + N * H * W:] == 0xAB).all()
    assert (i[:32] == -7).all() and (i[32 + N:] == -7).all()
    assert (d[:G] == 99).all() and (d[G + N * H * W:] == 99).all()
    assert (o[:G] == 0xCD).all() and (o[G + N * H * W:] == 0xCD).all()
    for n in range(N):
        want, want_it = rr.thin(host[n])
        assert np.array_equal(s[G + n * H * W:G + (n + 1) * H * W].reshape(H, W), want) and i[32 + n] == want_it


def test_oversized_plane_is_refused_before_launch(cuda_device):
    with pytest.raises(_lib.RsbError, match="words"):
        F.road_thin_device(torch.zeros((1, 1024, 1024), dtype=torch.uint8, device=cuda_device))


def _dataset(tmp_path):
    path = tmp_path / "dataset.toml"
    path.write_text("[common]\nclasses = [%s]\ncolors = [%s]\n" % (", ".join("'%s'" % c for c in CLASSES), ", ".join("'%s'" % c for c in COLORS)))
    return str(path)


def _write_masks(root, cases):
    palette = [v for i in range(256) for v in (i, 255 - i, (7 * i) % 256)]
    for tile, labels in cases:
        d = os.path.join(root, str(tile.z), str(tile.x))
        os.makedirs(d, exist_ok=True)
        im = Image.fromarray(labels, mode="P")
        im.putpalette(palette)
        im.save(os.path.join(d, "%d.png" % tile.y))


def _run_features(tmp_path, masks, batch=64, name="roads"):
    from robosat_b200.tools import features as tool

    out = str(tmp_path / ("%s_%d.geojson" % (name, batch)))
    tool.main(argparse.Namespace(masks=masks, type="road", dataset=_dataset(tmp_path), out=out), batch=batch)
    with open(out) as fp:
        return json.load(fp)


def test_tool_matches_restatement_path(cuda_device, tmp_path):
    rng = np.random.RandomState(11)
    S = 512
    big = np.zeros((3 * S, 4 * S), np.uint8)
    big[rng.rand(*big.shape) < 0.02] = 1  # building speckle
    roads = road_plane(rng, 4 * S, roads=14)[:3 * S]
    big[roads == 1] = ROAD
    masks = {(70100 + i, 104000 + j): big[j * S:(j + 1) * S, i * S:(i + 1) * S].copy() for i in range(4) for j in range(3) if (i, j) != (2, 1)}
    cases = [(Tile(x, y, 18), m) for (x, y), m in masks.items()]
    root = str(tmp_path / "masks")
    _write_masks(root, cases)
    want = []
    for tile, _ in sorted(cases, key=lambda c: (c[0].z, c[0].x, c[0].y)):
        want.extend(rr.cpu_features(tile, rr.halo(masks, (tile.x, tile.y), ROAD), (S, S)))
    assert len(want) > 10
    for b in (64, 5):
        got = _run_features(tmp_path, root, b)
        assert got["type"] == "FeatureCollection"
        assert got["features"] == json.loads(json.dumps(want)), b


# --- purpose: seeded roads burned through rs rasterize come back as their centre lines ------------------------------------------

Z, S = 18, 512
WORLD = S * 2 ** Z


def to_lonlat(X, Y):
    return X / WORLD * 360.0 - 180.0, math.degrees(math.atan(math.sinh(math.pi * (1 - 2 * Y / WORLD))))


def to_pixels(lon, lat):
    y = (1 - math.log(math.tan(math.radians(lat)) + 1 / math.cos(math.radians(lat))) / math.pi) / 2
    return (lon + 180.0) / 360.0 * WORLD, y * WORLD


def capsule(a, b, w, k=12):
    """the polygon of all points within w / 2 of segment ab (global pixels), round ends of k vertices each"""
    (ax, ay), (bx, by) = a, b
    t = math.atan2(by - ay, bx - ax)
    ring = []
    for (cx, cy), t0 in (((bx, by), t - math.pi / 2), ((ax, ay), t + math.pi / 2)):
        for i in range(k + 1):
            u = t0 + math.pi * i / k
            ring.append(to_lonlat(cx + w / 2 * math.cos(u), cy + w / 2 * math.sin(u)))
    ring.append(ring[0])
    return {"type": "Feature", "geometry": {"type": "Polygon", "coordinates": [ring]}, "properties": {}}


def seeded_roads(x0, y0, nx, ny, seed):
    """non-touching, gently bending roads 8-40 px wide across a block of nx x ny tiles: [(polyline [(X, Y)], width)]"""
    rng = np.random.RandomState(seed)
    roads = []
    band = 170
    for k, y in enumerate(range(y0 * S + 90, (y0 + ny) * S - 60, band)):
        w = float(rng.uniform(8, 40))
        xs = np.linspace(x0 * S - 40, (x0 + nx) * S + 40, 9)
        ys = y + np.cumsum(rng.uniform(-12, 12, size=9))
        pts = list(zip(xs, ys))
        roads.append((pts if k % 2 == 0 else pts[::-1], w))
    return roads


def _seg_dist(p, a, b):
    p, a, b = np.asarray(p), np.asarray(a), np.asarray(b)
    ab = b - a
    t = np.clip(np.dot(p - a, ab) / max(np.dot(ab, ab), 1e-12), 0, 1)
    return float(np.hypot(*(p - (a + t * ab))))


def _poly_dist(p, line):
    return min(_seg_dist(p, a, b) for a, b in zip(line, line[1:]))


def _burn_and_extract(tmp_path, x0, y0, nx, ny, seed):
    from robosat_b200.tools import rasterize as rz_tool

    roads = seeded_roads(x0, y0, nx, ny, seed)
    feats = [capsule(a, b, w) for pts, w in roads for a, b in zip(pts, pts[1:])]
    src = tmp_path / "roads.geojson"
    src.write_text(json.dumps({"type": "FeatureCollection", "features": feats}))
    tiles = [Tile(x0 + i, y0 + j, Z) for i in range(nx) for j in range(ny)]
    csv = tmp_path / "tiles.csv"
    csv.write_text("".join("%d,%d,%d\n" % tuple(t) for t in tiles))
    labels = tmp_path / "labels"
    rz_tool.main(argparse.Namespace(features=str(src), tiles=str(csv), out=str(labels), dataset=_dataset(tmp_path), zoom=Z, size=S,
                                    class_name="road"))
    got = _run_features(tmp_path, str(labels))["features"]
    lines = [[to_pixels(lon, lat) for lon, lat in f["geometry"]["coordinates"]] for f in got]
    return roads, got, lines


def test_burned_roads_come_back_as_centre_lines(cuda_device, tmp_path):
    x0, y0, nx, ny = 70100, 104000, 4, 3
    roads, got, lines = _burn_and_extract(tmp_path, x0, y0, nx, ny, seed=5)
    assert got and all(f["geometry"]["type"] == "LineString" for f in got)
    box = (x0 * S, y0 * S, (x0 + nx) * S, (y0 + ny) * S)

    def near_end(p, w):  # the block of tiles cuts every road: its ends are there, and a flat cut end thins to a fork
        return min(p[0] - box[0], box[2] - p[0], p[1] - box[1], box[3] - p[1]) <= w

    dist = []
    for line in lines:
        for v in line:
            d, w = min((_poly_dist(v, pts), w) for pts, w in roads)
            if not near_end(v, w):
                dist.append((d, v))
    worst = max(dist)
    print("output vertices checked: %d of %d; worst distance to the centre line %.3f px at %s" % (
        len(dist), sum(map(len, lines)), worst[0], worst[1]))
    assert worst[0] <= 2.5, worst
    missed, checked = [], 0
    for pts, w in roads:
        for a, b in zip(pts, pts[1:]):
            for t in np.linspace(0, 1, int(math.hypot(b[0] - a[0], b[1] - a[1]) / 2) + 1):
                p = (a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1]))
                if near_end(p, w):
                    continue
                checked += 1
                if min(_poly_dist(p, line) for line in lines) > 2.5:
                    missed.append(p)
    assert checked > 1000 and not missed, (checked, missed[:5])


def test_line_ends_at_tile_borders(cuda_device, tmp_path):
    """Reports how many line ends on inner tile borders coincide exactly with an end in the neighbouring tile."""
    x0, y0, nx, ny = 70100, 104000, 4, 3
    _, got, lines = _burn_and_extract(tmp_path, x0, y0, nx, ny, seed=8)
    ends = [tuple(f["geometry"]["coordinates"][i]) for f in got for i in (0, -1)]
    count = {}
    for e in ends:
        count[e] = count.get(e, 0) + 1
    on_border = 0
    for (lon, lat), (X, Y) in zip(ends, [(lines[k][i]) for k in range(len(lines)) for i in (0, -1)]):
        fx, fy = X / S - x0, Y / S - y0
        inner_x = abs(fx - round(fx)) < 1e-6 and 0 < round(fx) < nx
        inner_y = abs(fy - round(fy)) < 1e-6 and 0 < round(fy) < ny
        if inner_x or inner_y:
            on_border += 1
    matched = sum(1 for e, c in count.items() if c >= 2)
    print("road line ends on inner tile borders: %d; ends shared exactly by two tiles: %d pairs" % (on_border, matched))
    assert on_border > 0
