"""`rs extract` on the H100: DenseNodes decode, locate / gather and ring validity against tests/extract_reference.py and
`features.polygon_is_valid`, the whole extraction and the tool against the restatement, and the purpose test: the golden
parking fixture written as OSM ways comes back exactly and rasterizes to the golden masks."""

import argparse
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import extract_reference as xr  # noqa: E402
import rasterize_reference as rr  # noqa: E402

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import extract as EX  # noqa: E402
from robosat_b200.features import polygon_is_valid  # noqa: E402

pytestmark = pytest.mark.gpu

INVALID = -2 ** 31


def _fix(n):
    return (n[0], n[1] if abs(n[1]) <= 1800000000 else INVALID, n[2] if abs(n[2]) <= 900000000 else INVALID)


def _decode(raw):
    """the device decode of every node block of a file -> [(id, x, y)] in file order"""
    data = np.frombuffer(raw, np.uint8)
    frames = EX.read_frames(data)
    buf, offs, sizes = EX.inflate(data, frames[frames[:, 0] == _lib.RSB_PBF_BLOB_DATA])
    p = EX.parse(buf, offs, sizes, _lib.RSB_PBF_NODES)
    segs = p["segs"]
    counts = segs[:, _lib.RSB_PBF_SEG_COUNT]
    segs[:, _lib.RSB_PBF_SEG_OUT_FIRST] = np.cumsum(counts) - counts
    n = int(counts.sum())
    ids = torch.full((n,), 7, dtype=torch.int64, device="cuda")
    xy = torch.full((n, 2), 7, dtype=torch.int32, device="cuda")
    status = torch.ones((1,), dtype=torch.int32, device="cuda")
    dense = segs[:, _lib.RSB_PBF_SEG_KIND] == 0
    blk = torch.from_numpy(buf).cuda()
    offs_dev = torch.from_numpy(offs).cuda()
    segs_dev = torch.from_numpy(np.ascontiguousarray(segs[dense])).cuda()
    _lib.check(_lib.load().rsb_pbf_dense_nodes(blk.data_ptr(), offs_dev.data_ptr(), segs_dev.data_ptr(), int(dense.sum()), ids.data_ptr(), xy.data_ptr(),
                                               status.data_ptr(), _lib.current_stream_ptr()), "dense")
    assert int(status.item()) == 0
    ids, xy = ids.cpu().numpy(), xy.cpu().numpy()
    for s in segs[~dense]:
        o, c, h = s[_lib.RSB_PBF_SEG_OUT_FIRST], s[_lib.RSB_PBF_SEG_COUNT], s[_lib.RSB_PBF_SEG_HOST_FIRST]
        ids[o: o + c], xy[o: o + c] = p["host_ids"][h: h + c], p["host_xy"][h: h + c]
    return [(int(i), int(x), int(y)) for i, (x, y) in zip(ids, xy)]


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_dense_nodes_match_the_reader(cuda_device, seed):
    rng = np.random.RandomState(seed)
    w = xr.Writer(compression=["zlib", "raw"][seed % 2])
    groups = [[(5, 1, -1)]]  # a single-node group
    nid = -(2 ** 62) if seed == 0 else 0
    for size in (8000, 1, 33, 257, 1000):
        g = []
        for _ in range(size):
            step = int(rng.choice([1, 2, 1000, 2 ** 40, 2 ** 61]))
            nid = nid + step if nid + step < 2 ** 62 else -(2 ** 62)  # extreme deltas, 10-byte zigzags
            g.append((nid, int(rng.randint(-2 ** 31, 2 ** 31)), int(rng.choice([rng.randint(-2 ** 31, 2 ** 31), 2 ** 50, -(2 ** 50)]))))
        groups.append(g)
    w.block(dense_groups=groups, granularity=[100, 1, 1000, 7][seed], lat_offset=[0, -123456, 5, 2 ** 40][seed], lon_offset=[0, 99, -7, -(2 ** 35)][seed])
    w.block(dense=[(1, 2, 3), (1, 4, 5)], nodes=[(9, 900000000, 1800000000), (10, 900000001, -1800000001)])
    raw = w.bytes()
    nodes, _ = xr.read(raw)
    got = _decode(raw)
    assert len(got) == len(nodes)
    assert got == [_fix(n) for n in nodes]


def _ids_file(path, nodes_blocks, ways):
    w = xr.Writer()
    for b in nodes_blocks:
        w.block(dense=b)
    w.block(ways=ways)
    return w.write(path)


def _run(path, kind, **kw):
    feats, warns = EX.extract_device(str(path), kind, **kw)
    want_f, want_w = xr.expected(open(str(path), "rb").read(), kind)
    assert warns == want_w
    assert feats == want_f
    assert json.dumps(feats) == xr.dumps(want_f)[len('{"type": "FeatureCollection", "features": '):-1]
    return feats, warns


def test_locate_gather_missing_duplicates_and_repeated_refs(cuda_device, tmp_path):
    sq = lambda i, x, y: (i, xr.raw_coord(y), xr.raw_coord(x))  # noqa: E731
    b1 = [sq(1, 0, 0), sq(2, 100, 0), sq(3, 100, 100), sq(4, 0, 100), sq(-7, 50, 50)]
    b2 = [sq(2, 200, 0), sq(8, 1, 1), sq(2, 300, 0)]  # node 2 repeated: the last one wins
    ways = [(10, [1, 2, 3, 4, 1], {"amenity": "parking"}),
            (11, [1, 2, 99, 4, 1], {"amenity": "parking"}),            # missing node
            (12, [1, 2, 3, 3, 4, 1], {"amenity": "parking"}),          # a repeated ref
            (-13, [-7, 1, 2, -7], {"amenity": "parking"}),             # a negative id
            (14, [1, 3, 2, 4, 1], {"amenity": "parking"})]             # a bow-tie
    path = _ids_file(tmp_path / "a.osm.pbf", [b1, b2], ways)
    feats, warns = _run(path, "parking")
    assert len(feats) == 3 and feats[0]["geometry"]["coordinates"][0][1] == [300 / 1e7, 0.0]
    assert warns == [xr.W_LOCATION.format(11), xr.W_INVALID.format(14), xr.W_LOCATION_SUMMARY.format(1)]


def _city(path, seed, n_nodes=100000, n_ways=10000, per_block=8000):
    """a seeded synthetic city: grid-ish nodes, closed ways of 4-12 refs, about a third of them parking or buildings, decoys"""
    rng = np.random.RandomState(seed)
    ids = np.cumsum(rng.randint(1, 5, n_nodes)) - 1000
    lat = rng.randint(520000000, 520400000, n_nodes)
    lon = rng.randint(133000000, 133600000, n_nodes)
    w = xr.Writer()
    for a in range(0, n_nodes, per_block):
        sl = slice(a, a + per_block)
        nodes = list(zip(ids[sl].tolist(), lat[sl].tolist(), lon[sl].tolist()))
        if (a // per_block) % 4 == 3:
            w.block(nodes=nodes[:300], dense=nodes[300:], granularity=100)
        else:
            w.block(dense=nodes)
    ways = []
    for k in range(n_ways):
        c = rng.randint(0, n_nodes - 20)
        m = rng.randint(3, 12)
        if rng.rand() < 0.3:  # consecutive nodes
            refs = [int(ids[c + j]) for j in range(m)]
            refs.append(refs[0])
        else:
            refs = [int(r) for r in ids[rng.randint(0, n_nodes, m)]]
            refs.append(refs[0] if rng.rand() < 0.9 else refs[1])
        if rng.rand() < 0.02:
            refs[1] = int(ids[-1] + 1000)  # missing
        tags = [{"amenity": "parking"}, {"amenity": "parking", "parking": "underground"}, {"building": "yes"}, {"building": "ruins"},
                {"building": "house", "location": "underwater"}, {"highway": "residential"}][rng.randint(6)]
        ways.append((int(k * 3 - 500), refs, tags))
    for a in range(0, n_ways, 2500):
        w.block(ways=ways[a: a + 2500])
    return w.write(str(path))


@pytest.mark.parametrize("kind", ["parking", "building"])
def test_city_end_to_end_and_determinism(cuda_device, tmp_path, kind):
    path = _city(tmp_path / "city.osm.pbf", 11)
    feats, warns = _run(path, kind)
    assert len(feats) > 100
    again = EX.extract_device(path, kind)
    assert json.dumps(again) == json.dumps((feats, warns))
    stats = {}
    small = EX.extract_device(path, kind, budget=1500000, stats=stats)  # several node chunks
    assert stats["nodes"] == 100000
    assert json.dumps(small) == json.dumps((feats, warns))
    with pytest.raises(_lib.RsbError, match="budget"):
        EX.extract_device(path, kind, budget=1000)


def test_tool_end_to_end(cuda_device, tmp_path, capsys):
    from robosat_b200.tools import extract as tool

    path = _city(tmp_path / "city.osm.pbf", 12, n_nodes=20000, n_ways=3000)
    want_f, want_w = xr.expected(open(path, "rb").read(), "building")
    os.makedirs(str(tmp_path / "out"))
    tool.main(argparse.Namespace(type="building", batch=100, map=path, out=str(tmp_path / "out" / "b.geojson")))
    assert capsys.readouterr().err.splitlines() == want_w
    files = sorted(tmp_path.glob("out/b-*.geojson"))
    assert len(files) == (len(want_f) + 99) // 100
    got = [json.load(open(str(f))) for f in files]
    assert sorted(len(g["features"]) for g in got) == sorted([100] * (len(want_f) // 100) + ([len(want_f) % 100] if len(want_f) % 100 else []))
    key = lambda f: json.dumps(f)  # noqa: E731
    assert sorted(key(f) for g in got for f in g["features"]) == sorted(key(f) for f in want_f)


# --- validity ---------------------------------------------------------------------------------------------------------------


def _valid(rings):
    """rsb_extract_valid on closed integer rings -> list of bools"""
    offs = np.zeros(len(rings) + 1, np.int64)
    offs[1:] = np.cumsum([len(r) for r in rings])
    verts = torch.from_numpy(np.concatenate([np.asarray(r, np.int32).reshape(-1, 2) for r in rings])).cuda()
    valid, _ = EX.valid_rings(verts, offs)
    return [bool(v) for v in valid.cpu().numpy()]


def _closed(r):
    return list(r) + [r[0]]


def test_valid_hand_cases(cuda_device):
    cases = {
        "square": [(0, 0), (10, 0), (10, 10), (0, 10)],
        "bow-tie": [(0, 0), (10, 10), (10, 0), (0, 10)],
        "spike": [(0, 0), (10, 0), (10, 10), (10, 20), (10, 10), (0, 10)],
        "self-touch at a vertex": [(0, 0), (10, 0), (5, 5), (10, 10), (0, 10), (5, 5)],
        "collinear overlap": [(0, 0), (10, 0), (5, 0), (5, 5)],
        "repeated points": [(0, 0), (0, 0), (10, 0), (10, 0), (10, 10), (0, 10), (0, 10)],
        "zero area": [(0, 0), (10, 0), (20, 0)],
        "3 distinct": [(0, 0), (10, 0), (0, 10)],
        "2 distinct": [(0, 0), (10, 0), (0, 0), (10, 0)],
        "near collinear": [(0, 0), (2000000000 // 2, 1), (1000000000 * 2 - 1, 2), (0, 5)],
        "extremes": [(-1800000000, -900000000), (1800000000, -900000000), (1800000000, 900000000), (-1800000000, 900000000)],
        "extreme bow-tie": [(-1800000000, -900000000), (1800000000, 900000000), (1800000000, -900000000), (-1800000000, 900000000)],
        "extreme sliver": [(-1800000000, -900000000), (1800000000, 900000000), (1799999999, 899999999), (-1800000000, -899999999)],
    }
    rings = [_closed(r) for r in cases.values()]
    got = _valid(rings)
    want = [polygon_is_valid([r]) for r in rings]
    assert got == want, [(k, g, w) for k, g, w in zip(cases, got, want) if g != w]
    assert dict(zip(cases, got))["square"] and not dict(zip(cases, got))["bow-tie"]


def test_valid_random_rings(cuda_device):
    rng = np.random.RandomState(3)
    rings = []
    for k in range(600):
        m = rng.randint(3, 12)
        span = [3, 10, 2 ** 20, 1800000000][k % 4]
        r = [(int(rng.randint(-span, span + 1)), int(rng.randint(-span // 2, span // 2 + 1))) for _ in range(m)]
        if k % 5 == 0:  # near-collinear triples
            a, b = r[0], r[1]
            r.insert(1, ((a[0] + b[0]) // 2, (a[1] + b[1]) // 2 + int(rng.randint(-1, 2))))
        if k % 7 == 0:  # a convex polygon: sorted angles
            t = np.sort(rng.uniform(0, 2 * np.pi, m))
            r = [(int(span * np.cos(a)), int(span / 2 * np.sin(a))) for a in t]
        rings.append(_closed(r))
    got = _valid(rings)
    want = [polygon_is_valid([r]) for r in rings]
    assert got == want
    assert 50 < sum(got) < 550


@pytest.mark.parametrize("n", [300, 2000, 10000])
def test_valid_long_rings(cuda_device, n):
    """long rings go through the pair tiles: a convex ring is valid; moving one vertex across the ring, adding a far-apart touch,
    or a collinear doubling back makes it invalid (each known by construction; polygon_is_valid agrees at 300)"""
    t = np.linspace(0, 2 * np.pi, n, endpoint=False)
    base = [(int(900000000 * np.cos(a)), int(450000000 * np.sin(a))) for a in t]
    crossing = list(base)
    crossing[n // 3] = (-crossing[n // 3][0], -crossing[n // 3][1])     # a vertex thrown across: edges cross
    touching = list(base)
    touching[n // 2] = touching[0]                                         # a vertex on a far vertex
    spike = base[: n // 4] + [base[n // 4], (base[n // 4][0] * 2, base[n // 4][1] * 2), base[n // 4]] + base[n // 4 + 1:]
    rings = [_closed(r) for r in (base, crossing, touching, spike)]
    got = _valid(rings)
    assert got == [True, False, False, False]
    if n <= 300:
        assert got == [polygon_is_valid([r]) for r in rings]


# --- purpose: OSM -> extract -> rasterize reproduces the golden labels ------------------------------------------------------


def test_golden_parking_round_trip(cuda_device, tmp_path, capsys):
    from robosat_b200 import rasterize as RZ
    from robosat_b200.tiles import Tile
    from robosat_b200.tools import extract as tool

    g = rr.load_golden()
    feats = g["features"]["features"]
    w = xr.Writer()
    nodes, ways, nid = [], [], 1000
    for k, f in enumerate(feats):
        assert f["geometry"]["type"] == "Polygon" and len(f["geometry"]["coordinates"]) == 1
        ring = f["geometry"]["coordinates"][0]
        refs = []
        for lon, lat in ring[:-1]:
            x, y = int(round(lon * 1e7)), int(round(lat * 1e7))
            assert x / 1e7 == lon and y / 1e7 == lat  # 7 decimals: the lattice holds them exactly
            nodes.append((nid, xr.raw_coord(y), xr.raw_coord(x)))
            refs.append(nid)
            nid += 1
        ways.append((5000 + k, refs + [refs[0]], {"amenity": "parking"}))
    sq = [(1, 0, 0), (2, 0, 1000), (3, 1000, 1000), (4, 1000, 0)]
    nodes += [(i, xr.raw_coord(520000000 + a), xr.raw_coord(133000000 + b)) for i, a, b in sq]
    decoys = [(9001, [1, 2, 3, 4, 1], {"amenity": "parking", "parking": "underground"}),
              (9002, [1, 2, 3, 4], {"amenity": "parking"}),
              (9003, [1, 3, 2, 4, 1], {"amenity": "parking"}),
              (9004, [1, 2, 3, 77777, 1], {"amenity": "parking"})]
    w.block(dense=nodes)
    w.block(ways=ways[:2] + decoys[:2] + ways[2:] + decoys[2:])
    path = w.write(str(tmp_path / "golden.osm.pbf"))
    out = tmp_path / "out"
    out.mkdir()
    tool.main(argparse.Namespace(type="parking", batch=100000, map=path, out=str(out / "parking.geojson")))
    assert capsys.readouterr().err.splitlines() == [xr.W_INVALID.format(9003), xr.W_LOCATION.format(9004), xr.W_LOCATION_SUMMARY.format(1)]
    (f,) = list(out.glob("parking-*.geojson"))
    got = json.load(open(str(f)))["features"]
    assert [x["geometry"]["coordinates"] for x in got] == [x["geometry"]["coordinates"] for x in feats]
    tiles = [Tile(*t) for t in g["masks"]]
    polygons = [p["coordinates"] for x in got for p in RZ.feature_to_mercator(x)]
    burned, _ = RZ.burn_device(tiles, polygons, 512)
    for i, t in enumerate(tiles):
        assert int((burned[i].cpu().numpy() != g["masks"][tuple(t)]).sum()) == 0, t
