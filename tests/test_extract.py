"""`rs extract` without a GPU: the wire format, the restatement's reader and rules, the library's host entry points (framing,
inflate, way decode, tag values, DenseNodes byte ranges, plain Nodes) against the reader, every format error, and the tool's
flags and output files."""

import argparse
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import extract_reference as xr  # noqa: E402

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import extract as EX  # noqa: E402


def test_known_byte_encodings():
    assert xr.varint(300) == b"\xac\x02"
    assert xr.varint(xr.zigzag(-1)) == b"\x01"
    assert xr.varint(xr.zigzag(1)) == b"\x02"
    assert xr.varint(-1) == b"\xff" * 9 + b"\x01"
    assert xr.varint(1 << 63) == b"\x80" * 9 + b"\x01"
    assert xr.read_varint(xr.varint(-1), 0) == ((1 << 64) - 1, 10)
    for v in (0, 1, -1, 2 ** 62, -(2 ** 63), 2 ** 63 - 1):
        assert xr.unzigzag(xr.read_varint(xr.varint(xr.zigzag(v)), 0)[0]) == v


def test_coordinate_rule():
    assert xr.to_fixed(123, 100, 0) == 123
    assert xr.to_fixed(-150, 1, 0) == -1           # -1.5 truncates toward zero, not to -2
    assert xr.to_fixed(150, 1, 0) == 1
    assert xr.to_fixed(7, 1000, 0) == 70
    assert xr.to_fixed(-7, 1000, 50) == -69        # (50 - 7000) / 100 = -69.5 -> -69
    assert xr.to_fixed(3, 100, -1000) == -7
    assert xr.valid_location(1800000000, -900000000) and not xr.valid_location(1800000001, 0) and not xr.valid_location(0, -900000001)


def _city():
    w = xr.Writer()
    nodes = [(i, xr.raw_coord(500000000 + 10 * i), xr.raw_coord(130000000 + 7 * (i % 5))) for i in range(1, 21)]
    w.block(dense=nodes[:10])
    w.block(nodes=nodes[10:], granularity=100)
    w.block(ways=[(100, [1, 2, 3, 1], {"amenity": "parking"}), (-5, [4, 5, 6, 7, 4], {"building": "yes", "name": "x"})])
    return w


def test_writer_reader_round_trip():
    w = _city()
    nodes, ways = xr.read(w.bytes())
    assert [n[0] for n in nodes] == list(range(1, 21))
    assert nodes[3] == (4, 130000000 + 7 * 4, 500000000 + 40)
    assert ways == [(100, [1, 2, 3, 1], {"amenity": "parking"}), (-5, [4, 5, 6, 7, 4], {"building": "yes", "name": "x"})]
    # unpacked fields, raw blobs, offsets and granularity read the same
    w2 = xr.Writer(compression="raw")
    w2.block(dense=[(-3, xr.raw_coord(-7, 10, 50), xr.raw_coord(90, 10, -30))], granularity=10, lat_offset=50, lon_offset=-30, packed=False)
    w2.block(ways=[(2 ** 40, [-3, -3, 5], {"k": "v"})], packed=False)
    nodes, ways = xr.read(w2.bytes())
    assert nodes == [(-3, 90, -7)]
    assert ways == [(2 ** 40, [-3, -3, 5], {"k": "v"})]


@pytest.mark.parametrize("kind,tags,want", [
    ("parking", {"amenity": "parking"}, True),
    ("parking", {"amenity": "parking", "parking": "surface"}, True),
    ("parking", {"amenity": "parking", "parking": "multi-storey"}, True),
    ("parking", {"amenity": "cafe"}, False),
    ("parking", {"parking": "surface"}, False),
    ("building", {"building": "yes"}, True),
    ("building", {"building": "house", "location": "overground"}, True),
    ("building", {"amenity": "parking"}, False),
] + [("parking", {"amenity": "parking", "parking": v}, False) for v in sorted(xr.PARKING_FILTER)]
  + [("building", {"building": v}, False) for v in sorted(xr.BUILDING_FILTER)]
  + [("building", {"building": "yes", "location": v}, False) for v in sorted(xr.LOCATION_FILTER)])
def test_handler_rules(kind, tags, want):
    assert xr.wanted(kind, tags) == want
    # the library's pass-1 decode and the vectorised rule agree
    w = xr.Writer()
    w.block(ways=[(1, [1, 2, 3, 1], tags), (2, [1, 2, 1], tags), (3, [1, 2, 3, 4], tags)])
    data = np.frombuffer(w.bytes(), np.uint8)
    frames = EX.read_frames(data)
    buf, offs, sizes = EX.inflate(data, frames[frames[:, 0] == _lib.RSB_PBF_BLOB_DATA])
    keys, anchor = EX.QUERIES[kind]
    p = EX.parse(buf, offs, sizes, _lib.RSB_PBF_WAYS, keys, anchor)
    kept = list(p["way_ids"][EX.select(kind, p)])
    assert kept == ([1] if want else [])


def test_is_polygon():
    assert xr.is_polygon([1, 2, 3, 1]) and not xr.is_polygon([1, 2, 1]) and not xr.is_polygon([1, 2, 3, 4]) and xr.is_polygon([1, 1, 1, 1])


def _seeded_file(rng, compression="zlib"):
    w = xr.Writer(compression=compression)
    nid = -50
    for b in range(4):
        dense = []
        for _ in range(rng.randint(1, 300)):
            nid += rng.randint(1, 1000)
            dense.append((nid, int(rng.randint(-900000000, 900000000)), int(rng.randint(-1800000000, 1800000000))))
        plain = [(nid + k + 1, int(rng.randint(-9e8, 9e8)), int(rng.randint(-1.8e9, 1.8e9))) for k in range(rng.randint(0, 5))]
        nid += 10
        ways = [(int(rng.randint(-2 ** 40, 2 ** 40)), [int(r) for r in rng.randint(-60, 2000, rng.randint(0, 12))],
                 {"building": ["yes", "ruins", "house"][rng.randint(3)], "location": ["underground", "x"][rng.randint(2)]} if rng.rand() < 0.7 else {"k": "v"})
                for _ in range(rng.randint(0, 30))]
        w.block(dense=dense, nodes=plain, ways=ways, granularity=[100, 1000, 7][b % 3], lat_offset=[0, 12345, -999][b % 3],
                lon_offset=[0, -5, 77][b % 3], packed=b != 2)
    return w


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_host_entry_points_against_the_reader(seed):
    rng = np.random.RandomState(seed)
    w = _seeded_file(rng, compression=["zlib", "raw", "zlib"][seed])
    raw = w.bytes()
    nodes, ways = xr.read(raw)
    data = np.frombuffer(raw, np.uint8)
    frames = EX.read_frames(data)
    assert list(frames[:, 0]) == [_lib.RSB_PBF_BLOB_HEADER] + [_lib.RSB_PBF_BLOB_DATA] * 4
    hb, ho, hs = EX.inflate(data, frames[:1])
    EX.check_header(hb[ho[0]: ho[0] + hs[0]])
    buf, offs, sizes = EX.inflate(data, frames[1:])
    # ways: every building way, with its refs and tag values
    p = EX.parse(buf, offs, sizes, _lib.RSB_PBF_WAYS, ("building", "location"))
    want = [wy for wy in ways if "building" in wy[2]]
    assert list(p["way_ids"]) == [wy[0] for wy in want]
    ro = p["ref_offsets"]
    for i, (wid, refs, tags) in enumerate(want):
        assert list(p["refs"][ro[i]: ro[i + 1]]) == refs
        assert p["strings"][p["tags"][i, 0]] == tags["building"]
        assert (p["tags"][i, 1] < 0) if "location" not in tags else p["strings"][p["tags"][i, 1]] == tags["location"]
    assert all(k & _lib.RSB_PBF_HAS_DENSE for k in p["kinds"])
    # nodes: DenseNodes ranges decoded here from the byte ranges, plain Nodes decoded by the library, in element order
    q = EX.parse(buf, offs, sizes, _lib.RSB_PBF_NODES)
    got = []
    for s in q["segs"]:
        if s[_lib.RSB_PBF_SEG_KIND] == 0:
            base = offs[s[_lib.RSB_PBF_SEG_BLOCK]]
            cols = []
            for f in range(3):
                o, n = base + s[_lib.RSB_PBF_SEG_ID_OFF + 2 * f], s[_lib.RSB_PBF_SEG_ID_LEN + 2 * f]
                b, i, acc, vals = bytes(buf[o: o + n]), 0, 0, []
                while i < len(b):
                    v, i = xr.read_varint(b, i)
                    acc += xr.unzigzag(v)
                    vals.append(acc)
                cols.append(vals)
            assert len(cols[0]) == s[_lib.RSB_PBF_SEG_COUNT]
            g, lo, la = s[_lib.RSB_PBF_SEG_GRANULARITY], s[_lib.RSB_PBF_SEG_LON_OFFSET], s[_lib.RSB_PBF_SEG_LAT_OFFSET]
            got += [(i_, xr.to_fixed(x, g, lo), xr.to_fixed(y, g, la)) for i_, y, x in zip(*cols)]
        else:
            h, c = s[_lib.RSB_PBF_SEG_HOST_FIRST], s[_lib.RSB_PBF_SEG_COUNT]
            for i_, (x, y) in zip(q["host_ids"][h: h + c], q["host_xy"][h: h + c]):
                got.append((int(i_), int(x), int(y)))
    fix = lambda n: (n[0], n[1] if abs(n[1]) <= 1800000000 else -2 ** 31, n[2] if abs(n[2]) <= 900000000 else -2 ** 31)  # noqa: E731
    assert [fix(g) for g in got] == [fix(n) for n in nodes]


def _error(data, match):
    data = np.frombuffer(data, np.uint8)
    with pytest.raises(_lib.RsbError, match=match):
        frames = EX.read_frames(data)
        buf, offs, sizes = EX.inflate(data, frames)
        for f, o, s in zip(frames, offs, sizes):
            if f[0] == _lib.RSB_PBF_BLOB_HEADER:
                EX.check_header(buf[o: o + s])


def test_format_errors():
    good = _city().bytes()
    _error(xr.Writer(required=("OsmSchema-V0.6", "HistoricalInformation")).bytes(), "HistoricalInformation")
    _error(xr.Writer(required=("OsmSchema-V0.6", "Sort.Type_then_ID", "LocationsOnWays")).bytes(), "Sort.Type_then_ID")
    for comp in ("lzma", "zstd", "lz4", "bzip2"):
        blob = xr.blob(b"\x00" * 10, comp)
        _error(good + xr.frame("OSMData", blob), comp)
    _error(good[:-3], "truncated")
    _error(good + b"\x00\x00", "truncated")
    hdr = xr.f_bytes(1, b"OSMData" + b"x" * 70000) + xr.f_varint(3, 0)
    _error(good + xr.struct.pack(">I", len(hdr)) + hdr, "64 KiB")
    _error(good + xr.frame("OSMData", b"", datasize=33 * 1024 * 1024), "32 MiB")
    _error(good + xr.frame("OSMData", xr.blob(b"x" * 10, "zlib", raw_size=40 * 1024 * 1024)), "32 MiB")
    bad = xr.f_varint(2, 10) + xr.f_bytes(3, b"\x78\x9c" + b"\xff" * 20)
    _error(good + xr.frame("OSMData", bad), "zlib")
    _error(good + xr.frame("OSMData", xr.blob(b"y" * 100, "zlib", raw_size=99)), "raw_size")
    _error(good + xr.frame("OSMData", xr.blob(b"y" * 100, "zlib", raw_size=101)), "raw_size")


def test_abi_constants_match_the_header():
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "rsb200.h")).read()
    for name in ("RSB_PBF_FRAME_FIELDS", "RSB_PBF_SEG_FIELDS", "RSB_PBF_OUT_COUNT", "RSB_PBF_SEG_OUT_FIRST", "RSB_PBF_INFLATE_PAD", "RSB_EXTRACT_WARP_RING",
                 "RSB_PBF_HAS_DENSE", "RSB_PBF_OUT_HOST_XY"):
        assert "#define %s %d\n" % (name, getattr(_lib, name)) in text, name


# --- the tool --------------------------------------------------------------------------------------------------------------


def _args(**kw):
    from robosat_b200.tools import __main__ as M

    sys_argv = sys.argv
    try:
        sys.argv = ["rs", "extract"] + [a for k, v in kw.items() if k not in ("map", "out") for a in ("--" + k, str(v))] + [kw["map"], kw["out"]]
        return M.add_parsers()
    finally:
        sys.argv = sys_argv


def test_tool_flags_and_road():
    from robosat_b200.tools import extract as tool

    a = _args(type="building", map="m.osm.pbf", out="o.geojson")
    assert (a.type, a.batch, a.map, a.out) == ("building", 100000, "m.osm.pbf", "o.geojson") and a.func is tool.main
    with pytest.raises(SystemExit):
        _args(type="water", map="m", out="o")
    with pytest.raises(SystemExit, match="road is not ported"):
        tool.main(_args(type="road", map="m", out="o"))
    with pytest.raises(SystemExit, match="--batch"):
        tool.main(_args(type="parking", batch=0, map="m", out="o"))


def test_tool_batches_names_and_warnings(tmp_path, monkeypatch, capsys):
    from robosat_b200.tools import extract as tool

    feats = [{"type": "Feature", "geometry": {"type": "Polygon", "coordinates": [[[i, 0.0], [i, 1.0], [i + 1, 0.5], [i, 0.0]]]}, "properties": {}} for i in range(7)]
    out = str(tmp_path / "sub" / "out.geojson")
    os.makedirs(os.path.dirname(out))
    paths = tool.save(feats, out, 3)
    assert [len(json.load(open(p))["features"]) for p in paths] == [3, 3, 1]
    assert [f for p in paths for f in json.load(open(p))["features"]] == feats
    for p in paths:
        base = os.path.basename(p)
        assert base.startswith("out-") and base.endswith(".geojson") and len(base) == len("out-.geojson") + 32
        int(base[4:36], 16)
        assert json.load(open(p))["type"] == "FeatureCollection"
    assert tool.save([], str(tmp_path / "empty.geojson"), 3) == [] and not list(tmp_path.glob("empty*"))
    # main: warnings to stderr, features to files (the device path replaced by a stub)
    import torch

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(_lib, "require_device", lambda: None)
    monkeypatch.setattr(EX, "extract_device", lambda path, kind, stats=None: (feats[:2], ["Warning: a", "Warning: b"]))
    tool.main(_args(type="parking", batch=1, map="m.osm.pbf", out=str(tmp_path / "p.json")))
    assert capsys.readouterr().err.splitlines() == ["Warning: a", "Warning: b"]
    assert len(list(tmp_path.glob("p-*.json"))) == 2
