"""JPEG (Compression 7) GeoTIFFs on the host: the numpy restatement (tests/jpeg_reference.py) against libjpeg-turbo (the golden
decodes, and PIL when it links libjpeg-turbo), PIL's whole-file reads of the writer's files against the restatement's crops, the
library's header parser against the restatement's parse, every rejection named at open, the ABI's argument checks before the device
check, and the plans' device bytes."""

import ctypes
import io
import os

import numpy as np
import pytest
from PIL import Image, features

import jpeg_reference as J
import jpeg_tiff_writer as jw
from robosat_b200 import _lib
from robosat_b200 import jpeg
from robosat_b200 import segment as SG
from robosat_b200 import tile as T
from robosat_b200.geotiff import GeoTiff

HERE = os.path.dirname(os.path.abspath(__file__))
turbo = pytest.mark.skipif(not features.check("libjpeg_turbo"), reason="PIL does not link libjpeg-turbo")


def test_restatement_equals_the_golden_decodes():
    g = np.load(os.path.join(HERE, "golden", "jpeg.npz"))
    n = len([k for k in g.files if k.startswith("stream_")])
    assert n >= 10
    for i in range(n):
        spp, photometric = g["layout_%d" % i].tolist()
        got = J.decode(g["stream_%d" % i].tobytes(), spp=spp, photometric=photometric)
        np.testing.assert_array_equal(got, g["pixels_%d" % i], err_msg="golden stream %d" % i)


FRAMES = [(1, 1), (7, 13), (17, 33), (150, 200), (257, 255)]


def _sweep():
    rng = np.random.default_rng(7)
    cases = []
    for H, W in FRAMES:
        for sub in (0, 1, 2):
            for opt in (False, True):
                rst = [None, dict(restart_marker_blocks=1), dict(restart_marker_blocks=7), dict(restart_marker_rows=1)][int(rng.integers(4))]
                cases.append((H, W, 3, 6, dict(quality=int(rng.integers(10, 101)), subsampling=sub, optimize=opt, **(rst or {}))))
        cases.append((H, W, 1, 1, dict(quality=int(rng.integers(10, 101)), restart_marker_blocks=7)))
        cases.append((H, W, 3, 2, dict(quality=int(rng.integers(10, 101)), restart_marker_rows=1)))
    for q in (10, 100):
        cases.append((40, 56, 3, 6, dict(quality=q, subsampling=2)))
    return cases


@turbo
@pytest.mark.parametrize("case", range(len(_sweep())))
def test_restatement_equals_pil(case):
    H, W, spp, photometric, kw = _sweep()[case]
    s = jw.encode(jw.image(H, W, spp, seed=case), photometric, **kw)
    want = np.asarray(Image.open(io.BytesIO(s))).reshape(H, W, spp)
    np.testing.assert_array_equal(J.decode(s, spp=spp, photometric=photometric), want)


FILES = {  # name -> write_jpeg_tiff keywords
    "tiles-420": dict(tile=(64, 48)),
    "tiles-tables": dict(tile=(32, 32), tables=True),
    "tiles-rst": dict(tile=(48, 32), settings=dict(subsampling=1, restart_marker_blocks=3, quality=90)),
    "strips-ragged": dict(rows_per_strip=24),
    "strips-padded": dict(rows_per_strip=24, pad_last_strip=True),
    "strips-tables-be": dict(rows_per_strip=40, tables=True, order=">"),
    "rgb": dict(rows_per_strip=16, photometric=2, settings=dict(quality=90)),
    "big": dict(tile=(32, 64), big=True, settings=lambda k: dict(quality=40 + 5 * k, optimize=k % 2 == 1)),
    "gray": dict(tile=(32, 32), spp=1),
    "gray-strips": dict(rows_per_strip=13, spp=1, tables=True),
    "strip-over-height": dict(rows_per_strip=160, pad_last_strip=True),  # one strip, its frame padded to a RowsPerStrip above the height
    # GDAL's default: JPEGTables holds the quantisation tables only, every tile carries its own optimised Huffman tables
    "gdal-style": dict(tile=(32, 32), tables="dqt", settings=dict(quality=75, optimize=True)),
}


def write(tmp_path, name, H=100, W=130, seed=0, **extra):
    kw = dict(FILES[name])
    spp = kw.pop("spp", 3)
    kw.update(extra)
    p, _ = jw.write_jpeg_tiff(str(tmp_path / ("%s.tif" % name)), jw.image(H, W, spp, seed), **jw.GEO_3857, **kw)
    return p


@pytest.mark.parametrize("name", sorted(FILES))
def test_pil_whole_file_equals_the_restatement(tmp_path, name):
    r = GeoTiff(write(tmp_path, name))
    want = np.asarray(Image.open(r.path)).reshape(r.height, r.width, r.spp)
    np.testing.assert_array_equal(J.decode_file(r), want)


@pytest.mark.parametrize("name", sorted(FILES))
def test_host_parser_equals_the_restatement(tmp_path, name):
    r = GeoTiff(write(tmp_path, name))
    data = open(r.path, "rb").read()
    tables = J.read_tables(r.jpeg_tables)
    n_chunks = len(r.offsets)
    assert r.jpeg_descs.shape == (n_chunks, jpeg.F) and (r.jpeg_descs[:, jpeg.SET] == -1).all()  # no table set is kept at open
    order = np.arange(n_chunks)[::-1].copy()  # a selection in any order, as the windows make
    sets = np.zeros((n_chunks, _lib.RSB_JPEG_SET_WORDS), np.int32)
    descs, nsets = jpeg.parse(r, r.file_bytes(), r.jpeg_tables, 4, select=order, sets=sets)
    np.testing.assert_array_equal(np.delete(descs, jpeg.SET, 1), np.delete(r.jpeg_descs[order], jpeg.SET, 1))
    seen = []
    for i, k in enumerate(order.tolist()):
        off, n = r.offsets[k], r.byte_counts[k]
        hdr = J.parse(data[off:off + n], tables, r.spp, r.photometric)
        d = descs[i]
        mx, my, bpm = J.geometry(hdr, r.spp)
        assert d.tolist() == [off + hdr["start"], hdr["end"] - hdr["start"], d[jpeg.SET], hdr["width"], hdr["height"], hdr["h"], hdr["v"],
                              hdr["restart"], mx * my * bpm, 0, k, 0]
        s = sets[d[jpeg.SET]]
        for c in range(r.spp):
            np.testing.assert_array_equal(s[c * 64:(c + 1) * 64], hdr["quant"][c].astype(np.int16))
            for ac, t in enumerate((hdr["dc"][c], hdr["ac"][c])):
                base = 192 + (2 * c + ac) * 548
                np.testing.assert_array_equal(s[base:base + 548], np.concatenate([t["lookup"], t["maxcode"], t["valoffset"], t["huffval"]]))
        seen.append(int(d[jpeg.SET]))
    firsts = [x for i, x in enumerate(seen) if x not in seen[:i]]
    assert firsts == list(range(nsets))  # numbered in order of first use
    if name == "gdal-style":
        assert nsets == n_chunks  # one set per tile


def _replace_marker(stream, marker, fn):
    """apply fn to the payload of the first segment with `marker` (the length is rewritten)"""
    out, found = b"\xff\xd8", False
    for m, seg in jw.segments(stream):
        if m == marker and not found:
            payload = fn(seg[4:])
            seg = bytes([0xFF, m]) + (len(payload) + 2).to_bytes(2, "big") + payload
            found = True
        out += seg if m != "data" else b""
        if m == "data":
            out += seg
    assert found
    return out


def _sof_sampling(factors):
    def fn(p):
        p = bytearray(p)
        for i, f in enumerate(factors):
            p[7 + 3 * i] = f
        return bytes(p)
    return fn


def _sof_marker(m):
    def fn(s):
        i = s.index(b"\xff\xc0")
        return s[:i + 1] + bytes([m]) + s[i + 2:]
    return fn


def _two_scans(s):
    segs = jw.segments(s)
    sos = [seg for m, seg in segs if m == 0xDA][0]
    data = segs[-1][1]
    return s[:-2] + sos + data


def _over_subscribed(s):
    def fn(p):  # the first table becomes two 1-bit codes: the second is the all-ones code
        n = sum(p[1:17])
        return p[:1] + bytes([2] + [0] * 15) + b"\x00\x01" + p[17 + n:]
    return _replace_marker(s, 0xC4, fn)


REJECTS = [  # (name, writer keywords, corrupt function, expected text)
    ("not-soi", {}, lambda s: b"\x00" + s[1:], "does not start with SOI"),
    ("progressive", {}, _sof_marker(0xC2), r"progressive frames \(SOF2\)"),
    ("lossless", {}, _sof_marker(0xC3), r"lossless frames \(SOF3\)"),
    ("arithmetic", {}, _sof_marker(0xC9), r"arithmetic or hierarchical frames \(SOF9\)"),
    ("12-bit", {}, lambda s: _replace_marker(s, 0xC0, lambda p: b"\x0c" + p[1:]), "precision 12"),
    ("two-scans", {}, _two_scans, "only one scan"),
    ("components", {}, lambda s: _replace_marker(s, 0xC0, lambda p: p[:5] + b"\x01" + p[6:9]), "1 components in a 3-band image"),
    ("440", {}, lambda s: _replace_marker(s, 0xC0, _sof_sampling([0x12, 0x11, 0x11])), "sampling 1x2,1x1,1x1"),
    ("chroma", {}, lambda s: _replace_marker(s, 0xC0, _sof_sampling([0x22, 0x21, 0x11])), "sampling 2x2,2x1,1x1"),
    ("undefined-table", {}, lambda s: _replace_marker(s, 0xC0, lambda p: p[:8] + b"\x03" + p[9:]), "quantisation table 3 is used but not defined"),
    ("over-subscribed", {}, _over_subscribed, "over-subscribed Huffman table"),
    ("frame-width", {}, lambda s: _replace_marker(s, 0xC0, lambda p: p[:3] + (33).to_bytes(2, "big") + p[5:]), "a frame 33 wide in chunks 32 wide"),
]


@pytest.mark.parametrize("name,kw,fn,text", REJECTS, ids=[r[0] for r in REJECTS])
def test_rejections_are_named_at_open(tmp_path, name, kw, fn, text):
    p, streams = jw.write_jpeg_tiff(str(tmp_path / "r.tif"), jw.image(64, 64), tile=(32, 32), corrupt=(2, fn), **jw.GEO_3857, **kw)
    with pytest.raises(_lib.RsbError, match=r"Compression 7 \(JPEG\) tile 2: .*" + text):
        GeoTiff(p)
    if name != "frame-width":  # the restatement's parse refuses the stream alone for the same reason
        with pytest.raises(J.Rejected, match=text):
            J.parse(streams[2], J.read_tables(None), 3, 6)


def test_rejected_layouts_and_tables(tmp_path):
    px = jw.image(64, 64)
    jw.write_jpeg_tiff(str(tmp_path / "b.tif"), px, tile=(32, 32), **jw.GEO_3857, tags={262: (3, [2])})  # 4:2:0 streams labelled RGB
    with pytest.raises(_lib.RsbError, match=r"Compression 7 \(JPEG\) tile 0: subsampled RGB \(sampling 2x2\)"):
        GeoTiff(str(tmp_path / "b.tif"))
    tables, _ = jw.abbreviate([jw.encode(px[:32, :32])])
    dri = tables[:2] + b"\xff\xdd\x00\x04\x00\x01" + tables[2:]
    jw.write_jpeg_tiff(str(tmp_path / "e.tif"), px, tile=(32, 32), **jw.GEO_3857, tags={347: (7, list(dri))})
    with pytest.raises(_lib.RsbError, match=r"Compression 7 \(JPEG\) DRI in JPEGTables"):
        GeoTiff(str(tmp_path / "e.tif"))
    with pytest.raises(J.Rejected, match="DRI in JPEGTables"):
        J.read_tables(dri)
    jw.write_jpeg_tiff(str(tmp_path / "f.tif"), px, tile=(32, 32), **jw.GEO_3857,
                       tags={277: (3, [4]), 258: (3, [8] * 4), 339: (3, [1] * 4), 338: (3, [2]), 262: (3, [2])})
    with pytest.raises(_lib.RsbError, match=r"Compression 7 \(JPEG\) with 4 bands"):
        GeoTiff(str(tmp_path / "f.tif"))
    jw.write_jpeg_tiff(str(tmp_path / "g.tif"), px, tile=(32, 32), **jw.GEO_3857, tags={259: (3, [6])})
    with pytest.raises(_lib.RsbError, match=r"Compression 6 \(old-style JPEG\)"):
        GeoTiff(str(tmp_path / "g.tif"))
    jw.write_jpeg_tiff(str(tmp_path / "h.tif"), jw.image(58, 40), rows_per_strip=29, **jw.GEO_3857, tags={278: (4, [30])})
    with pytest.raises(_lib.RsbError, match=r"strip 0: a frame 29 high in a strip of 30 rows \(RowsPerStrip 30\)"):
        GeoTiff(str(tmp_path / "h.tif"))
    # one strip whose RowsPerStrip exceeds the height, its frame padded to RowsPerStrip: accepted; one row more is not
    r = GeoTiff(jw.write_jpeg_tiff(str(tmp_path / "i.tif"), jw.image(21, 40), rows_per_strip=32, pad_last_strip=True, **jw.GEO_3857)[0])
    assert r.chunk_h == 21 and r.rows_per_strip == 32 and r.jpeg_descs[0, jpeg.HEIGHT] == 32
    np.testing.assert_array_equal(J.decode_file(r), J.decode(open(r.path, "rb").read()[r.offsets[0]:r.offsets[0] + r.byte_counts[0]])[:21])
    jw.write_jpeg_tiff(str(tmp_path / "j.tif"), jw.image(21, 40), rows_per_strip=33, pad_last_strip=True, **jw.GEO_3857, tags={278: (4, [32])})
    with pytest.raises(_lib.RsbError, match=r"strip 0: a frame 33 high in a strip of 21 rows \(RowsPerStrip 32\)"):
        GeoTiff(str(tmp_path / "j.tif"))
    # YCbCr without JPEG keeps today's message
    import tiff_writer as tw

    tw.write_tiff(str(tmp_path / "y.tif"), px, photometric=6, **jw.GEO_3857)
    with pytest.raises(_lib.RsbError, match=r"3 bands with Photometric 6 \(YCbCr\) are not supported; only RGB is"):
        GeoTiff(str(tmp_path / "y.tif"))


def test_predictor_is_ignored_and_photometric_kept(tmp_path):
    p = write(tmp_path, "tiles-420", predictor=2)
    r = GeoTiff(p)
    assert r.predictor == 1 and r.photometric == 6 and r.compression == 7


def _abi_args(**over):
    buf = (ctypes.c_uint8 * 4096)()
    a = dict(staged=ctypes.addressof(buf), staged_len=16, descs=ctypes.addressof(buf), n=1, sets=ctypes.addressof(buf), n_sets=1, width=64, height=64,
             cw=32, ch=32, tiled=1, spp=3, photometric=6, row0=0, rows=8, col0=0, cols=8, out=ctypes.addressof(buf), scratch=ctypes.addressof(buf) // 16 * 16 + 16,
             scratch_bytes=4096, blocks=6, errors=ctypes.addressof(buf), stream=None)
    a.update(over)
    return buf, list(a.values())


def test_abi_validates_before_the_device_check():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    for over, text in [(dict(staged=None), "null pointer"), (dict(n=0), "0 chunks"), (dict(spp=4), "4 bands"), (dict(photometric=2, spp=1), "1 bands"),
                       (dict(rows=0), "outside"), (dict(row0=60, rows=8), "outside"), (dict(n=2), "the window touches 1"),
                       (dict(scratch_bytes=100), "scratch of 100 bytes"), (dict(tiled=0), "tiled 0"), (dict(blocks=0), "0 blocks"),
                       (dict(scratch=1), "aligned")]:
        keep, args = _abi_args(**over)
        assert lib.rsb_jpeg_decode_window(*args) == -1, over
        assert text in _lib.last_error(), (over, _lib.last_error())
    keep, args = _abi_args()
    assert lib.rsb_jpeg_decode_window(*args) == -3  # valid, but no device
    assert lib.rsb_jpeg_scratch_bytes(10) == 10 * _lib.RSB_JPEG_SCRATCH_PER_BLOCK and lib.rsb_jpeg_scratch_bytes(-1) == -1
    n = ctypes.c_int32()
    assert lib.rsb_jpeg_parse_chunks(None, 0, None, 0, None, None, 1, 8, 8, 8, 8, 8, 1, 3, 6, None, 0, 1, None, None, 0, ctypes.byref(n), None) == -1
    keep, args = _abi_args()
    sel = (ctypes.c_int64 * 1)(5)  # a selected chunk outside the raster
    assert lib.rsb_jpeg_parse_chunks(args[0], 16, None, 0, args[0], args[0], 1, 8, 8, 8, 8, 8, 1, 3, 6, sel, 1, 1, args[0], None, 0, ctypes.byref(n),
                                     None) == -1
    assert "selected chunk 5" in _lib.last_error()


def test_read_window_needs_a_device(tmp_path):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = GeoTiff(write(tmp_path, "tiles-420"))
    with pytest.raises(_lib.RsbError):
        r.read_window(0, 4, 0, 4)
    with pytest.raises(_lib.RsbError, match="outside the 130 x 100 raster"):
        r.read_window(98, 4, 0, 4)


def test_plans_count_staged_bytes_and_scratch(tmp_path):
    r = GeoTiff(write(tmp_path, "tiles-420", H=300, W=400))
    box = (10, 100, 50, 90)
    idx = jpeg.touched(r, *box)
    assert sorted(idx.tolist()) == sorted({(y // 48) * 7 + x // 64 for y in range(10, 110) for x in range(50, 140)})
    d = r.jpeg_descs[idx]
    extra = int(d[:, jpeg.LENGTH].sum()) + len(idx) * (jpeg.F * 8 + 8 + _lib.RSB_JPEG_SET_WORDS * 4) + int(d[:, jpeg.BLOCKS].sum()) * 192
    assert T.source_bytes(r, box) == 100 * 90 * 3 + extra
    assert extra == jpeg.extra_bytes(r, *box)
    zoom, size = 18, 64
    cand = T.candidate_tiles(r, zoom, size)
    step = T.choose_step(r, zoom, size, cand)
    ws = T.plan(r, zoom, size, cand, step)
    for w in ws:
        assert w.device_bytes(r, size) == T.window_bytes(w.rows * w.cols * 3 + jpeg.extra_bytes(r, w.row0, w.rows, w.col0, w.cols), len(w.xs), size,
                                                         w.nodes.size * 8)
    one = max(T.window_bytes(T.source_bytes(r, (w.row0, w.rows, w.col0, w.cols)), 1, size, 0) for w in ws)
    small = T.plan(r, zoom, size, cand, step, budget=one + 10 ** 6, batch=1)
    assert len(small) == sum(len(w.xs) for w in ws)
    with pytest.raises(_lib.RsbError, match="more than the budget"):
        T.plan(r, zoom, size, cand, step, budget=1000)


def test_segment_plan_counts_the_decode(tmp_path):
    from robosat_b200 import mosaic as M

    r = GeoTiff(write(tmp_path, "tiles-420", H=300, W=400))
    grid = M.Grid(r.width, r.height, r.crs, r.geotransform)
    p = SG.plan(r, grid, 18, 64, batch=4)
    want = max(jpeg.extra_bytes(r, w.row0, w.rows, w.col0, w.cols) for w in p.warps)
    assert p.decode_bytes == want
    assert p.store_bytes == p.image_slots * 64 * 64 * 3 + p.plane_slots * 64 * 64 + want
    SG.plan(r, grid, 18, 64, batch=4, budget=p.store_bytes)
    with pytest.raises(_lib.RsbError, match="JPEG decode need"):
        SG.plan(r, grid, 18, 64, batch=4, budget=p.store_bytes - 1)
