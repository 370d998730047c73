"""JPEG GeoTIFFs on the H100: rsb_jpeg_decode_window's windows bit-identical to the numpy restatement (and PIL) for every fixture
kind, repeatable with the bytes around the output untouched, damaged entropy data refused with the chunk named, and `rs tile` /
`rs segment` on a JPEG ortho identical to the same tools on a deflate twin holding the restatement's decoded pixels."""

import argparse
import os

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_reference as J
import jpeg_tiff_writer as jw
import tiff_writer as tw
from test_segment_gpu import CLASSES, COLORS, ROTATED
from test_tile_gpu import georef
from test_tile_jpeg import FILES, write
from robosat_b200 import _lib
from robosat_b200 import jpeg
from robosat_b200 import mosaic as M
from robosat_b200 import segment as SEG
from robosat_b200 import synth
from robosat_b200 import tile as T
from robosat_b200.geotiff import GeoTiff
from robosat_b200.tools import segment, tile

pytestmark = pytest.mark.gpu


def windows(r):
    H, W, cw, ch = r.height, r.width, r.chunk_w, r.chunk_h
    return [(0, H, 0, W), (0, 1, 0, 1), (H - 1, 1, W - 1, 1), (ch - 3, min(7, H - ch + 3), cw - 5, min(11, W - cw + 5)),
            (H // 3, H - H // 3, W // 2, W - W // 2), (max(0, H - ch - 2), min(H, ch + 2), 0, min(W, cw + 1))]


@pytest.mark.parametrize("name", sorted(FILES))
def test_windows_equal_the_restatement(tmp_path, cuda_device, name):
    r = GeoTiff(write(tmp_path, name, H=130, W=150, seed=3))
    full = J.decode_file(r)
    if not (name == "big"):  # PIL's libtiff reads the whole file the same way
        np.testing.assert_array_equal(np.asarray(Image.open(r.path)).reshape(full.shape), full)
    for row0, rows, col0, cols in windows(r):
        got = r.read_window(row0, rows, col0, cols)
        np.testing.assert_array_equal(got, full[row0:row0 + rows, col0:col0 + cols], err_msg=str((row0, rows, col0, cols)))


def test_a_launch_of_over_a_thousand_chunks(tmp_path, cuda_device):
    # GDAL-style: JPEGTables holds DQT only and every tile has its own optimised Huffman tables, so every lane of a warp reads its own
    # table set
    p, _ = jw.write_jpeg_tiff(str(tmp_path / "k.tif"), jw.image(1024, 1040, 3, 5), tile=(32, 32), tables="dqt",
                              settings=lambda k: dict(quality=30 + k % 70, subsampling=k % 3, optimize=True, restart_marker_blocks=(k % 4) or None),
                              **jw.GEO_3857)
    r = GeoTiff(p)
    assert len(jpeg.touched(r, 0, r.height, 0, r.width)) >= 1000
    np.testing.assert_array_equal(r.read_window(0, r.height, 0, r.width), J.decode_file(r))


def test_repeats_are_identical_and_guard_bytes_untouched(tmp_path, cuda_device):
    r = GeoTiff(write(tmp_path, "tiles-rst", H=130, W=150))
    row0, rows, col0, cols = 5, 100, 7, 120
    n = rows * cols * 3
    dec = r.jpeg_decoder("cuda")
    data = torch.empty((1 << 20,), dtype=torch.uint8, pin_memory=True)
    descs = torch.empty((64 * jpeg.F,), dtype=torch.int64, pin_memory=True)
    sets = torch.empty((64 * _lib.RSB_JPEG_SET_WORDS,), dtype=torch.int32, pin_memory=True)
    errors = torch.empty((64,), dtype=torch.int64, pin_memory=True)
    st = jpeg.stage(r, row0, rows, col0, cols, data.numpy(), descs.numpy(), sets.numpy())
    outs = []
    for _ in range(3):
        buf = torch.full((n + 2048,), 0xA5, dtype=torch.uint8, device="cuda")
        keep = dec.decode(st, data, descs, sets, buf[1024:1024 + n], errors)
        torch.cuda.synchronize()
        del keep
        dec.check(st, errors)
        host = buf.cpu().numpy()
        assert (host[:1024] == 0xA5).all() and (host[1024 + n:] == 0xA5).all()
        outs.append(host[1024:1024 + n])
    assert all(np.array_equal(outs[0], o) for o in outs[1:])
    np.testing.assert_array_equal(outs[0].reshape(rows, cols, 3), J.decode_file(r, row0, rows, col0, cols))


def _codes(bits, vals):
    """symbol -> (code, length) of a canonical Huffman table"""
    out, code = {}, 0
    i = 0
    for l in range(1, 17):
        for _ in range(bits[l]):
            out[vals[i]] = (code, l)
            code += 1
            i += 1
        code <<= 1
    return out


def _entropy(stream):
    segs = jw.segments(stream)
    head = b"\xff\xd8" + b"".join(seg for m, seg in segs[:-1])
    return head, segs[-1][1][:-2]  # the entropy-coded bytes without the EOI


def _ac_past_63(stream):
    head, _ = _entropy(stream)
    dht = [seg for m, seg in jw.segments(stream) if m == 0xC4]
    tables = {}
    for seg in dht:
        p, i = seg[4:], 0
        while i < len(p):
            bits = [0] + list(p[i + 1:i + 17])
            n = sum(bits)
            tables[(p[i] >> 4, p[i] & 15)] = _codes(bits, list(p[i + 17:i + 17 + n]))
            i += 17 + n
    acc, nbits = 0, 0
    for code, l in [tables[(0, 0)][0]] + [tables[(1, 0)][0xF1], (1, 1)] * 5:
        acc, nbits = (acc << l) | code, nbits + l
    pad = (-nbits) % 8
    acc, nbits = (acc << pad) | ((1 << pad) - 1), nbits + pad
    data = acc.to_bytes(nbits // 8, "big").replace(b"\xff", b"\xff\x00")
    return head + data + b"\xff\xd9"


def _rst(stream, fn):
    head, data = _entropy(stream)
    i = data.index(b"\xff\xd0")
    return head + fn(data, i) + b"\xff\xd9"


DAMAGE = {  # name -> (encoder settings, corrupt function, restatement code, message)
    "bad-code": ({}, lambda s: _entropy(s)[0] + b"\xff\x00" * 40 + b"\xff\xd9", J.BAD_CODE, "invalid Huffman code at MCU 0"),
    "ac-past-63": ({}, _ac_past_63, J.AC_PAST_63, "AC coefficient index past 63 at MCU 0"),
    "rst-number": (dict(restart_marker_blocks=1), lambda s: _rst(s, lambda d, i: d[:i] + b"\xff\xd3" + d[i + 2:]), J.BAD_MARKER,
                   "unexpected marker or RST number at MCU 1"),
    "extraneous": (dict(restart_marker_blocks=1), lambda s: _rst(s, lambda d, i: d[:i] + b"\x55" + d[i:]), J.EXTRANEOUS,
                   "extraneous bytes before a marker at MCU 1"),
    "truncated": ({}, lambda s: _entropy(s)[0] + _entropy(s)[1][:len(_entropy(s)[1]) // 2].rstrip(b"\xff") + b"\xff\xd9", J.TRUNCATED,
                  "data ends before the last MCU"),
}


@pytest.mark.parametrize("name", sorted(DAMAGE))
def test_damaged_entropy_data_names_the_chunk(tmp_path, cuda_device, name):
    settings, fn, code, text = DAMAGE[name]
    p, streams = jw.write_jpeg_tiff(str(tmp_path / "d.tif"), jw.image(64, 96), tile=(32, 32), settings=settings, corrupt=(4, fn), **jw.GEO_3857)
    r = GeoTiff(p)
    with pytest.raises(J.DataError) as e:
        J.decode(streams[4])
    assert e.value.code == code
    with pytest.raises(_lib.RsbError, match="tile 4: " + text):
        r.read_window(0, 64, 0, 96)
    np.testing.assert_array_equal(r.read_window(0, 32, 0, 32), J.decode_file(r, 0, 32, 0, 32))  # the other chunks still decode
    if name == "bad-code":
        with pytest.raises(_lib.RsbError, match="tile 4: " + text):
            T.tile_device(r, 18, 64)


# ---- the deflate twin ----

def twin(tmp_path, kind, H, W, seed=1):
    """(JPEG raster, deflate raster) with the same georeferencing; the deflate one holds the restatement's decode of the JPEG one"""
    kw = ROTATED if kind == "rotated" else georef(kind)
    p, _ = jw.write_jpeg_tiff(str(tmp_path / "ortho.tif"), jw.image(H, W, 3, seed), tile=(256, 256), tables="dqt",
                              settings=dict(quality=90, optimize=True), **kw)
    r = GeoTiff(p)
    tw.write_tiff(str(tmp_path / "twin.tif"), J.decode_file(r), compression=8, tile=(128, 64), predictor=2, **kw)
    return r, GeoTiff(str(tmp_path / "twin.tif"))


@pytest.mark.parametrize("kind", ["3857", "utm", "rotated"])
def test_rs_tile_equals_the_deflate_twin(tmp_path, cuda_device, kind):
    r, d = twin(tmp_path, kind, 700, 600)
    for resampling in ("nearest", "bilinear", "average"):
        zoom = 19 if resampling == "average" else 18
        got = T.tile_device(r, zoom, 256, resampling, batch=3)
        want = T.tile_device(d, zoom, 256, resampling, batch=3)
        assert got.keys() == want.keys() and len(got) >= 2
        for k in got:
            assert got[k][1] == want[k][1]
            np.testing.assert_array_equal(got[k][0], want[k][0], err_msg="%s %s" % (resampling, k))
        # the tool writes the same file set with the same pixels
        for name, path in (("jpeg", r.path), ("twin", d.path)):
            tile.main(argparse.Namespace(zoom=zoom, size=256, tiles=None, resampling=resampling, raster=path, out=str(tmp_path / resampling / name)))
        a, b = tmp_path / resampling / "jpeg", tmp_path / resampling / "twin"
        files = sorted(os.path.relpath(os.path.join(q, f), a) for q, _, fs in os.walk(a) for f in fs)
        assert files == sorted(os.path.relpath(os.path.join(q, f), b) for q, _, fs in os.walk(b) for f in fs) and len(files) == len(got)
        for f in files:
            np.testing.assert_array_equal(np.asarray(Image.open(a / f)), np.asarray(Image.open(b / f)), err_msg=f)


def _segment(tmp_path, raster, out, budget):
    stats = {}
    segment.main(argparse.Namespace(zoom=18, size=256, overlap=32, batch_size=4, tiles=None, resampling="bilinear", output="masks", tta="none",
                                    nodata=None, model=str(tmp_path / "model.toml"), dataset=str(tmp_path / "dataset.toml"),
                                    checkpoint=str(tmp_path / "ckpt.pth"), raster=raster, out=str(tmp_path / out)), stats, budget)
    return stats


@pytest.mark.parametrize("kind", ["3857", "rotated"])
def test_rs_segment_equals_the_deflate_twin(tmp_path, cuda_device, monkeypatch, kind):
    monkeypatch.setenv("RSB_GPUS", "1")
    monkeypatch.setenv("RSB_QUIET", "1")
    r, d = twin(tmp_path, kind, 1000, 1100, seed=2)
    torch.save({"epoch": 1, "state_dict": synth.make_state_dict(2, seed=5), "optimizer": {}}, tmp_path / "ckpt.pth")
    (tmp_path / "model.toml").write_text("[common]\ncuda = true\nbatch_size = 2\nimage_size = 256\ncheckpoint = '%s'\n" % tmp_path)
    (tmp_path / "dataset.toml").write_text("[common]\ndataset = '%s'\nclasses = %r\ncolors = %r\n" % (tmp_path, CLASSES[2], COLORS[2]))
    budget = None
    if kind == "rotated":  # at exactly the planned peak, which counts the staged chunks and the decoder scratch
        p = SEG.plan(r, M.Grid(r.width, r.height, r.crs, r.geotransform), 18, 256, 4)
        assert p.decode_bytes > 0 and r.jpeg_descs[:, jpeg.BLOCKS].sum() > 0
        budget = p.store_bytes
    s1 = _segment(tmp_path, r.path, "jpeg.tif", budget)
    s2 = _segment(tmp_path, d.path, "deflate.tif", None)
    a, b = Image.open(tmp_path / "jpeg.tif"), Image.open(tmp_path / "deflate.tif")
    tags = (256, 257, 258, 262, 320, 33550, 33922, 34264, 34735, 42113)
    assert {t: a.tag_v2.get(t) for t in tags} == {t: b.tag_v2.get(t) for t in tags}
    np.testing.assert_array_equal(np.array(a), np.array(b))
    assert s1["existing"] == s2["existing"] > 0
    if budget is not None:
        with pytest.raises(SystemExit, match="need %d device bytes" % budget):
            _segment(tmp_path, r.path, "never.tif", budget - 1)
        assert not os.path.exists(tmp_path / "never.tif")
