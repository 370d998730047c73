"""The band rule of `rs tile` / `rs segment` on the host (DESIGN.md §8): rsb_tiff_decode_bands against the written arrays over bits,
byte order, strips / tiles, compression and predictor, planar configuration and band selection, and against OpenCV's (libtiff's) own
16-bit files; header acceptance and refusals, with GeoTiff(path) refusing what it refused before; the rendering formula and the
percentile rule of the restatement; the tools' refusals before any device use; and the new entry points' argument checks before
the device check."""

import argparse
import ctypes
import itertools
import re
from fractions import Fraction

import numpy as np
import pytest

import tiff_bands_writer as bw
import tile_bands_reference as ref
from robosat_b200 import _lib
from robosat_b200 import tile as T
from robosat_b200.geotiff import BandTiff, GeoTiff, open_bands

GEO = dict(geo=bw.geokeys(), scale=(0.5, 0.5, 0.0), tiepoint=(0, 0, 0, 1000.0, 2000.0, 0))


def samples(H, W, spp, bits, seed):
    rng = np.random.default_rng(seed)
    px = rng.integers(0, 1 << bits, (H, W, spp), dtype=np.uint8 if bits == 8 else np.uint16)
    px[H // 2] = px[H // 2, :1]  # a run, so that LZW and DEFLATE have repeats to code
    return px


# ---- decoder ----

LAYOUTS = {"strips": dict(rows_per_strip=5), "tiles": dict(tile=(16, 16)), "ragged": dict(tile=(16, 32))}
CODECS = [(1, 1), (1, 2), (5, 1), (5, 2), (8, 1), (8, 2)]
MATRIX = list(itertools.product((8, 16), ("<", ">"), list(LAYOUTS), CODECS, (1, 2)))


@pytest.mark.parametrize("case", range(len(MATRIX)), ids=lambda i: "%d-%s-%s-c%d-p%d-planar%d" % (
    MATRIX[i][0], "LE" if MATRIX[i][1] == "<" else "BE", MATRIX[i][2], MATRIX[i][3][0], MATRIX[i][3][1], MATRIX[i][4]))
def test_decoder_windows_equal_the_written_arrays(tmp_path, case):
    bits, order, layout, (comp, pred), planar = MATRIX[case]
    spp = 1 + case % 8
    H, W = 37, 45
    px = samples(H, W, spp, bits, case)
    rng = np.random.default_rng(100 + case)
    path = bw.write_bands_tiff(str(tmp_path / "b.tif"), px, planar=planar, order=order, big=case % 3 == 0, compression=comp, predictor=pred,
                               photometric=1, **LAYOUTS[layout], **GEO)
    nsel = 1 if spp < 3 else int(rng.choice([1, 3]))
    bands = [int(b) for b in rng.integers(1, spp + 1, nsel)]
    g = open_bands(path, bands)
    assert (g.bits, g.planar, g.byteorder, g.bands, g.alpha_band, g.k) == (bits, planar, order, [b - 1 for b in bands], None, nsel)
    want = px[..., [b - 1 for b in bands]]
    for r0, rows, c0, cols in ((0, H, 0, W), (3, 17, 5, 33), (H - 1, 1, W - 1, 1), (15, 9, 0, 1), (0, 1, 16, 16), (30, 7, 31, 14)):
        for threads in (1, 4):
            got = g.read_window(r0, rows, c0, cols, threads=threads)
            assert got.dtype == want.dtype and np.array_equal(got, want[r0:r0 + rows, c0:c0 + cols]), (r0, rows, c0, cols, threads)


def test_decoder_gathers_any_selection_with_alpha(tmp_path):
    px = samples(29, 31, 6, 16, 7)
    for planar in (1, 2):
        path = bw.write_bands_tiff(str(tmp_path / ("a%d.tif" % planar)), px, planar=planar, compression=8, predictor=2, tile=(16, 16),
                                   photometric=1, extra_samples=(0, 2, 0, 0, 0), **GEO)  # MinIsBlack: band 1 is the colour band, 2..6 extra
        for bands in ([1], [6], [4, 4, 1], [5, 2, 6], [3]):
            g = open_bands(path, bands)
            assert g.alpha_band == 2 and g.k == len(bands) + 1
            assert np.array_equal(g.read_window(0, 29, 0, 31), px[..., [b - 1 for b in bands] + [2]])


class _NoGeo(BandTiff):
    def _georeference(self):  # OpenCV writes no GeoKeys; the pixel layout is what is tested
        pass


@pytest.mark.parametrize("comp", [1, 5, 8])
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_decoder_reads_opencv_16_bit_files(tmp_path, comp, channels):
    cv2 = pytest.importorskip("cv2")
    a = np.random.default_rng(channels * 10 + comp).integers(0, 65536, (53, 61, channels), dtype=np.uint16)
    a[20:30] = 1234
    path = str(tmp_path / "cv.tif")
    assert cv2.imwrite(path, a[..., 0] if channels == 1 else a, [cv2.IMWRITE_TIFF_COMPRESSION, comp])
    back = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    back = back[..., None] if back.ndim == 2 else back
    rgb = back[..., [2, 1, 0, 3][:channels]] if channels > 1 else back  # OpenCV's BGR(A) order, undone
    g = _NoGeo(path, None)
    assert (g.bits, g.spp, g.compression) == (16, channels, comp)
    assert np.array_equal(g.read_window(0, 53, 0, 61), rgb[..., :1 if channels == 1 else 3])
    assert np.array_equal(g.read_window(11, 30, 7, 40), rgb[11:41, 7:47, :1 if channels == 1 else 3])
    if channels == 4:  # no ExtraSamples is written: the fourth band is plain data, read with --bands 4
        assert g.alpha_band is None
        assert np.array_equal(_NoGeo(path, [4]).read_window(0, 53, 0, 61), rgb[..., 3:])


@pytest.mark.parametrize("planar,chunk,text", [(1, 3, "tile 3"), (2, 4 + 1, "tile 5")])
def test_damaged_chunk_is_named(tmp_path, planar, chunk, text):
    px = samples(32, 32, 3, 16, 3)
    path = bw.write_bands_tiff(str(tmp_path / "bad.tif"), px, planar=planar, compression=8, tile=(16, 16), corrupt=(chunk, lambda b: b[:len(b) // 2]),
                               **GEO)
    g = open_bands(path, [1, 2, 3])
    with pytest.raises(_lib.RsbError, match=text):
        g.read_window(0, 32, 0, 32)
    assert g.read_window(0, 16, 0, 16).shape == (16, 16, 3)  # a window that does not touch the damaged chunk decodes
    if planar == 2:  # the damaged chunk is band 2's: a selection without it never reads it
        assert open_bands(path, [1, 3, 3]).read_window(0, 32, 0, 32).shape == (32, 32, 3)


# ---- header ----

def test_band_rule_headers(tmp_path):
    def write(name, px, **kw):
        return bw.write_bands_tiff(str(tmp_path / name), px, **{**GEO, **kw})

    p = write("rgb16.tif", samples(8, 8, 3, 16, 1), nodata="65535")
    g = open_bands(p)
    assert (g.bands, g.alpha_band, g.nodata, g.scale, g.k) == ([0, 1, 2], None, 65535, None, 3)
    with pytest.raises(_lib.RsbError, match="BitsPerSample 16,16,16 is not supported; only 8 is"):
        GeoTiff(p)
    p = write("nir.tif", samples(8, 8, 4, 8, 1), extra_samples=(0,))
    g = open_bands(p)
    assert (g.bands, g.alpha_band, g.scale) == ([0, 1, 2], None, [(0, 255)] * 3)
    with pytest.raises(_lib.RsbError, match="4 bands with ExtraSamples \\(0,\\) are not supported"):
        GeoTiff(p)
    p = write("graya.tif", samples(8, 8, 2, 8, 1), photometric=1, extra_samples=(2,))
    assert (open_bands(p).bands, open_bands(p).alpha_band, open_bands(p).k) == ([0], 1, 2)
    with pytest.raises(_lib.RsbError, match="2 bands"):
        GeoTiff(p)
    p = write("planar.tif", samples(8, 8, 3, 8, 1), planar=2)
    assert open_bands(p).planar == 2
    with pytest.raises(_lib.RsbError, match="PlanarConfiguration 2"):
        GeoTiff(p)
    p = write("stack.tif", samples(8, 8, 5, 16, 1), photometric=1)
    with pytest.raises(_lib.RsbError, match="5 bands \\(Photometric MinIsBlack\\) need --bands"):
        open_bands(p)
    assert open_bands(p, [5, 1, 2]).bands == [4, 0, 1]
    with pytest.raises(_lib.RsbError, match="band 6 is not in this raster of 5 bands"):
        open_bands(p, [6])
    with pytest.raises(_lib.RsbError, match="--bands takes 1 or 3 bands, not 2"):
        open_bands(p, [1, 2])
    px = samples(8, 8, 3, 8, 1)
    for name, kw, text in (("jpeg", dict(tags={259: (3, [7])}), "Compression 7 \\(JPEG\\)"), ("signed", dict(tags={339: (3, [2, 2, 2])}), "SampleFormat 2"),
                           ("float", dict(tags={339: (3, [3, 3, 3])}), "SampleFormat 3"), ("pred3", dict(tags={317: (3, [3])}), "Predictor 3"),
                           ("bits12", dict(tags={258: (3, [12, 12, 12])}), "BitsPerSample 12,12,12"),
                           ("mixed", dict(tags={258: (3, [8, 16, 8])}), "BitsPerSample 8,16,8"),
                           ("palette", dict(photometric=3), "Photometric 3 \\(palette\\)"), ("ycbcr", dict(photometric=6), "Photometric 6 \\(YCbCr\\)"),
                           ("crs", dict(geo=bw.geokeys(1, 27700)), "ProjectedCSTypeGeoKey 27700")):
        with pytest.raises(_lib.RsbError, match=text):
            open_bands(write(name + ".tif", px, **kw))
    # GDAL_NODATA up to 2^bits - 1
    assert open_bands(write("n8.tif", px, nodata="300")).nodata == -1
    assert open_bands(write("n16.tif", samples(8, 8, 1, 16, 1), nodata="300")).nodata == 300


# ---- the rule's arithmetic ----

def test_render_formula():
    for lo, hi in ((0, 255), (0, 1), (100, 103), (7, 65535), (1000, 3000)):
        s = np.array([0, lo - 1 if lo else 0, lo, lo + 1, (lo + hi) // 2, hi - 1, hi, hi + 1, 65535], np.int64)
        got = ref.scale_values(s, lo, hi)
        for x, v in zip(s.tolist(), got.tolist()):
            t = min(max(x, lo), hi) - lo
            want = int(Fraction(255 * t, hi - lo) + Fraction(1, 2))  # 255 t / d, rounded half up
            assert v == want, (lo, hi, x, v, want)
        assert got[2] == 0 and got[6] == 255 and got[1] == 0 and got[-1] == 255
    # half-way ties round up: d = 2 puts t = 1 at 127.5
    assert ref.scale_values(np.array([1]), 0, 2)[0] == 128
    assert ref.scale_values(np.array([3]), 0, 6)[0] == 128
    # the identity scale of 8-bit rasters is the identity
    assert np.array_equal(ref.scale_values(np.arange(256), 0, 255), np.arange(256))
    # nodata is tested on the raw samples: a valid pixel scaled to 0 stays valid, a nodata pixel inside LO..HI is invalid
    raw = np.array([[[5], [50], [60]]], np.uint16)
    out = ref.render(raw, 1, False, 50, [(10, 100)])
    assert out[0, :, 3].tolist() == [255, 0, 255] and out[0, 0, :3].tolist() == [0, 0, 0]


@pytest.mark.parametrize("n", [1, 2, 7, 100, 1001])
def test_stretch_scale_is_the_percentile_rule(n):
    rng = np.random.default_rng(n)
    raw = rng.integers(0, 40, (1, n, 3)).astype(np.uint16)  # ties everywhere
    raw[0, :, 2] = 9  # a flat band
    hist = ref.histogram(raw, 3, False, -1, 16)
    for q_lo, q_hi in ((0, 10000), (200, 9800), (1, 9999), (5000, 5001), (0, 1), (9999, 10000)):
        got = T.stretch_scale(hist, q_lo, q_hi)
        assert got == ref.stretch(raw, 3, False, -1, 16, q_lo, q_hi)
        for b in range(2):
            v = np.sort(raw[0, :, b])
            lo, hi = v[max(1, -(-q_lo * n // 10000)) - 1], v[max(1, -(-q_hi * n // 10000)) - 1]
            assert got[b] == ((lo, hi) if hi > lo else (lo, lo + 1))
        assert got[2] == (9, 10)
    assert T.stretch_scale(hist, 0, 10000)[0] == (raw[0, :, 0].min(), raw[0, :, 0].max() + (raw[0, :, 0].min() == raw[0, :, 0].max()))
    top = np.zeros((1, 256), np.int64)
    top[0, 255] = 4
    assert T.stretch_scale(top, 200, 9800) == [(254, 255)]
    with pytest.raises(_lib.RsbError, match="no valid pixel"):
        T.stretch_scale(np.zeros((1, 256), np.int64), 200, 9800)


# ---- tools ----

def _parse(tool, argv):
    from robosat_b200.tools import segment, tile

    parser = argparse.ArgumentParser()
    sub = parser.add_subparsers()
    {"tile": tile, "segment": segment}[tool].add_parser(sub)
    return parser.parse_args([tool] + argv)


SEG_ARGS = ["--model", "m.toml", "--dataset", "d.toml", "--checkpoint", "c.pth"]


def test_parser_takes_the_band_options():
    a = _parse("tile", ["--zoom", "19", "--bands", "3,2,1", "--stretch", "2,98", "r.tif", "o"])
    assert (a.bands, a.scale, a.stretch) == ("3,2,1", None, "2,98")
    a = _parse("segment", ["--zoom", "19", "--bands", "1", "--scale", "10,4000"] + SEG_ARGS + ["r.tif", "o.tif"])
    assert (a.bands, a.scale, a.stretch) == ("1", "10,4000", None)
    a = _parse("tile", ["--zoom", "19", "r.tif", "o"])
    assert (a.bands, a.scale, a.stretch) == (None, None, None)


@pytest.mark.parametrize("tool", ["tile", "segment"])
def test_tool_refusals_before_device_use(tmp_path, monkeypatch, tool):
    import torch

    from robosat_b200.tools import segment, tile

    called = []
    monkeypatch.setattr(torch.cuda, "is_available", lambda: called.append(1) or False)
    main = {"tile": tile.main, "segment": segment.main}[tool]
    (tmp_path / "d.toml").write_text("[common]\ndataset = '.'\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n")
    (tmp_path / "m.toml").write_text("[common]\ncuda = true\n")
    extra = ["--model", str(tmp_path / "m.toml"), "--dataset", str(tmp_path / "d.toml"), "--checkpoint", "c.pth"] if tool == "segment" else []
    out = str(tmp_path / ("o.tif" if tool == "segment" else "o"))
    r16 = bw.write_bands_tiff(str(tmp_path / "r16.tif"), samples(8, 8, 4, 16, 1), photometric=1, **GEO)
    rgb = bw.write_bands_tiff(str(tmp_path / "rgb.tif"), samples(8, 8, 3, 16, 1), **GEO)
    jpg = bw.write_bands_tiff(str(tmp_path / "j.tif"), samples(8, 8, 3, 8, 1), tags={259: (3, [7])}, **GEO)
    for argv, text in ((["--bands", "1", rgb], "16-bit samples need --scale LO,HI or --stretch P_LO,P_HI"),
                       (["--scale", "0,100", "--stretch", "2,98", rgb], "--scale and --stretch are exclusive"),
                       (["--bands", "5", "--scale", "0,9", r16], "band 5 is not in this raster of 4 bands"),
                       (["--bands", "1,2", "--scale", "0,9", r16], "--bands takes 1 band \\(gray\\) or 3 \\(R,G,B\\), not 2"),
                       (["--bands", "0", "--scale", "0,9", r16], "1-based"),
                       (["--bands", "x", r16], "--bands 'x' is not a list of integers"),
                       (["--scale", "0,9", jpg], "Compression 7 \\(JPEG\\)"),
                       (["--scale", "0,9,1", rgb], "not 3 values"),
                       (["--scale", "0,9,1,5", rgb], "not 4 values"),
                       (["--bands", "1", "--scale", "0,9,1,5,3,4", r16], "3 pairs for 1 bands"),
                       (["--scale", "9,9", rgb], "--scale 9,9 is not 0 <= LO < HI <= 65535"),
                       (["--scale", "0,256", str(jpg).replace("j.tif", "rgb8.tif")], None),
                       (["--stretch", "2,98.123", rgb], "at most two decimals"),
                       (["--stretch", "50,50", rgb], "P_LO < P_HI"),
                       (["--stretch", "2,101", rgb], "P_HI <= 100"),
                       (["--bands", "1", r16], "need --scale")):
        if text is None:  # an 8-bit raster: the scale is checked against 255
            bw.write_bands_tiff(argv[-1], samples(8, 8, 3, 8, 1), **GEO)
            text = "--scale 0,256 is not 0 <= LO < HI <= 255"
        with pytest.raises(SystemExit, match=text):
            main(_parse(tool, ["--zoom", "19"] + extra + argv[:-1] + [argv[-1], out]))
        assert not called, (argv, text)
    # a valid band run gets as far as the device check
    with pytest.raises(SystemExit, match="CUDA requested but not available"):
        main(_parse(tool, ["--zoom", "19"] + extra + ["--bands", "4,3,2", "--stretch", "2,98", r16, out]))


def test_stretch_percent_parsing():
    from robosat_b200.tools.tile import _basis_points

    assert [_basis_points(v) for v in ("0", "2", "2.5", "2.05", "99.99", "100", "100.0")] == [0, 200, 250, 205, 9999, 10000, 10000]
    assert [_basis_points(v) for v in ("2.005", "-1", "1e2", "", "abc")] == [None] * 5


# ---- ABI ----

def test_abi_validates_before_the_device_check():
    import torch

    lib = _lib.load()
    src = np.zeros(64, np.uint16)
    out = np.zeros(64, np.uint32)
    scale = np.array([0, 255, 0, 255, 0, 255], np.int32)
    hist = np.zeros(3 * 65536, np.int64)
    p = src.ctypes.data
    base = [p, 2, 4, 16, 3, 1, -1, scale.ctypes.data, out.ctypes.data, 16, None]
    for k, bad in ((0, None), (0, p + 2), (3, 12), (4, 2), (5, 2), (6, 65536), (1, 0), (2, 0), (7, None), (8, None), (9, 15), (9, 14),
                   (8, out.ctypes.data + 2)):
        args = list(base)
        args[k] = bad
        assert lib.rsb_tile_render(*args) == -1, (k, bad)
    bad_scale = np.array([5, 5, 0, 255, 0, 255], np.int32)
    assert lib.rsb_tile_render(*(base[:7] + [bad_scale.ctypes.data] + base[8:])) == -1
    base8 = [p, 2, 4, 8, 3, 0, 255, scale.ctypes.data, out.ctypes.data, 16, None]
    high = np.array([0, 256, 0, 255, 0, 255], np.int32)
    assert lib.rsb_tile_render(*(base8[:7] + [high.ctypes.data] + base8[8:])) == -1
    hbase = [p, 2, 4, 16, 3, 1, -1, hist.ctypes.data, None]
    for k, bad in ((0, None), (0, p + 8), (3, 32), (4, 0), (5, -1), (6, -2), (1, -1), (7, None), (7, hist.ctypes.data + 4)):
        args = list(hbase)
        args[k] = bad
        assert lib.rsb_band_histogram(*args) == -1, (k, bad)
    if not torch.cuda.is_available():
        assert lib.rsb_tile_render(*base) == -3
        assert lib.rsb_band_histogram(*hbase) == -3
    # the host decoder checks its selection, bits and planar layout
    buf = (ctypes.c_uint8 * 64)()
    off, cnt = np.zeros(3, np.int64), np.zeros(3, np.int64)
    sel = np.array([0, 1, 2], np.int32)
    args = [ctypes.addressof(buf), 64, off.ctypes.data, cnt.ctypes.data, 3, 4, 4, 4, 4, 0, 3, 8, 2, 0, 1, 1, sel.ctypes.data, 3, 0, 4, 0, 4,
            out.ctypes.data, 1, None]
    assert lib.rsb_tiff_decode_bands(*args) == -1 and "holds fewer bytes than its pixels" in _lib.last_error()  # the chunks are empty
    for k, bad, text in ((11, 12, "12 bits"), (12, 3, "planar 3"), (17, 0, "0 selected bands"), (17, 5, "5 selected bands"),
                         (4, 1, "1 chunks, the raster needs 3"), (19, 5, "outside the 4 x 4 raster"), (16, None, "selected bands")):
        a = list(args)
        a[k] = bad
        assert lib.rsb_tiff_decode_bands(*a) == -1, (k, bad)
        assert text in _lib.last_error(), (k, bad, _lib.last_error())
    sel[1] = 3
    assert lib.rsb_tiff_decode_bands(*args) == -1
    assert re.search("band 3 of a raster of 3", _lib.last_error())
