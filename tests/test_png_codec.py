"""Host-side PNG codec of librsb200.so (csrc/rsb_png.cpp) against PIL -- the reference's own reader / writer for the files
either side of the predict path (robosat/tiles.py:150-159,181; robosat/tools/predict.py:105-113). CPU only."""

import io

import numpy as np
import pytest
from PIL import Image

from robosat_b200 import _lib, colors, synth


def _decode(raw, w, h):
    out = np.zeros((h, w, 3), dtype=np.uint8)
    rc = _lib.load().rsb_png_decode_rgb(raw, len(raw), out.ctypes.data, w, h)
    return rc, out


@pytest.mark.parametrize("level", [0, 1, 6, 9])
def test_decode_rgb_matches_pil_for_every_filter_mix(level):
    u8 = synth.make_tiles_u8(2, 256, seed=3).numpy()
    for arr in u8:
        b = io.BytesIO()
        Image.fromarray(arr).save(b, format="PNG", compress_level=level)  # PIL picks adaptive filters per scanline for RGB
        rc, out = _decode(b.getvalue(), 256, 256)
        assert rc == 0, _lib.last_error()
        assert np.array_equal(out, np.asarray(Image.open(io.BytesIO(b.getvalue())).convert("RGB")))


def test_decode_handles_the_modes_convert_rgb_accepts():
    base = Image.fromarray(synth.make_tiles_u8(1, 128, seed=4).numpy()[0])
    for name, im in (("L", base.convert("L")), ("LA", base.convert("LA")), ("RGBA", base.convert("RGBA")), ("P", base.quantize(37)),
                     ("rect", base.crop((0, 0, 128, 96)))):
        b = io.BytesIO()
        im.save(b, format="PNG")
        rc, out = _decode(b.getvalue(), im.size[0], im.size[1])
        assert rc == 0, (name, _lib.last_error())
        assert np.array_equal(out, np.asarray(Image.open(io.BytesIO(b.getvalue())).convert("RGB"))), name


def test_decode_reports_what_it_does_not_handle():
    a16 = (np.arange(64 * 64, dtype=np.uint16).reshape(64, 64) * 7)
    b = io.BytesIO()
    Image.fromarray(a16).save(b, format="PNG")
    rc, _ = _decode(b.getvalue(), 64, 64)
    assert rc == _lib.RSB_E_UNSUPPORTED  # 16-bit: the caller falls back to PIL (robosat_b200/stitch.py:decode_rgb)
    rc, _ = _decode(b"\xff\xd8\xff\xe0" + b"\0" * 64, 64, 64)
    assert rc == _lib.RSB_E_UNSUPPORTED  # a JPEG
    ok = io.BytesIO()
    Image.fromarray(np.zeros((64, 64, 3), np.uint8)).save(ok, format="PNG")
    rc, _ = _decode(ok.getvalue(), 32, 32)
    assert rc == -1 and "expected 32x32" in _lib.last_error()  # wrong tile size is an error, as in the reference's asserts
    rc, _ = _decode(ok.getvalue()[:60], 64, 64)
    assert rc == -1


@pytest.mark.parametrize("level", [1, 6])
def test_encode_p8_round_trips_through_pil(level, tmp_path):
    pal = colors.continuous_palette_for_color("pink", 256)
    rs = np.random.RandomState(0)
    for arr in (rs.randint(0, 256, (256, 256)).astype(np.uint8), np.clip(np.add.outer(np.arange(200), np.arange(312)) // 2, 0, 255).astype(np.uint8)):
        h, w = arr.shape
        path = str(tmp_path / ("m%d_%d.png" % (level, w)))
        _lib.check(_lib.load().rsb_png_write_p8(path.encode(), arr.ctypes.data, w, h, bytes(pal), 256, level), "write")
        im = Image.open(path)
        assert im.mode == "P" and im.size == (w, h)
        assert np.array_equal(np.asarray(im), arr)
        assert im.getpalette()[:768] == pal  # what `rs masks` / a viewer reads back is what predict.py:105-108 would have written


def test_save_batch_writes_each_callers_palette(tmp_path):
    """tools/predict.py's writers get a fresh palette list per call (`rs rasterize` after `rs predict` in one process): each
    file carries the palette it was written with, even when a new list takes the address of a freed one"""
    from robosat_b200.tools.predict import _save_batch, _save_png

    q = np.zeros((2, 8, 8), np.uint8)
    q[:, 2:5, 3:6] = 1
    cases = [("pink", None), ("denim", "orange"), ("pink", None), ("dark", "gray"), ("denim", "orange"), ("teal", "red")] * 3
    for i, (a, b) in enumerate(cases):
        want = colors.continuous_palette_for_color(a, 256) if b is None else colors.make_palette(a, b)
        if i % 2:
            _save_batch(str(tmp_path), list(want), [(i, 0, 1), (i, 1, 1)], q, 2)
        else:
            for y in range(2):
                _save_png(str(tmp_path), list(want), i, y, 1, q[y])
        for y in range(2):
            im = Image.open(str(tmp_path / "1" / str(i) / ("%d.png" % y)))
            assert im.getpalette()[:len(want)] == want, (i, a, b)
            assert np.array_equal(np.asarray(im), q[y])


def test_encode_strategy_follows_the_content(tmp_path):
    """noise-like masks skip deflate's string matcher (Z_RLE) without growing; compressible masks keep the default strategy"""
    import os
    import zlib

    pal = colors.continuous_palette_for_color("pink", 256)
    rs = np.random.RandomState(1)
    noisy = rs.randint(0, 256, (256, 256)).astype(np.uint8)
    yy, xx = np.mgrid[0:256, 0:256]
    soft = np.clip((np.sin(xx / 31.0) + np.cos(yy / 23.0)) * 400 + 128, 0, 255).astype(np.uint8)
    for name, arr, same_as_default in (("noisy", noisy, False), ("soft", soft, True)):
        path = str(tmp_path / (name + ".png"))
        _lib.check(_lib.load().rsb_png_write_p8(path.encode(), arr.ctypes.data, 256, 256, bytes(pal), 256, 6), "write")
        assert np.array_equal(np.asarray(Image.open(path)), arr)
        raw = np.concatenate([np.zeros((256, 1), np.uint8), arr], 1).tobytes()
        default = len(zlib.compress(raw, 6))
        overhead = 8 + 3 * 12 + 13 + 768 + 12  # signature, IHDR / PLTE / IDAT / IEND framing
        if same_as_default:
            assert os.path.getsize(path) == default + overhead
        else:
            assert os.path.getsize(path) <= 1.01 * default + overhead


def test_tools_use_the_native_codec_and_agree_with_pil(tmp_path, monkeypatch):
    from robosat_b200 import stitch
    from robosat_b200.tools import predict

    arr = synth.make_tiles_u8(1, 64, seed=8).numpy()[0]
    p = str(tmp_path / "t.png")
    Image.fromarray(arr).save(p)
    assert np.array_equal(stitch.decode_rgb(p, 64), arr)
    j = str(tmp_path / "t.webp")
    Image.fromarray(arr).save(j, lossless=True)
    assert np.array_equal(stitch.decode_rgb(j, 64), arr)  # non-PNG formats stay with PIL
    pal = colors.continuous_palette_for_color("pink", 256)
    q = (arr[..., 0]).copy()
    predict._save_png(str(tmp_path / "a"), pal, 1, 2, 3, q)
    monkeypatch.setattr(predict, "NATIVE_PNG", False)
    predict._save_png(str(tmp_path / "b"), pal, 1, 2, 3, q)
    a, b = Image.open(tmp_path / "a" / "3" / "1" / "2.png"), Image.open(tmp_path / "b" / "3" / "1" / "2.png")
    assert a.mode == b.mode == "P" and np.array_equal(np.asarray(a), np.asarray(b)) and a.getpalette()[:768] == b.getpalette()[:768]


def _own_inflate(stream, n):
    out = np.empty(max(n, 1), dtype=np.uint8)
    rc = _lib.load().rsb_zlib_inflate(stream, len(stream), out.ctypes.data, n)
    return rc, out[:n].tobytes()


def test_own_inflate_matches_zlib_on_every_block_type_and_strategy():
    """csrc/rsb_inflate.cpp (the PNG reader's DEFLATE decoder) against zlib: stored / fixed / dynamic blocks, literal-only and
    match-heavy data, long runs (distance 1), maximum distances, multi-block streams"""
    import os
    import zlib

    rs = np.random.RandomState(0)
    text = open(__file__, "rb").read()
    cases = [b"", b"a", b"hello hello hello hello hello", bytes(70000), os.urandom(70000), bytes(rs.randint(0, 4, 200000).astype(np.uint8)),
             (b"abcdefgh" * 5000) + os.urandom(1000) + (b"xy" * 40000), text * 20,
             bytes(rs.randint(0, 256, 40000).astype(np.uint8)) * 3]  # repeats at distance 40 000 > 32 K: literals again
    for i, c in enumerate(cases):
        for level in (0, 1, 6, 9):
            for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
                co = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
                stream = co.compress(c) + co.flush()
                rc, got = _own_inflate(stream, len(c))
                assert rc == 0 and got == c, (i, level, strategy, _lib.last_error())


def test_own_inflate_rejects_damaged_streams_and_the_reader_falls_back():
    """A flipped bit, a truncated stream or a wrong expected size is an error, never a silent wrong answer (Adler-32 is verified) and
    never an out-of-bounds access; window sizes / dictionaries the decoder does not take are left to zlib by the PNG reader."""
    import zlib

    rs = np.random.RandomState(1)
    text = open(__file__, "rb").read() * 4
    stream = zlib.compress(text, 6)
    for _ in range(400):
        b = bytearray(stream)
        b[rs.randint(2, len(b))] ^= 1 << rs.randint(0, 8)
        rc, got = _own_inflate(bytes(b), len(text))
        assert rc != 0 or got == text
    for cut in (6, 10, 100, len(stream) // 2, len(stream) - 1):
        assert _own_inflate(stream[:cut], len(text))[0] != 0
    assert _own_inflate(stream, len(text) - 1)[0] != 0 and _own_inflate(stream, len(text) + 1)[0] != 0


def test_png_reader_is_identical_with_either_inflate(monkeypatch):
    """the same tiles through the library inflate (default) and through zlib (RSB_INFLATE=zlib, read once per process: checked in
    a child) decode to the same pixels as PIL"""
    import subprocess
    import sys

    code = ("import io, sys, numpy as np\n"
            "from PIL import Image\n"
            "from robosat_b200 import _lib, synth\n"
            "u8 = synth.make_tiles_u8(3, 256, seed=5).numpy()\n"
            "for arr in u8:\n"
            "    for level in (1, 6, 9):\n"
            "        b = io.BytesIO(); Image.fromarray(arr).save(b, format='PNG', compress_level=level); raw = b.getvalue()\n"
            "        out = np.zeros((256, 256, 3), np.uint8)\n"
            "        assert _lib.load().rsb_png_decode_rgb(raw, len(raw), out.ctypes.data, 256, 256) == 0\n"
            "        assert np.array_equal(out, arr)\n"
            "print('ok')\n")
    import os

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for mode in ("own", "zlib"):
        env = dict(os.environ, RSB_INFLATE=mode, PYTHONPATH=root)
        res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
        assert res.returncode == 0 and res.stdout.strip().endswith("ok"), (mode, res.stderr[-800:])
