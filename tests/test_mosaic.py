"""`rs mosaic` without a GPU: the lattice step and the windows against the numpy restatement, the budget refusal, the GeoTIFF
writer and the library's tile encoder read back through PIL and `GeoTiff`, the header-only grid read, the ABI's argument validation
and the tool's parser and refusals."""

import argparse
import ctypes
import os

import numpy as np
import pytest
from PIL import Image

import mosaic_reference as ref
import tiff_writer as tw
from robosat_b200 import _lib
from robosat_b200 import mosaic as M
from robosat_b200 import tile as T
from robosat_b200.geotiff import GeoTiff, read_grid


def utm_grid(zone=32, south=False, W=700, H=500, res=0.3):
    lon0 = 6 * zone - 183
    E, N = T.tm_forward(lon0 + 1.1, -33.0 if south else 47.2, lon0, fn=1e7 if south else 0.0)
    return M.Grid(W, H, ("utm", zone, south), (float(E), res, 0.0, float(N), 0.0, -res))


def grids():
    return {
        "3857": M.Grid(600, 450, "3857", (1113300.3, 0.37, 0.0, 6106900.7, 0.0, -0.37)),
        "4326": M.Grid(500, 600, "4326", (10.0003, 3e-6, 0.0, 48.0004, 0.0, -2.5e-6)),
        "utm": utm_grid(),
        "utm-south": utm_grid(19, True),
        "rotated": M.Grid(400, 300, "3857", (1113300.3, 0.4, 0.06, 6106900.7, 0.05, -0.4)),
    }


def test_lattice_step_meets_the_bound_on_every_cell():
    seen = set()
    coarse = M.Grid(300, 2000, "4326", (5.0, 0.02, 0.0, 75.0, 0.0, -0.02))  # latitude is not linear in Mercator Y
    for name, g, zoom in [(n, g, 18) for n, g in grids().items()] + [("coarse", coarse, 8), ("coarse", coarse, 10)]:
        step = M.choose_step(g, zoom, 256)
        assert step == ref.choose_step(g, zoom, 256), name
        assert M.step_error(g, zoom, 256, step) <= M.TOLERANCE
        assert M.step_error(g, zoom, 256, step, rows=3) == M.step_error(g, zoom, 256, step)
        if step < 64:
            assert M.step_error(g, zoom, 256, 2 * step) > M.TOLERANCE
        seen.add(step)
    assert 64 in seen and len(seen) > 1


def existing_tiles(g, zoom, size, holes=3):
    """the tiles the grid's corners span, minus a few (holes)"""
    gx, gy = M.global_coords(g, zoom, size, np.array([0, g.width, 0, g.width]), np.array([0, 0, g.height, g.height]))
    xs = range(int(gx.min() // size) - 1, int(gx.max() // size) + 2)
    ys = range(int(gy.min() // size) - 1, int(gy.max() // size) + 2)
    t = [(x, y) for x in xs for y in ys]
    return np.array([p for k, p in enumerate(t) if k % 7 != holes], np.int64)


def smallest_budget(g, zoom, size, tiles, step):
    """the smallest budget `plan` accepts: that of the costliest single chunk, so that most windows hold one chunk"""
    lo, hi = 1, max(w.device_bytes(size) for w in M.plan(g, zoom, size, tiles, step) if w.reach is not None)
    while lo < hi:
        mid = (lo + hi) // 2
        try:
            M.plan(g, zoom, size, tiles, step, mid)
            hi = mid
        except _lib.RsbError:
            lo = mid + 1
    return lo


@pytest.mark.parametrize("name", ["3857", "4326", "utm", "rotated"])
@pytest.mark.parametrize("tiny", [False, True])
def test_windows_hold_every_reachable_sample(name, tiny):
    g = grids()[name]
    zoom, size = 18, 64
    tiles = existing_tiles(g, zoom, size)
    step = M.choose_step(g, zoom, size)
    budget = smallest_budget(g, zoom, size, tiles, step) if tiny else M.DEFAULT_BUDGET
    windows = M.plan(g, zoom, size, tiles, step, budget)
    if tiny:
        assert all(w.device_bytes(size) <= budget for w in windows if w.reach is not None)
        assert len(windows) > -(-g.height // M.CHUNK)
    n = ref.nodes(g, zoom, size, step)
    have = {tuple(t) for t in tiles.tolist()}
    seen = np.zeros((g.height, g.width), int)
    for w in windows:
        assert w.row0 % M.CHUNK == 0 and w.col0 % M.CHUNK == 0 and w.rows == min(M.CHUNK, g.height - w.row0)
        seen[w.row0:w.row0 + w.rows, w.col0:w.col0 + w.cols] += 1
        i, j = np.arange(w.col0, w.col0 + w.cols), np.arange(w.row0, w.row0 + w.rows)
        IX, IY = np.meshgrid(i // step, j // step)
        FX, FY = np.meshgrid((i % step) / step, (j % step) / step)
        gx = ref._lerp(ref._lerp(n[IY, IX, 0], n[IY, IX + 1, 0], FX), ref._lerp(n[IY + 1, IX, 0], n[IY + 1, IX + 1, 0], FX), FY)
        gy = ref._lerp(ref._lerp(n[IY, IX, 1], n[IY, IX + 1, 1], FX), ref._lerp(n[IY + 1, IX, 1], n[IY + 1, IX + 1, 1], FX), FY)
        if w.reach is None:  # no existing tile within reach of any sample
            for du in (-1, 0, 1):
                for dv in (-1, 0, 1):
                    assert not any((int(a) // size, int(b) // size) in have for a, b in zip((gx + du).ravel(), (gy + dv).ravel()))
            continue
        # the window's nodes are the restatement's, bit for bit
        assert np.array_equal(w.nodes, n[w.ky0:w.ky0 + w.nodes.shape[0], w.kx0:w.kx0 + w.nodes.shape[1]])
        tx0, ty0, tx1, ty1 = w.reach
        assert {tuple(t) for t in w.tiles.tolist()} == {t for t in have if tx0 <= t[0] <= tx1 and ty0 <= t[1] <= ty1}
        for du in (-0.5, 0.0, 0.5):  # every tap of both resamplings lies in the slot table's range
            for dv in (-0.5, 0.0, 0.5):
                a = np.clip(np.floor(gx + du), 0, 2 ** zoom * size - 1) // size
                b = np.clip(np.floor(gy + dv), 0, 2 ** zoom * size - 1) // size
                assert (a >= tx0).all() and (a <= tx1).all() and (b >= ty0).all() and (b <= ty1).all()
    assert (seen == 1).all()


def test_a_chunk_over_the_budget_is_refused_before_any_allocation():
    g = grids()["utm"]
    with pytest.raises(_lib.RsbError, match="more than the budget"):
        M.plan(g, 18, 256, existing_tiles(g, 18, 256), 64, budget=10000)


# ---- the GeoTIFF writer ----

class Win:
    def __init__(self, row0, rows, col0, cols):
        self.row0, self.rows, self.col0, self.cols = row0, rows, col0, cols


def write_raster(path, px, grid, palette=None, nodata=None, big=None, empty=()):
    """px uint8 [H, W] through TiffWriter, in windows of one or two chunks; chunk rows listed in `empty` as all-nodata windows"""
    w = M.TiffWriter(path, grid, palette, nodata, big=big)
    H, W = px.shape
    for r0 in range(0, H, M.CHUNK):
        rows = min(M.CHUNK, H - r0)
        for c0 in range(0, W, 2 * M.CHUNK):
            cols = min(2 * M.CHUNK, W - c0)
            if r0 // M.CHUNK in empty:
                w.write(Win(r0, rows, c0, cols), None)
            else:
                block = np.zeros((rows, cols + 5), np.uint8)  # a pitch wider than the window
                block[:, :cols] = px[r0:r0 + rows, c0:c0 + cols]
                w.write(Win(r0, rows, c0, cols), block[:, :cols])
    w.close()
    return w


@pytest.mark.parametrize("big", [False, True])
@pytest.mark.parametrize("kind", ["palette", "gray"])
@pytest.mark.parametrize("shape", [(256, 512), (300, 777), (17, 5)])
@pytest.mark.parametrize("nodata", [None, 7])
def test_writer_round_trips_through_pil(tmp_path, big, kind, shape, nodata):
    rng = np.random.default_rng(sum(shape))
    H, W = shape
    px = rng.integers(0, 4, (H, W), dtype=np.uint8)
    px[H // 3:] = 1
    empty = (1,) if H > 256 else ()
    if empty:
        px[256:] = 0 if nodata is None else nodata
    palette = rng.integers(0, 256, (256, 3), dtype=np.uint8) if kind == "palette" else None
    path = str(tmp_path / "o.tif")
    g = grids()["3857"]
    write_raster(path, px, M.Grid(W, H, g.crs, g.geotransform), palette, nodata, big=big, empty=empty)
    with open(path, "rb") as fp:
        assert fp.read(4) == (b"II+\0" if big else b"II*\0")
    im = Image.open(path)
    assert im.mode == ("P" if kind == "palette" else "L") and im.size == (W, H)
    assert np.array_equal(np.array(im), px)
    if palette is not None:
        assert np.array_equal(np.array(im.getpalette()[:768], np.uint8).reshape(256, 3), palette)
    assert (42113 in im.tag_v2) == (nodata is not None)
    if nodata is not None:
        assert im.tag_v2[42113].strip("\0") == "7"
    assert im.tag_v2[322] == 256 and im.tag_v2[259] == 8
    assert not [f for f in os.listdir(tmp_path) if f.endswith(".tmp")]


@pytest.mark.parametrize("name", ["3857", "4326", "utm", "utm-south", "rotated"])
def test_gray_output_reads_back_with_its_grid(tmp_path, name):
    g = grids()[name]
    px = np.random.default_rng(1).integers(0, 256, (g.height, g.width), dtype=np.uint8)
    path = str(tmp_path / "g.tif")
    write_raster(path, px, g)
    r = GeoTiff(path)
    assert (r.width, r.height, r.crs, r.geotransform, r.spp, r.tiled) == (g.width, g.height, g.crs, g.geotransform, 1, True)
    assert np.array_equal(r.read_window(0, g.height, 0, g.width)[..., 0], px)
    assert read_grid(path) == (g.width, g.height, g.crs, g.geotransform)


def test_encoder_pads_edge_chunks_with_the_fill_value():
    lib = _lib.load()
    cap = lib.rsb_tiff_deflate_bound(256 * 256)
    assert cap >= 256 * 256
    px = np.arange(40 * 300, dtype=np.uint32).astype(np.uint8).reshape(40, 300)
    out = np.empty(2 * cap, np.uint8)
    sizes = np.empty(2, np.int64)
    assert lib.rsb_tiff_encode_chunks(px.ctypes.data, 300, 40, 300, 256, 9, 6, out.ctypes.data, cap, sizes.ctypes.data, 2) == 0
    import zlib

    for k in range(2):
        chunk = np.frombuffer(zlib.decompress(bytes(out[k * cap:k * cap + sizes[k]])), np.uint8).reshape(256, 256)
        want = np.full((256, 256), 9, np.uint8)
        part = px[:, k * 256:(k + 1) * 256]
        want[:40, :part.shape[1]] = part
        assert np.array_equal(chunk, want)
    for args in ((px.ctypes.data, 299, 40, 300, 256, 9, 6, out.ctypes.data, cap, sizes.ctypes.data, 2),  # pitch < cols
                 (px.ctypes.data, 300, 257, 300, 256, 9, 6, out.ctypes.data, cap, sizes.ctypes.data, 2),  # rows > chunk
                 (px.ctypes.data, 300, 40, 300, 250, 9, 6, out.ctypes.data, cap, sizes.ctypes.data, 2),  # chunk not a multiple of 16
                 (px.ctypes.data, 300, 40, 300, 256, 256, 6, out.ctypes.data, cap, sizes.ctypes.data, 2),
                 (px.ctypes.data, 300, 40, 300, 256, 9, 6, out.ctypes.data, 100, sizes.ctypes.data, 2)):
        assert lib.rsb_tiff_encode_chunks(*args) == -1


# ---- the grid read ----

GEO_UTM = dict(geo=tw.geokeys(1, 32632), scale=(0.3, 0.3, 0.0), tiepoint=(0, 0, 0, 500000.0, 5300000.0, 0))


@pytest.mark.parametrize("name,kw,bands", [
    ("jpeg", dict(tags={259: (3, [7])}), 3),
    ("16-bit", dict(tags={258: (3, [16])}), 1),
    ("palette", dict(photometric=3, tags={320: (3, [0] * 768)}), 1),
])
def test_grid_read_takes_layouts_geotiff_rejects(tmp_path, name, kw, bands):
    p = tw.write_tiff(str(tmp_path / "l.tif"), np.zeros((20, 30, bands), np.uint8), **GEO_UTM, **kw)
    with pytest.raises(_lib.RsbError):
        GeoTiff(p)
    assert read_grid(p) == (30, 20, ("utm", 32, False), (500000.0, 0.3, 0.0, 5300000.0, 0.0, -0.3))


def test_grid_read_names_an_unsupported_crs(tmp_path):
    p = tw.write_tiff(str(tmp_path / "c.tif"), np.zeros((4, 4, 1), np.uint8), geo=tw.geokeys(1, 27700), scale=(1, 1, 0), tiepoint=(0, 0, 0, 0, 0, 0))
    with pytest.raises(_lib.RsbError, match="ProjectedCSTypeGeoKey 27700"):
        read_grid(p)


# ---- ABI and tool ----

def test_abi_validates_before_the_device_check():
    import torch

    lib = _lib.load()
    buf = (ctypes.c_uint8 * 64)()
    nodes = np.zeros(64, np.float64)
    slots = np.zeros(4, np.int32)
    b = ctypes.addressof(buf)
    base = [b, 64, 1, slots.ctypes.data, 0, 0, 1, 1, 3, 8, nodes.ctypes.data, 0, 0, 2, 2, 64, 0, 0, 4, 4, 0, 0, b, 4, b, b, None]
    for k, bad in ((0, None), (1, 63), (2, 0), (3, None), (4, 8), (6, 0), (7, 9), (8, 31), (9, 0), (9, 4097), (10, None), (13, 1), (15, 3),
                   (15, 128), (18, 0), (19, 0), (20, 2), (21, 256), (21, -1), (23, 3), (16, -1)):
        args = list(base)
        args[k] = bad
        assert lib.rsb_mosaic_warp(*args) == -1, (k, bad)
    if not torch.cuda.is_available():
        assert lib.rsb_mosaic_warp(*base) == -3


def _parse(argv):
    from robosat_b200.tools import mosaic

    parser = argparse.ArgumentParser()
    sub = parser.add_subparsers()
    mosaic.add_parser(sub)
    return parser.parse_args(argv)


def test_parser():
    a = _parse(["mosaic", "--zoom", "18", "masks", "out.tif"])
    assert (a.zoom, a.like, a.resampling, a.nodata, a.masks, a.out) == (18, None, "nearest", None, "masks", "out.tif")
    a = _parse(["mosaic", "--zoom", "18", "--like", "o.tif", "--resampling", "bilinear", "--nodata", "255", "probs", "p.tif"])
    assert (a.like, a.resampling, a.nodata) == ("o.tif", "bilinear", 255)
    with pytest.raises(SystemExit):
        _parse(["mosaic", "--zoom", "18", "--resampling", "mode", "m", "o.tif"])
    with pytest.raises(SystemExit):
        _parse(["mosaic", "m", "o.tif"])  # --zoom is required
    from robosat_b200.tools import __main__ as main

    assert "mosaic.add_parser" in open(main.__file__).read()


def save_png(path, array, palette=None, **kw):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    im = Image.fromarray(array, "L")
    if palette is not None:
        im = im.convert("P")
        im.putpalette(palette)
    im.save(path, **kw)


def test_tool_refusals_come_before_the_device_check(tmp_path, monkeypatch):
    import torch

    from robosat_b200.tools import mosaic

    calls = []
    monkeypatch.setattr(_lib, "require_device", lambda: calls.append(1))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: calls.append(0) or False)
    out = str(tmp_path / "o.tif")
    m = tmp_path / "m"

    def refuse(text, *extra, root=m):
        with pytest.raises(SystemExit, match=text):
            mosaic.main(_parse(["mosaic", "--zoom", "18"] + list(extra) + [str(root), out]))

    refuse("--nodata must be in 0..255", "--nodata", "256")
    refuse("--nodata must be in 0..255", "--nodata", "-1")
    refuse("no tiles at zoom 18")
    gray = np.zeros((32, 32), np.uint8)
    pal = [0, 0, 0, 255, 0, 0]
    save_png(str(m / "18" / "5" / "7.png"), gray, pal)
    save_png(str(m / "18" / "5" / "8.png"), gray + 1, pal + [0, 255, 0])
    (m / "18" / "6").mkdir()
    (m / "18" / "6" / "7.png").write_bytes(b"GIF89a" + b"\0" * 40)
    refuse("6/7.png is not a PNG file")
    Image.fromarray(np.zeros((32, 32, 3), np.uint8), "RGB").save(str(m / "18" / "6" / "7.png"))
    refuse("6/7.png is a PNG of colour type 2")
    save_png(str(m / "18" / "6" / "7.png"), np.zeros((16, 16), np.uint8), pal)
    refuse("6/7.png is 16x16, .*5/7.png is 32x32")
    save_png(str(m / "18" / "6" / "7.png"), gray)
    refuse("6/7.png is a gray PNG, .*5/7.png is a palette PNG")
    save_png(str(m / "18" / "6" / "7.png"), gray, [0, 0, 0, 255, 0, 1])
    refuse("6/7.png: palette entry 1 is \\(255, 0, 1\\), another tile's is \\(255, 0, 0\\)")
    save_png(str(m / "18" / "6" / "7.png"), gray, pal + [0, 255, 0, 9, 9, 9])
    like = tw.write_tiff(str(tmp_path / "like.tif"), np.zeros((4, 4, 1), np.uint8), geo=tw.geokeys(1, 2056), scale=(1, 1, 0), tiepoint=(0, 0, 0, 0, 0, 0))
    refuse("--like .*ProjectedCSTypeGeoKey 2056", "--like", like)
    assert calls == []
    refuse("CUDA requested but not available")
    assert calls == [0] and not os.path.exists(out)


def test_palette_union_and_gray(tmp_path):
    pal = [0, 0, 0, 255, 0, 0]
    tiles = {}
    for k, p in enumerate((pal, pal + [0, 255, 0], pal + [0, 255, 0, 1, 2, 3])):
        tiles[(k, 0)] = str(tmp_path / ("%d.png" % k))
        save_png(tiles[(k, 0)], np.full((8, 8), k, np.uint8), p, optimize=True)
    size, union = M.check_tiles(tiles)
    assert size == 8 and union[:4].tolist() == [[0, 0, 0], [255, 0, 0], [0, 255, 0], [1, 2, 3]] and not union[4:].any()
    gray = {(0, 0): str(tmp_path / "g.png")}
    save_png(gray[(0, 0)], np.zeros((8, 8), np.uint8))
    assert M.check_tiles(gray) == (8, None)
