"""`rs tile` without a GPU: the TIFF decoder against PIL (libtiff), the GeoTIFF header parser and its named rejections, the
projections against published and independent values, the lattice step, the windows and the candidate tiles, the ABI's argument
validation and the tool's parser and refusals."""

import argparse
import ctypes
import math

import numpy as np
import pytest
from PIL import Image, TiffImagePlugin

import tile_reference as ref
import tiff_writer as tw
from robosat_b200 import _lib
from robosat_b200 import tile as T
from robosat_b200.cover import xy as cover_xy
from robosat_b200.geotiff import GeoTiff
from robosat_b200.rasterize import project

GEO_3857 = dict(geo=tw.geokeys(), scale=(0.5, 0.5, 0.0), tiepoint=(0, 0, 0, 1000.0, 2000.0, 0))


def pixels(H, W, spp, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (H, W, spp), dtype=np.uint8)


def pil_pixels(path):
    a = np.array(Image.open(path))
    return a[..., None] if a.ndim == 2 else a


# ---- decoder ----

CASES = [  # (big, order, layout, compression, predictor, spp)
    (False, "<", ("strip", 7), 1, 1, 3),
    (True, ">", ("strip", 5), 1, 1, 1),
    (False, ">", ("tile", 16, 32), 1, 1, 4),
    (True, "<", ("tile", 32, 16), 8, 1, 3),
    (False, "<", ("strip", 11), 8, 2, 4),
    (False, ">", ("tile", 16, 16), 8, 2, 1),
    (True, ">", ("strip", 3), 5, 1, 3),
    (False, "<", ("tile", 16, 48), 5, 2, 3),
    (True, "<", ("strip", 64), 5, 2, 4),
    (False, ">", ("tile", 48, 16), 5, 1, 1),
    (False, "<", ("strip", 37), 32946, 1, 3),
]


def _write_case(path, case, H=37, W=45, seed=1):
    big, order, layout, comp, pred, spp = case
    px = pixels(H, W, spp, seed)
    px[H // 2] = 7  # runs, so that LZW and DEFLATE have repeats to code
    kw = dict(big=big, order=order, compression=comp, predictor=pred, **GEO_3857)
    if layout[0] == "tile":
        kw["tile"] = layout[1:]
    else:
        kw["rows_per_strip"] = layout[1]
    tw.write_tiff(path, px, **kw)
    return px


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%s-%s-%s-c%d-p%d-b%d" % ("big" if c[0] else "classic", "LE" if c[1] == "<" else "BE", c[2][0], c[3], c[4], c[5]))
def test_decoder_windows_equal_pil_crops(tmp_path, case):
    path = str(tmp_path / "a.tif")
    px = _write_case(path, case)
    if case[0] and case[1] == ">":  # Pillow does not open big-endian BigTIFF: read the little-endian twin of the same pixels
        _write_case(str(tmp_path / "le.tif"), (True, "<") + case[2:])
        pil = pil_pixels(str(tmp_path / "le.tif"))
    else:
        pil = pil_pixels(path)
    assert np.array_equal(pil, px)  # the writer wrote what PIL (libtiff) reads
    g = GeoTiff(path)
    H, W = px.shape[:2]
    for r0, rows, c0, cols in ((0, H, 0, W), (3, 17, 5, 33), (H - 1, 1, W - 1, 1), (15, 9, 0, 1), (0, 1, 16, 16), (30, 7, 31, 14)):
        for threads in (1, 4):
            got = g.read_window(r0, rows, c0, cols, threads=threads)
            assert np.array_equal(got, pil[r0:r0 + rows, c0:c0 + cols]), (r0, rows, c0, cols, threads)


def _pil_geo_info():
    ifd = TiffImagePlugin.ImageFileDirectory_v2()
    for tag, typ, val in ((34735, 3, tuple(tw.geokeys())), (33550, 12, (0.5, 0.5, 0.0)), (33922, 12, (0.0, 0.0, 0.0, 1000.0, 2000.0, 0.0))):
        ifd[tag] = val
        ifd.tagtype[tag] = typ
    return ifd


@pytest.mark.parametrize("compression", ["tiff_adobe_deflate", "tiff_lzw"])
@pytest.mark.parametrize("mode", ["RGB", "L", "RGBA"])
def test_decoder_reads_pil_written_files(tmp_path, compression, mode):
    spp = {"RGB": 3, "L": 1, "RGBA": 4}[mode]
    px = pixels(123, 77, spp, seed=5)
    px[40:60] = 200
    path = str(tmp_path / "pil.tif")
    Image.fromarray(px[..., 0] if spp == 1 else px, mode).save(path, compression=compression, tiffinfo=_pil_geo_info())
    g = GeoTiff(path)
    assert (g.width, g.height, g.spp, g.compression) == (77, 123, spp, 8 if "deflate" in compression else 5)
    assert np.array_equal(g.read_window(0, 123, 0, 77), pil_pixels(path))
    assert np.array_equal(g.read_window(50, 40, 10, 20), pil_pixels(path)[50:90, 10:30])


@pytest.mark.parametrize("comp,layout,damage,text", [
    (8, ("tile", 16, 16), lambda b: b[:len(b) // 2], "tile 3"),
    (8, ("strip", 8), lambda b: b[:-6] + bytes([b[-6] ^ 0xff]) + b[-5:], "strip 3"),
    (5, ("strip", 8), lambda b: b[:3], "strip 3"),
    (5, ("tile", 16, 16), lambda b: b[:2] + b"\xff\xff\xff\xff" + b[6:], "tile 3"),
    (1, ("strip", 8), lambda b: b[:10], "strip 3"),
])
def test_damaged_chunk_is_named(tmp_path, comp, layout, damage, text):
    path = str(tmp_path / "bad.tif")
    kw = dict(compression=comp, corrupt=(3, damage), **GEO_3857)
    if layout[0] == "tile":
        kw["tile"] = layout[1:]
    else:
        kw["rows_per_strip"] = layout[1]
    tw.write_tiff(path, pixels(40, 40, 3), **kw)
    g = GeoTiff(path)
    with pytest.raises(_lib.RsbError, match=text):
        g.read_window(0, 40, 0, 40)
    # a window that does not touch the damaged chunk decodes
    assert g.read_window(0, 8, 0, 16).shape == (8, 16, 3)


def test_lzw_past_table_resets(tmp_path):
    # 200 000 bytes of four symbols need more than 4094 codes, so the stream carries Clear codes mid-strip
    px = np.random.default_rng(3).integers(0, 4, (400, 500, 1), dtype=np.uint8)
    path = tw.write_tiff(str(tmp_path / "l.tif"), px, compression=5, **GEO_3857)
    assert np.array_equal(GeoTiff(path).read_window(0, 400, 0, 500), px)
    assert np.array_equal(pil_pixels(path), px)


# ---- header ----

def test_header_crs_and_georeferencing(tmp_path):
    px = pixels(10, 20, 3)
    for epsg, model, crs in ((3857, 1, "3857"), (4326, 2, "4326"), (32633, 1, ("utm", 33, False)), (32760, 1, ("utm", 60, True)),
                             (32601, 1, ("utm", 1, False))):
        p = tw.write_tiff(str(tmp_path / ("%d.tif" % epsg)), px, geo=tw.geokeys(model, epsg), scale=(2.0, 3.0, 0.0), tiepoint=(1, 2, 0, 100.0, 200.0, 0))
        g = GeoTiff(p)
        assert g.crs == crs and g.epsg == epsg
        c, a, b, f, d, e = g.geotransform
        assert (a, b, d, e) == (2.0, 0.0, 0.0, -3.0) and (c + a * 1, f + e * 2) == (100.0, 200.0)
    # PixelIsPoint: the tiepoint is the centre of pixel (1, 2), so the corner of pixel (0, 0) is 1.5 / 2.5 pixels away
    p = tw.write_tiff(str(tmp_path / "pt.tif"), px, geo=tw.geokeys(raster_type=2), scale=(2.0, 3.0, 0.0), tiepoint=(1, 2, 0, 100.0, 200.0, 0))
    c, a, b, f, d, e = GeoTiff(p).geotransform
    assert (c, f) == (100.0 - 1.5 * 2.0, 200.0 + 2.5 * 3.0)
    # ModelTransformation, with a rotation
    m = (0.5, 0.1, 0, 1000.0, 0.2, -0.5, 0, 2000.0, 0, 0, 0, 0, 0, 0, 0, 1)
    p = tw.write_tiff(str(tmp_path / "m.tif"), px, geo=tw.geokeys(), matrix=m)
    assert GeoTiff(p).geotransform == (1000.0, 0.5, 0.1, 2000.0, 0.2, -0.5)
    p = tw.write_tiff(str(tmp_path / "mp.tif"), px, geo=tw.geokeys(raster_type=2), matrix=m)
    assert GeoTiff(p).geotransform == (1000.0 - 0.5 * 0.6, 0.5, 0.1, 2000.0 - 0.5 * -0.3, 0.2, -0.5)
    # GDAL_NODATA
    for text, value in (("0", 0), ("255", 255), (" 17.0 ", 17), ("-9999", -1), ("nan", -1), ("1.5", -1)):
        p = tw.write_tiff(str(tmp_path / "n.tif"), px, nodata=text, **GEO_3857)
        assert GeoTiff(p).nodata == value, text
    p = tw.write_tiff(str(tmp_path / "a.tif"), pixels(4, 4, 4), **GEO_3857)
    assert GeoTiff(p).alpha and GeoTiff(p).nodata == -1
    # units that are stated and supported
    p = tw.write_tiff(str(tmp_path / "u.tif"), px, geo=tw.geokeys(1, 32633, extra=[(3076, 9001), (2054, 9102)]), scale=(1, 1, 0), tiepoint=(0, 0, 0, 0, 0, 0))
    assert GeoTiff(p).crs == ("utm", 33, False)


REJECTED = [
    ("JPEG", dict(tags={259: (3, [7])}), "Compression 7 \\(JPEG\\)"),
    ("PackBits", dict(tags={259: (3, [32773])}), "Compression 32773"),
    ("planar", dict(tags={284: (3, [2])}), "PlanarConfiguration 2"),
    ("16-bit", dict(tags={258: (3, [16, 16, 16])}), "BitsPerSample 16,16,16"),
    ("signed", dict(tags={339: (3, [2, 2, 2])}), "SampleFormat 2"),
    ("YCbCr", dict(tags={262: (3, [6])}), "Photometric 6 \\(YCbCr\\)"),
    ("predictor3", dict(tags={317: (3, [3])}), "Predictor 3"),
    ("crs", dict(geo=tw.geokeys(1, 27700)), "ProjectedCSTypeGeoKey 27700"),
    ("user-crs", dict(geo=tw.geokeys(1, 32767)), "user-defined"),
    ("geographic", dict(geo=tw.geokeys(2, 4269)), "GeographicTypeGeoKey 4269"),
    ("3857-as-geographic", dict(geo=tw.geokeys(2, 3857)), "GeographicTypeGeoKey 3857"),
    ("feet", dict(geo=tw.geokeys(1, 32633, extra=[(3076, 9002)])), "ProjLinearUnitsGeoKey 9002"),
    ("grads", dict(geo=tw.geokeys(2, 4326, extra=[(2054, 9105)])), "GeogAngularUnitsGeoKey 9105"),
    ("geocentric", dict(geo=tw.geokeys(3, 4978)), "GTModelTypeGeoKey 3"),
    ("no-geokeys", dict(geo=None), "no GeoKeyDirectory"),
    ("two-tiepoints", dict(tiepoint=(0, 0, 0, 1, 2, 0, 5, 5, 0, 3, 4, 0)), "2 tiepoints"),
    ("no-scale", dict(scale=None), "no georeferencing"),
]


@pytest.mark.parametrize("name,kw,text", REJECTED, ids=[r[0] for r in REJECTED])
def test_rejected_headers_are_named(tmp_path, name, kw, text):
    args = dict(GEO_3857)
    args.update(kw)
    p = tw.write_tiff(str(tmp_path / "r.tif"), pixels(8, 8, 3), **args)
    with pytest.raises(_lib.RsbError, match=text):
        GeoTiff(p)


def test_rejected_band_layouts(tmp_path):
    p = tw.write_tiff(str(tmp_path / "pal.tif"), pixels(8, 8, 1), photometric=3, tags={320: (3, [0] * 768)}, **GEO_3857)
    with pytest.raises(_lib.RsbError, match="Photometric 3 \\(palette\\)"):
        GeoTiff(p)
    p = tw.write_tiff(str(tmp_path / "two.tif"), pixels(8, 8, 2), photometric=1, extra_samples=2, **GEO_3857)
    with pytest.raises(_lib.RsbError, match="2 bands"):
        GeoTiff(p)
    p = tw.write_tiff(str(tmp_path / "ex0.tif"), pixels(8, 8, 4), extra_samples=0, **GEO_3857)
    with pytest.raises(_lib.RsbError, match="ExtraSamples \\(0,\\)"):
        GeoTiff(p)
    p = tw.write_tiff(str(tmp_path / "white.tif"), pixels(8, 8, 1), photometric=0, **GEO_3857)
    with pytest.raises(_lib.RsbError, match="MinIsWhite"):
        GeoTiff(p)
    (tmp_path / "x.tif").write_bytes(b"GIF89a....")
    with pytest.raises(_lib.RsbError, match="not a TIFF"):
        GeoTiff(str(tmp_path / "x.tif"))
    p = tw.write_tiff(str(tmp_path / "old.tif"), pixels(8, 8, 3), compression=5, corrupt=(0, lambda b: b"\x00\x01" + b[2:]), **GEO_3857)
    with pytest.raises(_lib.RsbError, match="strip 0.*old-style"):
        GeoTiff(p).read_window(0, 8, 0, 8)


# ---- projections ----

def test_transverse_mercator_matches_epsg_guidance_note_7_2():
    # OSGB 1936 / British National Grid on Airy 1830: 50°30'N 0°30'E -> E 577 274.99, N 69 740.50 (the published figures are rounded
    # and come from a lower-order formula)
    E, N = T.tm_forward(0.5, 50.5, -2.0, k0=0.9996012717, fe=400000.0, fn=-100000.0, lat0=49.0, a=6377563.396, f=1 / 299.3249646)
    assert abs(E - 577274.99) < 0.02 and abs(N - 69740.50) < 0.02


def test_northing_on_the_central_meridian_is_the_meridian_arc():
    from scipy.integrate import quad

    a, f = T.WGS84_A, T.WGS84_F
    e2 = f * (2 - f)
    for lat in (-79.0, -45.5, -10.0, 0.001, 12.0, 47.3, 66.6, 84.0):
        arc = quad(lambda p: a * (1 - e2) / (1 - e2 * math.sin(p) ** 2) ** 1.5, 0, math.radians(lat), epsabs=0, epsrel=1e-13)[0]
        E, N = T.tm_forward(15.0, lat, 15.0)
        assert abs(E - 500000.0) < 1e-9
        assert abs(N - T.UTM_K0 * arc) <= 1e-9 * abs(arc), lat


def test_forward_inverse_round_trip():
    rng = np.random.default_rng(7)
    lat = rng.uniform(-80, 84, 20000)
    lon = 9.0 + rng.uniform(-3.5, 3.5, 20000)
    E, N = T.tm_forward(lon, lat, 9.0)
    lo, la = T.tm_inverse(E, N, 9.0)
    E2, N2 = T.tm_forward(lo, la, 9.0)
    assert np.abs(E2 - E).max() < 1e-6 and np.abs(N2 - N).max() < 1e-6
    Es, Ns = T.tm_forward(lon, lat, 9.0, fn=1e7)
    assert np.array_equal(Ns - 1e7, N) or np.abs(Ns - 1e7 - N).max() < 1e-8


def test_conformal_scale_factors_agree():
    a, f = T.WGS84_A, T.WGS84_F
    e2 = f * (2 - f)
    h = 1e-4  # degrees
    for lat in (-60.0, -20.0, 0.5, 35.0, 70.0):
        for dlon in (-3.0, 0.7, 3.4):
            lon = 21.0 + dlon
            phi = math.radians(lat)
            rho = a * (1 - e2) / (1 - e2 * math.sin(phi) ** 2) ** 1.5
            nu = a / math.sqrt(1 - e2 * math.sin(phi) ** 2)
            En, Nn = T.tm_forward(lon, lat + h, 21.0)
            Es, Ns = T.tm_forward(lon, lat - h, 21.0)
            Ee, Ne = T.tm_forward(lon + h, lat, 21.0)
            Ew, Nw = T.tm_forward(lon - h, lat, 21.0)
            ky = math.hypot(En - Es, Nn - Ns) / (rho * math.radians((lat + h) - (lat - h)))
            kx = math.hypot(Ee - Ew, Ne - Nw) / (nu * math.cos(phi) * math.radians((lon + h) - (lon - h)))
            assert abs(kx - ky) <= 1e-9 * ky, (lat, dlon, kx, ky)


def test_4326_and_3857_agree_with_cover_and_rasterize():
    rng = np.random.default_rng(2)
    lon, lat = rng.uniform(-179, 179, 500), rng.uniform(-85, 85, 500)
    X, Y = T.lonlat_to_mercator(lon, lat)
    assert np.array_equal(np.stack([X, Y], axis=1), project(np.stack([lon, lat], axis=1)))
    for lo, la, x, y in zip(lon, lat, X, Y):
        cx, cy = cover_xy(lo, la)
        assert abs(cx - x) <= 1e-9 * max(1.0, abs(x)) and abs(cy - y) <= 1e-8 * max(1.0, abs(y))
    lo2, la2 = T.model_of_mercator("4326", X, Y)
    assert np.abs(lo2 - lon).max() < 1e-9 and np.abs(la2 - lat).max() < 1e-9
    assert T.model_of_mercator("3857", X, Y) == (X, Y) or np.array_equal(T.model_of_mercator("3857", X, Y)[0], X)


# ---- planning ----

class Raster:
    """the attributes of a GeoTiff that planning reads"""

    def __init__(self, crs, gt, W, H, spp=3, alpha=False, nodata=-1):
        self.crs, self.geotransform, self.width, self.height, self.spp, self.alpha, self.nodata = crs, gt, W, H, spp, alpha, nodata


def utm_raster(zone=32, south=False, W=900, H=700, res=0.6):
    lon0 = 6 * zone - 183
    E, N = T.tm_forward(lon0 + 1.2, -33.0 if south else 47.0, lon0, fn=1e7 if south else 0.0)
    return Raster(("utm", zone, south), (float(E), res, 0.0, float(N), 0.0, -res), W, H)


def rasters():
    return {
        "3857": Raster("3857", (1234567.0, 0.3, 0.0, 6543210.0, 0.0, -0.3), 700, 500),
        "4326": Raster("4326", (10.001, 4e-6, 0.0, 48.002, 0.0, -3e-6), 600, 800),
        "utm": utm_raster(),
        "utm-south": utm_raster(19, True),
        "rotated": Raster("3857", (1234567.0, 0.3, 0.05, 6543210.0, 0.04, -0.3), 400, 300),
    }


@pytest.mark.parametrize("name", ["3857", "4326", "utm", "utm-south", "rotated"])
def test_candidates_equal_a_brute_force_scan(name):
    r = rasters()[name]
    for zoom, size in ((16, 256), (18, 512), (19, 100)):
        got = [tuple(t) for t in T.candidate_tiles(r, zoom, size).tolist()]
        assert got == ref.candidates_brute_force(r, zoom, size)
        assert got == sorted(got) and len(got) > 0


def test_lattice_step_meets_the_bound_on_every_cell():
    # a tall lon/lat raster of fine pixels at a coarse zoom needs a step below 64: latitude is not linear in Mercator Y
    r = Raster("4326", (5.0, 0.01, 0.0, 70.0, 0.0, -0.01), 500, 2000)
    seen = set()
    for name, rr, zoom, size in [(n, x, 18, 512) for n, x in rasters().items()] + [("wide", r, 4, 512), ("wide", r, 6, 256)]:
        tiles = T.candidate_tiles(rr, zoom, size)
        step = T.choose_step(rr, zoom, size, tiles)
        assert step == ref.choose_step(rr, zoom, size, tiles.tolist()), name
        assert all(T.step_error(rr, zoom, size, step, run) <= T.TOLERANCE for run in T.runs(tiles))
        if step < 64:
            assert any(T.step_error(rr, zoom, size, 2 * step, run) > T.TOLERANCE for run in T.runs(tiles))
        seen.add(step)
    assert 64 in seen and len(seen) > 1


@pytest.mark.parametrize("name", ["3857", "4326", "utm", "rotated"])
@pytest.mark.parametrize("tiny", [False, True])
def test_windows_cover_every_reachable_sample(name, tiny):
    r = rasters()[name]
    zoom, size = 18, 128
    tiles = T.candidate_tiles(r, zoom, size)
    step = T.choose_step(r, zoom, size, tiles)
    # tiny: the budget of the costliest single tile, so that most windows hold one tile
    budget = max(w.device_bytes(r, size) for w in T.plan(r, zoom, size, tiles, step, batch=1)) if tiny else None
    windows = T.plan(r, zoom, size, tiles, step, budget=budget or T.DEFAULT_BUDGET, batch=7)
    assert all(len(w.xs) <= 7 for w in windows)
    if budget:
        assert all(w.device_bytes(r, size) <= budget for w in windows) and len(windows) > len(T.runs(tiles))
    placed = set()
    for w in windows:
        assert w.xs == list(range(w.xs[0], w.xs[-1] + 1))
        for x in w.xs:
            assert (x, w.y) not in placed
            placed.add((x, w.y))
            kx0, ky0, n = ref.tile_nodes(r, zoom, size, step, x, w.y)
            # the window's lattice holds this tile's nodes, bit for bit
            sub = w.nodes[ky0 - w.ky0:ky0 - w.ky0 + n.shape[0], kx0 - w.kx0:kx0 - w.kx0 + n.shape[1]]
            assert np.array_equal(sub, n, equal_nan=True)
            gx = x * size + np.arange(size)
            gy = w.y * size + np.arange(size)
            FX, FY = np.meshgrid((gx % step) / step, (gy % step) / step)
            IX, IY = np.meshgrid(gx // step - kx0, gy // step - ky0)
            u = ref._lerp(ref._lerp(n[IY, IX, 0], n[IY, IX + 1, 0], FX), ref._lerp(n[IY + 1, IX, 0], n[IY + 1, IX + 1, 0], FX), FY)
            v = ref._lerp(ref._lerp(n[IY, IX, 1], n[IY, IX + 1, 1], FX), ref._lerp(n[IY + 1, IX, 1], n[IY + 1, IX + 1, 1], FX), FY)
            inside = (u >= 0) & (u < r.width) & (v >= 0) & (v < r.height)
            # every tap of both resamplings, clamped to the raster, lies in the window
            for du in (-0.5, 0.0, 0.5):
                for dv in (-0.5, 0.0, 0.5):
                    i = np.clip(np.floor(u[inside] + du), 0, r.width - 1)
                    j = np.clip(np.floor(v[inside] + dv), 0, r.height - 1)
                    assert (i >= w.col0).all() and (i < w.col0 + w.cols).all() and (j >= w.row0).all() and (j < w.row0 + w.rows).all()
    # tiles left out of every window sample nothing
    for x, y in set(map(tuple, tiles.tolist())) - placed:
        _, _, n = ref.tile_nodes(r, zoom, size, step, x, y)
        assert T.source_box(n, r) is None


def test_a_tile_over_the_budget_is_refused_before_any_allocation():
    r = rasters()["3857"]
    tiles = T.candidate_tiles(r, 18, 512)
    with pytest.raises(_lib.RsbError, match="more than the budget"):
        T.plan(r, 18, 512, tiles, 64, budget=1000)


# ---- ABI and tool ----

def test_abi_validates_before_the_device_check():
    import torch

    lib = _lib.load()
    buf = (ctypes.c_uint8 * 64)()
    nodes = np.zeros(64, np.float64)
    tiles = np.zeros(2, np.int64)
    base = [ctypes.addressof(buf), 30, 0, 0, 10, 10, 10, 10, 3, 0, -1, nodes.ctypes.data, 0, 0, 2, 2, 64, tiles.ctypes.data, 1, 4, 1,
            ctypes.addressof(buf), 48, ctypes.addressof(buf), ctypes.addressof(buf), None]
    for k, bad in ((8, 2), (9, 1), (10, 256), (16, 48), (16, 128), (18, 0), (19, 0), (19, 4097), (20, 2), (22, 47), (1, 29), (4, 11), (0, None)):
        args = list(base)
        args[k] = bad
        assert lib.rsb_tile_warp(*args) == -1, (k, bad)
    if not torch.cuda.is_available():
        assert lib.rsb_tile_warp(*base) == -3
    out = (ctypes.c_uint8 * 16)()
    off, cnt = np.zeros(1, np.int64), np.zeros(1, np.int64)
    args = [ctypes.addressof(buf), 64, off.ctypes.data, cnt.ctypes.data, 1, 4, 4, 4, 4, 0, 1, 1, 1, 0, 4, 0, 4, ctypes.addressof(out), 1, None]
    assert lib.rsb_tiff_decode_window(*args) == -1  # chunk_w != width for strips
    args[7], args[8] = 4, 4
    args[10] = 2
    assert lib.rsb_tiff_decode_window(*args) == -1
    args[10], args[11] = 1, 7
    assert lib.rsb_tiff_decode_window(*args) == -1
    args[11], args[13] = 1, 1
    assert lib.rsb_tiff_decode_window(*args) == -1  # the window leaves the raster


def _parse(argv):
    from robosat_b200.tools import tile

    parser = argparse.ArgumentParser()
    sub = parser.add_subparsers()
    tile.add_parser(sub)
    return parser.parse_args(argv)


def test_parser():
    a = _parse(["tile", "--zoom", "19", "ortho.tif", "out"])
    assert (a.zoom, a.size, a.tiles, a.resampling, a.raster, a.out) == (19, 512, None, "bilinear", "ortho.tif", "out")
    a = _parse(["tile", "--zoom", "3", "--size", "256", "--tiles", "t.csv", "--resampling", "nearest", "r.tif", "o"])
    assert (a.size, a.tiles, a.resampling) == (256, "t.csv", "nearest")
    with pytest.raises(SystemExit):
        _parse(["tile", "--zoom", "3", "--resampling", "cubic", "r.tif", "o"])
    from robosat_b200.tools import __main__ as M

    assert "tile" in open(M.__file__).read()


def test_tool_refusals(tmp_path, monkeypatch):
    import torch

    from robosat_b200.tools import tile

    csv = tmp_path / "t.csv"
    csv.write_text("1,2,19\n3,4,18\n")
    with pytest.raises(SystemExit, match="row 2 is tile \\(3, 4, 18\\), not at --zoom 19"):
        tile.main(_parse(["tile", "--zoom", "19", "--tiles", str(csv), "r.tif", str(tmp_path)]))
    with pytest.raises(SystemExit, match="--size"):
        tile.main(_parse(["tile", "--zoom", "19", "--size", "0", "r.tif", str(tmp_path)]))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit, match="^Error: CUDA requested but not available$"):
        tile.main(_parse(["tile", "--zoom", "19", "r.tif", str(tmp_path)]))
