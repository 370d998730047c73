"""rsb_tile_warp and `rs tile` on the H100: output tiles and covered counts bit-identical to the numpy restatement
(tests/tile_reference.py) for every CRS, both resamplings, 1/3/4 bands with alpha and nodata, ragged rasters, batches of 1, 7 and 64
tiles and a tiny budget; a raster aligned to the tile grid comes back as its pixel slices; analytically drawn 4326 and UTM rasters
agree with `rs rasterize` of the same polygons; and the tool writes the expected PNGs."""

import argparse
import math
import os

import numpy as np
import pytest
from PIL import Image

import tile_reference as ref
import tiff_writer as tw
from robosat_b200 import stitch
from robosat_b200 import tile as T
from robosat_b200.geotiff import GeoTiff
from robosat_b200.rasterize import CE, PolygonSet, rasterize_device

pytestmark = pytest.mark.gpu

ZOOM, SIZE = 18, 128


def utm_origin(zone, south, lon, lat):
    E, N = T.tm_forward(lon, lat, 6 * zone - 183, fn=1e7 if south else 0.0)
    return float(E), float(N)


def georef(kind):
    """write_tiff keyword arguments placing a raster near (10 E, 48 N) or (-69 E, 33 S)"""
    if kind == "3857":
        return dict(geo=tw.geokeys(), scale=(0.45, 0.45, 0.0), tiepoint=(0, 0, 0, 1113312.7, 6106910.3, 0))
    if kind == "4326":
        return dict(geo=tw.geokeys(2, 4326), scale=(5e-6, 3.5e-6, 0.0), tiepoint=(0, 0, 0, 10.00031, 48.00042, 0))
    if kind == "utm":
        E, N = utm_origin(32, False, 10.2, 47.3)
        return dict(geo=tw.geokeys(1, 32632), scale=(0.4, 0.4, 0.0), tiepoint=(0, 0, 0, E, N, 0))
    if kind == "utm-south":
        E, N = utm_origin(19, True, -69.4, -33.1)
        return dict(geo=tw.geokeys(1, 32719), scale=(0.5, 0.5, 0.0), tiepoint=(0, 0, 0, E, N, 0))
    if kind == "rotated":
        return dict(geo=tw.geokeys(raster_type=2), matrix=(0.4, 0.07, 0, 1113312.7, 0.05, -0.4, 0, 6106910.3, 0, 0, 0, 0, 0, 0, 0, 1))
    raise ValueError(kind)


def noise(H, W, spp, seed):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (H // 8 + 2, W // 8 + 2, spp), dtype=np.uint8)
    smooth = np.repeat(np.repeat(base, 8, 0), 8, 1)[:H, :W].astype(np.int16)  # blocks, so that bilinear mixes distinct values
    return np.clip(smooth + rng.integers(-20, 21, (H, W, spp)), 0, 255).astype(np.uint8)


def write(tmp_path, name, px, kind, **kw):
    return GeoTiff(tw.write_tiff(str(tmp_path / (name + ".tif")), px, compression=8, tile=(64, 32), predictor=2, **georef(kind), **kw))


def check_against_reference(g, resampling, zoom=ZOOM, size=SIZE, **kw):
    stats = {}
    got = T.tile_device(g, zoom, size, resampling, stats=stats, **kw)
    cand = T.candidate_tiles(g, zoom, size)
    want, step = ref.render(g.read_window(0, g.height, 0, g.width), g, zoom, size, cand.tolist(), resampling)
    assert stats["step"] == step
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k][1] == want[k][1], k
        assert np.array_equal(got[k][0], want[k][0]), (k, int((got[k][0] != want[k][0]).any(axis=-1).sum()))
    assert len(got) > 1
    return got


@pytest.mark.parametrize("kind", ["3857", "4326", "utm", "utm-south", "rotated"])
@pytest.mark.parametrize("resampling", ["nearest", "bilinear"])
def test_restatement_per_crs(tmp_path, cuda_device, kind, resampling):
    g = write(tmp_path, kind, noise(237, 301, 3, 1), kind)
    check_against_reference(g, resampling)


@pytest.mark.parametrize("bands", ["gray-nodata", "rgb-nodata", "rgba"])
@pytest.mark.parametrize("resampling", ["nearest", "bilinear"])
def test_restatement_bands_alpha_and_nodata(tmp_path, cuda_device, bands, resampling):
    spp = {"gray-nodata": 1, "rgb-nodata": 3, "rgba": 4}[bands]
    px = noise(199, 257, spp, 2)
    kw = {}
    if bands == "rgba":
        px[..., 3] = 255
        px[40:90, 30:200, 3] = 0
        px[::7, ::5, 3] = 0
    else:
        px[50:80, 60:150] = 0  # a nodata hole
        px[::9, ::4] = 0
        kw["nodata"] = "0"
    g = write(tmp_path, bands, px, "utm", **kw)
    got = check_against_reference(g, resampling)
    assert any(c < SIZE * SIZE for _, c in got.values())


@pytest.mark.parametrize("batch", [1, 7, 64])
def test_batches_tiny_budget_and_repeats(tmp_path, cuda_device, batch):
    # a long, thin ragged raster: 80-odd tiles of 32 px per tile row at zoom 22, straddling the raster edges
    z = 22
    g = write(tmp_path, "long", noise(83, 1501, 3, 3), "4326")
    base = check_against_reference(g, "bilinear", zoom=z, size=32, batch=batch)
    again = T.tile_device(g, z, 32, "bilinear", batch=batch)
    assert sorted(again) == sorted(base) and all(np.array_equal(again[k][0], base[k][0]) for k in base)
    cand = T.candidate_tiles(g, z, 32)
    assert max(len(w.xs) for w in T.plan(g, z, 32, cand, T.choose_step(g, z, 32, cand), batch=batch)) == batch
    step = T.choose_step(g, z, 32, cand)
    tiny = max(w.device_bytes(g, 32) for w in T.plan(g, z, 32, cand, step, batch=1))
    stats = {}
    small = T.tile_device(g, z, 32, "bilinear", budget=tiny, batch=batch, stats=stats)
    assert stats["windows"] >= len(base) // 2
    assert sorted(small) == sorted(base) and all(np.array_equal(small[k][0], base[k][0]) and small[k][1] == base[k][1] for k in base)


@pytest.mark.parametrize("resampling", ["nearest", "bilinear"])
def test_aligned_raster_comes_back_as_its_pixel_slices(tmp_path, cuda_device, resampling):
    z, S = 17, 64
    x0, y0 = 68500, 45300
    px_size = CE / (2 ** z * S)
    left, top = x0 * CE / 2 ** z - CE / 2, CE / 2 - y0 * CE / 2 ** z
    H, W = 2 * S + 5, 3 * S + 10
    px = noise(H, W, 3, 4)
    g = GeoTiff(tw.write_tiff(str(tmp_path / "al.tif"), px, geo=tw.geokeys(), scale=(px_size, px_size, 0.0), tiepoint=(0, 0, 0, left, top, 0),
                              rows_per_strip=16))
    got = T.tile_device(g, z, S, resampling)
    assert sorted(got) == [(x0 + i, y0 + j) for i in range(4) for j in range(3)]
    for (x, y), (im, count) in got.items():
        i, j = x - x0, y - y0
        part = px[j * S:(j + 1) * S, i * S:(i + 1) * S]
        assert count == part.shape[0] * part.shape[1]
        assert np.array_equal(im[:part.shape[0], :part.shape[1]], part)
        assert not im[part.shape[0]:].any() and not im[:, part.shape[1]:].any()


def _polygons(rng, lon0, lat0, dlon, dlat, n=6):
    """seeded convex polygons (lon, lat rings) inside the box [lon0, lon0 + dlon] x [lat0 - dlat, lat0]"""
    polys = []
    for _ in range(n):
        cx, cy = lon0 + rng.uniform(0.2, 0.8) * dlon, lat0 - rng.uniform(0.2, 0.8) * dlat
        r = rng.uniform(0.06, 0.14) * min(dlon, dlat)
        a = np.sort(rng.uniform(0, 2 * np.pi, rng.integers(3, 8)))
        ring = [(cx + r * math.cos(t) * dlon / min(dlon, dlat), cy + r * math.sin(t) * dlat / min(dlon, dlat)) for t in a]
        polys.append(ring + [ring[0]])
    return polys


def _inside(lon, lat, polys):
    inside = np.zeros(lon.shape, bool)
    for ring in polys:
        p = np.asarray(ring)
        odd = np.zeros(lon.shape, bool)
        for (x1, y1), (x2, y2) in zip(p[:-1], p[1:]):
            cross = (y1 > lat) != (y2 > lat)
            with np.errstate(divide="ignore", invalid="ignore"):
                xc = x1 + (lat - y1) * (x2 - x1) / (y2 - y1)
            odd ^= cross & (lon < xc)
        inside |= odd
    return inside


def _segment_distance(P, A, B):
    d = B - A
    t = np.clip(((P - A) @ d) / (d @ d), 0, 1)
    return np.hypot(*(P - (A + t[:, None] * d)).T)


@pytest.mark.parametrize("kind", ["4326", "utm"])
def test_georeferencing_agrees_with_rasterize(tmp_path, cuda_device, kind):
    z, S = 19, 256
    H, W = 700, 900
    kw = georef(kind)
    g0 = GeoTiff(tw.write_tiff(str(tmp_path / "probe.tif"), np.zeros((H, W, 1), np.uint8), **kw))
    c, a, b, f, d, e = g0.geotransform
    jj, ii = np.mgrid[0:H, 0:W] + 0.5
    mx, my = c + a * ii + b * jj, f + d * ii + e * jj
    if kind == "4326":
        lon, lat = mx, my
    else:
        lon, lat = T.tm_inverse(mx, my, 6 * 32 - 183)
    rng = np.random.default_rng(11)
    polys = _polygons(rng, lon.min(), lat.max(), lon.max() - lon.min(), lat.max() - lat.min())
    white = np.where(_inside(lon, lat, polys), 255, 0).astype(np.uint8)
    g = GeoTiff(tw.write_tiff(str(tmp_path / "poly.tif"), white[..., None], compression=8, tile=(128, 128), **kw))
    got = T.tile_device(g, z, S, "nearest")
    tiles = sorted(got)
    merc = [[np.stack(T.lonlat_to_mercator(np.asarray(r)[:, 0], np.asarray(r)[:, 1]), axis=1)] for r in polys]
    masks, _ = rasterize_device(PolygonSet(merc, cuda_device), [(x, y, z) for x, y in tiles], S)
    masks = masks.cpu().numpy()
    # one source pixel in Mercator metres at the raster centre (the longer side)
    X0, Y0 = T.mercator_of_model(g.crs, np.array([c + a * W / 2, c + a * (W / 2 + 1), c + a * W / 2 + b]),
                                 np.array([f + e * H / 2, f + e * H / 2 + d, f + e * (H / 2 + 1)]))
    src_px = max(math.hypot(X0[1] - X0[0], Y0[1] - Y0[0]), math.hypot(X0[2] - X0[0], Y0[2] - Y0[0]))
    edges = [(np.asarray(m[0][k]), np.asarray(m[0][k + 1])) for m in merc for k in range(len(m[0]) - 1)]
    inter = union = 0
    px = CE / (2 ** z * S)
    for n, (x, y) in enumerate(tiles):
        mine = got[(x, y)][0][..., 0] == 255
        theirs = masks[n] == 1
        inter += int((mine & theirs).sum())
        union += int((mine | theirs).sum())
        rr, cc = np.nonzero(mine != theirs)
        if len(rr):
            P = np.stack([-CE / 2 + (x * S + cc + 0.5) * px, CE / 2 - (y * S + rr + 0.5) * px], axis=1)
            dist = np.min([_segment_distance(P, A, B) for A, B in edges], axis=0)
            assert dist.max() <= src_px, (x, y, dist.max(), src_px)
    assert union > 0 and inter / union >= 0.98, inter / union


def test_tool_end_to_end(tmp_path, cuda_device, capsys):
    from robosat_b200.tools import tile as tool

    px = noise(300, 410, 3, 5)
    g = GeoTiff(tw.write_tiff(str(tmp_path / "ortho.tif"), px, compression=8, tile=(128, 64), predictor=2, **georef("utm")))
    want = T.tile_device(g, 19, 256, "bilinear")
    out = tmp_path / "out"
    stale = out / "19" / str(sorted(want)[0][0]) / ("%d.png" % sorted(want)[0][1])
    os.makedirs(stale.parent)
    stale.write_bytes(b"old")
    args = argparse.Namespace(zoom=19, size=256, tiles=None, resampling="bilinear", raster=str(tmp_path / "ortho.tif"), out=str(out))
    stats = {}
    tool.main(args, stats)
    files = sorted((int(x), int(os.path.splitext(y)[0])) for x in os.listdir(out / "19") for y in os.listdir(out / "19" / x))
    assert files == sorted(want) and stats["written"] == len(want)
    for (x, y), (im, _) in want.items():
        path = str(out / "19" / str(x) / ("%d.png" % y))
        assert np.array_equal(np.array(Image.open(path).convert("RGB")), im)
        assert np.array_equal(stitch.decode_rgb(path, 256), im)
    # --tiles: a listed tile outside the raster is reported once, the others are written
    keep = sorted(want)[:2]
    csv = tmp_path / "t.csv"
    csv.write_text("".join("%d,%d,19\n" % t for t in keep) + "1,1,19\n")
    out2 = tmp_path / "out2"
    tool.main(argparse.Namespace(zoom=19, size=256, tiles=str(csv), resampling="bilinear", raster=str(tmp_path / "ortho.tif"), out=str(out2)))
    files = sorted((int(x), int(os.path.splitext(y)[0])) for x in os.listdir(out2 / "19") for y in os.listdir(out2 / "19" / x))
    assert files == keep
    err = capsys.readouterr().err
    assert err.count("1 of the 3 listed tiles have no pixel inside the raster") == 1
