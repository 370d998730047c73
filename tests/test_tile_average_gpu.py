"""rsb_tile_average, `rs tile --resampling average` and `rs segment --resampling average` on the H100: tiles and covered counts
bit-identical to the numpy restatement (tests/tile_average_reference.py) for every CRS at ratios below 1, around 2.6, 5.3 and 10,
1/3/4 bands with nodata or alpha, ragged rasters, batches of 1, 7 and 64 and a one-tile budget; an aligned raster comes back as its
pixels at ratio 1 and as block means at 2, 4 and 8; a checkerboard averages to grey where bilinear does not; the tools' outputs; and
a footprint over the cap stops both tools before any launch."""

import argparse
import os

import numpy as np
import pytest
from PIL import Image

import tiff_writer as tw
import tile_average_reference as ref
from robosat_b200 import mosaic as M
from robosat_b200 import segment as SEG
from robosat_b200 import stitch
from robosat_b200 import tile as T
from robosat_b200.geotiff import GeoTiff
from robosat_b200.rasterize import CE
from test_segment_gpu import fused, pipeline, read, setup
from test_tile_average import aligned_raster, check_block_means
from test_tile_gpu import georef, noise, write

pytestmark = pytest.mark.gpu

SIZE = 128
ZOOMS = {"below-1": 20, "2.6": 18, "5.3": 17, "10": 16}  # source pixels per tile pixel of the 0.45 m EPSG:3857 raster at 128² tiles


def check_against_reference(g, zoom, size=SIZE, **kw):
    stats = {}
    got = T.tile_device(g, zoom, size, "average", stats=stats, **kw)
    cand = T.candidate_tiles(g, zoom, size)
    want, step = ref.render(g.read_window(0, g.height, 0, g.width), g, zoom, size, cand.tolist())
    assert stats["step"] == step
    assert sorted(got) == sorted(want) and len(got) > 0
    for k in want:
        assert got[k][1] == want[k][1], k
        assert np.array_equal(got[k][0], want[k][0]), (k, int((got[k][0] != want[k][0]).any(axis=-1).sum()))
    return got


@pytest.mark.parametrize("kind", ["3857", "4326", "utm", "utm-south", "rotated"])
@pytest.mark.parametrize("ratio", list(ZOOMS))
def test_restatement_per_crs_and_ratio(tmp_path, cuda_device, kind, ratio):
    g = write(tmp_path, kind, noise(237, 301, 3, 1), kind)
    check_against_reference(g, ZOOMS[ratio])


@pytest.mark.parametrize("bands", ["gray-nodata", "rgb-nodata", "rgba"])
@pytest.mark.parametrize("zoom", [18, 17])
def test_restatement_bands_alpha_and_nodata(tmp_path, cuda_device, bands, zoom):
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
    got = check_against_reference(g, zoom)
    assert any(c < SIZE * SIZE for _, c in got.values())


@pytest.mark.parametrize("batch", [1, 7, 64])
def test_batches_tiny_budget_and_repeats(tmp_path, cuda_device, batch):
    # a long, thin ragged raster: 80-odd tiles of 32 px per tile row at zoom 22, straddling the raster edges
    z = 22
    g = write(tmp_path, "long", noise(83, 1501, 3, 3), "4326")
    base = check_against_reference(g, z, size=32, batch=batch)
    again = T.tile_device(g, z, 32, "average", batch=batch)
    assert sorted(again) == sorted(base) and all(np.array_equal(again[k][0], base[k][0]) for k in base)
    cand = T.candidate_tiles(g, z, 32)
    step = T.choose_step(g, z, 32, cand, corner=True)
    assert max(len(w.xs) for w in T.plan(g, z, 32, cand, step, batch=batch, corner=True)) == batch
    tiny = max(w.device_bytes(g, 32) for w in T.plan(g, z, 32, cand, step, batch=1, corner=True))
    stats = {}
    small = T.tile_device(g, z, 32, "average", budget=tiny, batch=batch, stats=stats)
    assert stats["windows"] >= len(base) // 2
    assert sorted(small) == sorted(base) and all(np.array_equal(small[k][0], base[k][0]) and small[k][1] == base[k][1] for k in base)


def aligned_tiff(tmp_path, px, r):
    c, a, _, f, _, e = r.geotransform
    return GeoTiff(tw.write_tiff(str(tmp_path / "al.tif"), px, geo=tw.geokeys(), scale=(a, -e, 0.0), tiepoint=(0, 0, 0, c, f, 0), rows_per_strip=16))


def test_aligned_raster_at_ratio_1_comes_back_as_its_pixel_slices(tmp_path, cuda_device):
    z, S = 17, 64
    x0, y0 = 68500, 45300
    r = aligned_raster(z, S, 1, 3, 2, x0, y0)
    px = noise(r.height, r.width, 3, 4)
    got = T.tile_device(aligned_tiff(tmp_path, px, r), z, S, "average")
    inner = [(x0 + i, y0 + j) for i in range(3) for j in range(2)]
    assert set(inner) <= set(got)
    for (x, y), (im, count) in got.items():
        if (x, y) in inner:
            i, j = x - x0, y - y0
            assert count == S * S and np.array_equal(im, px[j * S:(j + 1) * S, i * S:(i + 1) * S])
        else:  # a neighbour may catch a sliver of the raster's edge (the rounding of the corners): only in its row or column next to it
            rows, cols = np.nonzero(im.any(axis=-1))
            assert set(rows.tolist()) <= {0, S - 1} or set(cols.tolist()) <= {0, S - 1}, (x, y)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_aligned_raster_gives_block_means(tmp_path, cuda_device, k):
    z, S = 17, 64
    r = aligned_raster(z, S, k)
    px = noise(r.height, r.width, 3, k)
    got = T.tile_device(aligned_tiff(tmp_path, px, r), z, S, "average")
    for dx in (0, 1):
        for dy in (0, 1):
            im, count = got[(68500 + dx, 45300 + dy)]
            assert count == S * S
            check_block_means(im, px[dy * S * k:(dy + 1) * S * k, dx * S * k:(dx + 1) * S * k], k, S)


def test_checkerboard_averages_to_grey(tmp_path, cuda_device):
    """a 1-px checkerboard at 4 source pixels per tile pixel: every fully covered pixel is 127 or 128, bilinear is not. The raster is
    shifted by a quarter source pixel: on the exact alignment bilinear samples at pixel corners and averages 2 x 2 too."""
    z, S, k = 17, 64, 4
    r = aligned_raster(z, S, k)
    c, a, b, f, d, e = r.geotransform
    r.geotransform = (c + a / 4, a, b, f + e / 4, d, e)
    yy, xx = np.mgrid[0:r.height, 0:r.width]
    px = np.repeat((((xx + yy) % 2) * 255).astype(np.uint8)[..., None], 3, axis=-1)
    g = aligned_tiff(tmp_path, px, r)
    avg = T.tile_device(g, z, S, "average")
    bil = T.tile_device(g, z, S, "bilinear")
    step = T.choose_step(g, z, S, np.array(sorted(avg)), corner=True)
    full = 0
    for key, (im, _) in avg.items():
        u0, u1, v0, v1, nan = ref.footprints(ref.corners(g, z, S, step, *key))
        inside = ~nan & (u0 >= 0) & (u1 <= g.width) & (v0 >= 0) & (v1 <= g.height)
        if not inside.any():
            continue
        assert np.isin(im[inside], (127, 128)).all(), key
        assert not np.isin(bil[key][0][inside], (127, 128)).any(), key
        full += int(inside.sum())
    assert full >= 3 * S * S


def test_tool_end_to_end(tmp_path, cuda_device, capsys):
    from robosat_b200.tools import tile as tool

    px = noise(600, 820, 3, 5)
    g = GeoTiff(tw.write_tiff(str(tmp_path / "ortho.tif"), px, compression=8, tile=(128, 64), predictor=2, **georef("utm")))
    z, S = 17, 128
    assert T.coarse_ratio(g, z, S) > 2
    want = T.tile_device(g, z, S, "average")
    out = tmp_path / "out"
    stats = {}
    tool.main(argparse.Namespace(zoom=z, size=S, tiles=None, resampling="average", raster=str(tmp_path / "ortho.tif"), out=str(out)), stats)
    assert "aliases" not in capsys.readouterr().err
    files = sorted((int(x), int(os.path.splitext(y)[0])) for x in os.listdir(out / str(z)) for y in os.listdir(out / str(z) / x))
    assert files == sorted(want) and stats["written"] == len(want) and len(want) > 1
    for (x, y), (im, _) in want.items():
        path = str(out / str(z) / str(x) / ("%d.png" % y))
        assert np.array_equal(np.array(Image.open(path).convert("RGB")), im)
        assert np.array_equal(stitch.decode_rgb(path, S), im)
    tool.main(argparse.Namespace(zoom=z, size=S, tiles=None, resampling="bilinear", raster=str(tmp_path / "ortho.tif"), out=str(tmp_path / "b")))
    assert "use --resampling average" in capsys.readouterr().err


@pytest.mark.parametrize("case", ["masks-utm", "rotated-budget-at-peak"])
def test_segment_equals_the_four_tool_pipeline(tmp_path, cuda_device, monkeypatch, case):
    monkeypatch.setenv("RSB_GPUS", "1")
    monkeypatch.setenv("RSB_QUIET", "1")
    kind = "utm" if case == "masks-utm" else "rotated"
    setup(tmp_path, 2, kind)
    raster = GeoTiff(str(tmp_path / "ortho.tif"))
    grid = M.Grid(raster.width, raster.height, raster.crs, raster.geotransform)
    plan = SEG.plan(raster, grid, 18, 256, 4, None, resampling="average")
    assert plan.corner and 10 <= len(plan.tiles) <= 40
    budget = plan.store_bytes if case == "rotated-budget-at-peak" else None
    written = pipeline(tmp_path, 2, "masks", "average", "none", None, None)
    stats = fused(tmp_path, "masks", "average", "none", None, None, budget)
    want, mode_w, tags_w = read(tmp_path / "pipeline.tif")
    got, mode_g, tags_g = read(tmp_path / "fused.tif")
    assert mode_g == mode_w == "P" and got.shape == want.shape == (raster.height, raster.width)
    assert tags_g == tags_w
    diff = np.argwhere(got != want)
    assert len(diff) == 0, (len(diff), diff[:5].tolist())
    assert stats["existing"] == stats["predicted"] == written


def test_a_footprint_over_the_cap_stops_both_tools_before_any_launch(tmp_path, cuda_device, monkeypatch):
    from robosat_b200.tools import tile as tool

    def no_launch(*a, **k):
        raise AssertionError("a warp was launched")

    monkeypatch.setattr(T, "warp", no_launch)
    setup(tmp_path, 2, "3857")  # 0.45 m pixels: a zoom-12 pixel of 256² tiles spans about 85 of them
    z = 12
    with pytest.raises(SystemExit, match="may span .* source pixels, more than the 64 .* higher zoom"):
        tool.main(argparse.Namespace(zoom=z, size=256, tiles=None, resampling="average", raster=str(tmp_path / "ortho.tif"), out=str(tmp_path / "images")))
    assert not os.path.exists(tmp_path / "images")
    monkeypatch.setattr("test_segment_gpu.ZOOM", z)
    with pytest.raises(SystemExit, match="may span"):
        fused(tmp_path, "masks", "average", "none", None, None)
    assert not os.path.exists(tmp_path / "fused.tif") and not [f for f in os.listdir(tmp_path) if f.endswith(".tmp")]
