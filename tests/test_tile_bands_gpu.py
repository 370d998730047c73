"""The band rule on the H100 (DESIGN.md §8): rsb_tile_render bit-identical to the restatement (tests/tile_bands_reference.py) and
rsb_band_histogram equal to np.bincount, at ragged window sizes, 8 and 16 bits, k = 1..4, with nodata and alpha, over windows fed in
several launches; `rs tile` under --bands / --scale bit-identical to the restatement (render, then the plain rule of the RGBA raster)
for 3857, 4326 and UTM, nearest, bilinear and average, 16-bit with 3 and 4 bands and planar rasters; the identity property on 8-bit
1/3/4-band rasters; `--stretch` printing a --scale that reproduces its tiles; and `rs segment` under the band rule equal to
`rs tile → rs predict → rs masks → rs mosaic --like` with the same options."""

import argparse
import os
import re

import numpy as np
import pytest
import torch

import tiff_bands_writer as bw
import tile_average_reference as aref
import tile_bands_reference as ref
import tile_reference as pref
from robosat_b200 import _lib
from robosat_b200 import tile as T
from robosat_b200.geotiff import GeoTiff, open_bands
from test_segment_gpu import BATCH, OVERLAP, read, setup
from test_tile_gpu import georef, noise, write

pytestmark = pytest.mark.gpu

SIZE = 128
ZOOMS = {"nearest": 18, "bilinear": 18, "average": 17}


def smooth16(H, W, spp, seed, lo=800, hi=9000):
    """16-bit imagery: blocks plus noise, within lo..hi"""
    rng = np.random.default_rng(seed)
    base = rng.integers(lo, hi, (H // 8 + 2, W // 8 + 2, spp))
    px = np.repeat(np.repeat(base, 8, 0), 8, 1)[:H, :W] + rng.integers(-300, 301, (H, W, spp))
    return np.clip(px, 0, 65535).astype(np.uint16)


# ---- kernels ----

def _window(rows, cols, k, bits, seed, smooth=False):
    rng = np.random.default_rng(seed)
    top = (1 << bits) - 1
    if smooth:
        raw = np.full((rows, cols, k), top // 3, np.int64) + rng.integers(0, 3, (rows, cols, k))
    else:
        raw = rng.integers(0, top + 1, (rows, cols, k))
    raw = raw.astype(np.uint8 if bits == 8 else np.uint16)
    raw[::5, ::3, :k - (k in (2, 4))] = 17  # nodata pixels
    if k in (2, 4):
        raw[::4, ::2, -1] = 0  # alpha 0
    return raw


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_render_and_histogram_equal_the_restatement(cuda_device, bits, k):
    lib = _lib.load()
    nsel, alpha = (1 if k < 3 else 3), int(k in (2, 4))
    top = (1 << bits) - 1
    scale = [(0, top), (17, 18), (5, top // 2)][:nsel] if nsel == 3 else [(3, top - 7)]
    for rows, cols in ((1, 1), (1, 3), (3, 5), (37, 101), (200, 333), (64, 1024)):
        for nodata in (-1, 17):
            for smooth in (False, True):
                raw = _window(rows, cols, k, bits, rows * cols + k, smooth)
                src = torch.from_numpy(raw.reshape(-1).view(np.uint8).copy()).to(cuda_device)
                pitch = cols * 4 + 8
                out = torch.full((rows * pitch,), 0xAB, dtype=torch.uint8, device=cuda_device)
                sc = np.asarray(scale, np.int32).reshape(-1)
                _lib.check(lib.rsb_tile_render(src.data_ptr(), rows, cols, bits, nsel, alpha, nodata, sc.ctypes.data, out.data_ptr(), pitch,
                                               _lib.current_stream_ptr()), "rsb_tile_render")
                got = out.cpu().numpy().reshape(rows, pitch)
                assert np.array_equal(got[:, :cols * 4].reshape(rows, cols, 4), ref.render(raw, nsel, alpha, nodata, scale)), (rows, cols, nodata)
                assert (got[:, cols * 4:] == 0xAB).all()  # nothing past the row
                # the histogram, accumulated over the window fed in up to three launches of row bands
                hist = torch.zeros((nsel, 1 << bits), dtype=torch.int64, device=cuda_device)
                cuts = sorted({0, rows // 3, (2 * rows) // 3, rows})
                row_bytes = cols * k * (bits // 8)
                for a, b in zip(cuts[:-1], cuts[1:]):
                    part = torch.from_numpy(raw[a:b].reshape(-1).view(np.uint8).copy()).to(cuda_device)
                    assert part.data_ptr() % 16 == 0 and part.numel() == (b - a) * row_bytes
                    _lib.check(lib.rsb_band_histogram(part.data_ptr(), b - a, cols, bits, nsel, alpha, nodata, hist.data_ptr(),
                                                      _lib.current_stream_ptr()), "rsb_band_histogram")
                assert np.array_equal(hist.cpu().numpy(), ref.histogram(raw, nsel, alpha, nodata, bits)), (rows, cols, nodata, smooth)


# ---- rs tile ----

def check_band_raster(g, resampling, zoom=None, size=SIZE):
    zoom = zoom or ZOOMS[resampling]
    stats = {}
    got = T.tile_device(g, zoom, size, resampling, stats=stats)
    rgba, proxy = ref.rgba_of(g)
    cand = T.candidate_tiles(g, zoom, size).tolist()
    if resampling == "average":
        want, step = aref.render(rgba, proxy, zoom, size, cand)
    else:
        want, step = pref.render(rgba, proxy, zoom, size, cand, resampling)
    assert stats["step"] == step
    assert sorted(got) == sorted(want) and got  # one tile for the small 3857 and 4326 rasters at zoom 17
    for key in want:
        assert got[key][1] == want[key][1], key
        assert np.array_equal(got[key][0], want[key][0]), (key, int((got[key][0] != want[key][0]).any(axis=-1).sum()))
    return got


def _write16(tmp_path, name, px, kind, **kw):
    return bw.write_bands_tiff(str(tmp_path / (name + ".tif")), px, compression=8, predictor=2, tile=(64, 32), **georef(kind), **kw)


@pytest.mark.parametrize("kind", ["3857", "4326", "utm"])
@pytest.mark.parametrize("resampling", ["nearest", "bilinear", "average"])
def test_rs_tile_16_bit_equals_the_restatement(tmp_path, cuda_device, kind, resampling):
    px = smooth16(237, 301, 4, 1)
    px[60:90, 40:200] = 0  # a nodata hole
    g = open_bands(_write16(tmp_path, kind, px, kind, photometric=1, nodata="0"), [3, 2, 1])
    g.set_scale([(1000, 8000), (900, 8500), (1200, 7000)])
    got = check_band_raster(g, resampling)
    assert any(c < SIZE * SIZE for _, c in got.values())


@pytest.mark.parametrize("layout", ["rgb-alpha", "planar", "planar-gray-be"])
@pytest.mark.parametrize("resampling", ["nearest", "bilinear", "average"])
def test_rs_tile_16_bit_alpha_and_planar(tmp_path, cuda_device, layout, resampling):
    px = smooth16(199, 257, 4, 2)
    if layout == "rgb-alpha":
        px[..., 3] = 65535
        px[40:90, 30:200, 3] = 0
        px[::7, ::5, 3] = 0
        g = open_bands(_write16(tmp_path, layout, px, "utm", extra_samples=(2,)))
        assert g.alpha_band == 3 and g.bands == [0, 1, 2]
    elif layout == "planar":
        g = open_bands(_write16(tmp_path, layout, px, "utm", photometric=1, planar=2), [4, 2, 1])
    else:
        g = open_bands(bw.write_bands_tiff(str(tmp_path / "p.tif"), px, compression=5, predictor=2, rows_per_strip=13, planar=2, order=">", photometric=1,
                                           **georef("3857")), [2])
    g.set_scale([(500, 9500)])
    check_band_raster(g, resampling)


@pytest.mark.parametrize("bands", ["gray-nodata", "rgb-nodata", "rgba"])
@pytest.mark.parametrize("resampling", ["nearest", "bilinear", "average"])
def test_identity_property_on_8_bit_rasters(tmp_path, cuda_device, bands, resampling):
    spp = {"gray-nodata": 1, "rgb-nodata": 3, "rgba": 4}[bands]
    px = noise(199, 257, spp, 2)
    kw = {}
    if bands == "rgba":
        px[..., 3] = 255
        px[40:90, 30:200, 3] = 0
        px[::7, ::5, 3] = 0
    else:
        px[50:80, 60:150] = 0
        px[::9, ::4] = 0
        kw["nodata"] = "0"
    plain = write(tmp_path, bands, px, "utm", **kw)
    banded = open_bands(plain.path)
    assert banded.scale == [(0, 255)] * len(banded.bands)
    want = T.tile_device(plain, ZOOMS[resampling], SIZE, resampling)
    got = T.tile_device(banded, ZOOMS[resampling], SIZE, resampling)
    assert sorted(got) == sorted(want) and len(got) > 1
    for key in want:
        assert got[key][1] == want[key][1] and np.array_equal(got[key][0], want[key][0]), key


def _tile_args(raster, out, **kw):
    a = dict(zoom=ZOOMS["bilinear"], size=SIZE, tiles=None, resampling="bilinear", raster=raster, out=out, bands=None, scale=None, stretch=None)
    a.update(kw)
    return argparse.Namespace(**a)


def _pngs(root):
    found = {}
    for d, _, files in os.walk(root):
        for f in files:
            found[os.path.relpath(os.path.join(d, f), root)] = open(os.path.join(d, f), "rb").read()
    return found


def test_stretch_prints_a_scale_that_reproduces_its_tiles(tmp_path, cuda_device, capsys):
    from robosat_b200.tools import tile

    px = smooth16(301, 333, 4, 5)
    px[100:130, 50:90] = 0
    path = _write16(tmp_path, "s", px, "utm", photometric=1, nodata="0")
    stats = {}
    tile.main(_tile_args(path, str(tmp_path / "a"), bands="3,2,1", stretch="2,98"), stats)
    err = capsys.readouterr().err
    m = re.search(r"--stretch 2,98 of bands 3,2,1: --scale (\S+)", err)
    assert m, err
    values = [int(v) for v in m.group(1).split(",")]
    raw = open_bands(path, [3, 2, 1]).read_window(0, 301, 0, 333)
    want = ref.stretch(raw, 3, False, 0, 16, 200, 9800)
    assert [tuple(values[i:i + 2]) for i in range(0, 6, 2)] == want
    assert stats["stats_s"] > 0 and stats["stats_bands"] >= 1
    tile.main(_tile_args(path, str(tmp_path / "b"), bands="3,2,1", scale=m.group(1)))
    a, b = _pngs(tmp_path / "a"), _pngs(tmp_path / "b")
    assert a == b and len(a) > 1
    # the stretch counts the whole raster in row bands under any budget: a small one gives the same histogram
    g = open_bands(path, [3, 2, 1])
    small = {}
    h = T.band_stats(g, budget=333 * 6 * 40, stats=small)
    assert small["stats_bands"] > 3 and np.array_equal(h, ref.histogram(raw, 3, False, 0, 16))


SEG_CASES = {"3857-bilinear": dict(kind="3857", resampling="bilinear"), "utm-average": dict(kind="utm", resampling="average")}


@pytest.mark.parametrize("case", list(SEG_CASES))
def test_segment_equals_the_four_tool_pipeline(tmp_path, cuda_device, monkeypatch, case):
    from robosat_b200.tools import masks, mosaic, predict, segment, tile

    c = SEG_CASES[case]
    monkeypatch.setenv("RSB_GPUS", "1")
    monkeypatch.setenv("RSB_QUIET", "1")
    setup(tmp_path, 2, c["kind"])  # weights and configuration files (and an 8-bit raster, replaced here)
    px = smooth16(1000, 1100, 4, 11)
    bw.write_bands_tiff(str(tmp_path / "ortho.tif"), px, compression=8, predictor=2, tile=(128, 64), photometric=1, **georef(c["kind"]))
    t = tmp_path
    zoom, size, opts = 18, 256, dict(bands="3,2,1", scale="900,9000,1000,8800,800,9100")
    if c["resampling"] == "average":
        zoom = 17
    tile.main(argparse.Namespace(zoom=zoom, size=size, tiles=None, resampling=c["resampling"], raster=str(t / "ortho.tif"), out=str(t / "images"), **opts))
    predict.main(argparse.Namespace(batch_size=BATCH, checkpoint=str(t / "ckpt.pth"), overlap=OVERLAP, tile_size=size, workers=0, tiles=str(t / "images"),
                                    probs=str(t / "probs"), model=str(t / "model.toml"), dataset=str(t / "dataset.toml"), tta="none"))
    masks.main(argparse.Namespace(masks=str(t / "masks"), probs=[str(t / "probs")], weights=None, dataset=None))
    mosaic.main(argparse.Namespace(zoom=zoom, like=str(t / "ortho.tif"), resampling="nearest", nodata=None, masks=str(t / "masks"), out=str(t / "pipeline.tif")))
    stats = {}
    segment.main(argparse.Namespace(zoom=zoom, size=size, overlap=OVERLAP, batch_size=BATCH, tiles=None, resampling=c["resampling"], output="masks", tta="none",
                                    nodata=None, model=str(t / "model.toml"), dataset=str(t / "dataset.toml"), checkpoint=str(t / "ckpt.pth"),
                                    raster=str(t / "ortho.tif"), out=str(t / "fused.tif"), **opts), stats)
    want, mode_w, tags_w = read(t / "pipeline.tif")
    got, mode_g, tags_g = read(t / "fused.tif")
    assert mode_g == mode_w == "P" and got.shape == want.shape == (1000, 1100)
    assert tags_g == tags_w
    diff = np.argwhere(got != want)
    assert len(diff) == 0, (len(diff), diff[:5].tolist())
    assert stats["existing"] == stats["predicted"] > 0 and stats["render_s"] > 0
    assert stats["store_bytes"] > stats["image_slots"] * size * size * 3 + stats["plane_slots"] * size * size  # the band windows count


def test_plain_rasters_plan_as_before(tmp_path):
    from robosat_b200 import mosaic as M
    from robosat_b200 import segment as SEG

    setup(tmp_path, 2, "3857")
    g = GeoTiff(str(tmp_path / "ortho.tif"))
    p = SEG.plan(g, M.Grid(g.width, g.height, g.crs, g.geotransform), 18, 256, BATCH)
    assert p.store_bytes == p.image_slots * 256 * 256 * 3 + p.plane_slots * 256 * 256 and not hasattr(p, "render_bytes")
