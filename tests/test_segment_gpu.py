"""`rs segment` on the H100: the fused tool's GeoTIFF has the pixels, size, CRS, geotransform, nodata tag and ColorMap of
`rs tile → rs predict → rs masks → rs mosaic --like` run with the same settings on the same seeded raster and weights. The pipeline
batches its tiles column-major and the fused tool row-major, so equal pixels also show that a tile's bins do not depend on the
other tiles of its batch."""

import argparse
import os

import numpy as np
import pytest
import torch
from PIL import Image

import tiff_writer as tw
from test_tile_gpu import georef, noise
from robosat_b200 import mosaic as M
from robosat_b200 import segment as SEG
from robosat_b200 import synth
from robosat_b200.geotiff import GeoTiff
from robosat_b200.tools import masks, mosaic, predict, segment, tile

pytestmark = pytest.mark.gpu

ZOOM, SIZE, OVERLAP, BATCH = 18, 256, 32, 4
TAGS = (256, 257, 258, 262, 320, 33550, 33922, 34264, 34735, 42113)
CLASSES = {2: ["background", "parking"], 3: ["background", "building", "road"]}
COLORS = {2: ["denim", "orange"], 3: ["denim", "orange", "teal"]}
ROTATED = dict(geo=tw.geokeys(raster_type=2), matrix=(0.33, 0.22, 0, 1113312.7, 0.2, -0.35, 0, 6106910.3, 0, 0, 0, 0, 0, 0, 0, 1))


def setup(tmp_path, classes, kind, shape=(1000, 1100)):
    """a seeded RGB raster, weights and configuration files"""
    px = noise(shape[0], shape[1], 3, 11)
    kw = ROTATED if kind == "rotated" else georef(kind)
    tw.write_tiff(str(tmp_path / "ortho.tif"), px, compression=8, tile=(128, 64), predictor=2, **kw)
    torch.save({"epoch": 1, "state_dict": synth.make_state_dict(classes, seed=5), "optimizer": {}}, tmp_path / "ckpt.pth")
    (tmp_path / "model.toml").write_text("[common]\ncuda = true\nbatch_size = 2\nimage_size = 256\ncheckpoint = '%s'\n" % tmp_path)
    (tmp_path / "dataset.toml").write_text("[common]\ndataset = '%s'\nclasses = %r\ncolors = %r\n" % (tmp_path, CLASSES[classes], COLORS[classes]))


def pipeline(tmp_path, classes, output, resampling, tta, tiles, nodata):
    """the four tools, as a user would run them"""
    t = tmp_path
    tile.main(argparse.Namespace(zoom=ZOOM, size=SIZE, tiles=tiles, resampling=resampling, raster=str(t / "ortho.tif"), out=str(t / "images")))
    predict.main(argparse.Namespace(batch_size=BATCH, checkpoint=str(t / "ckpt.pth"), overlap=OVERLAP, tile_size=SIZE, workers=0, tiles=str(t / "images"),
                                    probs=str(t / "probs"), model=str(t / "model.toml"), dataset=str(t / "dataset.toml"), tta=tta))
    src = t / "probs"
    if output == "masks":
        masks.main(argparse.Namespace(masks=str(t / "masks"), probs=[str(src)], weights=None, dataset=str(t / "dataset.toml") if classes > 2 else None))
        src = t / "masks"
    mosaic.main(argparse.Namespace(zoom=ZOOM, like=str(t / "ortho.tif"), resampling="nearest", nodata=nodata, masks=str(src), out=str(t / "pipeline.tif")))
    return len(M.scan(str(t / "images"), ZOOM))


def fused(tmp_path, output, resampling, tta, tiles, nodata, budget=None):
    t = tmp_path
    stats = {}
    segment.main(argparse.Namespace(zoom=ZOOM, size=SIZE, overlap=OVERLAP, batch_size=BATCH, tiles=tiles, resampling=resampling, output=output, tta=tta,
                                    nodata=nodata, model=str(t / "model.toml"), dataset=str(t / "dataset.toml"), checkpoint=str(t / "ckpt.pth"),
                                    raster=str(t / "ortho.tif"), out=str(t / "fused.tif")), stats, budget)
    return stats


def read(path):
    im = Image.open(path)
    return np.array(im), im.mode, {t: im.tag_v2.get(t) for t in TAGS}


CASES = {
    "masks-3857-nearest": dict(classes=2, kind="3857", output="masks", resampling="nearest"),
    "probs-utm-bilinear": dict(classes=2, kind="utm", output="probs", resampling="bilinear"),
    "masks-4326-3-classes": dict(classes=3, kind="4326", output="masks", resampling="bilinear"),
    "tta-flip": dict(classes=2, kind="utm", output="masks", resampling="bilinear", tta="flip"),
    "tiles-holes-nodata": dict(classes=2, kind="3857", output="masks", resampling="bilinear", holes=True, nodata=255),
    "rotated-budget-at-peak": dict(classes=2, kind="rotated", output="masks", resampling="bilinear", at_peak=True),
    "fast-precision": dict(classes=2, kind="4326", output="probs", resampling="nearest", fast=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_equals_the_four_tool_pipeline(tmp_path, cuda_device, monkeypatch, case):
    c = CASES[case]
    monkeypatch.setenv("RSB_GPUS", "1")
    monkeypatch.setenv("RSB_QUIET", "1")
    if c.get("fast"):
        monkeypatch.setenv("RSB_PRECISION", "fast")
    setup(tmp_path, c["classes"], c["kind"])
    raster = GeoTiff(str(tmp_path / "ortho.tif"))
    grid = M.Grid(raster.width, raster.height, raster.crs, raster.geotransform)
    tiles = None
    if c.get("holes"):
        from robosat_b200 import tile as T

        cand = T.candidate_tiles(raster, ZOOM, SIZE).tolist()
        (tmp_path / "tiles.csv").write_text("".join("%d,%d,%d\n" % (x, y, ZOOM) for i, (x, y) in enumerate(cand) if i % 3 != 1))
        tiles = str(tmp_path / "tiles.csv")
    plan = SEG.plan(raster, grid, ZOOM, SIZE, BATCH, None)
    assert 10 <= len(plan.tiles) <= 40, len(plan.tiles)
    budget = plan.store_bytes if c.get("at_peak") else None
    if c.get("at_peak"):
        assert plan.plane_slots > 2 * max(len(w.xs) for w in plan.warps)  # output chunk rows reach many tile rows
    written = pipeline(tmp_path, c["classes"], c["output"], c["resampling"], c.get("tta", "none"), tiles, c.get("nodata"))
    stats = fused(tmp_path, c["output"], c["resampling"], c.get("tta", "none"), tiles, c.get("nodata"), budget)
    want, mode_w, tags_w = read(tmp_path / "pipeline.tif")
    got, mode_g, tags_g = read(tmp_path / "fused.tif")
    assert mode_g == mode_w == "P" and got.shape == want.shape == (raster.height, raster.width)
    assert tags_g == tags_w
    diff = np.argwhere(got != want)
    assert len(diff) == 0, (len(diff), diff[:5].tolist())
    assert stats["existing"] == stats["predicted"] == written
    if c.get("nodata") is not None:
        assert (got == c["nodata"]).any() and (got != c["nodata"]).any()


def test_budget_under_the_peak_leaves_no_file(tmp_path, cuda_device):
    setup(tmp_path, 2, "3857")
    raster = GeoTiff(str(tmp_path / "ortho.tif"))
    plan = SEG.plan(raster, M.Grid(raster.width, raster.height, raster.crs, raster.geotransform), ZOOM, SIZE, BATCH)
    with pytest.raises(SystemExit, match="need %d device bytes" % plan.store_bytes):
        fused(tmp_path, "masks", "bilinear", "none", None, None, plan.store_bytes - 1)
    assert not os.path.exists(tmp_path / "fused.tif") and not [f for f in os.listdir(tmp_path) if f.endswith(".tmp")]
