"""`rs segment` planning on the CPU: on grid-only raster stand-ins (EPSG:3857, 4326, UTM and a rotated model transformation) every
output window runs after the last batch that predicts a tile of its reach, no image or plane leaves its ring before its last reader,
the planned peaks equal a brute-force recount of the live sets, a budget one byte under the peak is refused, the output palette is
the one `rs mosaic` reads from the pipeline's tiles, and the tool refuses bad arguments before it looks for a device."""

import argparse
import os

import numpy as np
import pytest

from robosat_b200 import _lib
from robosat_b200 import mosaic as M
from robosat_b200 import segment as SEG
from robosat_b200 import tile as T
from robosat_b200.colors import continuous_palette_for_color, make_palette
from robosat_b200.stitch import NEIGHBOURS

ZOOM, SIZE = 18, 256


class Raster:
    """the grid of a GeoTiff without its pixels"""

    def __init__(self, crs, gt, W, H):
        self.crs, self.geotransform, self.width, self.height, self.spp, self.alpha, self.nodata = crs, gt, W, H, 3, False, -1


def raster_of(kind):
    """rasters of a few tens of zoom-18 tiles of 256² near (10 E, 48 N)"""
    if kind == "3857":
        return Raster("3857", (1113312.7, 0.45, 0.0, 6106910.3, 0.0, -0.45), 1500, 1100)
    if kind == "4326":
        return Raster("4326", (10.00031, 5e-6, 0.0, 48.00042, 0.0, -3.5e-6), 1300, 1200)
    if kind == "utm":
        E, N = T.tm_forward(10.2, 47.3, 9.0)
        return Raster(("utm", 32, False), (float(E), 0.4, 0.0, float(N), 0.0, -0.4), 1400, 1300)
    if kind == "rotated":
        return Raster("3857", (1113312.7, 0.4, 0.12, 6106910.3, 0.1, -0.4), 1200, 1100)
    raise ValueError(kind)


def grid_of(r):
    return M.Grid(r.width, r.height, r.crs, r.geotransform)


KINDS = ["3857", "4326", "utm", "rotated"]


@pytest.fixture(scope="module", params=KINDS)
def planned(request):
    r = raster_of(request.param)
    return r, SEG.plan(r, grid_of(r), ZOOM, SIZE, batch=4)


def reads(p, kind, number):
    """the indices an op reads: a batch's 3 x 3 neighbourhoods, an output window's reach"""
    if kind == "predict":
        a, b = p.batches[number]
        nb = p.neighbours[a:b]
        return nb[nb >= 0]
    if kind == "mosaic" and p.reach[number] is not None:
        r = p.reach[number]
        return r[r >= 0]
    return np.zeros(0, np.int64)


def test_plan_covers_the_tiles_of_rs_tile(planned):
    r, p = planned
    cand = T.candidate_tiles(r, ZOOM, SIZE)
    windows = T.plan(r, ZOOM, SIZE, cand, T.choose_step(r, ZOOM, SIZE, cand))
    assert p.tiles.tolist() == [[x, w.y] for w in windows for x in w.xs]
    assert 10 <= len(p.tiles) <= 60
    assert p.tiles.tolist() == sorted(p.tiles.tolist(), key=lambda t: (t[1], t[0]))  # row-major
    at = {tuple(t): i for i, t in enumerate(p.tiles.tolist())}
    for i, (x, y) in enumerate(p.tiles.tolist()):
        assert p.neighbours[i].tolist() == [at.get((x + dx, y + dy), -1) for dx, dy in NEIGHBOURS]
    assert len(p.windows) == len(M.plan(grid_of(r), ZOOM, SIZE, p.tiles, M.choose_step(grid_of(r), ZOOM, SIZE)))
    kinds = [o[0] for o in p.ops]
    assert sorted(o[1] for o in p.ops if o[0] == "warp") == list(range(len(p.warps)))
    assert [o[1] for o in p.ops if o[0] == "predict"] == list(range(len(p.batches)))
    assert sorted(o[1] for o in p.ops if o[0] == "mosaic") == list(range(len(p.windows)))
    assert kinds.count("warp") == len(p.warps)


def test_every_read_follows_its_writes(planned):
    """a batch runs after the warps of every neighbour; an output window after the batches of its reach (so after the last tile row
    of its reach)"""
    _, p = planned
    warped, predicted = set(), set()
    for kind, number, *_ in p.ops:
        if kind == "warp":
            warped.update(range(p.first[number], p.first[number + 1]))
        elif kind == "predict":
            assert set(reads(p, kind, number).tolist()) <= warped
            predicted.update(range(*p.batches[number]))
        else:
            idx = reads(p, kind, number)
            assert set(idx.tolist()) <= predicted
            if len(idx):
                last_row = p.tiles[idx, 1].max()
                assert set(np.flatnonzero(p.tiles[:, 1] <= last_row).tolist()) <= predicted | set(range(idx.max() + 1, len(p.tiles)))


def test_nothing_leaves_a_ring_before_its_last_reader(planned):
    _, p = planned
    prev = (0, 0, 0, 0)
    for kind, number, img_lo, img_hi, pl_lo, pl_hi in p.ops:
        if kind != "mosaic" or p.reach[number] is not None and (p.reach[number] >= 0).any():
            assert img_lo >= prev[0] and img_hi >= prev[1] and pl_lo >= prev[2] and pl_hi >= prev[3]  # FIFO: both rings
            prev = (img_lo, img_hi, pl_lo, pl_hi)
        assert img_hi - img_lo <= p.image_slots and pl_hi - pl_lo <= p.plane_slots
        idx = reads(p, kind, number)
        if kind == "predict":
            a, b = p.batches[number]
            assert ((idx >= img_lo) & (idx < img_hi)).all()
            assert pl_lo <= a and pl_hi == b
        elif kind == "mosaic" and len(idx):
            assert ((idx >= pl_lo) & (idx < pl_hi)).all()
    # a warp that reuses image slots waits for the last stitch that read their previous tiles
    for kind, k, *_ in p.ops:
        if kind != "warp":
            continue
        a, b = int(p.first[k]), int(p.first[k + 1])
        old = set(range(max(0, a - p.image_slots), max(0, b - p.image_slots)))
        readers = [j for j in range(len(p.batches)) if old & set(reads(p, "predict", j).tolist())]
        assert (max(readers) if readers else None) == p.wait.get(k)


def recount(p):
    """the peaks from the op list alone: at every op, the slots from the lowest index a later (or this) op still reads to the highest
    one written so far"""
    img_peak = pl_peak = 0
    warped_hi = produced_hi = 0
    for t, (kind, number, *_) in enumerate(p.ops):
        if kind == "warp":
            warped_hi = int(p.first[number + 1])
        if kind == "predict":
            produced_hi = p.batches[number][1]
        later = p.ops[t:]
        img_need = [i for o in later if o[0] == "predict" for i in reads(p, "predict", o[1]).tolist() if i < warped_hi]
        if kind == "warp":
            img_need.extend(range(int(p.first[number]), warped_hi))
        if img_need:
            img_peak = max(img_peak, warped_hi - min(img_need))
        pl_need = [i for o in later if o[0] == "mosaic" for i in reads(p, "mosaic", o[1]).tolist() if i < produced_hi]
        if kind == "predict":
            pl_need.extend(range(*p.batches[number]))
        if pl_need:
            pl_peak = max(pl_peak, produced_hi - min(pl_need))
    return img_peak, pl_peak


def test_peaks_equal_a_recount(planned):
    _, p = planned
    assert (p.image_slots, p.plane_slots) == recount(p)
    assert p.store_bytes == p.image_slots * SIZE * SIZE * 3 + p.plane_slots * SIZE * SIZE


@pytest.mark.parametrize("batch", [1, 3, 64])
def test_peaks_equal_a_recount_across_batches(batch):
    r = raster_of("rotated")
    p = SEG.plan(r, grid_of(r), ZOOM, SIZE, batch=batch)
    assert (p.image_slots, p.plane_slots) == recount(p)
    if batch >= len(p.tiles):
        assert p.image_slots == p.plane_slots == len(p.tiles)


def test_holes_from_a_tiles_list():
    r = raster_of("utm")
    cand = T.candidate_tiles(r, ZOOM, SIZE)
    listed = [tuple(t) for i, t in enumerate(cand.tolist()) if i % 4 != 1]
    p = SEG.plan(r, grid_of(r), ZOOM, SIZE, batch=4, tiles=listed)
    assert set(map(tuple, p.tiles.tolist())) <= set(listed)
    assert (p.image_slots, p.plane_slots) == recount(p)
    missing = {tuple(t) for t in cand.tolist()} - set(listed)
    at = {tuple(t) for t in p.tiles.tolist()}
    for i, (x, y) in enumerate(p.tiles.tolist()):
        for (dx, dy), j in zip(NEIGHBOURS, p.neighbours[i]):
            assert (j == -1) == ((x + dx, y + dy) not in at)
            if (x + dx, y + dy) in missing:
                assert j == -1


def test_rotated_raster_keeps_more_rows_live():
    north = SEG.plan(raster_of("3857"), grid_of(raster_of("3857")), ZOOM, SIZE, batch=4)
    rot = SEG.plan(raster_of("rotated"), grid_of(raster_of("rotated")), ZOOM, SIZE, batch=4)
    assert north.plane_slots < len(north.tiles)
    assert rot.plane_slots / len(rot.tiles) > north.plane_slots / len(north.tiles)


def test_budget_one_byte_under_the_peak_is_refused(planned, tmp_path):
    r, p = planned
    again = SEG.plan(r, grid_of(r), ZOOM, SIZE, batch=4, budget=p.store_bytes)
    assert again.store_bytes == p.store_bytes
    with pytest.raises(_lib.RsbError, match="need %d device bytes.*--tiles" % p.store_bytes):
        SEG.plan(r, grid_of(r), ZOOM, SIZE, batch=4, budget=p.store_bytes - 1)


def test_output_palette_is_what_rs_mosaic_reads(tmp_path):
    """the union palette `rs mosaic` builds from the pipeline's tiles: rs masks (PIL, optimize) and rs predict (the library)"""
    from robosat_b200.tiles import Tile
    from robosat_b200.tools import masks, predict

    mask = np.zeros((SIZE, SIZE), np.uint8)
    mask[3:9, 5:7] = 1
    for name, flat in (("two", make_palette("denim", "orange")), ("three", make_palette("denim", "orange", "teal"))):
        masks._save(str(tmp_path / name), flat, Tile(5, 7, ZOOM), mask)
        _, palette = M.check_tiles(M.scan(str(tmp_path / name), ZOOM))
        assert np.array_equal(palette, SEG.output_palette(flat))
    pink = continuous_palette_for_color("pink", 256)
    predict._save_png(str(tmp_path / "probs"), pink, 5, 7, ZOOM, mask)
    _, palette = M.check_tiles(M.scan(str(tmp_path / "probs"), ZOOM))
    assert np.array_equal(palette, SEG.output_palette(pink))


def _args(tmp_path, classes, **kw):
    (tmp_path / "model.toml").write_text("[common]\ncuda = true\nbatch_size = 2\nimage_size = 256\ncheckpoint = '%s'\n" % tmp_path)
    colors = ["denim", "orange", "teal", "red"][:len(classes)]
    (tmp_path / "dataset.toml").write_text("[common]\ndataset = '%s'\nclasses = %r\ncolors = %r\n" % (tmp_path, classes, colors))
    base = dict(zoom=ZOOM, size=256, overlap=32, batch_size=4, tiles=None, resampling="bilinear", output="masks", tta="none", nodata=None,
                model=str(tmp_path / "model.toml"), dataset=str(tmp_path / "dataset.toml"), checkpoint=str(tmp_path / "none.pth"),
                raster=str(tmp_path / "none.tif"), out=str(tmp_path / "out.tif"))
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw, classes, message", [
    (dict(output="probs"), ["background", "building", "road"], "--output probs .* two-class models only; the dataset has 3 classes"),
    (dict(zoom=31), ["background", "parking"], "--zoom must be in 0..30"),
    (dict(zoom=-1), ["background", "parking"], "--zoom must be in 0..30"),
    (dict(size=0), ["background", "parking"], "--size must be in 1..4096"),
    (dict(size=4097), ["background", "parking"], "--size must be in 1..4096"),
    (dict(overlap=300), ["background", "parking"], "--overlap must be in 0..--size"),
    (dict(size=250), ["background", "parking"], "multiple of 64"),
    (dict(batch_size=0), ["background", "parking"], "--batch_size must be at least 1"),
    (dict(nodata=256), ["background", "parking"], "--nodata must be in 0..255"),
    (dict(), ["background", "1", "road"], "class '1' is an integer"),
])
def test_tool_refuses_before_any_work(tmp_path, kw, classes, message):
    from robosat_b200.tools import segment as tool

    with pytest.raises(SystemExit, match=message):
        tool.main(_args(tmp_path, classes, **kw))
    assert not os.path.exists(tmp_path / "out.tif")


def test_parser():
    import sys

    from robosat_b200.tools import __main__ as cli

    argv = sys.argv
    try:
        sys.argv = ["rs", "segment", "--zoom", "18", "--model", "m.toml", "--dataset", "d.toml", "--checkpoint", "c.pth", "in.tif", "out.tif"]
        args = cli.add_parsers()
    finally:
        sys.argv = argv
    assert (args.size, args.overlap, args.batch_size, args.resampling, args.output, args.tta, args.nodata, args.tiles) == (
        512, 32, 32, "bilinear", "masks", "none", None, None)
    assert args.func.__module__ == "robosat_b200.tools.segment"
