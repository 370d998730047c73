"""`rs tile --resampling average` without a GPU: the restatement's weights against exact overlap areas, its vectorised sums against
a per-pixel loop, block means on an aligned raster, the corner lattice's step, the windows holding every weighted source pixel, the
footprint cap's host bound and refusal, the ABI's argument validation, both parsers and `rs segment`'s plan on the corner lattice."""

import argparse
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest

import test_segment as TS
import tile_average_reference as ref
from robosat_b200 import _lib
from robosat_b200 import segment as SEG
from robosat_b200 import tile as T
from robosat_b200.rasterize import CE
from test_tile import Raster, rasters

KINDS = ["3857", "4326", "utm", "utm-south", "rotated"]


def clipped_weights(u0, u1, v0, v1, W, H):
    """{(i, j): wx_i * wy_j as a Fraction} of one footprint, clipped to a W x H raster as the rule clips it (None: uncovered)"""
    a0, a1, b0, b1 = max(u0, 0.0), min(u1, float(W)), max(v0, 0.0), min(v1, float(H))
    if not (a0 < a1 and b0 < b1):
        return None
    i0, wx = ref.axis_weights(a0, a1)
    j0, wy = ref.axis_weights(b0, b1)
    return {(i0 + a, j0 + b): Fraction(float(x)) * Fraction(float(y)) for b, y in enumerate(wy) for a, x in enumerate(wx)}


def exact_overlaps(u0, u1, v0, v1, W, H):
    """{(i, j): area of [i, i + 1] x [j, j + 1] within the box and the raster} with non-zero area, in exact arithmetic"""
    U0, U1, V0, V1 = (Fraction(t) for t in (u0, u1, v0, v1))
    got = {}
    for j in range(max(0, math.floor(v0) - 1), min(H, math.ceil(v1) + 1)):
        for i in range(max(0, math.floor(u0) - 1), min(W, math.ceil(u1) + 1)):
            w = max(Fraction(0), min(U1, i + 1) - max(U0, i)) * max(Fraction(0), min(V1, j + 1) - max(V0, j))
            if w:
                got[(i, j)] = w
    return got


BOXES = [  # (u0, u1, v0, v1) on a 10 x 8 raster
    (2.25, 5.75, 1.5, 3.125),  # inside
    (-1.5, 2.25, 3.0, 4.5),  # over the left edge
    (8.75, 11.0, 0.5, 1.25),  # over the right edge
    (2.0, 3.5, -0.75, 0.5),  # over the top edge
    (4.125, 6.0, 7.5, 9.0),  # over the bottom edge
    (-2.0, 12.0, -1.0, 9.0),  # over every edge
    (3.25, 3.5, 5.0625, 5.125),  # inside one source pixel
    (4.875, 5.125, 2.9, 3.1),  # smaller than a pixel, across a pixel corner
    (9.9, 10.3, 7.7, 8.2),  # smaller than a pixel, in the raster's last pixel
    (1.3, 7.7, 2.1, 6.9),  # non-dyadic: the subtractions are still exact (Sterbenz) away from column and row 0
]


@pytest.mark.parametrize("box", BOXES)
def test_weights_are_the_exact_overlap_areas(box):
    assert clipped_weights(*box, 10, 8) == exact_overlaps(*box, 10, 8)


def test_empty_clipped_footprints_are_uncovered():
    for box in ((-3.0, -0.5, 1.0, 2.0), (10.0, 12.0, 1.0, 2.0), (1.0, 2.0, 8.0, 8.5), (2.0, 2.0, 1.0, 3.0)):
        assert clipped_weights(*box, 10, 8) is None


@pytest.mark.parametrize("kind", ["rotated", "4326"])
def test_weights_of_real_footprints_are_the_overlap_areas(kind):
    """the corners of tiles inside and across the raster edges (about 4 source pixels per tile pixel): every pixel's weights against
    exact areas, within one rounding at column or row 0, where 1 - a0 can round"""
    r = rasters()[kind]
    zoom, size = 21, 16
    tiles = T.candidate_tiles(r, zoom, size).tolist()
    step = ref.choose_step(r, zoom, size, tiles)
    checked = 0
    for x, y in tiles[::len(tiles) // 8]:
        u0, u1, v0, v1, nan = ref.footprints(ref.corners(r, zoom, size, step, x, y))
        for k in zip(*np.nonzero(~nan)):
            box = (float(u0[k]), float(u1[k]), float(v0[k]), float(v1[k]))
            mine = clipped_weights(*box, r.width, r.height)
            if mine is None:
                continue
            exact = exact_overlaps(*box, r.width, r.height)
            assert set(exact) <= set(mine)
            for key, w in mine.items():
                assert abs(w - exact.get(key, 0)) <= Fraction(1, 2 ** 52), (x, y, k, key)
            checked += 1
    assert checked > 100


def scalar_render(pixels, raster, zoom, size, step, x, y):
    """the rule pixel by pixel with Python floats, in the kernel's order"""
    H, W = pixels.shape[:2]
    valid = ref.valid_mask(pixels, raster.alpha, raster.nodata)
    u0, u1, v0, v1, nan = ref.footprints(ref.corners(raster, zoom, size, step, x, y))
    out = np.zeros((size, size, 3), np.uint8)
    covered = 0
    for r in range(size):
        for c in range(size):
            if nan[r, c]:
                continue
            a0, a1, b0, b1 = max(float(u0[r, c]), 0.0), min(float(u1[r, c]), float(W)), max(float(v0[r, c]), 0.0), min(float(v1[r, c]), float(H))
            if not (a0 < a1 and b0 < b1):
                continue
            A, Ws = [0.0, 0.0, 0.0], 0.0
            for j in range(math.floor(b0), math.ceil(b1)):
                wy = min(j + 1.0, b1) - max(float(j), b0)
                R, Rw = [0.0, 0.0, 0.0], 0.0
                for i in range(math.floor(a0), math.ceil(a1)):
                    if not valid[j, i]:
                        continue
                    wx = min(i + 1.0, a1) - max(float(i), a0)
                    p = pixels[j, i]
                    rgb = (p[0], p[0], p[0]) if pixels.shape[-1] == 1 else p[:3]
                    R = [R[b] + wx * float(rgb[b]) for b in range(3)]
                    Rw += wx
                A = [A[b] + wy * R[b] for b in range(3)]
                Ws += wy * Rw
            if Ws > 0:
                out[r, c] = [min(255, max(0, math.floor(A[b] / Ws + 0.5))) for b in range(3)]
                covered += 1
    return out, covered


@pytest.mark.parametrize("kind,spp", [("rotated", 3), ("utm", 1), ("4326", 4)])
def test_vectorised_restatement_equals_a_per_pixel_loop(kind, spp):
    r = rasters()[kind]
    rng = np.random.default_rng(3)
    px = rng.integers(0, 256, (r.height, r.width, spp), dtype=np.uint8)
    r = Raster(r.crs, r.geotransform, r.width, r.height, spp=spp, alpha=spp == 4, nodata=7 if spp != 4 else -1)
    px[::5, ::3, :min(spp, 3)] = 7
    if spp == 4:
        px[::4, ::2, 3] = 0
    zoom, size = 20, 12  # 3.6 to 10 source pixels per tile pixel
    tiles = T.candidate_tiles(r, zoom, size).tolist()
    step = ref.choose_step(r, zoom, size, tiles)
    for x, y in tiles[::max(1, len(tiles) // 4)]:
        want = scalar_render(px, r, zoom, size, step, x, y)
        got = ref.render_tile(px, r, zoom, size, step, x, y)
        assert got[1] == want[1] and np.array_equal(got[0], want[0]), (x, y)


def aligned_raster(zoom, size, k, tiles_w=2, tiles_h=2, x0=68500, y0=45300):
    """an EPSG:3857 raster whose pixels are the zoom's tile pixels split k x k, starting at the corner of tile (x0, y0)"""
    px = CE / (2 ** zoom * size) / k
    left, top = x0 * CE / 2 ** zoom - CE / 2, CE / 2 - y0 * CE / 2 ** zoom
    return Raster("3857", (left, px, 0.0, top, 0.0, -px), tiles_w * size * k, tiles_h * size * k)


def check_block_means(got, px, k, size):
    """got uint8 [size, size, 3] of the tile over px [size k, size k, 3]: each pixel the k x k block mean rounded half up, either
    neighbour where the mean is a half-integer"""
    blocks = px.reshape(size, k, size, k, 3).astype(np.int64).sum(axis=(1, 3))
    twice = 2 * blocks  # 2 k^2 mean
    lo = (twice + k * k) // (2 * k * k)  # floor(mean + 1/2)
    half = (twice % (2 * k * k)) == k * k
    ok = (got == lo) | (half & (got == lo - 1))
    assert ok.all(), int((~ok).sum())


@pytest.mark.parametrize("k", [2, 4, 8])
def test_aligned_raster_gives_block_means(k):
    zoom, size = 17, 16
    r = aligned_raster(zoom, size, k)
    px = np.random.default_rng(k).integers(0, 256, (r.height, r.width, 3), dtype=np.uint8)
    step = ref.choose_step(r, zoom, size, [(68500, 45300)])
    for dx, dy in ((0, 0), (1, 0), (1, 1)):
        im, covered = ref.render_tile(px, r, zoom, size, step, 68500 + dx, 45300 + dy)
        assert covered == size * size
        check_block_means(im, px[dy * size * k:(dy + 1) * size * k, dx * size * k:(dx + 1) * size * k], k, size)


LATTICE_CASES = [(n, 18, 512) for n in KINDS] + [(n, 15, 256) for n in KINDS]


@pytest.mark.parametrize("name,zoom,size", LATTICE_CASES)
def test_corner_lattice_step_meets_the_bound_on_every_cell(name, zoom, size):
    r = rasters()[name]
    tiles = T.candidate_tiles(r, zoom, size)
    step = T.choose_step(r, zoom, size, tiles, corner=True)
    assert step == ref.choose_step(r, zoom, size, tiles.tolist())
    assert all(T.step_error(r, zoom, size, step, run, corner=True) <= T.TOLERANCE for run in T.runs(tiles))
    if step < 64:
        assert any(T.step_error(r, zoom, size, 2 * step, run, corner=True) > T.TOLERANCE for run in T.runs(tiles))


def test_a_tall_lon_lat_raster_needs_a_finer_corner_lattice():
    r = Raster("4326", (5.0, 0.01, 0.0, 70.0, 0.0, -0.01), 500, 2000)
    tiles = T.candidate_tiles(r, 6, 256)
    assert T.choose_step(r, 6, 256, tiles, corner=True) == ref.choose_step(r, 6, 256, tiles.tolist()) < 64


@pytest.mark.parametrize("name", KINDS)
@pytest.mark.parametrize("tiny", [False, True])
def test_windows_hold_every_weighted_source_pixel(name, tiny):
    r = rasters()[name]
    zoom, size = 17, 64
    tiles = T.candidate_tiles(r, zoom, size)
    step = T.choose_step(r, zoom, size, tiles, corner=True)
    budget = max(w.device_bytes(r, size) for w in T.plan(r, zoom, size, tiles, step, batch=1, corner=True)) if tiny else T.DEFAULT_BUDGET
    windows = T.plan(r, zoom, size, tiles, step, budget=budget, batch=5, corner=True)
    if tiny:
        assert all(w.device_bytes(r, size) <= budget for w in windows) and len(windows) > len(T.runs(tiles))
        with pytest.raises(_lib.RsbError, match="more than the budget"):
            T.plan(r, zoom, size, tiles, step, budget=budget - 1, batch=1, corner=True)
    placed = set()
    for w in windows:
        for x in w.xs:
            placed.add((x, w.y))
            kx0, ky0, n = ref.tile_nodes(r, zoom, size, step, x, w.y)
            sub = w.nodes[ky0 - w.ky0:ky0 - w.ky0 + n.shape[0], kx0 - w.kx0:kx0 - w.kx0 + n.shape[1]]
            assert np.array_equal(sub, n, equal_nan=True)
            u0, u1, v0, v1, nan = ref.footprints(ref.corners(r, zoom, size, step, x, w.y))
            with np.errstate(invalid="ignore"):
                a0, a1 = np.maximum(u0, 0.0), np.minimum(u1, float(r.width))
                b0, b1 = np.maximum(v0, 0.0), np.minimum(v1, float(r.height))
                ok = ~nan & (a0 < a1) & (b0 < b1)
            # the first and last column and row with a non-zero weight
            assert (np.floor(a0[ok]) >= w.col0).all() and (np.ceil(a1[ok]) <= w.col0 + w.cols).all()
            assert (np.floor(b0[ok]) >= w.row0).all() and (np.ceil(b1[ok]) <= w.row0 + w.rows).all()
    for x, y in set(map(tuple, tiles.tolist())) - placed:  # left out: nothing to sum
        u0, u1, v0, v1, nan = ref.footprints(ref.corners(r, zoom, size, step, x, y))
        with np.errstate(invalid="ignore"):
            assert not (~nan & (np.maximum(u0, 0) < np.minimum(u1, r.width)) & (np.maximum(v0, 0) < np.minimum(v1, r.height))).any()


@pytest.mark.parametrize("name", KINDS)
def test_footprint_bound_holds_every_extent(name):
    r = rasters()[name]
    for zoom, size in ((18, 64), (14, 32)):
        tiles = T.candidate_tiles(r, zoom, size).tolist()
        step = ref.choose_step(r, zoom, size, tiles)
        for x, y in tiles:
            _, _, n = ref.tile_nodes(r, zoom, size, step, x, y)
            extent = ref.largest_extent(r, zoom, size, step, [(x, y)])
            assert T.footprint_bound(n, step) >= extent > 0, (zoom, x, y)


def test_a_run_over_the_cap_is_refused_before_any_device_work(monkeypatch):
    import torch

    r = rasters()["3857"]  # 0.3 m pixels: a zoom-12 tile pixel of 256² tiles spans about 127 of them
    tiles = T.candidate_tiles(r, 12, 256)
    step = T.choose_step(r, 12, 256, tiles, corner=True)
    with pytest.raises(_lib.RsbError, match="tile \\(\\d+, \\d+, 12\\) may span 1\\d\\d\\.\\d source pixels, more than the 64 .* higher zoom"):
        T.plan(r, 12, 256, tiles, step, corner=True)
    T.plan(r, 12, 256, tiles, step)  # the centre lattice has no cap
    T.plan(r, 14, 256, T.candidate_tiles(r, 14, 256), 64, corner=True)  # about 32 pixels: under it

    def no_device(*a, **k):
        raise AssertionError("device work")

    monkeypatch.setattr(torch.cuda, "synchronize", no_device)
    monkeypatch.setattr(torch.cuda, "current_stream", no_device)
    with pytest.raises(_lib.RsbError, match="may span"):
        T.run(r, 12, 256, "average")
    with pytest.raises(_lib.RsbError, match="may span"):
        SEG.plan(r, TS.grid_of(r), 12, 256, resampling="average")


def test_abi_validates_before_the_device_check():
    import torch

    lib = _lib.load()
    buf = (ctypes.c_uint8 * 64)()
    nodes = np.zeros(64, np.float64)
    tiles = np.zeros(2, np.int64)
    base = [ctypes.addressof(buf), 30, 0, 0, 10, 10, 10, 10, 3, 0, -1, nodes.ctypes.data, 0, 0, 2, 2, 64, tiles.ctypes.data, 1, 4,
            ctypes.addressof(buf), 48, ctypes.addressof(buf), ctypes.addressof(buf), None]
    for k, bad in ((8, 2), (9, 1), (10, 256), (10, -2), (14, 1), (12, -1), (16, 48), (16, 128), (16, 0), (18, 0), (18, 65536), (19, 0),
                   (19, 4097), (21, 47), (1, 29), (4, 11), (5, 11), (2, -1), (0, None), (11, None), (17, None), (20, None), (22, None),
                   (23, None)):
        args = list(base)
        args[k] = bad
        assert lib.rsb_tile_average(*args) == -1, (k, bad)
    args = list(base)
    args[11] = nodes.ctypes.data + 8  # nodes must be 16-byte aligned
    assert lib.rsb_tile_average(*args) == -1
    if not torch.cuda.is_available():
        assert lib.rsb_tile_average(*base) == -3


def test_parsers_accept_average():
    import sys

    from robosat_b200.tools import __main__ as cli
    from robosat_b200.tools import tile

    parser = argparse.ArgumentParser()
    tile.add_parser(parser.add_subparsers())
    assert parser.parse_args(["tile", "--zoom", "19", "--resampling", "average", "r.tif", "o"]).resampling == "average"
    assert parser.parse_args(["tile", "--zoom", "19", "r.tif", "o"]).resampling == "bilinear"
    argv = sys.argv
    try:
        sys.argv = ["rs", "segment", "--zoom", "18", "--resampling", "average", "--model", "m.toml", "--dataset", "d.toml", "--checkpoint", "c.pth",
                    "in.tif", "out.tif"]
        assert cli.add_parsers().resampling == "average"
    finally:
        sys.argv = argv


@pytest.mark.parametrize("kind", TS.KINDS)
def test_segment_plan_on_the_corner_lattice(kind):
    r = TS.raster_of(kind)
    p = SEG.plan(r, TS.grid_of(r), TS.ZOOM, TS.SIZE, batch=4, resampling="average")
    cand = T.candidate_tiles(r, TS.ZOOM, TS.SIZE)
    step = T.choose_step(r, TS.ZOOM, TS.SIZE, cand, corner=True)
    assert p.corner and p.step == step
    windows = T.plan(r, TS.ZOOM, TS.SIZE, cand, step, corner=True)
    assert [(w.y, w.xs, w.row0, w.rows, w.col0, w.cols) for w in p.warps] == [(w.y, w.xs, w.row0, w.rows, w.col0, w.cols) for w in windows]
    assert all(np.array_equal(a.nodes, b.nodes, equal_nan=True) for a, b in zip(p.warps, windows))
    # the schedule invariants test_segment.py checks on the centre lattice
    TS.test_every_read_follows_its_writes((r, p))
    TS.test_nothing_leaves_a_ring_before_its_last_reader((r, p))
    TS.test_peaks_equal_a_recount((r, p))
    with pytest.raises(_lib.RsbError, match="need %d device bytes" % p.store_bytes):
        SEG.plan(r, TS.grid_of(r), TS.ZOOM, TS.SIZE, batch=4, budget=p.store_bytes - 1, resampling="average")


def test_segment_run_refuses_a_resampling_its_plan_was_not_made_for():
    r = TS.raster_of("utm")
    avg = SEG.plan(r, TS.grid_of(r), TS.ZOOM, TS.SIZE, batch=4, resampling="average")
    centre = SEG.plan(r, TS.grid_of(r), TS.ZOOM, TS.SIZE, batch=4)
    assert not centre.corner
    with pytest.raises(ValueError, match="lattice is for average, not bilinear"):
        SEG.run(r, avg, None, "bilinear")
    with pytest.raises(ValueError, match="lattice is for nearest or bilinear, not average"):
        SEG.run(r, centre, None, "average")
    with pytest.raises(ValueError, match="resampling must be one of"):
        SEG.plan(r, TS.grid_of(r), TS.ZOOM, TS.SIZE, resampling="cubic")
