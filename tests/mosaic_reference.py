"""numpy float64 restatement of `rs mosaic`'s rule (DESIGN.md §8), over the whole output raster and without windows, for
bit-identity tests of rsb_mosaic_warp and robosat_b200.mosaic.

The rule is `rs tile`'s with the roles swapped: the tiles of zoom z are a raster of 2^z S pixels in EPSG:3857 and a global pixel is
valid when its tile's file exists. Output pixel (i, j) is centred at raster coordinates (i + 1/2, j + 1/2); the exact transform to
global pixel coordinates (gx, gy) is `robosat_b200.mosaic.global_coords` (the grid's geotransform, then `tile.mercator_of_model`,
whose projections test_tile.py checks). Everything after it is restated here: the lattice step, the per-pixel interpolation in the
kernel's operation order, the coverage test and both resamplings."""

import numpy as np

from robosat_b200 import mosaic as M


def _lerp(a, b, t):
    return a + t * (b - a)  # three separately rounded operations, as __dadd_rn(a, __dmul_rn(t, __dsub_rn(b, a)))


def nodes(grid, zoom, size, step):
    """(gx, gy) at the centres of output pixels (kG, lG) for every node the raster's cells need"""
    kx1, ky1 = (grid.width - 1) // step + 1, (grid.height - 1) // step + 1
    u, v = np.meshgrid(np.arange(kx1 + 1) * step + 0.5, np.arange(ky1 + 1) * step + 0.5)
    gx, gy = M.global_coords(grid, zoom, size, u, v)
    return np.stack([gx, gy], axis=-1)


def choose_step(grid, zoom, size):
    """the largest G of 64, 32, ..., 1 with |exact - interpolated| <= 1/8 tile pixel in gx and gy at every cell centre"""
    for step in (64, 32, 16, 8, 4, 2, 1):
        n = nodes(grid, zoom, size, step)
        mid = _lerp(_lerp(n[:-1, :-1], n[:-1, 1:], 0.5), _lerp(n[1:, :-1], n[1:, 1:], 0.5), 0.5)
        u, v = np.meshgrid(np.arange(n.shape[1] - 1) * step + step / 2 + 0.5, np.arange(n.shape[0] - 1) * step + step / 2 + 0.5)
        gx, gy = M.global_coords(grid, zoom, size, u, v)
        with np.errstate(invalid="ignore"):
            err = np.maximum(np.abs(gx - mid[..., 0]), np.abs(gy - mid[..., 1]))
        if not (err[np.isfinite(err)] > 0.125).any():
            return step
    return 1


def render(planes, grid, zoom, size, resampling, nodata=0, step=None):
    """planes {(x, y): uint8 [size, size]} -> (uint8 [height, width] output, covered pixels, step)"""
    step = step or choose_step(grid, zoom, size)
    world = 2 ** zoom * size
    keys = np.array(sorted(planes), np.int64).reshape(-1, 2)
    (ex0, ey0), (ex1, ey1) = keys.min(axis=0), keys.max(axis=0)
    index = np.full((ey1 - ey0 + 1, ex1 - ex0 + 1), -1, np.int64)
    index[keys[:, 1] - ey0, keys[:, 0] - ex0] = np.arange(len(keys))
    stack = np.stack([planes[(int(x), int(y))] for x, y in keys]).astype(np.float64)

    def lookup(gi, gj):
        """(valid, value) of global pixels (inside the world)"""
        tx, ty = gi // size - ex0, gj // size - ey0
        inside = (tx >= 0) & (tx < index.shape[1]) & (ty >= 0) & (ty < index.shape[0])
        slot = np.where(inside, index[np.clip(ty, 0, index.shape[0] - 1), np.clip(tx, 0, index.shape[1] - 1)], -1)
        ok = slot >= 0
        return ok, stack[np.where(ok, slot, 0), gj % size, gi % size]

    n = nodes(grid, zoom, size, step)
    i, j = np.arange(grid.width), np.arange(grid.height)
    IX, IY = np.meshgrid(i // step, j // step)
    FX, FY = np.meshgrid((i % step) / step, (j % step) / step)
    n00, n10, n01, n11 = n[IY, IX], n[IY, IX + 1], n[IY + 1, IX], n[IY + 1, IX + 1]
    gx = _lerp(_lerp(n00[..., 0], n10[..., 0], FX), _lerp(n01[..., 0], n11[..., 0], FX), FY)
    gy = _lerp(_lerp(n00[..., 1], n10[..., 1], FX), _lerp(n01[..., 1], n11[..., 1], FX), FY)
    with np.errstate(invalid="ignore"):
        inside = (gx >= 0) & (gx < world) & (gy >= 0) & (gy < world)
    gi = np.where(inside, gx, 0).astype(np.int64)
    gj = np.where(inside, gy, 0).astype(np.int64)
    valid, value = lookup(gi, gj)
    covered = inside & valid
    out = np.full((grid.height, grid.width), nodata, np.uint8)
    if resampling == "nearest":
        out[covered] = value[covered].astype(np.uint8)
        return out, int(covered.sum()), step
    a, b = np.where(covered, gx, 0.5) - 0.5, np.where(covered, gy, 0.5) - 0.5
    fa0, fb0 = np.floor(a), np.floor(b)
    fa, fb = a - fa0, b - fb0
    ga, gb = 1.0 - fa, 1.0 - fb
    i0, j0 = fa0.astype(np.int64), fb0.astype(np.int64)
    ia, ib = np.clip(i0, 0, world - 1), np.clip(i0 + 1, 0, world - 1)
    ja, jb = np.clip(j0, 0, world - 1), np.clip(j0 + 1, 0, world - 1)
    acc = np.zeros(gx.shape)
    ws = np.zeros(gx.shape)
    for ti, tj, w in ((ia, ja, ga * gb), (ib, ja, fa * gb), (ia, jb, ga * fb), (ib, jb, fa * fb)):  # this order, on the device too
        ok, val = lookup(ti, tj)
        acc = np.where(ok, acc + w * val, acc)
        ws = np.where(ok, ws + w, ws)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.clip(np.floor(acc / ws + 0.5), 0, 255)
    out[covered] = q[covered].astype(np.uint8)
    return out, int(covered.sum()), step
