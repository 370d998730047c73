"""numpy float64 restatement of `rs tile`'s rule (DESIGN.md §8), per tile and without windows, for bit-identity tests of
rsb_tile_warp and robosat_b200.tile.

The exact transform at the lattice nodes is `robosat_b200.tile.lattice` (`source_coords`), whose projections test_tile.py checks
against EPSG's worked example, a numerical meridian arc, a round trip and conformality. Everything after it is restated here: the
lattice step, the per-pixel interpolation in the kernel's operation order, the coverage test, both resamplings and the candidate
tiles."""

import math

import numpy as np

from robosat_b200 import tile as T
from robosat_b200.rasterize import CE


def _lerp(a, b, t):
    return a + t * (b - a)  # three separately rounded operations, as __dadd_rn(a, __dmul_rn(t, __dsub_rn(b, a)))


def tile_nodes(raster, zoom, size, step, x, y):
    """(kx0, ky0, nodes) of the lattice cells tile (x, y) reads: nodes of global pixel centres kG, kx0 <= k <= kx1 + 1"""
    kx0, kx1 = (x * size) // step, ((x + 1) * size - 1) // step + 1
    ky0, ky1 = (y * size) // step, ((y + 1) * size - 1) // step + 1
    return kx0, ky0, T.lattice(raster, zoom, size, step, kx0, kx1, ky0, ky1)


def choose_step(raster, zoom, size, tiles):
    """the largest G of 64, 32, ..., 1 with |exact - interpolated| <= 1/8 px in u and v at every cell centre of every tile"""
    for step in (64, 32, 16, 8, 4, 2, 1):
        ok = True
        for x, y in tiles:
            kx0, ky0, n = tile_nodes(raster, zoom, size, step, int(x), int(y))
            mid = _lerp(_lerp(n[:-1, :-1], n[:-1, 1:], 0.5), _lerp(n[1:, :-1], n[1:, 1:], 0.5), 0.5)
            px = CE / (2.0 ** zoom * size)
            X = -CE / 2 + ((kx0 + np.arange(n.shape[1] - 1)) * step + step / 2 + 0.5) * px
            Y = CE / 2 - ((ky0 + np.arange(n.shape[0] - 1)) * step + step / 2 + 0.5) * px
            u, v = T.source_coords(raster, *np.meshgrid(X, Y))
            err = np.maximum(np.abs(u - mid[..., 0]), np.abs(v - mid[..., 1]))
            if (err[np.isfinite(err)] > 0.125).any():
                ok = False
                break
        if ok:
            return step
    return 1


def valid_mask(pixels, alpha, nodata):
    """bool [H, W]: alpha (4th sample) non-zero when alpha, and not every colour sample equal to nodata (-1: none)"""
    colour = pixels[..., :3] if pixels.shape[-1] >= 3 else pixels[..., :1]
    ok = np.ones(pixels.shape[:2], bool)
    if alpha:
        ok &= pixels[..., 3] != 0
    if nodata >= 0:
        ok &= ~(colour == nodata).all(axis=-1)
    return ok


def render_tile(pixels, raster, zoom, size, step, x, y, resampling):
    """pixels uint8 [H, W, spp] (the whole raster) -> (uint8 [size, size, 3], covered pixels) of tile (x, y)"""
    H, W = pixels.shape[:2]
    rgb = np.repeat(pixels[..., :1], 3, axis=-1) if pixels.shape[-1] == 1 else pixels[..., :3]
    rgb = rgb.astype(np.float64)
    valid = valid_mask(pixels, raster.alpha, raster.nodata)
    kx0, ky0, n = tile_nodes(raster, zoom, size, step, x, y)
    gx = x * size + np.arange(size, dtype=np.int64)
    gy = y * size + np.arange(size, dtype=np.int64)
    ix, iy = gx // step - kx0, gy // step - ky0
    fx = (gx - (gx // step) * step) / step
    fy = (gy - (gy // step) * step) / step
    IX, IY = np.meshgrid(ix, iy)
    FX, FY = np.meshgrid(fx, fy)
    n00, n10, n01, n11 = n[IY, IX], n[IY, IX + 1], n[IY + 1, IX], n[IY + 1, IX + 1]
    u = _lerp(_lerp(n00[..., 0], n10[..., 0], FX), _lerp(n01[..., 0], n11[..., 0], FX), FY)
    v = _lerp(_lerp(n00[..., 1], n10[..., 1], FX), _lerp(n01[..., 1], n11[..., 1], FX), FY)
    with np.errstate(invalid="ignore"):
        inside = (u >= 0) & (u < W) & (v >= 0) & (v < H)
    i = np.where(inside, u, 0).astype(np.int64)
    j = np.where(inside, v, 0).astype(np.int64)
    covered = inside & valid[j, i]
    out = np.zeros((size, size, 3), np.uint8)
    if resampling == "nearest":
        out[covered] = rgb[j, i][covered].astype(np.uint8)
        return out, int(covered.sum())
    a, b = np.where(covered, u, 0.5) - 0.5, np.where(covered, v, 0.5) - 0.5
    fa0, fb0 = np.floor(a), np.floor(b)
    fa, fb = a - fa0, b - fb0
    ga, gb = 1.0 - fa, 1.0 - fb
    i0, j0 = fa0.astype(np.int64), fb0.astype(np.int64)
    ia, ib = np.clip(i0, 0, W - 1), np.clip(i0 + 1, 0, W - 1)
    ja, jb = np.clip(j0, 0, H - 1), np.clip(j0 + 1, 0, H - 1)
    acc = np.zeros((size, size, 3))
    ws = np.zeros((size, size))
    for ti, tj, w in ((ia, ja, ga * gb), (ib, ja, fa * gb), (ia, jb, ga * fb), (ib, jb, fa * fb)):  # this order, on the device too
        ok = valid[tj, ti]
        acc = np.where(ok[..., None], acc + w[..., None] * rgb[tj, ti], acc)
        ws = np.where(ok, ws + w, ws)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.clip(np.floor(acc / ws[..., None] + 0.5), 0, 255)
    out[covered] = q[covered].astype(np.uint8)
    return out, int(covered.sum())


def render(pixels, raster, zoom, size, tiles, resampling, step=None):
    """{(x, y): (image, covered)} of the tiles with covered pixels, and the step used"""
    step = step or choose_step(raster, zoom, size, tiles)
    got = {}
    for x, y in tiles:
        im, c = render_tile(pixels, raster, zoom, size, step, int(x), int(y), resampling)
        if c:
            got[(int(x), int(y))] = (im, c)
    return got, step


def candidates_brute_force(raster, zoom, size, pad=4):
    """every tile near the footprint whose Mercator box meets it widened by one tile pixel, by a scan of tile boxes"""
    fp = T.footprint(raster)
    px = CE / (2.0 ** zoom * size)
    box = (fp[0] - px, fp[1] - px, fp[2] + px, fp[3] + px)
    side = CE / 2 ** zoom
    lo_x, hi_x = int(math.floor((box[0] + CE / 2) / side)) - pad, int(math.floor((box[2] + CE / 2) / side)) + pad
    lo_y, hi_y = int(math.floor((CE / 2 - box[3]) / side)) - pad, int(math.floor((CE / 2 - box[1]) / side)) + pad
    out = []
    for x in range(max(0, lo_x), min(2 ** zoom - 1, hi_x) + 1):
        for y in range(max(0, lo_y), min(2 ** zoom - 1, hi_y) + 1):
            left, top = x * side - CE / 2, CE / 2 - y * side
            if left <= box[2] and left + side >= box[0] and top - side <= box[3] and top >= box[1]:
                out.append((x, y))
    return sorted(out)
