"""numpy float64 restatement of `rs tile --resampling average` (DESIGN.md §8), per tile and without windows, for bit-identity tests
of rsb_tile_average, robosat_b200.tile and robosat_b200.segment.

The rule, as the kernel applies it:
1. The exact (u, v) of `tile.source_coords` at the corners (kG, lG) of global pixels (the lattice of `tile.lattice(corner=True)`);
   tile (x, y) reads nodes k = floor(xS / G) .. floor((x + 1) S / G) + 1, and the same in y. G is the largest of 64 .. 1 for which
   the exact transform at every cell centre is within 1/8 source pixel of the interpolation.
2. Integer corner (gx, gy) interpolates its cell with fx = (gx - kG) / G, fy likewise, as lerp(lerp(n00, n10, fx), lerp(n01, n11,
   fx), fy), every operation rounded separately.
3. Pixel (gx, gy)'s footprint is the bounding box [u0, u1] x [v0, v1] of its corners (gx, gy) .. (gx + 1, gy + 1); a NaN corner
   leaves it uncovered. Clipped to a0 = max(u0, 0), a1 = min(u1, W), b0 = max(v0, 0), b1 = min(v1, H); empty -> uncovered.
4. wx_i = min(i + 1, a1) - max(i, a0) for i = floor(a0) .. ceil(a1) - 1, one rounded subtraction; wy_j likewise.
5. For j ascending: r_c = sum_i wx_i p_c(i, j), r_w = sum_i wx_i over valid (i, j), i ascending; A_c += wy_j r_c, Wsum += wy_j r_w.
6. Covered iff Wsum > 0; each band is floor(A_c / Wsum + 1/2) clamped to [0, 255].
7. The unclipped extent u1 - u0 or v1 - v0 may not exceed RSB_TILE_MAX_FOOTPRINT (the host refuses such runs)."""

import numpy as np

from robosat_b200 import _lib
from robosat_b200 import tile as T
from robosat_b200.rasterize import CE
from tile_reference import _lerp, valid_mask


def tile_nodes(raster, zoom, size, step, x, y):
    """(kx0, ky0, nodes) of the corner lattice cells tile (x, y) reads"""
    kx0, kx1 = (x * size) // step, ((x + 1) * size) // step + 1
    ky0, ky1 = (y * size) // step, ((y + 1) * size) // step + 1
    return kx0, ky0, T.lattice(raster, zoom, size, step, kx0, kx1, ky0, ky1, corner=True)


def choose_step(raster, zoom, size, tiles):
    """the largest G of 64, 32, ..., 1 with |exact - interpolated| <= 1/8 px in u and v at every corner-lattice cell centre"""
    for step in (64, 32, 16, 8, 4, 2, 1):
        ok = True
        for x, y in tiles:
            kx0, ky0, n = tile_nodes(raster, zoom, size, step, int(x), int(y))
            mid = _lerp(_lerp(n[:-1, :-1], n[:-1, 1:], 0.5), _lerp(n[1:, :-1], n[1:, 1:], 0.5), 0.5)
            px = CE / (2.0 ** zoom * size)
            X = -CE / 2 + ((kx0 + np.arange(n.shape[1] - 1)) * step + step / 2) * px
            Y = CE / 2 - ((ky0 + np.arange(n.shape[0] - 1)) * step + step / 2) * px
            u, v = T.source_coords(raster, *np.meshgrid(X, Y))
            err = np.maximum(np.abs(u - mid[..., 0]), np.abs(v - mid[..., 1]))
            if (err[np.isfinite(err)] > 0.125).any():
                ok = False
                break
        if ok:
            return step
    return 1


def corners(raster, zoom, size, step, x, y):
    """float64 [size + 1, size + 1, 2]: (u, v) of integer corner (x size + c, y size + r) at [r, c]"""
    kx0, ky0, n = tile_nodes(raster, zoom, size, step, x, y)
    gx = x * size + np.arange(size + 1, dtype=np.int64)
    gy = y * size + np.arange(size + 1, dtype=np.int64)
    IX, IY = np.meshgrid(gx // step - kx0, gy // step - ky0)
    FX, FY = np.meshgrid((gx - (gx // step) * step) / step, (gy - (gy // step) * step) / step)
    n00, n10, n01, n11 = n[IY, IX], n[IY, IX + 1], n[IY + 1, IX], n[IY + 1, IX + 1]
    u = _lerp(_lerp(n00[..., 0], n10[..., 0], FX), _lerp(n01[..., 0], n11[..., 0], FX), FY)
    v = _lerp(_lerp(n00[..., 1], n10[..., 1], FX), _lerp(n01[..., 1], n11[..., 1], FX), FY)
    return np.stack([u, v], axis=-1)


def footprints(C):
    """corners [h + 1, w + 1, 2] -> (u0, u1, v0, v1), each [h, w], and bool [h, w]: a corner is NaN"""
    def quad(a):
        return a[:-1, :-1], a[:-1, 1:], a[1:, :-1], a[1:, 1:]

    uq, vq = quad(C[..., 0]), quad(C[..., 1])
    nan = np.zeros(uq[0].shape, bool)
    for a in uq + vq:
        nan |= np.isnan(a)
    with np.errstate(invalid="ignore"):
        return (np.minimum(np.minimum(uq[0], uq[1]), np.minimum(uq[2], uq[3])), np.maximum(np.maximum(uq[0], uq[1]), np.maximum(uq[2], uq[3])),
                np.minimum(np.minimum(vq[0], vq[1]), np.minimum(vq[2], vq[3])), np.maximum(np.maximum(vq[0], vq[1]), np.maximum(vq[2], vq[3])), nan)


def axis_weights(lo, hi):
    """one pixel's clipped footprint [lo, hi] along one axis -> (first index, float64 weights): w_i = min(i + 1, hi) - max(i, lo)"""
    i = np.arange(int(np.floor(lo)), int(np.ceil(hi)), dtype=np.int64)
    return int(i[0]), np.minimum(i + 1.0, hi) - np.maximum(i.astype(np.float64), lo)


def render_tile(pixels, raster, zoom, size, step, x, y):
    """pixels uint8 [H, W, spp] (the whole raster) -> (uint8 [size, size, 3], covered pixels) of tile (x, y)"""
    H, W = pixels.shape[:2]
    rgb = (np.repeat(pixels[..., :1], 3, axis=-1) if pixels.shape[-1] == 1 else pixels[..., :3]).astype(np.float64)
    valid = valid_mask(pixels, raster.alpha, raster.nodata)
    u0, u1, v0, v1, nan = footprints(corners(raster, zoom, size, step, x, y))
    with np.errstate(invalid="ignore"):
        a0, a1, b0, b1 = np.maximum(u0, 0.0), np.minimum(u1, float(W)), np.maximum(v0, 0.0), np.minimum(v1, float(H))
        ok = ~nan & (a0 < a1) & (b0 < b1)
        assert not (ok & ((u1 - u0 > _lib.RSB_TILE_MAX_FOOTPRINT) | (v1 - v0 > _lib.RSB_TILE_MAX_FOOTPRINT))).any(), "over the footprint cap"
    a0, a1, b0, b1 = (np.where(ok, t, d) for t, d in ((a0, 0.0), (a1, 1.0), (b0, 0.0), (b1, 1.0)))
    i0, j0 = np.floor(a0).astype(np.int64), np.floor(b0).astype(np.int64)
    ni = np.where(ok, np.ceil(a1).astype(np.int64) - i0, 0)
    nj = np.where(ok, np.ceil(b1).astype(np.int64) - j0, 0)
    A = np.zeros((size, size, 3))
    Wsum = np.zeros((size, size))
    for dj in range(int(nj.max(initial=0))):  # rows ascending, per pixel
        j = j0 + dj
        row = dj < nj
        jc = np.clip(j, 0, H - 1)
        wy = np.minimum(j + 1.0, b1) - np.maximum(j.astype(np.float64), b0)
        R = np.zeros((size, size, 3))
        Rw = np.zeros((size, size))
        for di in range(int(ni.max(initial=0))):  # columns ascending
            i = i0 + di
            ic = np.clip(i, 0, W - 1)
            take = row & (di < ni) & valid[jc, ic]
            wx = np.minimum(i + 1.0, a1) - np.maximum(i.astype(np.float64), a0)
            R = np.where(take[..., None], R + wx[..., None] * rgb[jc, ic], R)
            Rw = np.where(take, Rw + wx, Rw)
        A = np.where(row[..., None], A + wy[..., None] * R, A)
        Wsum = np.where(row, Wsum + wy * Rw, Wsum)
    covered = ok & (Wsum > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.clip(np.floor(A / Wsum[..., None] + 0.5), 0, 255)
    out = np.zeros((size, size, 3), np.uint8)
    out[covered] = q[covered].astype(np.uint8)
    return out, int(covered.sum())


def render(pixels, raster, zoom, size, tiles, step=None):
    """{(x, y): (image, covered)} of the tiles with covered pixels, and the step used"""
    step = step or choose_step(raster, zoom, size, tiles)
    got = {}
    for x, y in tiles:
        im, c = render_tile(pixels, raster, zoom, size, step, int(x), int(y))
        if c:
            got[(int(x), int(y))] = (im, c)
    return got, step


def largest_extent(raster, zoom, size, step, tiles):
    """the largest unclipped extent (u1 - u0 or v1 - v0) of any pixel footprint of `tiles` without a NaN corner"""
    worst = 0.0
    for x, y in tiles:
        u0, u1, v0, v1, nan = footprints(corners(raster, zoom, size, step, int(x), int(y)))
        e = np.maximum(u1 - u0, v1 - v0)[~nan]
        worst = max(worst, float(e.max(initial=0.0)))
    return worst
