"""`rs tile`: slippy-map RGB tiles cut from a GeoTIFF, with the reprojection and the resampling on the GPU.

The rule is this project's own (the reference gets imagery only by downloading tiles) and is written down in DESIGN.md §8 and
restated in tests/tile_reference.py:

- Pixel (c, r) of tile (x, y, z) of S x S pixels is global pixel (gx, gy) = (x S + c, y S + r), centred at
  X = -CE/2 + (gx + 1/2) CE / (2^z S), Y = CE/2 - (gy + 1/2) CE / (2^z S) in EPSG:3857 (the frame of `rasterize.xy_bounds`).
- `source_coords` maps EPSG:3857 to the raster's CRS (the identity, spherical lon/lat, or lon/lat and then the WGS 84 transverse
  Mercator of a UTM zone as Krüger's series to order n^6, Karney 2011) and then through the inverse geotransform to raster
  coordinates (u, v); pixel (i, j) covers [i, i + 1) x [j, j + 1).
- The exact (u, v) is computed here, in numpy, only at the nodes of a lattice of every G global pixels (shared by neighbouring
  tiles); `rsb_tile_warp` interpolates them bilinearly per pixel. G is the largest of 64, 32, ..., 1 for which the exact transform
  at every lattice cell centre of the candidate tiles is within 1/8 source pixel of the interpolated one.
- A pixel is covered when (floor(u), floor(v)) is a valid pixel of the raster; nearest takes that pixel, bilinear the four
  neighbours of (u - 1/2, v - 1/2) clamped to the raster with invalid ones dropped and the weights renormalised. Uncovered pixels
  are (0, 0, 0).
- Candidate tiles are those whose Mercator box meets the raster footprint (the box of the raster boundary sampled at every edge
  pixel corner, widened by one tile pixel); a tile is produced only when it has a covered pixel.
- Area averaging (`average`, `rsb_tile_average`) takes the lattice at pixel corners instead (`corner=True` below): each pixel
  averages the source pixels under the bounding box of its four interpolated corners, weighted by their overlap with it. A footprint
  may span at most RSB_TILE_MAX_FOOTPRINT source pixels; `plan` refuses a run that could exceed it.

Work goes in windows: a run of at most `batch` adjacent tiles of one tile row, whose source rows and columns (from the lattice,
plus 2 pixels) and output fit `budget` device bytes. The next window is decoded on a host thread while the current one is warped,
and a caller's sink (the PNG writer of the tool) runs on another thread.
"""

import math
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from robosat_b200 import _lib
from robosat_b200.rasterize import CE, R

WGS84_A = 6378137.0
WGS84_F = 1 / 298.257223563
UTM_K0 = 0.9996
DEFAULT_BUDGET = 1 << 30
DEFAULT_BATCH = 64
STEPS = (64, 32, 16, 8, 4, 2, 1)
TOLERANCE = 0.125  # source pixels between the exact transform and the lattice interpolation at every cell centre
MARGIN = 2  # source pixels added around a window's lattice range
RESAMPLING = {"nearest": 0, "bilinear": 1}  # the codes of rsb_tile_warp
RESAMPLINGS = ("nearest", "bilinear", "average")  # average runs rsb_tile_average on the corner lattice
W_COARSE = "Warning: a zoom {} pixel spans {:.1f} raster pixels; bilinear resampling aliases above 2 (use --resampling average)"
FOOTPRINT_SLACK = 1e-6  # source pixels added to the host's bound of a footprint's extent, for the rounding of the interpolation


# ---- projections (numpy float64, elementwise) ----

def tm_series(f):
    """n, the rectifying radius factor A / a and Krüger's alpha and beta coefficients 1..6 (Karney 2011, eqs. 14, 35, 36)"""
    n = f / (2 - f)
    n2, n3, n4, n5, n6 = n ** 2, n ** 3, n ** 4, n ** 5, n ** 6
    A = (1 + n2 / 4 + n4 / 64 + n6 / 256) / (1 + n)
    alpha = (n / 2 - 2 * n2 / 3 + 5 * n3 / 16 + 41 * n4 / 180 - 127 * n5 / 288 + 7891 * n6 / 37800,
             13 * n2 / 48 - 3 * n3 / 5 + 557 * n4 / 1440 + 281 * n5 / 630 - 1983433 * n6 / 1935360,
             61 * n3 / 240 - 103 * n4 / 140 + 15061 * n5 / 26880 + 167603 * n6 / 181440,
             49561 * n4 / 161280 - 179 * n5 / 168 + 6601661 * n6 / 7257600,
             34729 * n5 / 80640 - 3418889 * n6 / 1995840,
             212378941 * n6 / 319334400)
    beta = (n / 2 - 2 * n2 / 3 + 37 * n3 / 96 - n4 / 360 - 81 * n5 / 512 + 96199 * n6 / 604800,
            n2 / 48 + n3 / 15 - 437 * n4 / 1440 + 46 * n5 / 105 - 1118711 * n6 / 3870720,
            17 * n3 / 480 - 37 * n4 / 840 - 209 * n5 / 4480 + 5569 * n6 / 90720,
            4397 * n4 / 161280 - 11 * n5 / 504 - 830251 * n6 / 7257600,
            4583 * n5 / 161280 - 108847 * n6 / 3991680,
            20648693 * n6 / 638668800)
    return n, A, alpha, beta


def _tm_xy(phi, lam, e, alpha):
    """conformal latitude, then Krüger's series: (eta, xi) on the unit rectifying sphere"""
    s = np.sin(phi)
    t = np.sinh(np.arctanh(s) - e * np.arctanh(e * s))
    xi_p = np.arctan2(t, np.cos(lam))
    eta_p = np.arctanh(np.sin(lam) / np.sqrt(1 + t * t))
    xi, eta = xi_p.copy(), eta_p.copy()
    for j, a in enumerate(alpha, 1):
        xi = xi + a * np.sin(2 * j * xi_p) * np.cosh(2 * j * eta_p)
        eta = eta + a * np.cos(2 * j * xi_p) * np.sinh(2 * j * eta_p)
    return eta, xi


def tm_forward(lon, lat, lon0, k0=UTM_K0, fe=500000.0, fn=0.0, lat0=0.0, a=WGS84_A, f=WGS84_F):
    """transverse Mercator (degrees -> easting, northing in metres) as Krüger's series of order n^6"""
    _, A, alpha, _ = tm_series(f)
    e = math.sqrt(f * (2 - f))
    eta, xi = _tm_xy(np.radians(np.asarray(lat, np.float64)), np.radians(np.asarray(lon, np.float64) - lon0), e, alpha)
    xi0 = 0.0
    if lat0:
        xi0 = float(_tm_xy(np.radians(np.float64(lat0)), np.float64(0.0), e, alpha)[1])
    return fe + k0 * a * A * eta, fn + k0 * a * A * (xi - xi0)


def tm_inverse(easting, northing, lon0, k0=UTM_K0, fe=500000.0, fn=0.0, a=WGS84_A, f=WGS84_F):
    """inverse of `tm_forward` with lat0 = 0 -> (lon, lat) in degrees (Karney 2011, eqs. 11, 15, 18-21)"""
    _, A, _, beta = tm_series(f)
    e = math.sqrt(f * (2 - f))
    eta = (np.asarray(easting, np.float64) - fe) / (k0 * a * A)
    xi = (np.asarray(northing, np.float64) - fn) / (k0 * a * A)
    xi_p, eta_p = xi.copy(), eta.copy()
    for j, b in enumerate(beta, 1):
        xi_p = xi_p - b * np.sin(2 * j * xi) * np.cosh(2 * j * eta)
        eta_p = eta_p - b * np.cos(2 * j * xi) * np.sinh(2 * j * eta)
    tau_p = np.sin(xi_p) / np.sqrt(np.sinh(eta_p) ** 2 + np.cos(xi_p) ** 2)
    lam = np.arctan2(np.sinh(eta_p), np.cos(xi_p))
    tau = tau_p.copy()
    e2 = e * e
    for _ in range(5):  # Newton on tau' (tau) = tau_p
        sig = np.sinh(e * np.arctanh(e * tau / np.sqrt(1 + tau * tau)))
        tp = tau * np.sqrt(1 + sig * sig) - sig * np.sqrt(1 + tau * tau)
        tau = tau + (tau_p - tp) / np.sqrt(1 + tp * tp) * (1 + (1 - e2) * tau * tau) / ((1 - e2) * np.sqrt(1 + tau * tau))
    return lon0 + np.degrees(lam), np.degrees(np.arctan(tau))


def mercator_to_lonlat(X, Y):
    return np.degrees(np.asarray(X, np.float64) / R), np.degrees(np.arctan(np.sinh(np.asarray(Y, np.float64) / R)))


def lonlat_to_mercator(lon, lat):
    """rasterize.project on arrays; latitudes beyond ±90 give NaN"""
    with np.errstate(invalid="ignore", divide="ignore"):
        return R * np.radians(lon), R * np.log(np.tan(np.pi / 4 + np.radians(lat) / 2))


def utm_params(crs):
    _, zone, south = crs
    return 6.0 * zone - 183.0, 10000000.0 if south else 0.0


def model_of_mercator(crs, X, Y):
    """EPSG:3857 -> the raster's CRS (GeoTiff.crs)"""
    X, Y = np.asarray(X, np.float64), np.asarray(Y, np.float64)
    if crs == "3857":
        return X, Y
    lon, lat = mercator_to_lonlat(X, Y)
    if crs == "4326":
        return lon, lat
    lon0, fn = utm_params(crs)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return tm_forward(lon, lat, lon0, fn=fn)


def mercator_of_model(crs, mx, my):
    """the raster's CRS -> EPSG:3857"""
    mx, my = np.asarray(mx, np.float64), np.asarray(my, np.float64)
    if crs == "3857":
        return mx, my
    if crs == "4326":
        return lonlat_to_mercator(mx, my)
    lon0, fn = utm_params(crs)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return lonlat_to_mercator(*tm_inverse(mx, my, lon0, fn=fn))


def inverse_geotransform(gt):
    c, a, b, f, d, e = gt
    det = a * e - b * d
    ia, ib, id_, ie = e / det, -b / det, -d / det, a / det
    return -(ia * c + ib * f), ia, ib, -(id_ * c + ie * f), id_, ie


def source_coords(raster, X, Y):
    """EPSG:3857 (X, Y) -> raster coordinates (u, v) of `raster` (a GeoTiff, or anything with .crs and .geotransform); the exact
    transform the lattice nodes take"""
    mx, my = model_of_mercator(raster.crs, X, Y)
    c, a, b, f, d, e = inverse_geotransform(raster.geotransform)
    return c + a * mx + b * my, f + d * mx + e * my


def pixel_centre(g, zoom, size, corner=False):
    """global pixel index -> Mercator coordinate of its centre (its left corner when `corner`) along x (Y is its negation)"""
    g = np.asarray(g, np.float64)
    return -CE / 2 + (g if corner else g + 0.5) * (CE / (2.0 ** zoom * size))


def lattice(raster, zoom, size, step, kx0, kx1, ky0, ky1, corner=False):
    """float64 [ky1 - ky0 + 1, kx1 - kx0 + 1, 2]: (u, v) at the centres (the top-left corners when `corner`) of global pixels
    (k step, l step), kx0 <= k <= kx1, ky0 <= l <= ky1"""
    X = pixel_centre(np.arange(kx0, kx1 + 1, dtype=np.int64) * step, zoom, size, corner)
    Y = -pixel_centre(np.arange(ky0, ky1 + 1, dtype=np.int64) * step, zoom, size, corner)
    u, v = source_coords(raster, *np.meshgrid(X, Y))
    return np.ascontiguousarray(np.stack([u, v], axis=-1))


def last_node(t, size, lg, corner=False):
    """the last lattice node tile t (along one axis) reads: its last pixel's centre, or its far corner, lies in the cell before it"""
    return (((t + 1) * size - (0 if corner else 1)) >> lg) + 1


def run_nodes(raster, zoom, size, step, y, xa, xb, corner=False):
    """(kx0, ky0, nodes) of the lattice that tiles xa..xb of tile row y read"""
    lg = step.bit_length() - 1
    kx0, kx1 = (xa * size) >> lg, last_node(xb, size, lg, corner)
    ky0, ky1 = (y * size) >> lg, last_node(y, size, lg, corner)
    return kx0, ky0, lattice(raster, zoom, size, step, kx0, kx1, ky0, ky1, corner)


# ---- planning ----

def footprint(raster):
    """(xmin, ymin, xmax, ymax) in EPSG:3857 of the raster boundary sampled at every edge pixel corner"""
    W, H = raster.width, raster.height
    i, j = np.arange(W + 1, dtype=np.float64), np.arange(H + 1, dtype=np.float64)
    u = np.concatenate([i, i, np.zeros(H + 1), np.full(H + 1, float(W))])
    v = np.concatenate([np.zeros(W + 1), np.full(W + 1, float(H)), j, j])
    c, a, b, f, d, e = raster.geotransform
    X, Y = mercator_of_model(raster.crs, c + a * u + b * v, f + d * u + e * v)
    ok = np.isfinite(X) & np.isfinite(Y)
    if not ok.any():
        return None
    return X[ok].min(), Y[ok].min(), X[ok].max(), Y[ok].max()


def tile_meets(x, y, zoom, box):
    """whether the closed Mercator box of tile (x, y) (rasterize.xy_bounds) meets `box`"""
    side = CE / 2 ** zoom
    left = x * side - CE / 2
    top = CE / 2 - y * side
    return (left <= box[2]) & (left + side >= box[0]) & (top - side <= box[3]) & (top >= box[1])


def candidate_tiles(raster, zoom, size):
    """int64 [n, 2] (x, y) sorted by (x, y): the tiles whose Mercator box meets the footprint widened by one tile pixel"""
    fp = footprint(raster)
    if fp is None:
        return np.zeros((0, 2), np.int64)
    px = CE / (2.0 ** zoom * size)
    box = (fp[0] - px, fp[1] - px, fp[2] + px, fp[3] + px)
    side, last = CE / 2 ** zoom, 2 ** zoom - 1

    def span(lo, hi):
        return max(0, int(math.floor(lo / side)) - 1), min(last, int(math.floor(hi / side)) + 1)

    x0, x1 = span(box[0] + CE / 2, box[2] + CE / 2)
    y0, y1 = span(CE / 2 - box[3], CE / 2 - box[1])
    if x0 > x1 or y0 > y1:
        return np.zeros((0, 2), np.int64)
    xs = np.arange(x0, x1 + 1, dtype=np.int64)
    ys = np.arange(y0, y1 + 1, dtype=np.int64)
    xs = xs[tile_meets(xs, np.full(len(xs), y0), zoom, (box[0], -np.inf, box[2], np.inf))]
    ys = ys[tile_meets(np.full(len(ys), x0), ys, zoom, (-np.inf, box[1], np.inf, box[3]))]
    gx, gy = np.meshgrid(xs, ys, indexing="ij")
    return np.stack([gx.ravel(), gy.ravel()], axis=1)


def runs(tiles):
    """(y, xa, xb) per run of adjacent tiles in one tile row, over tiles int64 [n, 2] of distinct tiles"""
    out = []
    t = np.asarray(tiles, np.int64).reshape(-1, 2)
    for y in np.unique(t[:, 1]):
        xs = np.sort(t[t[:, 1] == y, 0])
        breaks = np.flatnonzero(np.diff(xs) != 1)
        starts = np.concatenate([[0], breaks + 1])
        ends = np.concatenate([breaks, [len(xs) - 1]])
        out.extend((int(y), int(xs[s]), int(xs[e])) for s, e in zip(starts, ends))
    return out


def _lerp(a, b, t):
    return a + t * (b - a)


def step_error(raster, zoom, size, step, run, corner=False):
    """the largest |exact - interpolated| (u or v, source pixels) at the lattice cell centres of a run; NaN cells are skipped"""
    y, xa, xb = run
    kx0, ky0, nodes = run_nodes(raster, zoom, size, step, y, xa, xb, corner)
    mid = _lerp(_lerp(nodes[:-1, :-1], nodes[:-1, 1:], 0.5), _lerp(nodes[1:, :-1], nodes[1:, 1:], 0.5), 0.5)
    ny, nx = nodes.shape[0] - 1, nodes.shape[1] - 1
    X = pixel_centre((np.arange(kx0, kx0 + nx, dtype=np.int64) * step).astype(np.float64) + step / 2, zoom, size, corner)
    Y = -pixel_centre((np.arange(ky0, ky0 + ny, dtype=np.int64) * step).astype(np.float64) + step / 2, zoom, size, corner)
    u, v = source_coords(raster, *np.meshgrid(X, Y))
    err = np.maximum(np.abs(u - mid[..., 0]), np.abs(v - mid[..., 1]))
    err = err[np.isfinite(err)]
    return float(err.max()) if len(err) else 0.0


def choose_step(raster, zoom, size, tiles, corner=False):
    """the largest lattice step of STEPS that meets TOLERANCE on every run of `tiles`"""
    rs = runs(tiles)
    for step in STEPS:
        if all(step_error(raster, zoom, size, step, r, corner) <= TOLERANCE for r in rs):
            return step
    return 1


def footprint_bound(nodes, step):
    """an upper bound of the unclipped extent (u1 - u0 or v1 - v0, source pixels) of every pixel footprint inside a block of corner
    nodes [h, w, 2]: u is bilinear in each cell, so across one pixel (1 / step of a cell) it changes by at most (the largest |du| along
    the cell's x edges + the largest along its y edges) / step; FOOTPRINT_SLACK covers the rounding of the interpolation. 0 when no
    cell is finite."""
    dx = np.abs(nodes[:, 1:] - nodes[:, :-1])  # [h, w - 1, 2]
    dy = np.abs(nodes[1:] - nodes[:-1])  # [h - 1, w, 2]
    with np.errstate(invalid="ignore"):
        ext = (np.maximum(dx[:-1], dx[1:]) + np.maximum(dy[:, :-1], dy[:, 1:])) / step  # per cell and coordinate
    ext = ext[np.isfinite(ext)]
    return float(ext.max()) * (1 + 1e-12) + FOOTPRINT_SLACK if len(ext) else 0.0


def source_box(nodes, raster):
    """(row0, rows, col0, cols) of the raster a block of lattice nodes can sample (their range plus MARGIN pixels, clipped to the
    raster), or None when it samples nothing"""
    u, v = nodes[..., 0], nodes[..., 1]
    ok = np.isfinite(u) & np.isfinite(v)
    if not ok.any():
        return None
    c0 = max(0, int(math.floor(u[ok].min())) - MARGIN)
    c1 = min(raster.width, int(math.floor(u[ok].max())) + MARGIN + 1)
    r0 = max(0, int(math.floor(v[ok].min())) - MARGIN)
    r1 = min(raster.height, int(math.floor(v[ok].max())) + MARGIN + 1)
    if c0 >= c1 or r0 >= r1:
        return None
    return r0, r1 - r0, c0, c1 - c0


class Window:
    """tiles xs[0]..xs[-1] (adjacent) of tile row y, the lattice they read (nodes [h, w, 2] from node (kx0, ky0)) and the source
    rows [row0, row0 + rows) x columns [col0, col0 + cols) their samples can reach"""

    def __init__(self, y, xs, kx0, ky0, nodes, box):
        self.y, self.xs, self.kx0, self.ky0, self.nodes = y, xs, kx0, ky0, nodes
        self.row0, self.rows, self.col0, self.cols = box

    def device_bytes(self, raster, size):
        return window_bytes(source_bytes(raster, (self.row0, self.rows, self.col0, self.cols)), len(self.xs), size, self.nodes.size * 8)


def window_bytes(src_bytes, n, size, node_bytes):
    return src_bytes + n * size * size * 3 + node_bytes + n * 32 + 8


def is_jpeg(raster):
    return getattr(raster, "compression", None) == 7


def is_bands(raster):
    """whether `raster` is read under the band rule (geotiff.BandTiff): its windows are rendered to RGBA before the warp"""
    return hasattr(raster, "bands")


def raw_bytes(raster, rows, cols):
    """bytes of a decoded window of rows x cols pixels: spp samples per pixel, or for a band raster k samples of bits / 8 bytes"""
    return rows * cols * (raster.k * raster.sample_bytes if is_bands(raster) else raster.spp)


def source_bytes(raster, box):
    """device bytes of a source window (row0, rows, col0, cols): its pixels, plus for a JPEG raster the staged bytes and the decoder
    scratch of the chunks it touches (jpeg.extra_bytes), and for a band raster its RGBA rendering"""
    n = raw_bytes(raster, box[1], box[3])
    if is_bands(raster):
        n += box[1] * box[3] * 4
    if is_jpeg(raster):
        from robosat_b200 import jpeg

        n += jpeg.extra_bytes(raster, *box)
    return n


def plan(raster, zoom, size, tiles, step, budget=DEFAULT_BUDGET, batch=DEFAULT_BATCH, corner=False):
    """the windows of `tiles` (int64 [n, 2], distinct) on the centre lattice, or the corner lattice of area averaging when `corner`;
    tiles whose lattice samples no raster pixel are in no window. RsbError when one tile alone needs more than `budget` device
    bytes, and, on the corner lattice, when a footprint of a tile may span more than RSB_TILE_MAX_FOOTPRINT source pixels."""
    lg = step.bit_length() - 1
    windows = []
    for y, xa, xb in runs(tiles):
        kx0, ky0, nodes = run_nodes(raster, zoom, size, step, y, xa, xb, corner)
        cur = None
        for x in range(xa, xb + 1):
            a = ((x * size) >> lg) - kx0
            b = last_node(x, size, lg, corner) - kx0
            box = source_box(nodes[:, a:b + 1], raster)
            if box is None:
                cur = None
                continue
            if corner:
                extent = footprint_bound(nodes[:, a:b + 1], step)
                if extent > _lib.RSB_TILE_MAX_FOOTPRINT:
                    raise _lib.RsbError("a pixel of tile (%d, %d, %d) may span %.1f source pixels, more than the %d that area averaging sums; "
                                        "use a higher zoom (smaller tile pixels span fewer source pixels)" % (
                                            x, y, zoom, extent, _lib.RSB_TILE_MAX_FOOTPRINT))
            alone = window_bytes(source_bytes(raster, box), 1, size, nodes[:, a:b + 1].size * 8)
            if alone > budget:
                raise _lib.RsbError("tile (%d, %d, %d) needs %d device bytes (a %d x %d source window), more than the budget of %d bytes" % (
                    x, y, zoom, alone, box[3], box[1], budget))
            if cur is not None and len(cur.xs) < batch:
                r0, c0 = min(cur.row0, box[0]), min(cur.col0, box[2])
                merged = (r0, max(cur.row0 + cur.rows, box[0] + box[1]) - r0, c0, max(cur.col0 + cur.cols, box[2] + box[3]) - c0)
                ca = ((cur.xs[0] * size) >> lg) - kx0
                trial = Window(y, cur.xs + [x], kx0 + ca, ky0, nodes[:, ca:b + 1], merged)
                if trial.device_bytes(raster, size) <= budget:
                    windows[-1] = cur = trial
                    continue
            cur = Window(y, [x], kx0 + a, ky0, nodes[:, a:b + 1], box)
            windows.append(cur)
    return windows


def coarse_ratio(raster, zoom, size):
    """raster pixels per zoom pixel at the raster's centre (the longer of the two steps)"""
    c, a, b, f, d, e = raster.geotransform
    X, Y = mercator_of_model(raster.crs, c + a * raster.width / 2 + b * raster.height / 2, f + d * raster.width / 2 + e * raster.height / 2)
    px = CE / (2.0 ** zoom * size)
    u, v = source_coords(raster, np.array([X, X + px, X]), np.array([Y, Y, Y - px]))
    return float(max(math.hypot(u[1] - u[0], v[1] - v[0]), math.hypot(u[2] - u[0], v[2] - v[0])))


# ---- execution ----

def entry_point(resampling):
    return "rsb_tile_average" if resampling == "average" else "rsb_tile_warp"


def render(lib, raster, src, rows, cols, out):
    """rsb_tile_render of a band raster's decoded window `src` (rows x cols pixels) into `out`, RGBA rows of 4 cols bytes (device
    pointers), with the raster's scale, on the current stream"""
    if raster.scale is None:
        raise _lib.RsbError("%s: %d-bit samples need --scale or --stretch" % (raster.path, raster.bits))
    scale = np.asarray(raster.scale, np.int32).reshape(-1)
    _lib.check(lib.rsb_tile_render(src, rows, cols, raster.bits, len(raster.bands), int(raster.alpha), raster.nodata, scale.ctypes.data, out,
                                   cols * 4, _lib.current_stream_ptr()), "rsb_tile_render")


def warp_layout(raster):
    """(spp, alpha, nodata) of the pixels the warp reads: the raster's own, or RGBA with alpha validity for a band raster"""
    return (4, 1, -1) if is_bands(raster) else (raster.spp, int(raster.alpha), raster.nodata)


def warp(lib, resampling, src, w, raster, nodes, step, tiles, n, size, out, image_stride, covered, misses):
    """one launch of rsb_tile_warp or rsb_tile_average (device pointers) over Window `w`'s source (for a band raster, its RGBA
    rendering) and lattice, on the current stream"""
    spp, alpha, nodata = warp_layout(raster)
    args = (src, w.cols * spp, w.row0, w.col0, w.rows, w.cols, raster.width, raster.height, spp, alpha, nodata,
            nodes, w.kx0, w.ky0, w.nodes.shape[1], w.nodes.shape[0], step, tiles, n, size)
    tail = (out, image_stride, covered, misses, _lib.current_stream_ptr())
    if resampling == "average":
        _lib.check(lib.rsb_tile_average(*args, *tail), "rsb_tile_average")
    else:
        _lib.check(lib.rsb_tile_warp(*args, RESAMPLING[resampling], *tail), "rsb_tile_warp")


def _pinned(n):
    import torch

    return torch.empty((max(1, n),), dtype=torch.uint8, pin_memory=True)


def run(raster, zoom, size, resampling="bilinear", tiles=None, sink=None, budget=DEFAULT_BUDGET, batch=DEFAULT_BATCH, device="cuda", stats=None,
        threads=None):
    """Warp the candidate tiles of `raster` (a GeoTiff), intersected with `tiles` (iterable of (x, y)) when given. For every window,
    sink(xy int64 [n, 2], images uint8 [n, size, size, 3], covered int64 [n]) is called on a writer thread with the tiles that have
    covered pixels (the arrays are reused after the call returns). Returns the int64 [n, 2] candidate tiles. `stats`, a dict,
    receives the lattice step and seconds of decode, upload, render and warp (CUDA events) and sink. For a JPEG raster, decode is the
    staging of the chunks' entropy-coded bytes on the host and upload includes their decode on the device. A band raster
    (geotiff.BandTiff) is decoded to its raw samples, uploaded, and rendered to RGBA by rsb_tile_render before the warp."""
    import torch

    if resampling not in RESAMPLINGS:
        raise ValueError("resampling must be one of %s" % ", ".join(RESAMPLINGS))
    if not 0 <= zoom <= _lib.RSB_COVER_MAX_ZOOM or not 1 <= size <= _lib.RSB_TILE_MAX_SIZE:
        raise ValueError("zoom must be in 0..%d and size in 1..%d" % (_lib.RSB_COVER_MAX_ZOOM, _lib.RSB_TILE_MAX_SIZE))
    stats = stats if stats is not None else {}
    cand = candidate_tiles(raster, zoom, size)
    if tiles is not None:
        want = {(int(x), int(y)) for x, y in tiles}
        cand = cand[np.array([(int(x), int(y)) in want for x, y in cand], bool)] if len(cand) else cand
    corner = resampling == "average"
    step = choose_step(raster, zoom, size, cand, corner)
    windows = plan(raster, zoom, size, cand, step, budget, batch, corner)
    stats.update(step=step, candidates=len(cand), windows=len(windows), decode_s=0.0, upload_s=0.0, render_s=0.0, warp_s=0.0, sink_s=0.0,
                 written=0)
    if not windows:
        return cand
    from robosat_b200.cover import _alloc

    dev = torch.device(device)
    bands = is_bands(raster)
    jpeg_host = _jpeg_buffers(raster, windows, dev)
    if jpeg_host:
        src_host = jpeg_host["data"]
    else:
        src_host = [_pinned(max(raw_bytes(raster, w.rows, w.cols) for w in windows)) for _ in range(2)]
    nmax = max(len(w.xs) for w in windows)
    out_host = [_pinned(nmax * size * size * 3) for _ in range(2)]
    counts_host = [torch.empty((nmax,), dtype=torch.int64, pin_memory=True) for _ in range(2)]
    misses_host = torch.empty((1,), dtype=torch.int64, pin_memory=True)
    lib = _lib.load()

    def decode(k):
        t0 = time.perf_counter()
        w = windows[k]
        if jpeg_host:
            jpeg_host["staged"][k % 2] = _jpeg_stage(raster, w, jpeg_host, k % 2)
        else:
            raster.read_window(w.row0, w.rows, w.col0, w.cols, out=src_host[k % 2].numpy(), threads=threads)
        return time.perf_counter() - t0

    def deliver(k, n):
        t0 = time.perf_counter()
        w = windows[k]
        c = counts_host[k % 2].numpy()[:n].copy()
        keep = np.flatnonzero(c > 0)
        if len(keep) and sink is not None:
            images = out_host[k % 2].numpy()[:n * size * size * 3].reshape(n, size, size, 3)
            xy = np.stack([np.asarray(w.xs, np.int64), np.full(n, w.y, np.int64)], axis=1)
            if len(keep) < n:
                sink(xy[keep], images[keep], c[keep])
            else:
                sink(xy, images, c)
        return time.perf_counter() - t0, len(keep)

    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rendered = torch.cuda.Event(enable_timing=True)
    stream = torch.cuda.current_stream(dev)
    with ThreadPoolExecutor(1) as decoder, ThreadPoolExecutor(1) as writer:
        pending = decoder.submit(decode, 0)
        writes = [None, None]
        try:
            for k, w in enumerate(windows):
                stats["decode_s"] += pending.result()
                if k + 1 < len(windows):
                    pending = decoder.submit(decode, k + 1)  # into the other pinned buffer, while this window is warped
                n = len(w.xs)
                t0 = time.perf_counter()
                src = _alloc((raw_bytes(raster, w.rows, w.cols),), torch.uint8, dev, "the %d x %d source window" % (w.cols, w.rows))
                if jpeg_host:
                    keep = _jpeg_decode(jpeg_host, k % 2, src)
                else:
                    src.copy_(src_host[k % 2][:src.numel()], non_blocking=True)
                nodes = torch.from_numpy(np.ascontiguousarray(w.nodes)).to(dev)
                xy = torch.tensor([[x, w.y] for x in w.xs], dtype=torch.int64).to(dev)
                torch.cuda.synchronize(dev)
                if jpeg_host:
                    del keep
                    _jpeg_check(jpeg_host, k % 2)
                stats["upload_s"] += time.perf_counter() - t0
                out = _alloc((n, size, size, 3), torch.uint8, dev, "%d output tiles" % n)
                covered = torch.empty((n,), dtype=torch.int64, device=dev)
                misses = torch.empty((1,), dtype=torch.int64, device=dev)
                start.record(stream)
                pixels = src
                if bands:
                    pixels = _alloc((w.rows * w.cols * 4,), torch.uint8, dev, "the %d x %d RGBA window" % (w.cols, w.rows))
                    render(lib, raster, src.data_ptr(), w.rows, w.cols, pixels.data_ptr())
                rendered.record(stream)
                warp(lib, resampling, pixels.data_ptr(), w, raster, nodes.data_ptr(), step, xy.data_ptr(), n, size, out.data_ptr(), size * size * 3,
                     covered.data_ptr(), misses.data_ptr())
                end.record(stream)
                if writes[k % 2] is not None:  # the writer is done with this buffer pair before it is overwritten
                    dt, kept = writes[k % 2].result()
                    stats["sink_s"] += dt
                    stats["written"] += kept
                out_host[k % 2][:out.numel()].copy_(out.view(-1), non_blocking=True)
                counts_host[k % 2][:n].copy_(covered, non_blocking=True)
                misses_host.copy_(misses, non_blocking=True)
                torch.cuda.synchronize(dev)
                stats["render_s"] += start.elapsed_time(rendered) / 1e3
                stats["warp_s"] += rendered.elapsed_time(end) / 1e3
                if int(misses_host[0]):
                    raise _lib.RsbError("%s: %d samples of tiles %d..%d of row %d fell outside their source window (a planning error)" % (
                        entry_point(resampling), int(misses_host[0]), w.xs[0], w.xs[-1], w.y))
                del src, pixels, out
                writes[k % 2] = writer.submit(deliver, k, n)
        finally:
            for f in writes:
                if f is not None:
                    dt, kept = f.result()
                    stats["sink_s"] += dt
                    stats["written"] += kept
    return cand


def _jpeg_buffers(raster, windows, dev):
    """for a JPEG raster: the decoder and two sets of pinned staging buffers sized for the largest of `windows`; None otherwise"""
    import torch

    if not is_jpeg(raster):
        return None
    from robosat_b200 import jpeg

    nbytes, chunks = jpeg.stage_sizes(raster, [(w.row0, w.rows, w.col0, w.cols) for w in windows])
    return dict(decoder=raster.jpeg_decoder(dev), data=[_pinned(nbytes) for _ in range(2)],
                descs=[torch.empty((chunks * jpeg.F,), dtype=torch.int64, pin_memory=True) for _ in range(2)],
                sets=[torch.empty((chunks * _lib.RSB_JPEG_SET_WORDS,), dtype=torch.int32, pin_memory=True) for _ in range(2)],
                errors=[torch.empty((chunks,), dtype=torch.int64, pin_memory=True) for _ in range(2)], staged=[None, None])


def _jpeg_stage(raster, w, bufs, i):
    from robosat_b200 import jpeg

    return jpeg.stage(raster, w.row0, w.rows, w.col0, w.cols, bufs["data"][i].numpy(), bufs["descs"][i].numpy(), bufs["sets"][i].numpy())


def _jpeg_decode(bufs, i, src):
    """the upload and decode of staging buffer i into the device window `src`, on the current stream"""
    return bufs["decoder"].decode(bufs["staged"][i], bufs["data"][i], bufs["descs"][i], bufs["sets"][i], src, bufs["errors"][i])


def _jpeg_check(bufs, i):
    bufs["decoder"].check(bufs["staged"][i], bufs["errors"][i])


def tile_device(raster, zoom, size, resampling="bilinear", tiles=None, budget=DEFAULT_BUDGET, batch=DEFAULT_BATCH, stats=None):
    """`run` collected: {(x, y): (uint8 [size, size, 3] image, covered pixels)} of the tiles with covered pixels"""
    got = {}

    def sink(xy, images, counts):
        for (x, y), im, c in zip(xy.tolist(), images, counts.tolist()):
            got[(x, y)] = (im.copy(), c)

    run(raster, zoom, size, resampling, tiles, sink, budget, batch, stats=stats)
    return got


# ---- the band rule's contrast stretch ----

DEFAULT_STATS_BUDGET = 256 << 20  # bytes of one row band of decoded samples (two pinned host copies, one device copy)


def band_stats(raster, budget=DEFAULT_STATS_BUDGET, device="cuda", threads=None, stats=None):
    """int64 [len(raster.bands), 2^bits]: the count of every value of each selected band over the valid pixels of the whole band
    raster (geotiff.BandTiff), from rsb_band_histogram. The raster goes in full-width row bands of whole chunk rows under `budget`
    bytes; each band is decoded on a host thread while the previous one is counted. `stats`, a dict, receives stats_s (seconds,
    wall clock) and stats_bands (the row bands)."""
    import torch

    t0 = time.perf_counter()
    dev = torch.device(device)
    row_bytes = raw_bytes(raster, 1, raster.width)
    step = max(1, budget // row_bytes // raster.chunk_h) * raster.chunk_h  # whole chunk rows: each chunk is decoded once
    step = min(step, raster.height)
    spans = [(r, min(step, raster.height - r)) for r in range(0, raster.height, step)]
    host = [_pinned(step * row_bytes) for _ in range(min(2, len(spans)))]
    src = torch.empty((step * row_bytes,), dtype=torch.uint8, device=dev)
    hist = torch.zeros((len(raster.bands), 1 << raster.bits), dtype=torch.int64, device=dev)
    lib = _lib.load()

    def decode(i):
        r0, rows = spans[i]
        raster.read_window(r0, rows, 0, raster.width, out=host[i % 2].numpy(), threads=threads)

    with ThreadPoolExecutor(1) as decoder:
        pending = decoder.submit(decode, 0)
        for i, (r0, rows) in enumerate(spans):
            pending.result()
            if i + 1 < len(spans):
                pending = decoder.submit(decode, i + 1)  # into the other pinned buffer, while this band is counted
            n = rows * row_bytes
            src[:n].copy_(host[i % 2][:n], non_blocking=True)
            _lib.check(lib.rsb_band_histogram(src.data_ptr(), rows, raster.width, raster.bits, len(raster.bands), int(raster.alpha), raster.nodata,
                                              hist.data_ptr(), _lib.current_stream_ptr()), "rsb_band_histogram")
            torch.cuda.synchronize(dev)  # the next decode into this pinned buffer waits for its upload
    out = hist.cpu().numpy()
    if stats is not None:
        stats.update(stats_s=time.perf_counter() - t0, stats_bands=len(spans))
    return out


def stretch_scale(hist, q_lo, q_hi):
    """[(LO, HI)] per band of `hist` (int64 [bands, values], band_stats) at the percentiles q_lo < q_hi given in hundredths of a
    percent (0..10000): with N the band's count, rank = max(1, ceil(q N / 10000)), and the value is the smallest v whose cumulative
    count reaches the rank. HI = LO gives HI = LO + 1 (LO = HI - 1 at the top value). RsbError when there is no valid pixel."""
    hist = np.asarray(hist, np.int64)
    top = hist.shape[1] - 1
    pairs = []
    for h in hist:
        cum = np.cumsum(h)
        n = int(cum[-1])
        if n == 0:
            raise _lib.RsbError("the raster has no valid pixel to stretch")
        lo, hi = (int(np.searchsorted(cum, max(1, -(-q * n // 10000)), side="left")) for q in (int(q_lo), int(q_hi)))
        if hi == lo:
            lo, hi = (lo, lo + 1) if lo < top else (top - 1, top)
        pairs.append((lo, hi))
    return pairs
