"""`rs cover` (robosat/tools/cover.py): the slippy-map tiles that GeoJSON polygons touch, with the burn and the deduplication on
the GPU.

The reference calls supermercado's `burntiles.burn([feature], zoom)` once per feature: rasterio's `rasterize` with
`all_touched=True` on a grid of the feature's tile range, then a Python set over all features. Here each feature gets the same
grid (`grid`: mercantile 1.0.4's `tile`, `ul` and `xy` restated with `math`), its polygons are projected with
`rasterize.project` and uploaded once, and a batch of features is burned by `rsb_cover_polygons` (GDAL's scanline fill of `rs
rasterize` plus its all-touched line walk, DESIGN.md §8) into a bitmap of one bit per tile. The set tiles become int64 keys
(x << zoom) | y, which `rsb_sort_unique_u64` sorts and deduplicates on the device, so the cover comes out sorted by (x, y).
`mercantile`, `rasterio` and `supermercado` are not needed.

Memory is bounded by `budget`: features are burned in batches whose bitmap, keys and sort workspace fit in it, and a feature
larger than the budget is burned alone in bands of rows. The merged cover must fit on the device; when it cannot, `RsbError`
says so before anything is allocated.
"""

import math

import numpy as np

from robosat_b200 import _lib
from robosat_b200.rasterize import INVALID_ERRORS, W_INVALID, PolygonSet, fill_bands, polygon_to_mercator

R = 6378137.0
MAX_LAT = 85.0511287798066  # supermercado clamps the latitude extrema to Web Mercator's square
SHRINK = 1e-10  # supermercado shrinks the lon/lat extrema by this much on each side
DEFAULT_BUDGET = 1 << 30
# device bytes per grid cell of a batch, beyond its bitmap: an int64 key per cell at most, plus the sort's two padded key buffers
KEY_BYTES_PER_CELL = 25
W_GEOMETRY = "Warning: feature {} is a {}, not a Polygon or MultiPolygon, skipping"


def tile(lng, lat, zoom):
    """(x, y) of the tile containing (lng, lat): mercantile 1.0.4's `tile`, without clamping"""
    lat = math.radians(lat)
    n = 2.0 ** zoom
    x = int(math.floor((lng + 180.0) / 360.0 * n))
    y = int(math.floor((1.0 - math.log(math.tan(lat) + (1.0 / math.cos(lat))) / math.pi) / 2.0 * n))
    return x, y


def ul(x, y, zoom):
    """(lng, lat) of a tile's upper left corner: mercantile 1.0.4's `ul`"""
    n = 2.0 ** zoom
    lon_deg = x / n * 360.0 - 180.0
    lat_rad = math.atan(math.sinh(math.pi * (1 - 2 * y / n)))
    return lon_deg, math.degrees(lat_rad)


def xy(lng, lat):
    """EPSG:3857 (X, Y) of (lng, lat): mercantile 1.0.4's `xy`"""
    return R * math.radians(lng), R * math.log(math.tan((math.pi * 0.25) + (0.5 * math.radians(lat))))


def grid(extrema, zoom):
    """The grid a feature is burned on, from its lon/lat extrema (min lon, min lat, max lon, max lat) ->
    (xmin, ymin, W, H, (c0, c1, r0, r1)) with pixel coordinates px = c0 + X * c1, py = r0 + Y * r1 (GDAL's inverse of the
    geotransform supermercado builds). W = H = 0 when the shrunk extrema are empty (a feature thinner than 2e-10 degrees that
    straddles a tile border)."""
    west, south = extrema[0] + SHRINK, max(-MAX_LAT, extrema[1] + SHRINK)
    east, north = extrema[2] - SHRINK, min(MAX_LAT, extrema[3] - SHRINK)
    xmin, ymin = tile(west, north, zoom)
    xmax, ymax = tile(east, south, zoom)
    W, H = xmax - xmin + 1, ymax - ymin + 1
    if W < 1 or H < 1:
        return xmin, ymin, 0, 0, (0.0, 0.0, 0.0, 0.0)
    ulx, uly = xy(*ul(xmin, ymin, zoom))
    lrx, lry = xy(*ul(xmax + 1, ymax + 1, zoom))
    xcell = (lrx - ulx) / W
    ycell = (uly - lry) / H
    return xmin, ymin, W, H, (-ulx / xcell, 1 / xcell, uly / ycell, -1 / ycell)


def world_rows(ymin, H, zoom):
    """rows [lo, hi) of a grid that are tiles of the world (0 <= y < 2^zoom); the clamped latitude can round to y = -1 or 2^zoom"""
    return max(0, -ymin), max(0, min(H, 2 ** zoom - ymin))


class FeatureSet:
    """Polygon and MultiPolygon features packed for covering. `polyset` (a rasterize.PolygonSet) holds every polygon; a
    MultiPolygon's components are polygons of their own that share the feature's grid. Feature f owns polygons
    [feature_polys[f], feature_polys[f + 1]) and extrema[f] = (min lon, min lat, max lon, max lat) of all its positions.
    `warnings` lists the skipped features: other geometry types, and polygons that fail `rasterize`'s validity rule or have a
    longitude outside [-180, 180]."""

    def __init__(self, features, device=None):
        polygons, counts, extrema, self.warnings = [], [], [], []
        for i, feature in enumerate(features):
            geometry = feature.get("geometry") or {}
            kind = geometry.get("type")
            if kind not in ("Polygon", "MultiPolygon"):
                self.warnings.append(W_GEOMETRY.format(i, kind))
                continue
            try:
                components = [geometry["coordinates"]] if kind == "Polygon" else geometry["coordinates"]
                if not components:
                    raise ValueError("no polygons")
                merc = [polygon_to_mercator(c) for c in components]
                ll = np.concatenate([np.asarray([p[:2] for p in ring], np.float64) for c in components for ring in c])
                if ll[:, 0].min() < -180.0 or ll[:, 0].max() > 180.0:
                    raise ValueError("longitude outside [-180, 180]")
            except INVALID_ERRORS:
                self.warnings.append(W_INVALID.format(i))
                continue
            polygons.extend(merc)
            counts.append(len(merc))
            extrema.append((ll[:, 0].min(), ll[:, 1].min(), ll[:, 0].max(), ll[:, 1].max()))
        self.polyset = PolygonSet(polygons, device)
        self.feature_polys = np.zeros(len(counts) + 1, np.int32)
        np.cumsum(counts, out=self.feature_polys[1:])
        self.extrema = extrema

    def __len__(self):
        return len(self.extrema)


def _plan(grids, zoom, budget):
    """Batches of jobs (feature, row_lo, rows) of consecutive features whose device bytes fit in `budget`; a feature larger
    than the budget is split into bands of rows, one batch each."""
    batches, batch, used = [], [], 0
    for f, (xmin, ymin, W, H, _) in enumerate(grids):
        lo, hi = world_rows(ymin, H, zoom)
        if W > _lib.RSB_COVER_MAX_WIDTH:
            raise _lib.RsbError("feature %d spans %d tiles at zoom %d; a grid of more than %d columns is not supported" % (f, W, zoom, _lib.RSB_COVER_MAX_WIDTH))
        row_bytes = ((W + 31) // 32) * 4 + KEY_BYTES_PER_CELL * W
        cost = (hi - lo) * row_bytes
        if cost <= budget:
            if batch and used + cost > budget:
                batches.append(batch)
                batch, used = [], 0
            batch.append((f, lo, hi - lo))
            used += cost
            continue
        if batch:
            batches.append(batch)
            batch, used = [], 0
        band = budget // row_bytes
        if band < 1:
            raise _lib.RsbError("feature %d: one row of its %d x %d tile grid needs %d bytes, more than the budget of %d bytes" % (f, W, H, row_bytes, budget))
        for r in range(lo, hi, band):
            batches.append([(f, r, min(band, hi - r))])
    if batch:
        batches.append(batch)
    return batches


def _device_bytes_free(device):
    import torch

    free, _ = torch.cuda.mem_get_info(device)
    return free + torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)


def _alloc(shape, dtype, device, what):
    """torch.empty, but an allocation the device cannot hold is an RsbError that says what did not fit"""
    import torch

    nbytes = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
    if nbytes > _device_bytes_free(device):
        raise _lib.RsbError("%s needs %d bytes of device memory, more than the %d bytes free" % (what, nbytes, _device_bytes_free(device)))
    try:
        return torch.empty(shape, dtype=dtype, device=device)
    except torch.cuda.OutOfMemoryError as e:
        raise _lib.RsbError("%s needs %d bytes of device memory: %s" % (what, nbytes, e)) from None


def _sort_unique(keys, n, zoom, what):
    """sorts keys[:n] in place and drops duplicates -> the number of unique keys (synchronises)"""
    import torch

    lib = _lib.load()
    dev = keys.device
    ws = _alloc((max(1, lib.rsb_sort_unique_workspace_bytes(n)),), torch.uint8, dev, what + " sort workspace")
    count = torch.empty((1,), dtype=torch.int64, device=dev)
    _lib.check(lib.rsb_sort_unique_u64(keys.data_ptr(), n, 2 * zoom, ws.data_ptr(), ws.numel(), count.data_ptr(), _lib.current_stream_ptr()),
               "rsb_sort_unique_u64")
    return int(count.item())


def _batch_args(fs, grids, jobs):
    """the device arrays and sizes of rsb_cover_polygons for one batch of jobs, or None when the batch has no cells"""
    import torch

    ps = fs.polyset
    dev = ps.device
    F = len(jobs)
    f0 = jobs[0][0]
    feats = np.array([j[0] for j in jobs], np.int64)
    assert np.array_equal(feats, np.arange(f0, f0 + F)), "a batch is a run of consecutive features"
    fpolys = np.ascontiguousarray(fs.feature_polys[f0:f0 + F + 1])
    first = ps.ring_offsets[ps.poly_rings[fpolys]]
    vertex_offsets = np.zeros(F + 1, np.int64)
    np.cumsum(np.diff(first), out=vertex_offsets[1:])
    g = [grids[f] for f in feats]
    transforms = np.asarray([gi[4] for gi in g], np.float64).reshape(F, 4)
    rows = np.array([j[2] for j in jobs], np.int64)
    W = np.array([gi[2] for gi in g], np.int64)
    ints = np.stack([[gi[0] for gi in g], [gi[1] for gi in g], W, [gi[3] for gi in g], [j[1] for j in jobs], rows], axis=1).astype(np.int64)
    words = (W + 31) // 32
    bitmap_offsets = np.zeros(F + 1, np.int64)
    np.cumsum(rows * words, out=bitmap_offsets[1:])
    if bitmap_offsets[-1] == 0:
        return None
    bands, band_rows, max_words = fill_bands(rows, words)
    if len(bands) > 0x7fffffff:
        raise _lib.RsbError("%d fill bands in one batch" % len(bands))

    def up(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    a = dict(zip(("fpolys", "voff", "tr", "grids", "boff", "bands"), (up(x) for x in (fpolys, vertex_offsets, transforms, ints, bitmap_offsets, bands))))
    a.update(F=F, f0=f0, vertices=int(vertex_offsets[-1]), num_bands=len(bands), band_rows=band_rows, max_words=max_words, words=int(bitmap_offsets[-1]),
             cells=int((rows * W).sum()))
    a["bitmap"] = _alloc((a["words"],), torch.int32, dev, "the cover bitmap of %d features" % F)
    a["status"] = torch.empty((4,), dtype=torch.int64, device=dev)
    return a


def _burn(ps, a):
    """enqueue rsb_cover_polygons for the batch `a` (from _batch_args)"""
    _lib.check(_lib.load().rsb_cover_polygons(ps.d_vertices.data_ptr(), ps.d_ring_offsets.data_ptr(), ps.d_poly_rings.data_ptr(), len(ps),
                                              a["fpolys"].data_ptr(), a["voff"].data_ptr(), a["tr"].data_ptr(), a["grids"].data_ptr(), a["boff"].data_ptr(),
                                              a["F"], a["vertices"], a["bands"].data_ptr(), a["num_bands"], a["band_rows"], a["max_words"],
                                              a["bitmap"].data_ptr(), a["words"], a["status"].data_ptr(), _lib.current_stream_ptr()), "rsb_cover_polygons")


def _cover_batch(fs, grids, jobs, zoom):
    """sorted unique int64 keys (CUDA tensor) of one batch of jobs, or None when it has no cells"""
    import torch

    a = _batch_args(fs, grids, jobs)
    if a is None:
        return None
    _burn(fs.polyset, a)
    n, overflow = a["status"][:2].tolist()
    if overflow:
        raise _lib.RsbError("rsb_cover_polygons: an edge walk of features %d..%d did not finish (coordinates beyond float64 resolution)" % (a["f0"], a["f0"] + a["F"] - 1))
    if n == 0:
        return None
    keys = _alloc((n,), torch.int64, fs.polyset.device, "%d cover keys" % n)
    _lib.check(_lib.load().rsb_cover_emit_keys(a["bitmap"].data_ptr(), a["words"], a["boff"].data_ptr(), a["grids"].data_ptr(), a["F"], zoom, keys.data_ptr(), n,
                                               a["status"].data_ptr(), _lib.current_stream_ptr()), "rsb_cover_emit_keys")
    del a
    return keys[:_sort_unique(keys, n, zoom, "the batch's keys")]


def cover_device(features, zoom, budget=DEFAULT_BUDGET, device="cuda"):
    """The cover of `features` (GeoJSON features, or a FeatureSet) at `zoom` -> int64 CUDA tensor of the keys (x << zoom) | y,
    sorted (so tiles are in (x, y) order) and unique. `budget` bounds the device bytes of one batch (bitmap, keys and sort
    workspace); a single feature needs at least one row of its grid, about 25 bytes per tile of its width. Synchronises.

    Raises ValueError for a zoom outside 0..30, and RsbError when a feature is wider than RSB_COVER_MAX_WIDTH tiles, when one
    row of a feature does not fit in the budget, or when the device cannot hold a batch or the merged cover."""
    import torch

    if not isinstance(zoom, (int, np.integer)) or not 0 <= zoom <= _lib.RSB_COVER_MAX_ZOOM:
        raise ValueError("zoom must be an integer in 0..%d" % _lib.RSB_COVER_MAX_ZOOM)
    zoom = int(zoom)
    fs = features if isinstance(features, FeatureSet) else FeatureSet(features)
    if fs.polyset.device is None:
        fs.polyset.upload(torch.device(device))
    dev = fs.polyset.device
    grids = [grid(e, zoom) for e in fs.extrema]
    parts = [p for p in (_cover_batch(fs, grids, jobs, zoom) for jobs in _plan(grids, zoom, budget)) if p is not None]
    if not parts:
        return torch.empty((0,), dtype=torch.int64, device=dev)
    if len(parts) == 1:
        return parts[0]
    total = sum(len(p) for p in parts)
    merged = _alloc((total,), torch.int64, dev, "the merged cover of %d keys" % total)
    at = 0
    for p in parts:
        merged[at:at + len(p)].copy_(p)
        at += len(p)
    del parts
    return merged[:_sort_unique(merged, total, zoom, "the merged cover")]


def keys_to_tiles(keys, zoom):
    """int64 keys (numpy) -> int64 [n, 2] (x, y)"""
    keys = np.asarray(keys, np.int64)
    return np.stack([keys >> zoom, keys & ((1 << zoom) - 1)], axis=1)


def cover(features, zoom, budget=DEFAULT_BUDGET):
    """Drop-in for the reference's per-feature `burntiles.burn` plus set union: the (x, y, zoom) tiles touched by the Polygon
    and MultiPolygon features, as a list sorted by (x, y)."""
    xy_ = keys_to_tiles(cover_device(features, zoom, budget).cpu().numpy(), zoom)
    return [(int(x), int(y), zoom) for x, y in xy_]


def write_csv(path, keys, zoom):
    """rows `x,y,z` ending in CRLF (as csv.writer writes them), in key order; no rows for no keys"""
    xy_ = keys_to_tiles(keys, zoom)
    tail = ",%d\r\n" % zoom
    with open(path, "w", newline="") as fp:
        fp.write("".join(["%d,%d%s" % (x, y, tail) for x, y in xy_.tolist()]))
