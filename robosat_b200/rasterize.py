"""`rs rasterize` (robosat/tools/rasterize.py): GeoJSON polygons burned into slippy-map label masks, with the fill on the GPU.

The reference projects every feature with rasterio / PROJ, finds the tiles it covers with supermercado's `burntiles`, and calls
`rasterio.features.rasterize` (GDAL's scanline fill, all_touched=False) once per tile. Here the projection is the spherical
Web Mercator formula in float64, every polygon is uploaded once, polygons are binned to the requested tiles by their Mercator
bounding box, and one `rsb_rasterize_polygons` launch fills a whole batch of tiles with GDAL's rule restated (see DESIGN.md §8).
`mercantile`, `rasterio` and `supermercado` are not needed: `xy_bounds` restates mercantile's formula and the tile transform
restates `rasterio.transform.from_bounds`.
"""

import math

import numpy as np

from robosat_b200 import _lib

R = 6378137.0  # EPSG:3857 sphere radius
CE = 2 * math.pi * R


def project(lonlat):
    """[[lon, lat], ...] (degrees, EPSG:4326) -> float64 [n, 2] EPSG:3857 (X, Y)"""
    a = np.asarray(lonlat, dtype=np.float64)
    a = a.reshape(-1, a.shape[-1] if a.size else 2)[:, :2]  # positions may carry an altitude
    with np.errstate(invalid="ignore", divide="ignore"):  # |lat| > 90 projects to NaN
        return np.stack([R * np.radians(a[:, 0]), R * np.log(np.tan(np.pi / 4 + np.radians(a[:, 1]) / 2))], axis=1)


def feature_to_mercator(feature):
    """Yield {"coordinates": [ring [(X, Y), ...], ...], "type": "Polygon"} per polygon of a Polygon or MultiPolygon feature."""
    geometry = feature["geometry"]
    if geometry["type"] == "Polygon":
        components = [geometry["coordinates"]]
    elif geometry["type"] == "MultiPolygon":
        components = geometry["coordinates"]
    else:
        return
    for component in components:
        yield {"coordinates": [[tuple(p) for p in project(ring).tolist()] for ring in component], "type": "Polygon"}


def xy_bounds(tile):
    """(left, bottom, right, top) of a tile in EPSG:3857 metres, as mercantile.xy_bounds."""
    x, y, z = tile[0], tile[1], tile[2]
    side = CE / 2 ** z
    left = x * side - CE / 2
    top = CE / 2 - y * side
    return left, top - side, left + side, top


def tile_transform(tile, size):
    """(c0, c1, r0, r1) with px = c0 + X * c1 and py = r0 + Y * r1: the inverse of `from_bounds(*xy_bounds(tile), size, size)`."""
    left, bottom, right, top = xy_bounds(tile)
    a = (right - left) / size
    e = (bottom - top) / size
    return -left / a, 1 / a, -top / e, 1 / e


class PolygonSet:
    """Polygons (each a list of Mercator rings, outer ring first) packed once: float64 vertices [V, 2], int64 ring offsets,
    int32 polygon -> ring offsets and float64 bounding boxes [P, 4] (xmin, ymin, xmax, ymax) on the host; the first three are
    uploaded to `device` when one is given."""

    def __init__(self, polygons, device=None):
        rings = [np.asarray(r, dtype=np.float64).reshape(-1, 2) for poly in polygons for r in poly]
        self.vertices = np.ascontiguousarray(np.concatenate(rings) if rings else np.zeros((0, 2)), dtype=np.float64)
        self.ring_offsets = np.zeros(len(rings) + 1, np.int64)
        np.cumsum([len(r) for r in rings], out=self.ring_offsets[1:])
        self.poly_rings = np.zeros(len(polygons) + 1, np.int32)
        np.cumsum([len(p) for p in polygons], out=self.poly_rings[1:])
        self.bboxes = np.full((len(polygons), 4), np.nan)
        starts, ends = self.ring_offsets[self.poly_rings[:-1]], self.ring_offsets[self.poly_rings[1:]]
        full = np.flatnonzero(ends > starts)
        if len(full):  # the polygons between two non-empty ones have no vertices, so each reduceat run is one polygon
            self.bboxes[full, :2] = np.minimum.reduceat(self.vertices, starts[full])
            self.bboxes[full, 2:] = np.maximum.reduceat(self.vertices, starts[full])
        self.device = None
        if device is not None:
            self.upload(device)

    def __len__(self):
        return len(self.poly_rings) - 1

    def upload(self, device):
        import torch

        self.device = device
        # at least one row, so that the pointer is valid even when every ring is empty
        self.d_vertices = torch.from_numpy(self.vertices if len(self.vertices) else np.zeros((1, 2))).to(device)
        self.d_ring_offsets = torch.from_numpy(self.ring_offsets).to(device)
        self.d_poly_rings = torch.from_numpy(self.poly_rings).to(device)


def bin_polygons(tiles, bboxes):
    """Polygon ids per tile as CSR (offsets int32 [N + 1], ids int32): every polygon whose Mercator bounding box, widened by
    1e-6 of a tile on each side, meets the tile. A filled pixel centre lies in the box and at least 1 / (2 * 4096) of a tile inside
    its tile, far more than the rounding of the tile index, so this covers every tile where the polygon can fill a pixel, and
    burning with these lists gives the same masks as burning every polygon into every tile. Polygons without vertices (NaN
    boxes) meet no tile."""
    N = len(tiles)
    pairs_t, pairs_p = [], []
    tiles_arr = np.asarray([(int(t[0]), int(t[1]), int(t[2])) for t in tiles], dtype=np.int64).reshape(-1, 3)
    ok = ~np.isnan(bboxes).any(axis=1)
    for z in np.unique(tiles_arr[:, 2]):
        at_z = np.flatnonzero(tiles_arr[:, 2] == z)
        tx, ty = tiles_arr[at_z, 0], tiles_arr[at_z, 1]
        keys = (tx << 32) | ty
        order = np.argsort(keys, kind="stable")
        skeys = keys[order]
        side = CE / 2 ** int(z)
        ids = np.flatnonzero(ok)
        b = bboxes[ids]
        lim = 2 ** int(z) - 1
        eps = 1e-6
        x0 = np.clip(np.floor((b[:, 0] + CE / 2) / side - eps), 0, lim).astype(np.int64)
        x1 = np.clip(np.floor((b[:, 2] + CE / 2) / side + eps), 0, lim).astype(np.int64)
        y0 = np.clip(np.floor((CE / 2 - b[:, 3]) / side - eps), 0, lim).astype(np.int64)
        y1 = np.clip(np.floor((CE / 2 - b[:, 1]) / side + eps), 0, lim).astype(np.int64)
        count = (x1 - x0 + 1) * (y1 - y0 + 1)
        huge = count > len(at_z)
        for i in np.flatnonzero(huge):  # a box of more tiles than the list: scan the list instead of enumerating the box
            hit = np.flatnonzero((tx >= x0[i]) & (tx <= x1[i]) & (ty >= y0[i]) & (ty <= y1[i]))
            pairs_t.append(at_z[hit])
            pairs_p.append(np.full(len(hit), ids[i], np.int64))
        small = np.flatnonzero(~huge)
        if len(small):  # enumerate the boxes, look each tile up in the sorted keys
            cnt = count[small]
            rep = np.repeat(small, cnt)
            k = np.arange(len(rep)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
            w = (x1 - x0 + 1)[rep]
            qx, qy = x0[rep] + k % w, y0[rep] + k // w
            q = (qx << 32) | qy
            pos = np.minimum(np.searchsorted(skeys, q), len(skeys) - 1)
            found = skeys[pos] == q
            # a tile listed twice gets the polygon once per listing
            first, last = np.searchsorted(skeys, q[found], "left"), np.searchsorted(skeys, q[found], "right")
            dup = last - first
            tsel = np.repeat(first, dup) + (np.arange(dup.sum()) - np.repeat(np.cumsum(dup) - dup, dup))
            pairs_t.append(at_z[order[tsel]])
            pairs_p.append(np.repeat(ids[rep[found]], dup))
    t = np.concatenate(pairs_t) if pairs_t else np.zeros(0, np.int64)
    p = np.concatenate(pairs_p) if pairs_p else np.zeros(0, np.int64)
    order = np.lexsort((p, t))
    offsets = np.zeros(N + 1, np.int64)
    np.cumsum(np.bincount(t, minlength=N), out=offsets[1:])
    if offsets[-1] > np.iinfo(np.int32).max:
        raise ValueError("too many (tile, polygon) pairs for one batch: %d" % offsets[-1])
    return offsets.astype(np.int32), p[order].astype(np.int32)


def rasterize_device(polyset, tiles, size, csr=None, out=None):
    """Burn the PolygonSet (uploaded) into `tiles` -> (uint8 CUDA tensor [N, size, size] {0, 1}, int32 CUDA tensor [N] foreground
    counts). `csr` = (offsets, ids) from `bin_polygons` (computed here when None); `out` may be a preallocated uint8 CUDA tensor
    [N, size, size] with contiguous rows. Enqueued on the current stream, no synchronisation."""
    import torch

    if polyset.device is None:
        raise ValueError("rasterize_device needs a PolygonSet uploaded to a CUDA device")
    if not 1 <= size <= _lib.RSB_RASTER_MAX_SIZE:
        raise ValueError("size must be in 1..%d" % _lib.RSB_RASTER_MAX_SIZE)
    dev = polyset.device
    N = len(tiles)
    if out is None:
        out = torch.empty((N, size, size), dtype=torch.uint8, device=dev)
    elif out.dtype != torch.uint8 or not out.is_cuda or out.shape != (N, size, size) or out.stride(2) != 1 or out.stride(1) != size:
        raise ValueError("out must be a uint8 CUDA tensor [N, size, size] with contiguous rows")
    counts = torch.empty((N,), dtype=torch.int32, device=dev)
    if N == 0:
        return out, counts
    offsets, ids = csr if csr is not None else bin_polygons(tiles, polyset.bboxes)
    transforms = np.asarray([tile_transform(t, size) for t in tiles], dtype=np.float64)
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    d_offsets = torch.from_numpy(np.ascontiguousarray(offsets, dtype=np.int32)).to(dev)
    d_ids = torch.from_numpy(ids if len(ids) else np.zeros(1, np.int32)).to(dev)
    d_tr = torch.from_numpy(transforms).to(dev)
    _lib.check(_lib.load().rsb_rasterize_polygons(polyset.d_vertices.data_ptr(), polyset.d_ring_offsets.data_ptr(), polyset.d_poly_rings.data_ptr(),
                                                  len(polyset), d_offsets.data_ptr(), d_ids.data_ptr(), d_tr.data_ptr(), N, size, out.data_ptr(),
                                                  out.stride(0) if N > 1 else size * size, counts.data_ptr(), _lib.current_stream_ptr()),
               "rsb_rasterize_polygons")
    return out, counts


def burn_device(tiles, polygons, size, device="cuda"):
    """Batch path: `polygons` (lists of Mercator rings, as in `feature_to_mercator(...)["coordinates"]`) burned into every tile ->
    (uint8 CUDA tensor [N, size, size], int32 CUDA tensor [N] foreground counts)."""
    return rasterize_device(PolygonSet(polygons, device), tiles, size)


def burn(tile, features, size):
    """Drop-in for robosat.tools.rasterize.burn: uint8 [size, size] {0, 1} of the Polygon and MultiPolygon features (each
    MultiPolygon component is a polygon of its own) on `tile`."""
    polygons = [g["coordinates"] for f in features for g in feature_to_mercator(f)]
    out, _ = burn_device([tile], polygons, size)
    return out[0].cpu().numpy()


W_INVALID = "Warning: invalid feature {}, skipping"


def polygons_from_features(features):
    """The Polygon features `rs rasterize` burns, as Mercator rings -> (polygons, warnings).

    Other geometry types are skipped silently, as the reference does (rasterize.py:109). A Polygon that cannot be burned gets the
    reference's warning and is skipped: one without rings, a ring of fewer than 4 positions (a closed ring needs 3 distinct
    vertices and the repeated first one), a position that is not a number pair, or coordinates that do not project to finite
    Mercator values (e.g. latitudes beyond ±90°)."""
    polygons, warnings = [], []
    for i, feature in enumerate(features):
        geometry = feature.get("geometry") or {}
        if geometry.get("type") != "Polygon":
            continue
        try:
            rings = geometry["coordinates"]
            if not rings:
                raise ValueError("no rings")
            merc = []
            for ring in rings:
                if len(ring) < 4:
                    raise ValueError("ring with fewer than 4 positions")
                xy = project([p[:2] for p in ring])
                if not np.isfinite(xy).all():
                    raise ValueError("coordinates outside the projection")
                merc.append(xy)
        except (ValueError, TypeError, KeyError, IndexError):
            warnings.append(W_INVALID.format(i))
            continue
        polygons.append(merc)
    return polygons, warnings
