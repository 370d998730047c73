"""numpy restatement of GDAL's polygon fill (`rasterio.features.rasterize`, all_touched=False, merge "replace", burn value 1) as
`rs rasterize` uses it (robosat/tools/rasterize.py:64-83), on the same float64 numbers as rsb_rasterize_polygons.

Rule: every ring is closed implicitly. For row r the scanline is yc = r + 0.5. An edge (x1, y1)-(x2, y2) with y1 <= y2 crosses it
iff y1 <= yc < y2, at x = (yc - y1) * (x2 - x1) / (y2 - y1) + x1 (horizontal edges never cross). The crossings of one polygon
(outer ring and holes together) are sorted and paired; each pair (a, b) fills columns [floor(a + 0.5), floor(b + 0.5)) clipped
to [0, size). Polygons are OR-ed (burned one after another with "replace").
"""

import json
import math
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
R = 6378137.0


def project(lonlat):
    """[[lon, lat], ...] -> float64 [n, 2] EPSG:3857 coordinates"""
    a = np.asarray(lonlat, dtype=np.float64).reshape(-1, 2)
    return np.stack([R * np.radians(a[:, 0]), R * np.log(np.tan(np.pi / 4 + np.radians(a[:, 1]) / 2))], axis=1)


def xy_bounds(x, y, z):
    ce = 2 * math.pi * R
    side = ce / 2 ** z
    left = x * side - ce / 2
    top = ce / 2 - y * side
    return left, top - side, left + side, top


def transform(tile, size):
    """(c0, c1, r0, r1): px = c0 + X * c1, py = r0 + Y * r1"""
    left, bottom, right, top = xy_bounds(*tile)
    a = (right - left) / size
    e = (bottom - top) / size
    return -left / a, 1 / a, -top / e, 1 / e


def fill_polygon(rings_px, size):
    """bool [size, size]: even-odd fill of one polygon given as pixel-space rings (float64 [n, 2] each)"""
    x1s, y1s, x2s, y2s = [], [], [], []
    for ring in rings_px:
        if len(ring) == 0:
            continue
        nxt = np.roll(ring, -1, axis=0)
        x1s.append(ring[:, 0]), y1s.append(ring[:, 1]), x2s.append(nxt[:, 0]), y2s.append(nxt[:, 1])
    out = np.zeros((size, size), bool)
    if not x1s:
        return out
    x1, y1, x2, y2 = (np.concatenate(v) for v in (x1s, y1s, x2s, y2s))
    swap = y1 > y2
    x1, x2 = np.where(swap, x2, x1), np.where(swap, x1, x2)
    y1, y2 = np.where(swap, y2, y1), np.where(swap, y1, y2)
    # candidate rows per edge (a superset), then the exact test
    lo = np.clip(np.floor(y1 - 0.5), 0, size).astype(np.int64)
    hi = np.clip(np.ceil(y2 - 0.5) + 1, 0, size).astype(np.int64)
    n = np.maximum(hi - lo, 0)
    if n.sum() == 0:
        return out
    edge = np.repeat(np.arange(len(n)), n)
    row = lo[edge] + (np.arange(len(edge)) - np.repeat(np.cumsum(n) - n, n))
    yc = row + 0.5
    hit = (y1[edge] <= yc) & (yc < y2[edge])
    edge, row, yc = edge[hit], row[hit], yc[hit]
    x = (yc - y1[edge]) * (x2[edge] - x1[edge]) / (y2[edge] - y1[edge]) + x1[edge]
    order = np.lexsort((x, row))
    row, x = row[order], x[order]
    assert len(row) % 2 == 0 and np.array_equal(row[0::2], row[1::2]), "closed rings cross every scanline an even number of times"
    ca = np.clip(np.floor(x[0::2] + 0.5), 0, size).astype(np.int64)
    cb = np.clip(np.floor(x[1::2] + 0.5), 0, size).astype(np.int64)
    rows, slot = np.unique(row[0::2], return_inverse=True)
    diff = np.zeros((len(rows), size + 1), np.int64)
    np.add.at(diff, (slot, ca), 1)
    np.add.at(diff, (slot, cb), -1)
    out[rows] = np.cumsum(diff, axis=1)[:, :size] > 0
    return out


def to_pixels(ring_xy, tr):
    c0, c1, r0, r1 = tr
    ring_xy = np.asarray(ring_xy, dtype=np.float64).reshape(-1, 2)
    return np.stack([c0 + ring_xy[:, 0] * c1, r0 + ring_xy[:, 1] * r1], axis=1)


def burn_transform(tr, polygons, size):
    """uint8 [size, size]: the union of the polygons (each a list of Mercator rings) under the transform tr"""
    out = np.zeros((size, size), bool)
    for rings in polygons:
        out |= fill_polygon([to_pixels(r, tr) for r in rings], size)
    return out.astype(np.uint8)


def mercator_polygons(features):
    """GeoJSON features -> polygons as lists of Mercator rings (a MultiPolygon gives one polygon per component)"""
    polys = []
    for f in features:
        g = f["geometry"]
        comps = [g["coordinates"]] if g["type"] == "Polygon" else g["coordinates"] if g["type"] == "MultiPolygon" else []
        for comp in comps:
            polys.append([project(ring) for ring in comp])
    return polys


def burn(tile, features, size):
    return burn_transform(transform(tile, size), mercator_polygons(features), size)


def load_golden():
    """{"features": FeatureCollection, "tiles": [(x, y, z)], "masks": {(x, y, z): uint8 [512, 512]}}"""
    with open(os.path.join(GOLDEN, "rasterize.json")) as fp:
        meta = json.load(fp)
    arrays = np.load(os.path.join(GOLDEN, "rasterize.npz"))
    tiles = [tuple(t) for t in meta["tiles"]]
    masks = {tuple(t): arrays["mask_%d_%d_%d" % tuple(t)] for t in meta["labelled"]}
    return {"features": meta["features"], "tiles": tiles, "masks": masks}
