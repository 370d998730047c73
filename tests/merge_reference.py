"""`rs merge` restated in numpy for the tests: the steps the kernels take, written without their algorithms.

- Near: for every vertex of one shape and every edge of the other, the float64 point-to-segment distance of DESIGN.md §8
  (t = clamp(((p - a).(b - a)) / |b - a|^2, 0, 1), q = a + t (b - a), |p - q|^2 <= d * d), vectorised over all pairs; numpy
  rounds every operation on its own, as the kernel's intrinsics do.
- Intersects: `dedupe_reference`'s exact segment and point-in-polygon predicates, on the EPSG:3395 vertices.
- Components: a sequential union-find; the label is the smallest member.
- Fill: `rasterize_reference.fill_polygon` on the component's grid (the scanline rule of `rs rasterize` and `rs cover`), OR-ed
  over the member polygons.
- Closing: scipy.ndimage's binary dilation, then erosion, with the digital disk and cells outside the grid at 0.

The host steps (candidate pairs, grids, tracing) are the package's own and are tested on their own in test_merge.py."""

import numpy as np
import scipy.ndimage

import dedupe_reference as dr
import rasterize_reference as rr
from robosat_b200 import merge as MG


def rings_xy(feature):
    """EPSG:3395 rings (float64 [n, 2], unclosed) of every polygon of a feature, grouped by polygon"""
    g = feature["geometry"]
    polys = [g["coordinates"]] if g["type"] == "Polygon" else g["coordinates"]
    out = []
    for poly in polys:
        rings = []
        for ring in poly:
            r = MG.mercator([p[:2] for p in ring])
            if len(r) > 1 and (r[0] == r[-1]).all():
                r = r[:-1]
            rings.append(r)
        out.append(rings)
    return out


def _edges(rings):
    """(a, b) float64 [m, 2] arrays of the edges of closed rings, zero-length edges left out"""
    a = np.concatenate([r for r in rings if len(r)]) if rings else np.zeros((0, 2))
    b = np.concatenate([np.roll(r, -1, axis=0) for r in rings if len(r)]) if rings else np.zeros((0, 2))
    keep = ~(a == b).all(1)
    return a[keep], b[keep]


def point_segment_within(p, a, b, d):
    """bool [len(p), len(a)]: |p_i - q|^2 <= d * d, q the point of segment a_j b_j nearest to p_i"""
    p = p[:, None, :]
    dx, dy = b[None, :, 0] - a[None, :, 0], b[None, :, 1] - a[None, :, 1]
    len2 = dx * dx + dy * dy
    num = (p[..., 0] - a[None, :, 0]) * dx + (p[..., 1] - a[None, :, 1]) * dy
    with np.errstate(invalid="ignore", divide="ignore"):
        t = np.where(len2 > 0, num / len2, 0.0)
    t = np.minimum(np.maximum(t, 0.0), 1.0)
    qx, qy = a[None, :, 0] + t * dx, a[None, :, 1] + t * dy
    ex, ey = p[..., 0] - qx, p[..., 1] - qy
    return ex * ex + ey * ey <= d * d


def near_rings(rings_a, rings_b, d):
    """some vertex of one set of rings lies within d of some edge of the other"""
    a0, a1 = _edges(rings_a)
    b0, b1 = _edges(rings_b)
    if not len(a0) or not len(b0):
        return False
    return bool(point_segment_within(a0, b0, b1, d).any() or point_segment_within(b0, a0, a1, d).any())


def intersects_rings(polys_a, polys_b):
    """`rsb_dedupe_intersects`'s predicate on projected rings (grouped by polygon): edges meet, or the first exterior vertex of a
    polygon of one lies inside or on the other"""
    ea = [(tuple(map(float, a)), tuple(map(float, b))) for a, b in zip(*_edges([r for p in polys_a for r in p]))]
    eb = [(tuple(map(float, a)), tuple(map(float, b))) for a, b in zip(*_edges([r for p in polys_b for r in p]))]
    for a, b in ea:
        for c, d in eb:
            if dr.segments_meet(a, b, c, d):
                return True
    for polys, other in ((polys_a, eb), (polys_b, ea)):
        for poly in polys:
            if len(poly[0]) and dr.point_in(tuple(map(float, poly[0][0])), other) != "out":
                return True
    return False


def linked(features, d):
    """the linked pairs (i, j), i < j, over the candidate pairs of the parsed features (`MG.candidate_pairs`), as a sorted list"""
    shapes, _ = MG.parse(features)
    p, q = MG.candidate_pairs(shapes, d)
    polys = [rings_xy(features[i]) for i in shapes.index]
    out = []
    for i, j in zip(p.tolist(), q.tolist()):
        if intersects_rings(polys[i], polys[j]) or near_rings([r for x in polys[i] for r in x], [r for x in polys[j] for r in x], d):
            out.append((i, j))
    return out


def labels(n, pairs):
    """int [n]: the smallest node of each node's component"""
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x

    for i, j in pairs:
        a, b = find(i), find(j)
        if a != b:
            parent[max(a, b)] = min(a, b)
    return np.array([find(i) for i in range(n)], np.int32)


def disk(k):
    i, j = np.mgrid[-k:k + 1, -k:k + 1]
    return i * i + j * j <= k * k


def close(fill, k=MG.CELLS_PER_THRESHOLD):
    """erode(dilate(fill)) with the disk of radius k, cells outside the grid at 0"""
    s = disk(k)
    dil = scipy.ndimage.binary_dilation(fill, structure=s, border_value=0)
    return scipy.ndimage.binary_erosion(dil, structure=s, border_value=0)


def fill(comp, polys):
    """bool [H, W] fill of a Component's grid by the polygons (lists of EPSG:3395 rings)"""
    _, _, W, H = comp.grid
    S = max(W, H)
    out = np.zeros((H, W), bool)
    tr = comp.transform()
    for rings in polys:
        out |= rr.fill_polygon([rr.to_pixels(r, tr) for r in rings], S)[:H, :W]
    return out


def pipeline(features, d):
    """the restated components of `features` at threshold d -> [Component] in component order, with `fill` and `closed` set"""
    shapes, _ = MG.parse(features)
    lab = labels(len(shapes), linked(features, d))
    comps = MG.components(shapes, lab, d)
    for c in comps:
        if c.grid[2] == 0:
            continue
        polys = [p for f in c.members for p in rings_xy(features[shapes.index[f]])]
        c.fill = fill(c, polys)
        c.closed = close(c.fill)
        c.count = int(c.closed.sum())
    return comps


# ---- seeded workloads ----

def straddling(n, seed, z=18, origin=(137500, 91500)):
    """n seeded convex polygons (about 40-60 % of a tile across at zoom z, as tile units) and the z tiles each covers: even ones
    centred on a tile corner (2 x 2 tiles), odd ones on a tile centre and larger (3 x 3 tiles), 6 tiles apart -> (features,
    [[(x, y, z), ...] per polygon])"""
    import cover_reference as cr

    rng = np.random.default_rng(seed)
    feats, tiles = [], []
    for i in range(n):
        bx, by = origin[0] + 6 * (i % 20), origin[1] + 6 * (i // 20)
        if i % 2 == 0:
            cx, cy, r, span = bx + 1.0, by + 1.0, rng.uniform(0.25, 0.45), range(0, 2)
        else:
            cx, cy, r, span = bx + 1.5, by + 1.5, rng.uniform(0.6, 0.9), range(0, 3)
        k = int(rng.integers(5, 12))
        a = np.sort(rng.uniform(0, 2 * np.pi, k)) + rng.uniform(0, 2 * np.pi)
        rr_ = r * rng.uniform(0.85, 1.0)
        pts = list(zip(cx + rr_ * np.cos(a), cy + rr_ * rng.uniform(0.7, 1.0) * np.sin(a)))
        feats.append(cr.polygon_feature([pts], z))
        tiles.append([(bx + dx, by + dy, z) for dy in span for dx in span])
    return feats, tiles


def fragments(features, tiles, size=512):
    """`rs rasterize` of the features on their tiles, then `rs features --type parking` -> the per-tile parking features (on the
    device; needs a GPU)"""
    import collections

    import torch

    from robosat_b200 import features as FT
    from robosat_b200.rasterize import PolygonSet, rasterize_device, feature_to_mercator

    Tile = collections.namedtuple("Tile", "x y z")
    all_tiles = sorted({t for ts in tiles for t in ts})
    polys = [g["coordinates"] for f in features for g in feature_to_mercator(f)]
    masks, _ = rasterize_device(PolygonSet(polys, torch.device("cuda")), all_tiles, size)
    handler = FT.ParkingHandler()
    handler.apply_batch([Tile(*t) for t in all_tiles], masks, 1)
    return handler.features
