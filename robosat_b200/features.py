"""`rs features` post-processing (robosat/features/{core,parking}.py) with the mask morphology on the GPU.

The reference's parking handler spends nearly all its time in `denoise` + `grow`: an opening and then a closing with a 20 x 20
ellipse. Here that 4-op chain (erode, dilate, dilate, erode) is one `rsb_morph_binary` launch over a batch of label images,
bit-identical to OpenCV. The launch also counts each result's foreground, so empty tiles never reach the host. Contour tracing,
simplification and the hierarchy walk stay on the host with the reference's OpenCV calls. The ring order, the three warnings and
the skips are the reference's. `mercantile` and `shapely` are not needed: `bounds` restates mercantile's tile bounds, and
`polygon_is_valid` restates the OGC validity rules that the reference asks shapely for.

`BuildingHandler` is this project's building rule (the reference has none; DESIGN.md §8): a small opening, then connected
components on the device (`rsb_building_clean`) drop specks and fill small holes, and the host turns each outer contour and its
holes into one polygon.
"""

import collections
import json
import math
import sys

import numpy as np

from robosat_b200 import _lib

MorphOp = collections.namedtuple("MorphOp", ["dilate", "spans", "kw", "anchor"])
MorphOp.__doc__ = """One erosion (dilate=False) or dilation of a binary image: element rows as column runs `spans` [(j0, j1)] * kh
of a kh x kw element, anchor (ay, ax)."""


def ellipse_spans(k):
    """Rows of `cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (k, k))` as column runs [j0, j1).

    Row i of an ellipse of radius r = k // 2 centred at column c = k // 2 covers the columns within round(c * sqrt(1 - (i - r)^2 /
    r^2)) of c, clipped to the element; a row with |i - r| > r is empty. round() is round-half-to-even, as OpenCV's."""
    r = c = k // 2
    inv_r2 = 1.0 / (r * r) if r else 0.0
    spans = []
    for i in range(k):
        dy = i - r
        if abs(dy) > r:
            spans.append((0, 0))
            continue
        dx = int(round(c * math.sqrt((r * r - dy * dy) * inv_r2)))
        spans.append((max(c - dx, 0), min(c + dx + 1, k)))
    return spans


def ellipse_op(k, dilate):
    return MorphOp(dilate, ellipse_spans(k), k, (k // 2, k // 2))


def parking_chain(k_denoise=20, k_grow=20):
    """`grow(denoise(m, k_denoise), k_grow)` (core.py:65-92): MORPH_OPEN then MORPH_CLOSE = erode, dilate, dilate, erode."""
    return [ellipse_op(k_denoise, False), ellipse_op(k_denoise, True), ellipse_op(k_grow, True), ellipse_op(k_grow, False)]


def _op_struct(op):
    kh = len(op.spans)
    s = _lib.MorphOp(dilate=int(bool(op.dilate)), kh=kh, kw=op.kw, ay=op.anchor[0], ax=op.anchor[1])
    for i, (j0, j1) in enumerate(op.spans[:_lib.RSB_MORPH_MAX_K]):
        s.span[i][0], s.span[i][1] = j0, j1
    return s


def morph_device(labels, class_index, ops):
    """labels: uint8 CUDA tensor [N, H, W] (rows contiguous; the image stride may exceed H * W) -> (uint8 [N, H, W] {0, 1}
    result of the op chain on (labels == class_index), int32 [N] foreground counts), both on the device. Enqueued on the current
    stream, no synchronisation."""
    import torch

    if not labels.is_cuda or labels.dtype != torch.uint8 or labels.dim() != 3:
        raise ValueError("morph_device needs a uint8 CUDA tensor [N, H, W]")
    N, H, W = labels.shape
    if labels.stride(2) != 1 or labels.stride(1) != W:
        raise ValueError("morph_device needs contiguous rows of each image")
    if not 1 <= len(ops) <= _lib.RSB_MORPH_MAX_OPS:
        raise ValueError("morph_device takes 1..%d ops" % _lib.RSB_MORPH_MAX_OPS)
    if any(len(op.spans) > _lib.RSB_MORPH_MAX_K for op in ops):
        raise ValueError("structuring elements are limited to %d rows" % _lib.RSB_MORPH_MAX_K)
    arr = (_lib.MorphOp * len(ops))(*[_op_struct(op) for op in ops])
    out = torch.empty((N, H, W), dtype=torch.uint8, device=labels.device)
    counts = torch.empty((N,), dtype=torch.int32, device=labels.device)
    _lib.check(_lib.load().rsb_morph_binary(labels.data_ptr(), labels.stride(0) if N > 1 else H * W, N, H, W, int(class_index), arr, len(ops),
                                            out.data_ptr(), counts.data_ptr(), _lib.current_stream_ptr()), "rsb_morph_binary")
    return out, counts


def _planes(planes, what):
    import torch

    if not planes.is_cuda or planes.dtype != torch.uint8 or planes.dim() != 3:
        raise ValueError("%s needs a uint8 CUDA tensor [N, H, W]" % what)
    N, H, W = planes.shape
    if planes.stride(2) != 1 or planes.stride(1) != W:
        raise ValueError("%s needs contiguous rows of each image" % what)
    return N, H, W, planes.stride(0) if N > 1 else H * W


def components_device(planes, value, connectivity):
    """planes: uint8 CUDA tensor [N, H, W] (rows contiguous) -> (int32 [N, H, W] root of each pixel's component of
    (planes == value) under 4- or 8-connectivity, i.e. its smallest pixel index y * W + x in the image, or -1 off the plane;
    int32 [N, H, W] the area of that component, 0 off the plane). Enqueued on the current stream, no synchronisation."""
    import torch

    from robosat_b200.cover import _alloc

    N, H, W, stride = _planes(planes, "components_device")
    labels = _alloc((N, H, W), torch.int32, planes.device, "component labels")
    areas = _alloc((N, H, W), torch.int32, planes.device, "component areas")
    _lib.check(_lib.load().rsb_label_components(planes.data_ptr(), stride, N, H, W, int(value), int(connectivity), labels.data_ptr(),
                                                areas.data_ptr(), _lib.current_stream_ptr()), "rsb_label_components")
    return labels, areas


def building_open(k_denoise=5):
    """The building rule's denoise: MORPH_OPEN with a k x k ellipse = erode, dilate."""
    return [ellipse_op(k_denoise, False), ellipse_op(k_denoise, True)]


def building_clean_device(labels, class_index, k_denoise=5, min_area=64, min_hole_area=64):
    """labels: uint8 CUDA tensor [N, H, W] of class indices -> (uint8 [N, H, W] {0, 1} cleaned building masks, int32 [N] foreground
    counts), both on the device: the opening of (labels == class_index), then 8-connected components below min_area pixels dropped,
    then 4-connected background components below min_hole_area pixels that miss the tile border filled (DESIGN.md §8). Enqueued
    on the current stream, no synchronisation."""
    import torch

    from robosat_b200.cover import _alloc

    opened, _ = morph_device(labels, class_index, building_open(k_denoise))
    N, H, W = opened.shape
    work = _alloc((N, H, W), torch.int32, opened.device, "building component labels")
    stats = _alloc((N, H, W), torch.int32, opened.device, "building component areas")
    out = torch.empty((N, H, W), dtype=torch.uint8, device=opened.device)
    counts = torch.empty((N,), dtype=torch.int32, device=opened.device)
    _lib.check(_lib.load().rsb_building_clean(opened.data_ptr(), H * W, N, H, W, int(min_area), int(min_hole_area), work.data_ptr(),
                                              stats.data_ptr(), out.data_ptr(), counts.data_ptr(), _lib.current_stream_ptr()),
               "rsb_building_clean")
    return out, counts


# --- geo transform (mercantile.bounds, robosat/tiles.py:19-42 pixel_to_location) -----------------------------------------------

def _ul(x, y, z):
    n = 2.0 ** z
    return x / n * 360.0 - 180.0, math.degrees(math.atan(math.sinh(math.pi * (1 - 2 * y / n))))


def bounds(tile):
    """(west, south, east, north) in degrees of a Web Mercator tile, as mercantile.bounds."""
    west, north = _ul(tile.x, tile.y, tile.z)
    east, south = _ul(tile.x + 1, tile.y + 1, tile.z)
    return west, south, east, north


def pixel_to_location(tile, dx, dy):
    assert 0 <= dx <= 1, "x offset is in [0, 1]"
    assert 0 <= dy <= 1, "y offset is in [0, 1]"
    west, south, east, north = bounds(tile)

    def lerp(a, b, c):
        return a + c * (b - a)

    return lerp(west, east, dx), lerp(south, north, dy)


def featurize(tile, polygon, shape):
    """Pixel ring [(px, py)] -> closed [(lon, lat)] ring (core.py:37-62; shape = mask.shape[:2], i.e. (rows, cols))."""
    xmax, ymax = shape
    feature = [pixel_to_location(tile, px / xmax, 1. - py / ymax) for px, py in polygon]
    assert feature, "at least one location in polygon"
    feature.append(feature[0])
    return feature


# --- polygon validity on integer pixel rings --------------------------------------------------------------------------------

def _orient(a, b, c):
    v = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
    return (v > 0) - (v < 0)


def _on_segment(p, a, b):
    return (_orient(a, b, p) == 0 and min(a[0], b[0]) <= p[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= p[1] <= max(a[1], b[1]))


def _intersect(a, b, c, d):
    """How segments ab and cd meet: None, 'point' (one common point) or 'overlap' (a common piece of positive length)."""
    o1, o2, o3, o4 = _orient(a, b, c), _orient(a, b, d), _orient(c, d, a), _orient(c, d, b)
    if o1 == o2 == o3 == o4 == 0:
        # collinear: project on the dominant axis
        ax = 0 if (a[0] != b[0] or c[0] != d[0]) else 1
        lo = max(min(a[ax], b[ax]), min(c[ax], d[ax]))
        hi = min(max(a[ax], b[ax]), max(c[ax], d[ax]))
        if lo > hi:
            return None
        return "point" if lo == hi else "overlap"
    if o1 != o2 and o3 != o4:
        return "point"
    if (o1 == 0 and _on_segment(c, a, b)) or (o2 == 0 and _on_segment(d, a, b)) or \
       (o3 == 0 and _on_segment(a, c, d)) or (o4 == 0 and _on_segment(b, c, d)):
        return "point"
    return None


def _edges(ring):
    return [(ring[i], ring[(i + 1) % len(ring)]) for i in range(len(ring))]


def _inside(p2, ring2):
    """Even-odd test of a point (doubled coordinates) not on the ring's boundary (doubled coordinates)."""
    x, y = p2
    inside = False
    n = len(ring2)
    for i in range(n):
        (x1, y1), (x2, y2) = ring2[i], ring2[(i + 1) % n]
        if (y1 > y) != (y2 > y):
            # x of the edge at height y, compared without division
            lhs = (x - x1) * (y2 - y1)
            rhs = (x2 - x1) * (y - y1)
            if (lhs < rhs) == (y2 > y1):
                inside = not inside
    return inside


def _sides(a, b):
    """Where ring a lies relative to ring b: the set of {'in', 'out'} over a's vertices and pieces of a's edges not on b's
    boundary. Edges are split at every vertex of b they pass through, so each piece lies wholly on one side."""
    b2 = [(2 * x, 2 * y) for x, y in b]
    eb = _edges(b)
    on_b = lambda p: any(_on_segment(p, u, v) for u, v in eb)  # noqa: E731
    sides = set()
    for p, q in _edges(a):
        cuts = sorted({tuple(p), tuple(q)} | {tuple(v) for v in b if _on_segment(v, p, q)},
                      key=lambda v: (v[0] - p[0]) ** 2 + (v[1] - p[1]) ** 2)
        for u in cuts:
            if not on_b(u):
                sides.add("in" if _inside((2 * u[0], 2 * u[1]), b2) else "out")
        for u, v in zip(cuts, cuts[1:]):
            m2 = (u[0] + v[0], u[1] + v[1])
            if not any(_on_segment(m2, (2 * s[0], 2 * s[1]), (2 * t[0], 2 * t[1])) for s, t in eb):
                sides.add("in" if _inside(m2, b2) else "out")
    return sides


def _dedupe(ring):
    out = []
    for p in ring:
        p = (int(p[0]), int(p[1]))
        if not out or out[-1] != p:
            out.append(p)
    while len(out) > 1 and out[0] == out[-1]:
        out.pop()
    return out


def polygon_is_valid(rings):
    """OGC validity (what GEOS's `is_valid` checks for a Polygon) of a shell and holes given as integer vertex lists (unclosed).

    Every ring has >= 3 distinct vertices and non-zero area; no ring meets itself except consecutive edges at their common vertex;
    rings meet each other only in points (no crossing, no shared piece of edge); every hole lies in the shell and in no other hole;
    the interior is connected: no two rings touch in two or more points and the graph of touching rings has no cycle."""
    rings = [_dedupe(r) for r in rings]
    for r in rings:
        if len(set(r)) < 3:
            return False
        if sum(r[i][0] * r[(i + 1) % len(r)][1] - r[(i + 1) % len(r)][0] * r[i][1] for i in range(len(r))) == 0:
            return False
        e = _edges(r)
        n = len(e)
        for i in range(n):
            for j in range(i + 1, n):
                hit = _intersect(e[i][0], e[i][1], e[j][0], e[j][1])
                # consecutive edges meet in their common vertex; any more (a spike doubling back) is an overlap
                adjacent = j == i + 1 or (i == 0 and j == n - 1)
                if hit == "overlap" or (hit == "point" and not adjacent):
                    return False
    parent = list(range(len(rings)))

    def find(i):
        while parent[i] != i:
            parent[i] = parent[parent[i]]
            i = parent[i]
        return i

    for a in range(len(rings)):
        for b in range(a + 1, len(rings)):
            touches = set()
            for p, q in _edges(rings[a]):
                for u, v in _edges(rings[b]):
                    hit = _intersect(p, q, u, v)
                    if hit == "overlap":
                        return False
                    if hit == "point":
                        pts = [x for x in (p, q) if _on_segment(x, u, v)] + [x for x in (u, v) if _on_segment(x, p, q)]
                        if not pts:
                            return False  # the edges cross in their interiors
                        touches.update(pts)
            if len(touches) >= 2:
                return False
            if touches:
                ra, rb = find(a), find(b)
                if ra == rb:
                    return False
                parent[ra] = rb
    for h in range(1, len(rings)):
        if _sides(rings[h], rings[0]) != {"in"}:
            return False
        for g in range(1, len(rings)):
            if g != h and "in" in _sides(rings[h], rings[g]):
                return False
    return True


# --- the handler (robosat/features/parking.py) ------------------------------------------------------------------------------

def _parents_in_hierarchy(node, tree):
    up = tree[node][3]
    while up != -1:
        index = up
        up = tree[index][3]
        assert index != node, "upward path does not include starting node"
        yield index


W_SIMPLIFIED = "Warning: simplified feature no longer valid polygon, skipping"
W_TOO_DEEP = "Warning: polygon ring nesting level too deep, skipping"
W_INVALID = "Warning: extracted feature is not valid, skipping"


def polygons_from_grown(tile, grown, simplify_threshold=0.01):
    """Host half of `ParkingHandler.apply` (parking.py:39-100) on one grown {0, 1} uint8 mask.

    Returns (features, warnings): GeoJSON Feature dicts and the warning lines the reference prints, in the reference's order.
    Thread-safe: it prints nothing and OpenCV releases the GIL."""
    import cv2

    features, warnings = [], []
    multipolygons, hierarchy = cv2.findContours(grown, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
    if hierarchy is None:
        return features, warnings
    assert len(hierarchy) == 1, "always single hierarchy for all polygons in multipolygon"
    hierarchy = hierarchy[0]
    assert len(multipolygons) == len(hierarchy), "polygons and hierarchy in sync"
    assert 0 <= simplify_threshold <= 1, "approximation accuracy is percentage in [0, 1]"
    polygons = [cv2.approxPolyDP(p, epsilon=simplify_threshold * cv2.arcLength(p, closed=True), closed=True) for p in multipolygons]

    groups = collections.defaultdict(set)  # the reference's container: its iteration order is the ring order
    for i, (polygon, node) in enumerate(zip(polygons, hierarchy)):
        if len(polygon) < 3:
            warnings.append(W_SIMPLIFIED)
            continue
        ancestors = list(_parents_in_hierarchy(i, hierarchy))
        if len(ancestors) > 1:
            warnings.append(W_TOO_DEEP)
            continue
        root = ancestors[-1] if ancestors else i
        groups[root].add(i)

    for outer, inner in groups.items():
        ring_ids = [outer] + list(inner.difference(set([outer])))
        pixel_rings = [[tuple(int(v) for v in pt[0]) for pt in polygons[r]] for r in ring_ids]
        if polygon_is_valid(pixel_rings):
            coords = [featurize(tile, ring, grown.shape[:2]) for ring in pixel_rings]
            features.append({"type": "Feature", "geometry": {"type": "Polygon", "coordinates": coords}, "properties": {}})
        else:
            warnings.append(W_INVALID)
    return features, warnings


class ParkingHandler:
    """Drop-in for robosat.features.parking.ParkingHandler: `apply(tile, mask)` per tile, `save(out)`; plus `apply_batch` for a
    batch of label images already on the device."""

    kernel_size_denoise = 20
    kernel_size_grow = 20
    simplify_threshold = 0.01

    def __init__(self):
        self.features = []

    def check_zoom(self, tile):
        if tile.z != 18:
            raise NotImplementedError("Parking lot post-processing thresholds are tuned for z18")

    def _gather(self, results):
        for features, warnings in results:
            for w in warnings:
                print(w, file=sys.stderr)
            self.features.extend(features)

    def apply(self, tile, mask):
        import torch

        self.check_zoom(tile)
        labels = torch.from_numpy(np.ascontiguousarray(mask, dtype=np.uint8)[None]).cuda()
        self.apply_batch([tile], labels, 1)

    def apply_batch(self, tiles, labels_device, class_index, pool=None):
        """tiles: N tiles; labels_device: uint8 CUDA tensor [N, H, W] of class indices. Features of (labels == class_index) are
        appended in tile order. Tiles whose grown mask is empty do no host work. `pool` (an Executor) runs the contour step."""
        for t in tiles:
            self.check_zoom(t)
        grown, counts = morph_device(labels_device, class_index, parking_chain(self.kernel_size_denoise, self.kernel_size_grow))
        full = np.flatnonzero(counts.cpu().numpy())
        if len(full) == 0:
            return
        import torch

        masks = grown[torch.from_numpy(full).to(grown.device)].cpu().numpy()
        work = [(tiles[i], m) for i, m in zip(full, masks)]
        run = lambda tm: polygons_from_grown(tm[0], tm[1], self.simplify_threshold)  # noqa: E731
        self._gather(pool.map(run, work) if pool is not None else map(run, work))

    def save(self, out):
        with open(out, "w") as fp:
            json.dump({"type": "FeatureCollection", "features": self.features}, fp)


# --- buildings (this project's rule; the reference has no building handler: DESIGN.md §8) ----------------------------------------

def polygons_from_filled(tile, filled, simplify_epsilon=1.0):
    """Host half of `BuildingHandler`: one Polygon per outer contour of a cleaned {0, 1} uint8 mask, with its holes.

    Contours are `cv2.findContours(RETR_CCOMP, CHAIN_APPROX_SIMPLE)`: outer contours in OpenCV's order, each followed by its child
    holes in list order. Every ring is simplified with `approxPolyDP(epsilon=simplify_epsilon)`; when a simplified ring has fewer
    than 3 vertices or the simplified polygon is not valid, the traced rings are used, and when those are not valid either the
    polygon is skipped with W_INVALID. Returns (features, warnings); thread-safe, as `polygons_from_grown`."""
    import cv2

    features, warnings = [], []
    contours, hierarchy = cv2.findContours(filled, cv2.RETR_CCOMP, cv2.CHAIN_APPROX_SIMPLE)
    if hierarchy is None:
        return features, warnings
    parents = hierarchy[0][:, 3]
    for outer in np.flatnonzero(parents == -1):
        ring_ids = [outer] + [int(h) for h in np.flatnonzero(parents == outer)]
        traced = [[tuple(int(v) for v in pt[0]) for pt in contours[r]] for r in ring_ids]
        simplified = [[tuple(int(v) for v in pt[0]) for pt in cv2.approxPolyDP(contours[r], simplify_epsilon, True)] for r in ring_ids]
        if all(len(r) >= 3 for r in simplified) and polygon_is_valid(simplified):
            rings = simplified
        elif polygon_is_valid(traced):
            rings = traced
        else:
            warnings.append(W_INVALID)
            continue
        coords = [featurize(tile, ring, filled.shape[:2]) for ring in rings]
        features.append({"type": "Feature", "geometry": {"type": "Polygon", "coordinates": coords}, "properties": {}})
    return features, warnings


class BuildingHandler(ParkingHandler):
    """Building footprints: `apply(tile, mask)` per tile, `apply_batch` for a batch of label images on the device, `save(out)`.

    The mask cleanup (an opening with a k_denoise x k_denoise ellipse, speck drop, small-hole fill) runs on the device in
    `building_clean_device`; the contours run on the host in `polygons_from_filled`. The thresholds are this project's choices
    for z18 tiles of 512 px (64 px is about 2.4 m square there), not tuned against imagery."""

    kernel_size_denoise = 5
    min_area = 64
    min_hole_area = 64
    simplify_epsilon = 1.0

    def check_zoom(self, tile):
        if tile.z != 18:
            raise NotImplementedError("Building post-processing thresholds are set for z18")

    def apply_batch(self, tiles, labels_device, class_index, pool=None):
        """tiles: N tiles; labels_device: uint8 CUDA tensor [N, H, W] of class indices. Features of (labels == class_index) are
        appended in tile order. Tiles whose cleaned mask is empty do no host work. `pool` (an Executor) runs the contour step."""
        for t in tiles:
            self.check_zoom(t)
        filled, counts = building_clean_device(labels_device, class_index, self.kernel_size_denoise, self.min_area, self.min_hole_area)
        full = np.flatnonzero(counts.cpu().numpy())
        if len(full) == 0:
            return
        import torch

        masks = filled[torch.from_numpy(full).to(filled.device)].cpu().numpy()
        work = [(tiles[i], m) for i, m in zip(full, masks)]
        run = lambda tm: polygons_from_filled(tm[0], tm[1], self.simplify_epsilon)  # noqa: E731
        self._gather(pool.map(run, work) if pool is not None else map(run, work))


# --- roads (this project's rule; the reference has no road handler: DESIGN.md §8) ------------------------------------------------

def road_thin_device(planes):
    """planes: uint8 CUDA tensor [N, H, W] (rows contiguous) -> (uint8 [N, H, W] {0, 1} Zhang-Suen skeleton of (planes != 0), int32
    [N] full iterations run, the last one that deleted nothing included). Refuses a plane of more than RSB_ROAD_MAX_WORDS 32-bit
    row words with an RsbError before any launch. Enqueued on the current stream, no synchronisation."""
    import torch

    N, H, W, stride = _planes(planes, "road_thin_device")
    skel = torch.empty((N, H, W), dtype=torch.uint8, device=planes.device)
    iterations = torch.empty((N,), dtype=torch.int32, device=planes.device)
    _lib.check(_lib.load().rsb_road_thin(planes.data_ptr(), stride, N, H, W, skel.data_ptr(), iterations.data_ptr(), _lib.current_stream_ptr()),
               "rsb_road_thin")
    return skel, iterations


def _contiguous(t, dtype, what):
    import torch

    if not t.is_cuda or t.dtype != getattr(torch, dtype) or t.dim() != 3 or not t.is_contiguous():
        raise ValueError("%s needs a contiguous %s CUDA tensor [N, H, W]" % (what, dtype))
    return t.shape


def road_degree_device(skel):
    """skel: contiguous uint8 CUDA tensor [N, H, W] {0, 1} -> int8 [N, H, W] m-degree of every skeleton pixel, -1 off it"""
    import torch

    N, H, W = _contiguous(skel, "uint8", "road_degree_device")
    deg = torch.empty((N, H, W), dtype=torch.int8, device=skel.device)
    _lib.check(_lib.load().rsb_road_degree(skel.data_ptr(), N, H, W, deg.data_ptr(), _lib.current_stream_ptr()), "rsb_road_degree")
    return deg


def road_prune_device(skel, deg, min_length):
    """skel, deg: contiguous [N, H, W] from road_thin_device / road_degree_device -> uint8 [N, H, W] skel without its spurs and
    short isolated pieces (fewer than min_length pixels, a spur's junction not counted), decided in one pass on (skel, deg)"""
    import torch

    N, H, W = _contiguous(skel, "uint8", "road_prune_device")
    if _contiguous(deg, "int8", "road_prune_device") != skel.shape:
        raise ValueError("road_prune_device: deg and skel differ in shape")
    out = torch.empty_like(skel)
    _lib.check(_lib.load().rsb_road_prune(skel.data_ptr(), deg.data_ptr(), N, H, W, int(min_length), out.data_ptr(), _lib.current_stream_ptr()),
               "rsb_road_prune")
    return out


def road_chains_device(skel, deg):
    """skel, deg: contiguous [N, H, W] -> per plane a list of int32 arrays, the pixel indices y * W + x of each chain of the graph
    (DESIGN.md §8), in (first pixel, second pixel) order. Synchronises once for the per-plane totals; planes without chains copy
    nothing back."""
    import torch

    from robosat_b200.cover import _alloc

    N, H, W = _contiguous(skel, "uint8", "road_chains_device")
    if _contiguous(deg, "int8", "road_chains_device") != skel.shape:
        raise ValueError("road_chains_device: deg and skel differ in shape")
    dev = skel.device
    lib, stream = _lib.load(), _lib.current_stream_ptr()
    labels, flags = components_device(skel, 1, 8)
    counts = _alloc((N, H, W), torch.int32, dev, "road chain counts")
    rows = torch.empty((N, H), dtype=torch.int64, device=dev)
    totals = torch.empty((N,), dtype=torch.int64, device=dev)
    _lib.check(lib.rsb_road_chain_count(skel.data_ptr(), deg.data_ptr(), labels.data_ptr(), flags.data_ptr(), N, H, W, counts.data_ptr(),
                                        rows.data_ptr(), totals.data_ptr(), stream), "rsb_road_chain_count")
    t = totals.cpu().numpy()
    nchains, npixels = (t >> 32).astype(np.int64), (t & 0xffffffff).astype(np.int64)
    out = [[] for _ in range(N)]
    if nchains.sum() == 0:
        return out
    chain_base = np.concatenate([[0], np.cumsum(nchains)[:-1]])
    pixel_base = np.concatenate([[0], np.cumsum(npixels)[:-1]])
    offsets = _alloc((int(nchains.sum()),), torch.int64, dev, "road chain offsets")
    pixels = _alloc((int(npixels.sum()),), torch.int32, dev, "road chain pixels")
    cb, pb = torch.from_numpy(chain_base).to(dev), torch.from_numpy(pixel_base).to(dev)
    _lib.check(lib.rsb_road_chain_write(skel.data_ptr(), deg.data_ptr(), labels.data_ptr(), flags.data_ptr(), N, H, W, counts.data_ptr(),
                                        rows.data_ptr(), cb.data_ptr(), pb.data_ptr(), offsets.data_ptr(), pixels.data_ptr(), stream),
               "rsb_road_chain_write")
    offsets, pixels = offsets.cpu().numpy(), pixels.cpu().numpy()
    ends = np.append(offsets[1:], len(pixels))
    for n in np.flatnonzero(nchains):
        c0, c1 = chain_base[n], chain_base[n] + nchains[n]
        out[n] = [pixels[offsets[c]:ends[c]] for c in range(c0, c1)]
    return out


def road_device(planes, min_area=256, min_hole_area=256, min_length=20):
    """planes: uint8 CUDA tensor [N, H, W] of halo'd binary road masks {0, 1} -> per plane the list of its chains (int32 pixel
    indices y * W + x of the plane): the cleanup (`rsb_building_clean`), the thinning, the spur pruning and the chains of what
    remains (DESIGN.md §8). Synchronises once."""
    import torch

    from robosat_b200.cover import _alloc

    N, H, W, stride = _planes(planes, "road_device")
    work = _alloc((N, H, W), torch.int32, planes.device, "road component labels")
    stats = _alloc((N, H, W), torch.int32, planes.device, "road component areas")
    clean = torch.empty((N, H, W), dtype=torch.uint8, device=planes.device)
    counts = torch.empty((N,), dtype=torch.int32, device=planes.device)
    _lib.check(_lib.load().rsb_building_clean(planes.data_ptr(), stride, N, H, W, int(min_area), int(min_hole_area), work.data_ptr(),
                                              stats.data_ptr(), clean.data_ptr(), counts.data_ptr(), _lib.current_stream_ptr()),
               "rsb_building_clean")
    del work, stats
    skel, _ = road_thin_device(clean)
    pruned = road_prune_device(skel, road_degree_device(skel), min_length)
    return road_chains_device(pruned, road_degree_device(pruned))


def halo_plane(center, neighbours, class_index, halo, out):
    """Writes the halo'd binary plane of one tile into out (uint8 [H + 2 halo, W + 2 halo]): (mask == class_index) of the tile and
    of the halo-px strips of its 8 neighbours; `neighbours[(dy, dx)]` is a neighbour's mask or None (background)."""
    H, W = center.shape
    h = halo
    out[:] = 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            m = center if (dy, dx) == (0, 0) else neighbours.get((dy, dx))
            if m is None:
                continue
            ys = slice(H - h, H) if dy < 0 else (slice(0, h) if dy > 0 else slice(0, H))
            xs = slice(W - h, W) if dx < 0 else (slice(0, h) if dx > 0 else slice(0, W))
            oy = 0 if dy < 0 else (h + H if dy > 0 else h)
            ox = 0 if dx < 0 else (h + W if dx > 0 else h)
            sub = m[ys, xs]
            np.equal(sub, class_index, out=out[oy:oy + sub.shape[0], ox:ox + sub.shape[1]].view(bool))


def _runs(chain, H, W, halo):
    """The maximal runs of a chain's pixels inside the tile -> [(points [(x, y)], closed)] in tile pixel coordinates: pixel centres,
    plus the midpoint of the two centres where a run continues to a pixel outside the tile"""
    Wp = W + 2 * halo
    y, x = chain // Wp - halo, chain % Wp - halo
    inside = (y >= 0) & (y < H) & (x >= 0) & (x < W)
    if not inside.any():
        return []
    cx, cy = x + 0.5, y + 0.5
    if inside.all() and chain[0] == chain[-1]:
        return [([(float(a), float(b)) for a, b in zip(cx[:-1], cy[:-1])], True)]
    out = []
    edges = np.flatnonzero(np.diff(np.concatenate([[0], inside.astype(np.int8), [0]])))
    for i, j in zip(edges[0::2], edges[1::2]):
        pts = [(float(a), float(b)) for a, b in zip(cx[i:j], cy[i:j])]
        if i > 0:
            pts.insert(0, (0.5 * float(cx[i - 1] + cx[i]), 0.5 * float(cy[i - 1] + cy[i])))
        if j < len(chain):
            pts.append((0.5 * float(cx[j - 1] + cx[j]), 0.5 * float(cy[j - 1] + cy[j])))
        if len(pts) >= 2:
            out.append((pts, False))
    return out


def lines_from_chains(tile, chains, shape, halo, simplify_epsilon=1.0):
    """Host half of `RoadHandler`: the chains of one halo'd plane (pixel indices of the plane) -> LineString features of the tile
    of `shape` (rows, cols): each chain cut into its runs inside the tile, simplified with `approxPolyDP(epsilon)` (closed for a
    whole cycle inside the tile, which then repeats its first point) and mapped to lon/lat. Thread-safe."""
    import cv2

    H, W = shape
    features = []
    for chain in chains:
        for pts, closed in _runs(np.asarray(chain, dtype=np.int64), H, W, halo):
            simple = cv2.approxPolyDP(np.array(pts, dtype=np.float32).reshape(-1, 1, 2), simplify_epsilon, closed).reshape(-1, 2)
            line = [(float(a), float(b)) for a, b in simple]
            if closed:
                line.append(line[0])
            if len(line) < 2:
                continue
            coords = [list(pixel_to_location(tile, a / W, 1. - b / H)) for a, b in line]
            features.append({"type": "Feature", "geometry": {"type": "LineString", "coordinates": coords}, "properties": {}})
    return features


class RoadHandler(ParkingHandler):
    """Road centre lines: `apply_batch` for a batch of halo'd binary road planes on the device, `save(out)`.

    The cleanup, the thinning, the spur pruning and the chains run on the device (`road_device`); the crop to the tile, the
    simplification and the transform to lon/lat run on the host in `lines_from_chains`. The thresholds are this project's choices
    for z18 tiles (DESIGN.md §8), not tuned against imagery."""

    halo = 64
    min_area = 256
    min_hole_area = 256
    min_length = 20
    simplify_epsilon = 1.0

    def check_zoom(self, tile):
        if tile.z != 18:
            raise NotImplementedError("Road post-processing thresholds are set for z18")

    def apply(self, tile, mask):
        raise NotImplementedError("roads need each tile's neighbours: use apply_batch with halo'd planes (rs features --type road)")

    def apply_batch(self, tiles, planes_device, pool=None):
        """tiles: N tiles; planes_device: uint8 CUDA tensor [N, H + 2 halo, W + 2 halo] of halo'd binary road planes (`halo_plane`).
        Features are appended in tile order. Planes without chains do no host work. `pool` (an Executor) runs the host step."""
        for t in tiles:
            self.check_zoom(t)
        chains = road_device(planes_device, self.min_area, self.min_hole_area, self.min_length)
        _, Hp, Wp = planes_device.shape
        shape = (Hp - 2 * self.halo, Wp - 2 * self.halo)
        work = [(tiles[i], c) for i, c in enumerate(chains) if c]
        run = lambda tc: (lines_from_chains(tc[0], tc[1], shape, self.halo, self.simplify_epsilon), [])  # noqa: E731
        self._gather(pool.map(run, work) if pool is not None else map(run, work))
