"""`rs dedupe` (robosat/tools/dedupe.py, robosat/spatial/core.py): drop the predicted features that OpenStreetMap already maps,
with the overlap test and the areas on the GPU.

For each predicted shape P the reference takes the OSM shapes whose lon/lat bounding boxes meet P's (an rtree query, closed
boxes), keeps those that P `intersects` (GEOS: not disjoint, touching included), and keeps P when there are none or when
IoU(P, U) < threshold, U being their union, with both shapes projected to Mollweide (ESRI:54009). Here:

- both collections are packed once (`ShapeSet`: `rasterize.PolygonSet`s of lon/lat and of projected vertices with the same
  offsets; rings cleaned of zero-length edges and oriented, exteriors counter-clockwise and holes clockwise);
- the candidate pairs come from a vectorised grid join of the closed lon/lat boxes (`candidate_pairs`);
- `rsb_dedupe_intersects` decides each pair exactly on the lon/lat vertices, and `rsb_dedupe_areas` integrates A(P),
  A(P ∩ U) and A(U) over boundary pieces on the projected vertices (csrc/rsb_dedupe.cu, DESIGN.md §8);
- IoU = I / (A(P) + A(U) - I) and the comparison with the threshold run on the host in float64, as the reference's Python does.

The projection is `mollweide`, this project's restatement of PROJ's `moll` on the sphere, applied to (lon, lat): the reference
hands pyproj (lon, lat) where it expects (lat, lon), which DESIGN.md §8 describes. shapely, rtree, pyproj and geojson are not
needed. Device work space is bounded by `budget`: predictions go in batches whose candidate pairs and edge work items fit in it.
"""

import math

import numpy as np

from robosat_b200 import _lib
from robosat_b200.cover import _alloc
from robosat_b200.rasterize import INVALID_ERRORS, W_INVALID, PolygonSet, polygon_to_mercator

R = 6378137.0  # the sphere of ESRI:54009 as restated here
DEFAULT_BUDGET = 1 << 30
# device bytes of a batch: per candidate pair (int32 pair + flag), per edge work item (two float64 terms), per prediction and
# per segment (its arrays)
PAIR_BYTES, ITEM_BYTES, PRED_BYTES, SEGMENT_BYTES = 9, 16, 64, 12
W_OSM_GEOMETRY = "Warning: {} OSM features are not a Polygon or MultiPolygon, ignoring them"
W_OSM_INVALID = "Warning: invalid OSM feature {}, ignoring"
MOLL_ITER, MOLL_TOL = 10, 1e-7  # PROJ's `moll`: Newton steps and tolerance
# a feature of at least INDEX_MIN_EDGES edges gets a y-band index of one band per EDGES_PER_BAND edges, so that a scan of its
# edges near another edge visits the bands that edge spans instead of every edge (DESIGN.md §8)
INDEX_MIN_EDGES, EDGES_PER_BAND = 256, 16


def mollweide(lonlat):
    """[[lon, lat], ...] (degrees) -> float64 [n, 2] Mollweide (x, y) in metres on the sphere R: theta solves
    2 theta + sin 2 theta = pi sin phi by PROJ's Newton loop (at most MOLL_ITER steps, stop when a step is below MOLL_TOL, +-pi/2
    when it does not converge), x = (2 sqrt 2 / pi) R lambda cos theta, y = sqrt 2 R sin theta."""
    a = np.asarray(lonlat, dtype=np.float64).reshape(-1, 2)
    lam, phi = np.radians(a[:, 0]), np.radians(a[:, 1])
    k = math.pi * np.sin(phi)
    u = phi.copy()  # u = 2 theta
    done = np.zeros(len(u), bool)
    with np.errstate(invalid="ignore", divide="ignore"):
        for _ in range(MOLL_ITER):
            v = (u + np.sin(u) - k) / (1.0 + np.cos(u))
            u = np.where(done, u, u - v)
            done |= np.abs(v) < MOLL_TOL
    theta = np.where(done, 0.5 * u, np.where(u < 0.0, -0.5 * math.pi, 0.5 * math.pi))
    return np.stack([(2.0 * math.sqrt(2.0) / math.pi) * R * lam * np.cos(theta), math.sqrt(2.0) * R * np.sin(theta)], axis=1)


def areal_polygons(geometry):
    """The lon/lat rings (float64 [n, 2] each) of each polygon of a Polygon or MultiPolygon geometry; raises one of
    INVALID_ERRORS when a polygon fails `rasterize.polygon_to_mercator`'s validity rule."""
    components = [geometry["coordinates"]] if geometry["type"] == "Polygon" else geometry["coordinates"]
    if not components:
        raise ValueError("no polygons")
    polygons = []
    for c in components:
        polygon_to_mercator(c)
        polygons.append([np.asarray([p[:2] for p in ring], np.float64) for ring in c])
    return polygons


def is_areal(feature):
    return ((feature.get("geometry") or {}).get("type")) in ("Polygon", "MultiPolygon")


class ShapeSet:
    """Areal features packed for dedupe. `index[f]` is the input position of packed feature f, which owns polygons
    [feature_polys[f], feature_polys[f + 1]) of `lonlat` and `xy` (rasterize.PolygonSets with the same offsets). Rings hold no
    two equal consecutive projected vertices and no closing repeat; `next[v]` is the vertex the edge from v ends at. Exterior
    rings run counter-clockwise and holes clockwise in (x, y). `feature_vertices`, `exterior_offsets` / `exteriors` and the
    per-feature boxes (`boxes_ll`, `boxes_xy`, NaN for a feature without vertices) are what the kernels read. `projection` maps
    lon/lat to the (x, y) of `xy`: Mollweide for dedupe, EPSG:3395 for `rs merge`."""

    def __init__(self, polygons_per_feature, index, projection=mollweide):
        self.index = np.asarray(index, np.int64)
        counts = [len(p) for p in polygons_per_feature]
        self.feature_polys = np.zeros(len(counts) + 1, np.int64)
        np.cumsum(counts, out=self.feature_polys[1:])
        raw = PolygonSet([p for ps in polygons_per_feature for p in ps])
        ro, V = raw.ring_offsets, raw.vertices
        nr = len(ro) - 1
        xy = projection(V)
        rid = np.repeat(np.arange(nr), np.diff(ro))
        idx = np.arange(len(V))
        succ = np.where(idx + 1 < ro[rid + 1], idx + 1, ro[rid])
        keep = ~(xy == xy[succ]).all(axis=1)  # equal lon/lat gives equal (x, y), so this drops every zero-length edge of both
        lens = np.bincount(rid[keep], minlength=nr)
        offsets = np.zeros(nr + 1, np.int64)
        np.cumsum(lens, out=offsets[1:])
        V, xy, rid = V[keep], xy[keep], rid[keep]
        j = np.arange(len(V))
        first, n = offsets[rid], lens[rid]
        succ = np.where(j + 1 < first + n, j + 1, first)
        rel = xy - xy[first]
        signed = np.bincount(rid, weights=rel[:, 0] * rel[succ, 1] - rel[succ, 0] * rel[:, 1], minlength=nr)
        exterior = np.zeros(nr, bool)
        exterior[raw.poly_rings[:-1][np.diff(raw.poly_rings) > 0]] = True
        flip = (exterior & (signed < 0)) | (~exterior & (signed > 0))
        src = np.where(flip[rid], first + (n - (j - first)) % np.maximum(n, 1), j)  # reversed, keeping the first vertex
        V, xy = V[src], xy[src]
        self.lonlat = PolygonSet.from_arrays(V, offsets, raw.poly_rings)
        self.xy = PolygonSet.from_arrays(xy, offsets, raw.poly_rings)
        if len(V) > np.iinfo(np.int32).max:
            raise _lib.RsbError("%d vertices in one collection; at most 2^31 - 1 are supported" % len(V))
        self.next = succ.astype(np.int32)
        self.feature_vertices = offsets[raw.poly_rings[self.feature_polys]]
        ext_rings = raw.poly_rings[:-1]
        has = lens[ext_rings] > 0 if nr else np.zeros(len(ext_rings), bool)
        poly_feature = np.repeat(np.arange(len(counts)), counts)
        self.exteriors = offsets[ext_rings[has]]
        self.exterior_offsets = np.zeros(len(counts) + 1, np.int64)
        np.cumsum(np.bincount(poly_feature[has], minlength=len(counts)), out=self.exterior_offsets[1:])
        self.boxes_ll = self._boxes(V)
        self.boxes_xy = self._boxes(xy)
        self._band_index(xy)
        self.device = None

    def _band_index(self, xy):
        """per feature of at least INDEX_MIN_EDGES edges: nb equal bands over its projected y range; band_ranges[f] = (y0, nb / height)
        maps y to band floor((y - y0) * that), clamped to [0, nb); band b of feature f lists, in band_edges[band_offsets[fb + b] ..
        band_offsets[fb + b + 1]) with fb = feature_bands[f], the edges (by first vertex) whose y ranges meet it"""
        n = self.edges()
        height = self.boxes_xy[:, 3] - self.boxes_xy[:, 1]
        nb = np.where((n >= INDEX_MIN_EDGES) & (height > 0), n // EDGES_PER_BAND, 0)
        self.feature_bands = np.zeros(len(n) + 1, np.int64)
        np.cumsum(nb, out=self.feature_bands[1:])
        self.band_ranges = np.zeros((len(n), 2))
        idx = np.flatnonzero(nb)
        self.band_ranges[idx, 0] = self.boxes_xy[idx, 1]
        self.band_ranges[idx, 1] = nb[idx] / height[idx]
        v = np.concatenate([np.arange(self.feature_vertices[f], self.feature_vertices[f + 1]) for f in idx]) if len(idx) else np.zeros(0, np.int64)
        f = np.repeat(idx, n[idx])
        y0, inv, last = self.band_ranges[f, 0], self.band_ranges[f, 1], (nb[f] - 1).astype(np.float64)
        ys = np.stack([xy[v, 1], xy[self.next[v], 1]], axis=1) if len(v) else np.zeros((0, 2))
        b0 = np.clip(np.floor((ys.min(1) - y0) * inv), 0.0, last).astype(np.int64)
        b1 = np.clip(np.floor((ys.max(1) - y0) * inv), 0.0, last).astype(np.int64)
        cnt = b1 - b0 + 1
        band = np.repeat(self.feature_bands[f] + b0, cnt) + (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt))
        order = np.argsort(band, kind="stable")
        self.band_edges = np.repeat(v, cnt)[order].astype(np.int32)
        self.band_offsets = np.zeros(self.feature_bands[-1] + 1, np.int64)
        np.cumsum(np.bincount(band, minlength=int(self.feature_bands[-1])), out=self.band_offsets[1:])

    def _boxes(self, v):
        b = np.full((len(self), 4), np.nan)
        starts, ends = self.feature_vertices[:-1], self.feature_vertices[1:]
        full = np.flatnonzero(ends > starts)
        if len(full):
            b[full, :2] = np.minimum.reduceat(v, starts[full])
            b[full, 2:] = np.maximum.reduceat(v, starts[full])
        return b

    def __len__(self):
        return len(self.index)

    def edges(self):
        return np.diff(self.feature_vertices)

    def upload(self, device):
        """copies the arrays to `device` (once; outside any batch budget) -> (lon/lat Shapes, projected Shapes) for the kernels"""
        if self.device is None:
            arrays = (("vll", self.lonlat.vertices, np.float64), ("vxy", self.xy.vertices, np.float64), ("next", self.next, np.int32),
                      ("fv", self.feature_vertices, np.int64), ("eo", self.exterior_offsets, np.int64), ("ext", self.exteriors, np.int64),
                      ("bll", self.boxes_ll, np.float64), ("bxy", self.boxes_xy, np.float64), ("fb", self.feature_bands, np.int64),
                      ("br", self.band_ranges, np.float64), ("bo", self.band_offsets, np.int64), ("be", self.band_edges, np.int32))
            self.d = {k: _upload(a, t, device, "the packed shapes (%d bytes)" % a.nbytes) for k, a, t in arrays}
            self.device = device
        d = self.d

        def shapes(v, b):
            return _lib.Shapes(v.data_ptr(), d["next"].data_ptr(), d["fv"].data_ptr(), d["eo"].data_ptr(), d["ext"].data_ptr(), b.data_ptr(),
                               d["fb"].data_ptr(), d["br"].data_ptr(), d["bo"].data_ptr(), d["be"].data_ptr(), len(self.next), len(self), 0)

        return shapes(d["vll"], d["bll"]), shapes(d["vxy"], d["bxy"])


def parse(features, osm):
    """GeoJSON features -> (ShapeSet of the valid areal ones, warnings). Predicted features (osm=False) that fail the validity
    rule get `rasterize`'s W_INVALID; other geometry types are not packed (the caller passes them through). OSM features that
    are not areal are counted in one summary warning, and invalid ones are ignored with W_OSM_INVALID."""
    polygons, index, warnings, other = [], [], [], 0
    for i, feature in enumerate(features):
        if not is_areal(feature):
            other += 1
            continue
        try:
            polygons.append(areal_polygons(feature["geometry"]))
        except INVALID_ERRORS:
            warnings.append((W_OSM_INVALID if osm else W_INVALID).format(i))
            continue
        index.append(i)
    if osm and other:
        warnings.insert(0, W_OSM_GEOMETRY.format(other))
    return ShapeSet(polygons, index), warnings


def candidate_pairs(pbox, qbox, cell=None):
    """(p, q) int64 index arrays, sorted, of the boxes (xmin, ymin, xmax, ymax) that meet as closed boxes (touching counts); NaN
    boxes meet nothing. A grid join: boxes of at most 64 cells of size `cell` (by default the median box extent) are listed in
    the cells they cover and looked up by cell; each larger one is compared with every box of the other side, one vectorised
    test per large box, so host memory stays linear in the number of boxes and pairs."""
    pbox, qbox = np.asarray(pbox, np.float64).reshape(-1, 4), np.asarray(qbox, np.float64).reshape(-1, 4)
    pid, qid = np.flatnonzero(~np.isnan(pbox).any(1)), np.flatnonzero(~np.isnan(qbox).any(1))
    empty = np.zeros(0, np.int64)
    if not len(pid) or not len(qid):
        return empty, empty
    if cell is None:
        ext = np.concatenate([pbox[pid, 2:] - pbox[pid, :2], qbox[qid, 2:] - qbox[qid, :2]]).max(1)
        cell = float(np.median(ext))
    lo = np.minimum(pbox[pid, :2].min(0), qbox[qid, :2].min(0))
    span = np.maximum(pbox[pid, 2:].max(0), qbox[qid, 2:].max(0)) - lo
    cell = max(cell, float(span.max()) / 2 ** 20, 1e-300)

    def cells(b):
        c0 = np.floor((b[:, :2] - lo) / cell).astype(np.int64)
        c1 = np.floor((b[:, 2:] - lo) / cell).astype(np.int64)
        return c0, c1, (c1[:, 0] - c0[:, 0] + 1) * (c1[:, 1] - c0[:, 1] + 1)

    def enumerate_cells(ids, c0, c1, cnt):
        rep = np.repeat(np.arange(len(ids)), cnt)
        k = np.arange(len(rep)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        w = (c1[:, 0] - c0[:, 0] + 1)[rep]
        return ids[rep], ((c0[rep, 0] + k % w) << 21) | (c0[rep, 1] + k // w)

    pc0, pc1, pcnt = cells(pbox[pid])
    qc0, qc1, qcnt = cells(qbox[qid])
    ps, qs = [], []
    pbig, qbig = pcnt > 64, qcnt > 64

    def meeting(b, other, ids):  # the boxes of `ids` that meet box b: memory per large box is one mask over the other side
        o = other[ids]
        return ids[(b[0] <= o[:, 2]) & (o[:, 0] <= b[2]) & (b[1] <= o[:, 3]) & (o[:, 1] <= b[3])]

    for i in pid[pbig]:  # a large prediction box against every OSM box
        hit = meeting(pbox[i], qbox, qid)
        ps.append(np.full(len(hit), i))
        qs.append(hit)
    for i in qid[qbig]:  # a large OSM box against every small prediction box (large ones were paired above)
        hit = meeting(qbox[i], pbox, pid[~pbig])
        ps.append(hit)
        qs.append(np.full(len(hit), i))
    small_q = ~qbig
    qi, qkey = enumerate_cells(qid[small_q], qc0[small_q], qc1[small_q], qcnt[small_q])
    order = np.argsort(qkey, kind="stable")
    qi, qkey = qi[order], qkey[order]
    pi, pkey = enumerate_cells(pid[~pbig], pc0[~pbig], pc1[~pbig], pcnt[~pbig])
    a, b = np.searchsorted(qkey, pkey, "left"), np.searchsorted(qkey, pkey, "right")
    n = b - a
    ps.append(np.repeat(pi, n))
    qs.append(qi[np.repeat(a, n) + (np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n))])
    p, q = np.concatenate(ps).astype(np.int64), np.concatenate(qs).astype(np.int64)
    meet = (pbox[p, 0] <= qbox[q, 2]) & (qbox[q, 0] <= pbox[p, 2]) & (pbox[p, 1] <= qbox[q, 3]) & (qbox[q, 1] <= pbox[p, 3])
    key = np.unique(p[meet] * len(qbox) + q[meet])
    return key // len(qbox), key % len(qbox)


def _plan(cost, budget):
    """[start, end) runs of consecutive predictions whose summed device bytes fit in `budget`"""
    big = np.flatnonzero(cost > budget)
    if len(big):
        raise _lib.RsbError("prediction %d needs %d bytes of device work space for its candidate pairs and edges, more than the budget of %d bytes"
                            % (big[0], cost[big[0]], budget))
    cum = np.concatenate([[0], np.cumsum(cost)])
    runs, start = [], 0
    while start < len(cost):
        end = int(np.searchsorted(cum, cum[start] + budget, "right")) - 1
        runs.append((start, max(end, start + 1)))
        start = runs[-1][1]
    return runs


def dedupe_device(predicted, osm, threshold, budget=DEFAULT_BUDGET, device="cuda", stats=None):
    """The dedupe decision for each predicted GeoJSON feature against the OSM ones -> (keep bool [n], areas float64 [n, 3] =
    (A(P), A(P ∩ U), A(U)) in m², NaN where no IoU was needed). See `decide`."""
    ps, _ = parse(predicted, False)
    qs, _ = parse(osm, True)
    return decide(ps, qs, threshold, [not is_areal(f) for f in predicted], budget, device, stats)


def dedupe(features_predicted, features_osm, threshold, budget=DEFAULT_BUDGET, device="cuda"):
    """Drop-in for the reference's `rs dedupe` loop: the kept predicted features, in input order, as GeoJSON Feature dicts with
    the reference's layout (`output_feature`: properties dropped, rings closed, coordinates as floats)."""
    keep, _ = dedupe_device(features_predicted, features_osm, threshold, budget, device)
    return kept_features(features_predicted, keep)


def output_geometry(geometry):
    """the geometry as `shapely.geometry.mapping` returns it for a kept feature: Polygon and MultiPolygon rings closed and
    coordinates as floats; other types unchanged"""
    def ring(r):
        out = [[float(c) for c in p] for p in r]
        if out and out[0] != out[-1]:
            out.append(list(out[0]))
        return out

    kind = geometry.get("type")
    if kind == "Polygon":
        return {"type": kind, "coordinates": [ring(r) for r in geometry["coordinates"]]}
    if kind == "MultiPolygon":
        return {"type": kind, "coordinates": [[ring(r) for r in c] for c in geometry["coordinates"]]}
    return geometry


def output_feature(feature):
    """`geojson.Feature(geometry=mapping(shape))` of the reference: {"type": "Feature", "geometry": …, "properties": {}}"""
    return {"type": "Feature", "geometry": output_geometry(feature.get("geometry") or {}), "properties": {}}


def kept_features(features, keep):
    return [output_feature(f) for f, k in zip(features, keep) if k]


def decide(ps, qs, threshold, passthrough, budget=DEFAULT_BUDGET, device="cuda", stats=None):
    """`dedupe_device` on parsed collections (`parse`). A prediction is kept when passthrough[i] (not a Polygon or MultiPolygon),
    when no OSM feature intersects it, or when IoU(P, U) < threshold; a zero-area P ∪ U counts as IoU 0. An invalid prediction
    is not kept. `budget` bounds the device bytes of a batch (the packed shapes, uploaded once, are outside it); a prediction
    that alone needs more raises RsbError before anything is uploaded, and an allocation the device cannot hold raises RsbError
    naming what did not fit. `stats` (a dict), when given, receives the candidate pair, intersecting and item
    counts and the kernel times (CUDA events). Synchronises."""
    import torch

    areas_ps = np.full((len(ps), 3), np.nan)
    pp, qq = candidate_pairs(ps.boxes_ll, qs.boxes_ll)
    stats = stats if stats is not None else {}
    stats.update(pairs=len(pp), items=0, intersects_ms=0.0, areas_ms=0.0, batches=0)
    if len(pp):
        pcount = np.bincount(pp, minlength=len(ps))
        pair_start = np.concatenate([[0], np.cumsum(pcount)])
        bound_items = ps.edges() + np.bincount(pp, weights=qs.edges()[qq], minlength=len(ps)).astype(np.int64)
        cost = PAIR_BYTES * pcount + ITEM_BYTES * bound_items + PRED_BYTES + SEGMENT_BYTES * (pcount + 1)
        cost[pcount == 0] = 0
        plan = _plan(cost, budget)  # raises before anything is uploaded
        dev = torch.device(device)
        p_ll, p_xy = ps.upload(dev)
        q_ll, q_xy = qs.upload(dev)
        lib = _lib.load()
        for start, end in plan:
            a, b = pair_start[start], pair_start[end]
            if a == b:
                continue
            stats["batches"] += 1
            hit = _intersects(lib, p_ll, q_ll, pp[a:b], qq[a:b], dev, stats)
            if hit.any():
                _areas(lib, ps, qs, p_xy, q_xy, pp[a:b][hit], qq[a:b][hit], dev, areas_ps, stats)
    a_p, a_i, a_u = areas_ps[:, 0], areas_ps[:, 1], areas_ps[:, 2]
    has = ~np.isnan(a_p)
    union = a_p + a_u - a_i
    iou = np.zeros(len(ps))
    ok = has & (union != 0.0)
    iou[ok] = a_i[ok] / union[ok]
    stats["intersecting"] = int(has.sum())
    keep = np.asarray(passthrough, bool).copy()
    keep[ps.index] = ~has | (iou < threshold)
    areas = np.full((len(keep), 3), np.nan)
    areas[ps.index] = areas_ps
    return keep, areas


def _upload(a, dtype, device, what):
    """a copy of numpy `a` on the device (one element at least, so the pointer is valid), allocated by cover._alloc so that an
    allocation the device cannot hold is an RsbError naming `what`"""
    import torch

    a = np.ascontiguousarray(a, dtype=dtype)
    d = _alloc((max(1, len(a)),) + a.shape[1:], torch.from_numpy(a[:0]).dtype, device, what)
    if len(a):
        d[:len(a)].copy_(torch.from_numpy(a))
    return d


def _intersects(lib, p_ll, q_ll, p, q, dev, stats):
    """flags of the candidate pairs (p, q): not disjoint, on the device"""
    import torch

    pairs = np.stack([p, q], axis=1).astype(np.int32)
    d_pairs = _upload(pairs, np.int32, dev, "%d candidate pairs" % len(pairs))
    out = _alloc((len(pairs),), torch.uint8, dev, "%d intersect flags" % len(pairs))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    _lib.check(lib.rsb_dedupe_intersects(p_ll, q_ll, d_pairs.data_ptr(), len(pairs), out.data_ptr(), _lib.current_stream_ptr()), "rsb_dedupe_intersects")
    ev[1].record()
    flags = out.cpu().numpy().astype(bool)
    stats["intersects_ms"] += ev[0].elapsed_time(ev[1])
    return flags


def _areas(lib, ps, qs, p_xy, q_xy, p, q, dev, areas_out, stats):
    """(A(P), A(P ∩ U), A(U)) of the predictions in p (sorted, with their intersecting OSM features q) into areas_out"""
    import torch

    preds, m = np.unique(p, return_counts=True)
    B = len(preds)
    set_offsets = np.zeros(B + 1, np.int64)
    np.cumsum(m, out=set_offsets[1:])
    seg_items = np.empty(B + len(q), np.int64)
    pseg = np.arange(B) + set_offsets[:-1]
    qmask = np.ones(len(seg_items), bool)
    qmask[pseg] = False
    seg_items[pseg] = ps.edges()[preds]
    seg_items[qmask] = qs.edges()[q]
    item_offsets = np.zeros(len(seg_items) + 1, np.int64)
    np.cumsum(seg_items, out=item_offsets[1:])
    seg_pred = np.repeat(np.arange(B), m + 1).astype(np.int32)
    box = ps.boxes_xy[preds]
    origins = np.stack([0.5 * (box[:, 0] + box[:, 2]), 0.5 * (box[:, 1] + box[:, 3])], axis=1)
    items = int(item_offsets[-1])

    d = [_upload(x, t, dev, "the batch's segment arrays") for x, t in ((preds, np.int32), (origins.reshape(-1), np.float64), (set_offsets, np.int64), (q, np.int32), (item_offsets, np.int64), (seg_pred, np.int32))]
    terms = _alloc((max(1, 2 * items),), torch.float64, dev, "the edge terms of %d work items" % items)
    out = _alloc((B, 3), torch.float64, dev, "the areas of %d predictions" % B)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    _lib.check(lib.rsb_dedupe_areas(p_xy, q_xy, B, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), len(seg_items), d[4].data_ptr(), d[5].data_ptr(),
                                    items, terms.data_ptr(), out.data_ptr(), _lib.current_stream_ptr()), "rsb_dedupe_areas")
    ev[1].record()
    areas_out[preds] = out.cpu().numpy()
    stats["areas_ms"] += ev[0].elapsed_time(ev[1])
    stats["items"] += items
