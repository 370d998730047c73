"""`rs merge` (robosat/tools/merge.py, robosat/graph/core.py, robosat/spatial/core.py): join the features that lie within
`threshold` metres of each other, such as the fragments `rs features` leaves on both sides of a tile border, with the
adjacency test, the components and the closing on the GPU.

The reference buffers every shape by the threshold in EPSG:3395, links shape i to t when buffer(i) intersects t, takes the
connected components, and writes buffer(union of the buffered members, -threshold) with its area. GEOS's buffer is not
restated; this project defines the rule instead (DESIGN.md §8). With d the threshold:

- the shapes are projected to EPSG:3395 (`mercator`, PROJ's `merc` on WGS84) and packed once (`dedupe.ShapeSet`);
- candidate pairs are the closed boxes, widened by d, that meet (`dedupe.candidate_pairs`); a pair is linked when
  `rsb_dedupe_intersects` finds the shapes not disjoint or `rsb_merge_near` finds a vertex of one within d of an edge of the
  other (float64, every operation rounded on its own);
- `rsb_merge_components` labels every shape with the smallest index of its component; components go out in that order, the
  order of the reference's `UndirectedGraph.components()`;
- each component is filled on a lattice of square cells of side d / CELLS_PER_THRESHOLD (cell centres inside a member polygon,
  `rs rasterize`'s scanline rule) by `rsb_merge_fill`, and `rsb_merge_close` takes the closing erode(dilate(fill)) with the
  digital disk of radius CELLS_PER_THRESHOLD;
- on the host, the closed cells are traced into polygons (4-connected foreground), simplified by Douglas-Peucker at one cell
  unless that breaks validity, mapped back to lon/lat and written with their Mollweide area.

shapely, rtree, pyproj and geojson are not needed. Device work space for the grids is bounded by `budget`.
"""

import concurrent.futures
import math
import os

import numpy as np

from robosat_b200 import _lib
from robosat_b200 import dedupe as DD
from robosat_b200 import features as FT
from robosat_b200.cover import _alloc
# FILL_WORDS, the band budget of rsb_merge_fill, is defined once in rasterize and stays readable as merge.FILL_WORDS
from robosat_b200.rasterize import FILL_WORDS, INVALID_ERRORS, W_INVALID, fill_bands  # noqa: F401

A = 6378137.0  # WGS84
FLATTENING = 1 / 298.257223563
E = math.sqrt(FLATTENING * (2 - FLATTENING))
PHI2_ITER, PHI2_TOL = 15, 1e-10  # PROJ's pj_phi2
CELLS_PER_THRESHOLD = 4  # K: cells per threshold distance, and the radius of the closing's disk in cells
MARGIN = CELLS_PER_THRESHOLD + 2  # cells around a component's box, so that the dilation never reaches the grid edge
DEFAULT_BUDGET = 1 << 30
TILE_ROWS, TILE_WORDS = 32, 32  # a closing CTA's tile
COMPONENT_BYTES = 64  # device bytes per component beyond its two bitmaps: transforms, grid, offsets, bands, tiles (upper bound)
W_GEOMETRY = "Warning: {} features are not a Polygon or MultiPolygon, skipping them"
W_NOT_POLYGON = "Warning: merged feature is neither Polygon nor MultiPoylgon, skipping"  # the reference's spelling
W_NOT_VALID = "Warning: merged feature is not valid, skipping"


def mercator(lonlat):
    """[[lon, lat], ...] (degrees) -> float64 [n, 2] EPSG:3395 (x, y) in metres: PROJ's `merc` on WGS84,
    x = a lambda, y = a (atanh(sin phi) - e atanh(e sin phi))"""
    p = np.asarray(lonlat, dtype=np.float64).reshape(-1, 2)
    s = np.sin(np.radians(p[:, 1]))
    with np.errstate(invalid="ignore", divide="ignore"):
        y = A * (np.arctanh(s) - E * np.arctanh(E * s))
    return np.stack([A * np.radians(p[:, 0]), y], axis=1)


def inverse_mercator(xy):
    """EPSG:3395 (x, y) -> float64 [n, 2] (lon, lat) in degrees: lambda = x / a and PROJ's pj_phi2 iteration for phi (at most
    PHI2_ITER steps, stopping once a step is at most PHI2_TOL)"""
    p = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    ts = np.exp(-p[:, 1] / A)
    phi = 0.5 * math.pi - 2.0 * np.arctan(ts)
    done = np.zeros(len(p), bool)
    for _ in range(PHI2_ITER):
        con = E * np.sin(phi)
        dphi = 0.5 * math.pi - 2.0 * np.arctan(ts * ((1.0 - con) / (1.0 + con)) ** (0.5 * E)) - phi
        phi = np.where(done, phi, phi + dphi)
        done |= np.abs(dphi) <= PHI2_TOL
        if done.all():
            break
    return np.stack([np.degrees(p[:, 0] / A), np.degrees(phi)], axis=1)


def parse(features):
    """GeoJSON features -> (dedupe.ShapeSet on EPSG:3395 of the valid Polygon and MultiPolygon features, warnings). A polygon that
    fails `rasterize.polygon_to_mercator`'s rule, or does not project to finite EPSG:3395 values, gets `rs rasterize`'s warning;
    other geometry types are counted in one summary warning."""
    polygons, index, warnings, other = [], [], [], 0
    for i, feature in enumerate(features):
        if not DD.is_areal(feature):
            other += 1
            continue
        try:
            polys = DD.areal_polygons(feature["geometry"])
            if not all(np.isfinite(mercator(r)).all() for p in polys for r in p):
                raise ValueError("coordinates outside EPSG:3395")
        except INVALID_ERRORS:
            warnings.append(W_INVALID.format(i))
            continue
        polygons.append(polys)
        index.append(i)
    if other:
        warnings.insert(0, W_GEOMETRY.format(other))
    return DD.ShapeSet(polygons, index, projection=mercator), warnings


def candidate_pairs(shapes, d):
    """(i, j) int64 arrays, i < j, sorted: the features whose closed EPSG:3395 boxes, one widened by d on every side, meet"""
    box = shapes.boxes_xy
    p, q = DD.candidate_pairs(box + np.array([-d, -d, d, d]), box)
    keep = p < q
    return p[keep], q[keep]


def _check_threshold(d):
    if not (isinstance(d, (int, float, np.integer, np.floating)) and math.isfinite(d) and d > 0):
        raise ValueError("threshold must be a positive distance in metres, got %r" % (d,))
    return float(d)


def _events():
    import torch

    return [torch.cuda.Event(enable_timing=True) for _ in range(2)]


def _polygon_arrays(shapes, dev):
    """the EPSG:3395 polygon arrays of rsb_merge_fill on the device (once)"""
    if getattr(shapes, "merge_d", None) is None:
        xy = shapes.xy
        shapes.merge_d = [DD._upload(a, t, dev, "the packed polygons (%d bytes)" % a.nbytes)
                          for a, t in ((xy.vertices, np.float64), (xy.ring_offsets, np.int64), (xy.poly_rings, np.int32))]
    return shapes.merge_d


def link(shapes, d, device="cuda", stats=None):
    """linked pairs of the parsed features -> (i, j) int64 arrays of the candidate pairs whose shapes intersect or lie within d
    (on the device)"""
    import torch

    d = _check_threshold(d)
    stats = stats if stats is not None else {}
    p, q = candidate_pairs(shapes, d)
    stats.update(pairs=len(p), intersects_ms=0.0, near_ms=0.0)
    if not len(p):
        return p, q
    dev = torch.device(device)
    lib = _lib.load()
    _, s_xy = shapes.upload(dev)
    hit = DD._intersects(lib, s_xy, s_xy, p, q, dev, stats)
    rest = np.flatnonzero(~hit)
    stats["intersecting"] = int(hit.sum())
    if len(rest):
        pairs = np.stack([p[rest], q[rest]], axis=1).astype(np.int32)
        d_pairs = DD._upload(pairs, np.int32, dev, "%d candidate pairs" % len(pairs))
        out = _alloc((len(pairs),), torch.uint8, dev, "%d near flags" % len(pairs))
        ev = _events()
        ev[0].record()
        _lib.check(lib.rsb_merge_near(s_xy, d_pairs.data_ptr(), len(pairs), d, out.data_ptr(), _lib.current_stream_ptr()), "rsb_merge_near")
        ev[1].record()
        hit[rest] = out.cpu().numpy().astype(bool)
        stats["near_ms"] += ev[0].elapsed_time(ev[1])
    return p[hit], q[hit]


def components_device(n, p, q, device="cuda", stats=None):
    """int32 [n] labels: the smallest node of each node's component under the links (p, q), from rsb_merge_components"""
    import torch

    stats = stats if stats is not None else {}
    if n == 0:
        return np.zeros(0, np.int32)
    dev = torch.device(device)
    pairs = np.stack([p, q], axis=1).astype(np.int32)
    d_pairs = DD._upload(pairs, np.int32, dev, "%d linked pairs" % len(pairs))
    linked = _alloc((max(1, len(pairs)),), torch.uint8, dev, "%d link flags" % len(pairs))
    linked.fill_(1)
    parent = _alloc((n,), torch.int32, dev, "the union-find of %d features" % n)
    labels = _alloc((n,), torch.int32, dev, "the labels of %d features" % n)
    ev = _events()
    ev[0].record()
    _lib.check(_lib.load().rsb_merge_components(d_pairs.data_ptr(), linked.data_ptr(), len(pairs), n, parent.data_ptr(), labels.data_ptr(),
                                                _lib.current_stream_ptr()), "rsb_merge_components")
    ev[1].record()
    out = labels.cpu().numpy()
    stats["components_ms"] = stats.get("components_ms", 0.0) + ev[0].elapsed_time(ev[1])
    return out


class Component:
    """One merged component: `members` (indices into the parsed ShapeSet, ascending), its cell grid (u0, v1, W, H): column k is
    cell u = u0 + k and row r (from the top) is cell v = v1 - r of side `cell` metres, and after `close_device` the closed cells
    `closed` (bool [H, W]) and their count."""

    def __init__(self, members, grid, cell):
        self.members, self.grid, self.cell = members, grid, cell
        self.closed, self.count = None, 0

    def transform(self):
        """(c0, c1, r0, r1): px = c0 + X * c1, py = r0 + Y * r1 maps EPSG:3395 to the grid's cell coordinates"""
        u0, v1, _, _ = self.grid
        return (-float(u0), 1.0 / self.cell, float(v1 + 1), -1.0 / self.cell)

    def words(self):
        return (self.grid[2] + 31) // 32

    def device_bytes(self):
        return 8 * self.grid[3] * self.words() + COMPONENT_BYTES


def components(shapes, labels, d):
    """the Components of the labelled features, in ascending order of label, each with its grid"""
    cell = d / CELLS_PER_THRESHOLD
    if not len(labels):
        return []
    order = np.argsort(labels, kind="stable")
    cuts = np.flatnonzero(np.diff(labels[order])) + 1
    out = []
    for members in np.split(order, cuts):
        box = shapes.boxes_xy[members]
        box = box[~np.isnan(box).any(1)]
        if not len(box):
            out.append(Component(members, (0, 0, 0, 0), cell))
            continue
        u0 = int(math.floor(box[:, 0].min() / cell)) - MARGIN
        u1 = int(math.floor(box[:, 2].max() / cell)) + MARGIN
        v0 = int(math.floor(box[:, 1].min() / cell)) - MARGIN
        v1 = int(math.floor(box[:, 3].max() / cell)) + MARGIN
        out.append(Component(members, (u0, v1, u1 - u0 + 1, v1 - v0 + 1), cell))
    return out


def plan(comps, budget):
    """[start, end) runs of consecutive components whose grids fit in `budget` device bytes; a component that alone needs more
    raises RsbError"""
    runs, start, used = [], 0, 0
    for i, c in enumerate(comps):
        cost = c.device_bytes()
        if cost > budget:
            raise _lib.RsbError("component %d (%d features, a %d x %d cell grid) needs %d bytes of device work space, more than the budget of %d bytes"
                                % (i, len(c.members), c.grid[2], c.grid[3], cost, budget))
        if i > start and used + cost > budget:
            runs.append((start, i))
            start, used = i, 0
        used += cost
    if start < len(comps):
        runs.append((start, len(comps)))
    return runs


def close_device(shapes, comps, device="cuda", stats=None, keep_fill=False):
    """fills and closes the grids of `comps` (one batch) on the device and sets each one's `closed` and `count` (and `fill`
    with keep_fill)"""
    import torch

    stats = stats if stats is not None else {}
    comps = [c for c in comps if c.grid[2] > 0]
    if not comps:
        return
    dev = torch.device(device)
    vertices, ring_offsets, poly_rings = _polygon_arrays(shapes, dev)
    C = len(comps)
    W = np.array([c.grid[2] for c in comps], np.int64)
    H = np.array([c.grid[3] for c in comps], np.int64)
    words = (W + 31) // 32
    offsets = np.zeros(C + 1, np.int64)
    np.cumsum(H * words, out=offsets[1:])
    fp = shapes.feature_polys
    polys = [np.concatenate([np.arange(fp[f], fp[f + 1]) for f in c.members]) for c in comps]
    poly_offsets = np.zeros(C + 1, np.int64)
    np.cumsum([len(x) for x in polys], out=poly_offsets[1:])
    bands, band_rows, max_words = fill_bands(H, words)
    tr, tw = (H + TILE_ROWS - 1) // TILE_ROWS, (words + TILE_WORDS - 1) // TILE_WORDS
    nt = tr * tw
    tc = np.repeat(np.arange(C), nt)
    k = np.arange(len(tc)) - np.repeat(np.cumsum(nt) - nt, nt)
    tiles = np.stack([tc, (k // tw[tc]) * TILE_ROWS, (k % tw[tc]) * TILE_WORDS], axis=1)
    if len(bands) > 0x7fffffff or len(tiles) > 0x7fffffff:
        raise _lib.RsbError("%d fill bands / %d closing tiles in one batch" % (len(bands), len(tiles)))
    arrays = [(poly_offsets, np.int32), (np.concatenate(polys), np.int32), (np.array([c.transform() for c in comps]), np.float64),
              (np.stack([W, H], axis=1), np.int64), (offsets, np.int64), (bands, np.int32), (tiles, np.int32)]
    d_po, d_polys, d_tr, d_grids, d_off, d_bands, d_tiles = [DD._upload(a, t, dev, "the batch's component arrays") for a, t in arrays]
    total = int(offsets[-1])
    fill = _alloc((total,), torch.int32, dev, "the fill bitmaps of %d components" % C)
    closed = _alloc((total,), torch.int32, dev, "the closed bitmaps of %d components" % C)
    counts = _alloc((C,), torch.int64, dev, "the cell counts of %d components" % C)
    lib = _lib.load()
    ev = _events() + _events()
    ev[0].record()
    _lib.check(lib.rsb_merge_fill(vertices.data_ptr(), ring_offsets.data_ptr(), poly_rings.data_ptr(), len(shapes.xy), d_po.data_ptr(), d_polys.data_ptr(),
                                  d_tr.data_ptr(), d_grids.data_ptr(), d_off.data_ptr(), C, d_bands.data_ptr(), len(bands), band_rows, max_words,
                                  fill.data_ptr(), total, _lib.current_stream_ptr()), "rsb_merge_fill")
    ev[1].record()
    ev[2].record()
    _lib.check(lib.rsb_merge_close(fill.data_ptr(), d_grids.data_ptr(), d_off.data_ptr(), C, d_tiles.data_ptr(), len(tiles), CELLS_PER_THRESHOLD,
                                   closed.data_ptr(), counts.data_ptr(), _lib.current_stream_ptr()), "rsb_merge_close")
    ev[3].record()
    host = closed.cpu().numpy().view(np.uint32)
    cnt = counts.cpu().numpy()
    host_fill = fill.cpu().numpy().view(np.uint32) if keep_fill else None
    stats["fill_ms"] = stats.get("fill_ms", 0.0) + ev[0].elapsed_time(ev[1])
    stats["close_ms"] = stats.get("close_ms", 0.0) + ev[2].elapsed_time(ev[3])
    stats["cells"] = stats.get("cells", 0) + int((W * H).sum())
    for i, c in enumerate(comps):
        c.closed = unpack(host[offsets[i]:offsets[i + 1]], c.grid[3], c.grid[2])
        c.count = int(cnt[i])
        if keep_fill:
            c.fill = unpack(host_fill[offsets[i]:offsets[i + 1]], c.grid[3], c.grid[2])


def unpack(words, H, W):
    """uint32 [H * ceil(W / 32)] bit rows (bit b of word w = column 32 w + b) -> bool [H, W]"""
    w = (W + 31) // 32
    bits = np.unpackbits(np.ascontiguousarray(words, np.uint32).view(np.uint8).reshape(H, w * 4), axis=1, bitorder="little")
    return bits[:, :W].astype(bool)


def merge_device(features, threshold, budget=DEFAULT_BUDGET, device="cuda", stats=None):
    """The merged components of `features` (GeoJSON features, or a ShapeSet from `parse`) -> (ShapeSet, [Component] in
    component order, each with its closed cells). `budget` bounds the device bytes of one batch of grids (two bitmaps of one bit
    per cell); the packed shapes and the pair arrays are outside it. A component that alone needs more raises RsbError before
    anything is allocated. `stats` (a dict) receives counts and kernel times (CUDA events). Synchronises."""
    d = _check_threshold(threshold)
    shapes = features if isinstance(features, DD.ShapeSet) else parse(features)[0]
    stats = stats if stats is not None else {}
    p, q = link(shapes, d, device, stats)
    labels = components_device(len(shapes), p, q, device, stats)
    comps = components(shapes, labels, d)
    runs = plan(comps, budget)  # raises before any grid is allocated
    stats.update(features=len(shapes), linked=len(p), components=len(comps), batches=len(runs))
    for start, end in runs:
        close_device(shapes, comps[start:end], device, stats)
    return shapes, comps


# ---- host: tracing, simplification, output -------------------------------------------------------------------------------

_STEP = np.array([(1, 0), (0, 1), (-1, 0), (0, -1)], np.int64)  # edge directions: +x, +y, -x, -y
# cells ahead-left and ahead-right of an edge's end point P, as offsets of (cx, cy) from P (cell (cx, cy) is [cx, cx + 1] x [cy, cy + 1])
_AHEAD_LEFT = np.array([(0, 0), (-1, 0), (-1, -1), (0, -1)], np.int64)
_AHEAD_RIGHT = np.array([(0, -1), (0, 0), (-1, 0), (-1, -1)], np.int64)


def trace(cells):
    """bool [H, W] cells (row 0 at the top) -> polygons [[exterior, hole, ...], ...] as int64 [n, 2] rings of lattice points
    (x = column, y = rows from the bottom edge of the grid), one polygon per 4-connected region of set cells, ordered by the
    region's first cell in row-major order from the top.

    The boundary of the union of the set cells as closed squares is walked with the cells on the left, so exterior rings run
    counter-clockwise and holes clockwise. Where two set cells meet only at a corner, the walk turns left (around the cell it
    follows) when they belong to different regions, so those polygons touch at the vertex, and right when they belong to the
    same region, so that a hole touching the shell or another hole at a point becomes a ring of its own. Rings hold no
    collinear vertices and start at their lexicographically smallest (x, y); holes follow the exterior in that order."""
    import scipy.ndimage

    G = np.asarray(cells, bool)
    H, W = G.shape
    lab, n = scipy.ndimage.label(G)
    if n == 0:
        return []
    Fp = np.zeros((H + 2, W + 2), np.int64)  # y up, padded: Fp[y + 1, x + 1] is the region of cell (x, y), 0 for none
    Fp[1:-1, 1:-1] = lab[::-1]
    fg = Fp > 0
    c = fg[1:-1, 1:-1]
    starts, dirs, regs = [], [], []
    for d, (nb, sx, sy) in enumerate(((fg[:-2, 1:-1], 0, 0), (fg[1:-1, 2:], 1, 0), (fg[2:, 1:-1], 1, 1), (fg[1:-1, :-2], 0, 1))):
        y, x = np.nonzero(c & ~nb)
        starts.append(np.stack([x + sx, y + sy], axis=1))
        dirs.append(np.full(len(x), d, np.int64))
        regs.append(Fp[y + 1, x + 1])
    S, D, reg = np.concatenate(starts), np.concatenate(dirs), np.concatenate(regs)
    P = S + _STEP[D]
    al = Fp[P[:, 1] + _AHEAD_LEFT[D, 1] + 1, P[:, 0] + _AHEAD_LEFT[D, 0] + 1]
    ar = Fp[P[:, 1] + _AHEAD_RIGHT[D, 1] + 1, P[:, 0] + _AHEAD_RIGHT[D, 0] + 1]
    turn = np.where(al == 0, np.where((ar > 0) & (ar == reg), 3, 1), np.where(ar == 0, 0, 3))
    ND = (D + turn) % 4
    key = (S[:, 1] * (W + 2) + S[:, 0]) * 4 + D
    order = np.argsort(key)
    nxt = order[np.searchsorted(key[order], (P[:, 1] * (W + 2) + P[:, 0]) * 4 + ND)].tolist()
    seen = bytearray(len(S))
    rings = {}
    for s in range(len(S)):
        if seen[s]:
            continue
        ring, i = [], s
        while not seen[i]:
            seen[i] = 1
            ring.append(i)
            i = nxt[i]
        idx = np.asarray(ring)
        dd = D[idx]
        pts = S[idx[dd != np.roll(dd, 1)]]
        first = np.lexsort((pts[:, 1], pts[:, 0]))[0]
        pts = np.roll(pts, -first, axis=0)
        rings.setdefault(int(reg[ring[0]]), []).append(pts)
    return [sorted(rings[r], key=lambda a: (_area2(a) < 0, int(a[0, 0]), int(a[0, 1]))) for r in range(1, n + 1)]


def _area2(ring):
    """twice the signed area of an integer ring (exact)"""
    x, y = ring[:, 0], ring[:, 1]
    return int((x * np.roll(y, -1) - np.roll(x, -1) * y).sum())


def _segment_distances(pts, a, b):
    """float64 distances of integer points to the segment ab; exact enough that `> 1` is decided exactly"""
    ab = (b - a).astype(np.float64)
    ap = (pts - a).astype(np.float64)
    len2 = float(ab @ ab)
    if len2 == 0.0:
        return np.sqrt((ap * ap).sum(1))
    t = ap @ ab
    cross = np.abs(ap[:, 0] * ab[1] - ap[:, 1] * ab[0])
    bp = (pts - b).astype(np.float64)
    return np.where(t <= 0, np.sqrt((ap * ap).sum(1)), np.where(t >= len2, np.sqrt((bp * bp).sum(1)), cross / math.sqrt(len2)))


def _douglas_peucker(chain, tol):
    """bool mask of the vertices of an open chain that Douglas-Peucker keeps (ends always; a vertex farther than tol from the
    current segment splits it at the farthest one, the first on ties)"""
    keep = np.zeros(len(chain), bool)
    keep[0] = keep[-1] = True
    stack = [(0, len(chain) - 1)]
    while stack:
        i, j = stack.pop()
        if j <= i + 1:
            continue
        dist = _segment_distances(chain[i + 1:j], chain[i], chain[j])
        k = int(np.argmax(dist))
        if dist[k] > tol:
            k += i + 1
            keep[k] = True
            stack += [(i, k), (k, j)]
    return keep


def simplify_ring(ring, tol=1.0):
    """Douglas-Peucker of a closed ring (int64 [n, 2], unclosed) at `tol`, split at its first vertex and at the vertex farthest
    from it -> the kept vertices in order, starting at the first"""
    n = len(ring)
    if n < 4:
        return ring
    d2 = ((ring - ring[0]) ** 2).sum(1)
    far = int(np.argmax(d2))
    a = ring[:far + 1]
    b = np.concatenate([ring[far:], ring[:1]])
    return np.concatenate([a[_douglas_peucker(a, tol)][:-1], b[_douglas_peucker(b, tol)][:-1]])


def _polygons_meet_in_points(polygons):
    """the polygons (integer rings, exteriors first) share no piece of boundary, cross nowhere and none has a vertex strictly
    inside another's exterior and outside its holes"""
    for i in range(len(polygons)):
        for j in range(i + 1, len(polygons)):
            ea = [e for r in polygons[i] for e in FT._edges([tuple(p) for p in r.tolist()])]
            eb = [e for r in polygons[j] for e in FT._edges([tuple(p) for p in r.tolist()])]
            for p, q in ea:
                for u, v in eb:
                    hit = FT._intersect(p, q, u, v)
                    if hit == "overlap":
                        return False
                    if hit == "point" and not (FT._on_segment(p, u, v) or FT._on_segment(q, u, v) or FT._on_segment(u, p, q) or FT._on_segment(v, p, q)):
                        return False
            for a, b in ((polygons[i], polygons[j]), (polygons[j], polygons[i])):
                for p in a[0].tolist():
                    if any(FT._on_segment(tuple(p), u, v) for r in b for u, v in FT._edges([tuple(x) for x in r.tolist()])):
                        continue
                    inside = FT._inside((2 * p[0], 2 * p[1]), [(2 * x, 2 * y) for x, y in b[0].tolist()])
                    if inside and not any(FT._inside((2 * p[0], 2 * p[1]), [(2 * x, 2 * y) for x, y in h.tolist()]) for h in b[1:]):
                        return False
                    break
    return True


def simplified(polygons):
    """the polygons with every ring simplified at one cell, or the polygons unchanged when a simplified ring has fewer than 4
    positions (3 vertices), changes orientation, or the result is not OGC-valid (each polygon `features.polygon_is_valid`, and
    polygons meeting only in points)"""
    out = [[simplify_ring(r) for r in poly] for poly in polygons]
    for poly in out:
        if any(len(r) < 3 for r in poly) or _area2(poly[0]) <= 0 or any(_area2(h) >= 0 for h in poly[1:]):
            return polygons
        if not FT.polygon_is_valid([[tuple(p) for p in r.tolist()] for r in poly]):
            return polygons
    if len(out) > 1 and not _polygons_meet_in_points(out):
        return polygons
    return out


def ring_area(lonlat):
    """signed Mollweide area (m²) of a closed or unclosed lon/lat ring: positive counter-clockwise"""
    xy = DD.mollweide(lonlat)
    xy = xy - xy.mean(0)
    x, y = xy[:, 0], xy[:, 1]
    return 0.5 * float((x * np.roll(y, -1) - np.roll(x, -1) * y).sum())


def _well_formed(polygons):
    """every ring has at least 3 vertices, exteriors run counter-clockwise and holes clockwise"""
    return all(len(r) >= 3 for p in polygons for r in p) and all(_area2(p[0]) > 0 and all(_area2(h) < 0 for h in p[1:]) for p in polygons)


def component_feature(comp):
    """(GeoJSON Feature dict or None, warning or None) of a closed Component"""
    if comp.closed is None or comp.count == 0:
        return None, W_NOT_POLYGON
    polygons = simplified(trace(comp.closed))
    if not _well_formed(polygons):
        return None, W_NOT_VALID
    u0, v1, _, H = comp.grid
    v0 = v1 - H + 1
    coords, area = [], 0.0
    for poly in polygons:
        rings = []
        for r in poly:
            ll = inverse_mercator((r + np.array([u0, v0])).astype(np.float64) * comp.cell)
            area += ring_area(ll)
            ll = ll.tolist()
            rings.append(ll + [ll[0]])
        coords.append(rings)
    geometry = {"type": "Polygon", "coordinates": coords[0]} if len(coords) == 1 else {"type": "MultiPolygon", "coordinates": coords}
    return {"type": "Feature", "geometry": geometry, "properties": {"area": int(round(area))}}, None


def merge_shapes(shapes, threshold, budget=DEFAULT_BUDGET, device="cuda", pool=None, stats=None):
    """`merge` on parsed features (`parse`) -> (merged Feature dicts in component order, warnings of the merge step). `pool` (an
    Executor) traces the components; by default one thread per CPU. `stats` receives the counts, the kernel times and the
    seconds on the device and tracing."""
    import time

    stats = stats if stats is not None else {}
    t0 = time.perf_counter()
    _, comps = merge_device(shapes, threshold, budget, device, stats)
    t1 = time.perf_counter()
    own = pool is None
    if own:
        pool = concurrent.futures.ThreadPoolExecutor(os.cpu_count() or 1)
    try:
        results = list(pool.map(component_feature, comps))
    finally:
        if own:
            pool.shutdown()
    t2 = time.perf_counter()
    out, warnings = [], []
    for feature, warning in results:
        if warning:
            warnings.append(warning)
        else:
            out.append(feature)
    stats.update(device_s=t1 - t0, trace_s=t2 - t1)
    return out, warnings


def merge(features, threshold, budget=DEFAULT_BUDGET, device="cuda"):
    """Drop-in for the reference's `rs merge` loop: GeoJSON features -> (merged Feature dicts
    {"type": "Feature", "geometry": Polygon or MultiPolygon, "properties": {"area": m²}} in component order, warnings)"""
    shapes, warnings = parse(features)
    out, more = merge_shapes(shapes, threshold, budget, device)
    return out, warnings + more
