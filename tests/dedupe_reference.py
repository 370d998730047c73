"""`rs dedupe` restated in exact arithmetic: `fractions.Fraction` on the float64 inputs, sharing no algorithm with the kernels.

- Intersects: exact segment predicates (closed segments, touching counts) and exact point-in-polygon of one vertex per
  component, on lon/lat positions.
- Areas: slab decomposition on the Mollweide positions of `robosat_b200.dedupe.mollweide` (the one projection both sides use).
  The plane is cut at every vertex x and every x where two edges cross; inside a slab no two edges cross, so the edges spanning
  it are ordered by their y at the slab's middle, membership of each gap between consecutive edges follows from even-odd
  counts per feature, and the length of a region is linear in x across the slab: its area is the slab width times the length
  at the middle, exactly.

Features are GeoJSON dicts; a feature's shape is all rings of all its polygons, taken even-odd."""

from fractions import Fraction

import numpy as np

from robosat_b200.dedupe import mollweide


def polygons(feature):
    g = feature["geometry"]
    return [g["coordinates"]] if g["type"] == "Polygon" else g["coordinates"]


def rings_ll(feature):
    return [np.asarray([p[:2] for p in ring], np.float64) for poly in polygons(feature) for ring in poly]


def rings_xy(feature):
    return [mollweide(r) for r in rings_ll(feature)]


def _edges(rings):
    """[(a, b)] as float pairs, closing each ring, without zero-length edges"""
    out = []
    for r in rings:
        n = len(r)
        for i in range(n):
            a, b = tuple(map(float, r[i])), tuple(map(float, r[(i + 1) % n]))
            if a != b:
                out.append((a, b))
    return out


def orient(a, b, c):
    """exact sign of (b - a) x (c - a)"""
    ax, ay, bx, by, cx, cy = (Fraction(v) for v in (a[0], a[1], b[0], b[1], c[0], c[1]))
    d = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax)
    return (d > 0) - (d < 0)


def _on(a, b, p):
    return min(a[0], b[0]) <= p[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= p[1] <= max(a[1], b[1])


def segments_meet(a, b, c, d):
    if max(a[0], b[0]) < min(c[0], d[0]) or max(c[0], d[0]) < min(a[0], b[0]) or max(a[1], b[1]) < min(c[1], d[1]) or max(c[1], d[1]) < min(a[1], b[1]):
        return False
    o1, o2, o3, o4 = orient(a, b, c), orient(a, b, d), orient(c, d, a), orient(c, d, b)
    if o1 * o2 < 0 and o3 * o4 < 0:
        return True
    return (o1 == 0 and _on(a, b, c)) or (o2 == 0 and _on(a, b, d)) or (o3 == 0 and _on(c, d, a)) or (o4 == 0 and _on(c, d, b))


def point_in(p, edges):
    """'in', 'out' or 'on' for the even-odd region of `edges`"""
    inside = False
    for a, b in edges:
        if orient(a, b, p) == 0 and _on(a, b, p):
            return "on"
        if (a[1] > p[1]) != (b[1] > p[1]):
            o = orient(a, b, p)
            if (o > 0) == (b[1] > a[1]):
                inside = not inside
    return "in" if inside else "out"


def intersects(fp, fq):
    """GEOS `intersects` of two areal features, on lon/lat"""
    ep, eq = _edges(rings_ll(fp)), _edges(rings_ll(fq))
    for a, b in ep:
        for c, d in eq:
            if segments_meet(a, b, c, d):
                return True
    for f, other in ((fp, eq), (fq, ep)):
        for poly in polygons(f):
            p = tuple(map(float, poly[0][0][:2]))
            if point_in(p, other) != "out":
                return True
    return False


def _cross_x(e, f):
    """x of the single crossing point of segments e and f, or None"""
    (a, b), (c, d) = e, f
    if not segments_meet(a, b, c, d):
        return None
    ax, ay, bx, by, cx, cy, dx, dy = (Fraction(v) for v in (a[0], a[1], b[0], b[1], c[0], c[1], d[0], d[1]))
    den = (bx - ax) * (dy - cy) - (by - ay) * (dx - cx)
    if den == 0:
        return None  # parallel: collinear overlaps end at vertices, which are cut anyway
    t = ((cx - ax) * (dy - cy) - (cy - ay) * (dx - cx)) / den
    return ax + t * (bx - ax)


def areas(p_rings, q_rings_list, window=None):
    """exact (A(P), A(P ∩ U), A(U)) as Fractions, U the union of the features whose rings are q_rings_list, all in projected
    (x, y). With `window` = (x0, x1), only slabs inside it are summed (for A(P ∩ U) of a P inside the window, when the
    features are too large for the full sweep)."""
    feats = [_edges(p_rings)] + [_edges(r) for r in q_rings_list]
    edges = [(k, e) for k, es in enumerate(feats) for e in es]
    if window is not None:
        edges = [(k, e) for k, e in edges if max(e[0][0], e[1][0]) >= window[0] and min(e[0][0], e[1][0]) <= window[1]]
    xs = {Fraction(v[0]) for _, e in edges for v in e}
    if len(edges) > 1:
        box = np.array([[min(a[0], b[0]), min(a[1], b[1]), max(a[0], b[0]), max(a[1], b[1])] for _, (a, b) in edges])
        i, j = np.nonzero((box[:, None, 0] <= box[None, :, 2]) & (box[None, :, 0] <= box[:, None, 2]) & (box[:, None, 1] <= box[None, :, 3]) & (box[None, :, 1] <= box[:, None, 3]))
        for a, b in zip(i.tolist(), j.tolist()):
            if a < b:
                x = _cross_x(edges[a][1], edges[b][1])
                if x is not None:
                    xs.add(x)
    if window is not None:
        xs = {x for x in xs if Fraction(window[0]) <= x <= Fraction(window[1])} | {Fraction(window[0]), Fraction(window[1])}
    xs = sorted(xs)
    # sweep: non-vertical edges by their left end
    span = sorted(((Fraction(min(a[0], b[0])), Fraction(max(a[0], b[0])), k, a, b) for k, (a, b) in edges if a[0] != b[0]), key=lambda s: s[0])
    active, ptr = [], 0
    total = [Fraction(0)] * 3
    nq = len(feats) - 1
    for xl, xr in zip(xs[:-1], xs[1:]):
        while ptr < len(span) and span[ptr][0] <= xl:
            active.append(span[ptr])
            ptr += 1
        active = [s for s in active if s[1] >= xr]
        if not active:
            continue
        xm = (xl + xr) / 2
        ys = []
        for _, _, k, a, b in active:
            ax, ay, bx, by = Fraction(a[0]), Fraction(a[1]), Fraction(b[0]), Fraction(b[1])
            ys.append((ay + (xm - ax) * (by - ay) / (bx - ax), k))
        ys.sort()
        parity = [False] * (nq + 1)
        length = [Fraction(0)] * 3
        for (y0, k), (y1, _) in zip(ys[:-1], ys[1:]):
            parity[k] = not parity[k]
            if y1 == y0:
                continue
            in_p, in_u = parity[0], any(parity[1:])
            if in_p:
                length[0] += y1 - y0
            if in_p and in_u:
                length[1] += y1 - y0
            if in_u:
                length[2] += y1 - y0
        for r in range(3):
            total[r] += (xr - xl) * length[r]
    return tuple(total)


def iou(a_p, a_i, a_u):
    union = a_p + a_u - a_i
    return Fraction(0) if union == 0 else a_i / union


def is_areal(feature):
    return ((feature.get("geometry") or {}).get("type")) in ("Polygon", "MultiPolygon")


def intersecting(fp, osm):
    """indices of the areal OSM features whose closed lon/lat boxes meet fp's and that fp intersects"""
    def box(f):
        v = np.concatenate(rings_ll(f))
        return v[:, 0].min(), v[:, 1].min(), v[:, 0].max(), v[:, 1].max()

    bp = box(fp)
    out = []
    for i, q in enumerate(osm):
        if not is_areal(q):
            continue
        bq = box(q)
        if bp[0] <= bq[2] and bq[0] <= bp[2] and bp[1] <= bq[3] and bq[1] <= bp[3] and intersects(fp, q):
            out.append(i)
    return out


def perturbed(features, seed, jitter, shift, drop):
    """OSM-like copies of areal features: each vertex moved by up to `jitter` degrees, each feature shifted by up to `shift`,
    and a `drop` fraction of the features left out (seeded)"""
    rng = np.random.default_rng(seed)
    out = []
    for f in features:
        if rng.uniform() < drop:
            continue
        d = rng.uniform(-shift, shift, 2)

        def ring(r):
            a = np.asarray(r, np.float64)[:-1]
            a = a + d + rng.uniform(-jitter, jitter, a.shape)
            return np.concatenate([a, a[:1]]).tolist()

        out.append({"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [ring(r) for r in polygons(f)[0]]}})
    return out


def boundary_squares(feature, count, half, seed):
    """`count` squares of half-side `half` degrees centred on random vertices of the feature's first ring"""
    rng = np.random.default_rng(seed)
    ring = polygons(feature)[0][0]
    out = []
    for i in rng.choice(len(ring) - 1, count, replace=False):
        x, y = ring[i][:2]
        sq = [[x - half, y - half], [x + half, y - half], [x + half, y + half], [x - half, y + half], [x - half, y - half]]
        out.append({"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [sq]}})
    return out


def split_disc(n_ring, n_border, centre=(10.0, 45.0), radius=0.5, amplitude=1e-4):
    """Two OSM polygons that share a jagged border: a regular n_ring-gon split along a diameter replaced by a zigzag of n_border
    points (offsets tapered to zero at its ends) -> (feature A, feature B, the disc as one ring, the border's points)"""
    a = np.linspace(0, 2 * np.pi, n_ring, endpoint=False)
    ring = np.stack([centre[0] + radius * np.cos(a), centre[1] + radius * np.sin(a)], 1)
    h = n_ring // 2
    s = np.linspace(0, 1, n_border + 2)[1:-1]
    offset = amplitude * np.sin(np.pi * s) * np.where(np.arange(n_border) % 2, 1.0, -1.0)
    border = np.stack([ring[h, 0] + s * (ring[0, 0] - ring[h, 0]), ring[h, 1] + offset], 1)  # from vertex h to vertex 0
    upper = np.concatenate([ring[:h + 1], border])                 # 0 .. h over the top, then back along the border
    lower = np.concatenate([ring[h:], ring[:1], border[::-1]])     # h .. n-1, 0 along the bottom, then back the other way

    def feature(r):
        return {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [np.concatenate([r, r[:1]]).tolist()]}}

    return feature(upper), feature(lower), ring, border


def squares_at(points, half):
    return [{"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [[
        [x - half, y - half], [x + half, y - half], [x + half, y + half], [x - half, y + half], [x - half, y - half]]]}} for x, y in points]


def shoelace(rings):
    """float area of rings about their first vertex, with math.fsum"""
    import math

    total = []
    for r in rings:
        v = r - r[0]
        total.extend((v[:, 0] * np.roll(v[:, 1], -1) - np.roll(v[:, 0], -1) * v[:, 1]).tolist())
    return 0.5 * math.fsum(total)


def dedupe(predicted, osm, threshold):
    """(keep [bool], areas [(A_P, A_I, A_U) as Fractions or None]) for valid inputs"""
    keep, out = [], []
    for fp in predicted:
        if not is_areal(fp):
            keep.append(True)
            out.append(None)
            continue
        s = intersecting(fp, osm)
        if not s:
            keep.append(True)
            out.append(None)
            continue
        a = areas(rings_xy(fp), [rings_xy(osm[i]) for i in s])
        keep.append(float(iou(*a)) < threshold)
        out.append(a)
    return keep, out
