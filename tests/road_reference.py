"""numpy restatement of the road rule of DESIGN.md §8 (halo'd plane, cleanup, Zhang-Suen thinning, m-adjacency graph, spur
pruning, chains) and the CPU path of `rs features --type road`, for the tests."""

import numpy as np
from scipy import ndimage

import building_reference as br
from robosat_b200.features import RoadHandler, lines_from_chains

# neighbour offsets in increasing pixel index; the diagonals are m-adjacent only without a common 4-neighbour
OFFSETS = [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1)]


def halo(masks, tile, class_index, h=RoadHandler.halo):
    """masks: {(x, y): label image} of one zoom -> the halo'd binary plane of tile (x, y), missing neighbours background"""
    H, W = masks[tile].shape
    big = np.zeros((3 * H, 3 * W), np.uint8)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            m = masks.get((tile[0] + dx, tile[1] + dy))
            if m is not None:
                big[(dy + 1) * H:(dy + 2) * H, (dx + 1) * W:(dx + 2) * W] = m == class_index
    return big[H - h:2 * H + h, W - h:2 * W + h].copy()


def clean(m, min_area=RoadHandler.min_area, min_hole_area=RoadHandler.min_hole_area):
    return br.fill(br.drop(m, min_area), min_hole_area)


def _shift(a, dy, dx):
    """b[y, x] = a[y + dy, x + dx], background outside"""
    H, W = a.shape
    b = np.zeros_like(a)
    b[max(0, -dy):H - max(0, dy), max(0, -dx):W - max(0, dx)] = a[max(0, dy):H + min(0, dy), max(0, dx):W + min(0, dx)]
    return b


def thin(m):
    """Zhang-Suen on (m != 0) -> (uint8 skeleton, full iterations run including the last, which deleted nothing)"""
    s = (np.asarray(m) != 0).astype(np.uint8)
    it = 0
    while True:
        it += 1
        changed = False
        for sub in (0, 1):
            P = [_shift(s, dy, dx) for dy, dx in ((-1, 0), (-1, 1), (0, 1), (1, 1), (1, 0), (1, -1), (0, -1), (-1, -1))]  # P2..P9
            B = sum(p.astype(np.int32) for p in P)
            A = sum(((P[i] == 0) & (P[(i + 1) % 8] == 1)).astype(np.int32) for i in range(8))
            p2, p4, p6, p8 = P[0], P[2], P[4], P[6]
            if sub == 0:
                c = (p2 * p4 * p6 == 0) & (p4 * p6 * p8 == 0)
            else:
                c = (p2 * p4 * p8 == 0) & (p2 * p6 * p8 == 0)
            delete = (s == 1) & (B >= 2) & (B <= 6) & (A == 1) & c
            if delete.any():
                changed = True
                s = s & ~delete
                s = s.astype(np.uint8)
        if not changed:
            return s, it


def degrees(s):
    """int8 m-degree of each pixel of s, -1 off it"""
    s = s.astype(bool)
    d = np.zeros(s.shape, np.int32)
    for dy, dx in OFFSETS:
        q = _shift(s, dy, dx)
        if dy and dx:
            q &= ~_shift(s, dy, 0) & ~_shift(s, 0, dx)
        d += q
    return np.where(s, d, -1).astype(np.int8)


def neighbours(s, p):
    H, W = s.shape
    y, x = divmod(p, W)
    out = []
    for dy, dx in OFFSETS:
        yy, xx = y + dy, x + dx
        if not (0 <= yy < H and 0 <= xx < W and s[yy, xx]):
            continue
        if dy and dx and (s[yy, x] or s[y, xx]):
            continue
        out.append(yy * W + xx)
    return out


def _walk(s, d, p, q):
    path = [p, q]
    while path[-1] != p and d.flat[path[-1]] == 2:
        a, b = neighbours(s, path[-1])
        path.append(a if b == path[-2] else b)
    return path


def prune(s, d, min_length=RoadHandler.min_length):
    """s without the endpoint-to-junction chains of fewer than min_length pixels (junction not counted) and the endpoint-to-
    endpoint chains of fewer than min_length pixels, decided on (s, d)"""
    out = s.copy()
    for e in np.flatnonzero(d.ravel() == 1):
        (q,) = neighbours(s, e)
        path = _walk(s, d, e, q)
        end = d.flat[path[-1]]
        body = path[:-1] if end >= 3 else path
        if len(body) < min_length:
            out.flat[body] = 0
    return out


def chains(s, d=None):
    """The chains of skeleton s: a list of pixel index lists in (first, second) order, each from its end with the smaller index"""
    if d is None:
        d = degrees(s)
    out = []
    flat = d.ravel()
    lab, _ = ndimage.label(s.astype(bool), structure=np.ones((3, 3), bool))
    has_node = np.zeros(lab.max() + 1, bool)
    has_node[lab.ravel()[(flat >= 0) & (flat != 2)]] = True
    seen = set()
    for p in np.flatnonzero(flat >= 0):
        p = int(p)
        if flat[p] != 2:
            for q in neighbours(s, p):
                path = _walk(s, d, p, q)
                if path[-1] > p or (path[-1] == p and q < path[-2]):
                    out.append(path)
        elif not has_node[lab.flat[p]] and lab.flat[p] not in seen:
            seen.add(lab.flat[p])  # p is the component's smallest pixel
            out.append(_walk(s, d, p, neighbours(s, p)[0]))
    return out


def skeleton_chains(plane, min_length=RoadHandler.min_length):
    """steps 2-5 on a halo'd binary plane -> (skeleton, iterations, pruned skeleton, chains)"""
    skel, it = thin(clean(plane))
    pruned = prune(skel, degrees(skel), min_length)
    return skel, it, pruned, chains(pruned)


def cpu_features(tile, plane, shape, h=RoadHandler.halo):
    """Features of one tile on the CPU: the restated steps 2-5, then the same host code as the device path"""
    return lines_from_chains(tile, skeleton_chains(plane)[3], shape, h, RoadHandler.simplify_epsilon)
