"""rsb_label_components, rsb_building_clean and `rs features --type building` on the H100: roots and areas bit-identical to the
scipy restatement (tests/building_reference.py) on hard shapes and patterns, run-to-run and batch-split identity, guard bytes,
the tool end to end against the CPU path, and seeded rectangles burned by `rs rasterize --class building` coming back one
feature each."""

import argparse
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

import building_reference as br
import rasterize_reference as rr
from robosat_b200 import _lib
from robosat_b200 import features as F
from robosat_b200.tiles import Tile

pytestmark = pytest.mark.gpu

SHAPES = [(512, 512), (509, 131), (1, 1), (1, 300), (300, 1)]
CLASSES = ["background", "parking", "building"]
COLORS = ["denim", "orange", "dark"]


def spiral(H, W):
    """a one-pixel-wide square spiral with one-pixel gaps from the top-left corner inwards, over the whole image"""
    m = np.zeros((H, W), np.uint8)
    dirs = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    y = x = d = 0
    m[0, 0] = 1

    def free(yy, xx):
        return 0 <= yy < H and 0 <= xx < W and not m[yy, xx]

    while True:
        for turn in range(2):
            dy, dx = dirs[d]
            ahead2 = (y + 2 * dy, x + 2 * dx)
            if free(y + dy, x + dx) and (free(*ahead2) or not (0 <= ahead2[0] < H and 0 <= ahead2[1] < W)):
                y, x = y + dy, x + dx
                m[y, x] = 1
                break
            d = (d + 1) % 4
        else:
            return m


def serpentine(H, W):
    """rows 0, 2, 4, ... joined alternately at the right and the left end: one path through the whole image"""
    m = np.zeros((H, W), np.uint8)
    m[0::2] = 1
    for r in range(1, H, 2):
        m[r, W - 1 if (r // 2) % 2 == 0 else 0] = 1
    return m


def patterns(H, W):
    yy, xx = np.mgrid[:H, :W]
    rng = np.random.RandomState(H * 7 + W)
    out = [np.zeros((H, W), np.uint8), np.ones((H, W), np.uint8), ((yy + xx) % 2).astype(np.uint8), spiral(H, W), serpentine(H, W),
           serpentine(W, H).T.copy()]
    out += [(rng.rand(H, W) < p).astype(np.uint8) for p in (0.3, 0.5, 0.6)]
    return out


def batch(H, W, N):
    base = patterns(H, W)
    rng = np.random.RandomState(N + H + W)
    imgs = [base[i] if i < len(base) else (rng.rand(H, W) < (0.3, 0.5, 0.6)[i % 3]).astype(np.uint8) for i in range(N)]
    return np.stack(imgs)


def _device(host, pad=37):
    """uint8 [N][H][W] on the device with an image stride of H*W + pad, and guard bytes between images"""
    N, H, W = host.shape
    buf = torch.full((N * (H * W + pad) + pad,), 7, dtype=torch.uint8)
    buf.as_strided((N, H, W), (H * W + pad, W, 1)).copy_(torch.from_numpy(host))
    return buf.cuda().as_strided((N, H, W), (H * W + pad, W, 1))


def _check_components(host, value, connectivity, roots, areas):
    roots, areas = roots.cpu().numpy(), areas.cpu().numpy()
    for n in range(host.shape[0]):
        want_root, want_area, _ = br.components(host[n], value, connectivity)
        assert np.array_equal(roots[n].reshape(-1), want_root.reshape(-1)), (n, value, connectivity)
        assert np.array_equal(areas[n], want_area), (n, value, connectivity)


@pytest.mark.parametrize("connectivity", [4, 8])
@pytest.mark.parametrize("shape", SHAPES)
def test_components_match_restatement(cuda_device, shape, connectivity):
    H, W = shape
    for N in (1, 7, 64):
        host = batch(H, W, N)
        planes = _device(host, pad=0 if N == 7 else 37)
        for value in (0, 1):
            roots, areas = F.components_device(planes, value, connectivity)
            _check_components(host, value, connectivity, roots, areas)


def test_every_pattern_alone(cuda_device):
    """N = 1 per pattern, so each one is also labelled without neighbours in the batch"""
    for H, W in SHAPES[:2]:
        for i, p in enumerate(patterns(H, W)):
            for connectivity in (4, 8):
                roots, areas = F.components_device(torch.from_numpy(p[None].copy()).cuda(), 1, connectivity)
                _check_components(p[None], 1, connectivity, roots, areas)
    checker = patterns(512, 512)[2]
    roots, areas = F.components_device(torch.from_numpy(checker[None].copy()).cuda(), 1, 8)
    assert int(areas[0].max()) == int(checker.sum())  # one 8-connected component
    roots, areas = F.components_device(torch.from_numpy(checker[None].copy()).cuda(), 0, 4)
    assert int(areas[0].max()) == 1  # every background pixel alone


def test_repeated_runs_and_batch_splits_agree(cuda_device):
    host = batch(512, 512, 64)
    planes = _device(host)
    for connectivity in (4, 8):
        r1, a1 = F.components_device(planes, 1, connectivity)
        r2, a2 = F.components_device(planes, 1, connectivity)
        assert torch.equal(r1, r2) and torch.equal(a1, a2)
        parts = [F.components_device(planes[i:j], 1, connectivity) for i, j in ((0, 29), (29, 64))]
        assert torch.equal(torch.cat([p[0] for p in parts]), r1) and torch.equal(torch.cat([p[1] for p in parts]), a1)
    labels = _device(building_labels(np.random.RandomState(3), 64, 512, 512))
    f1, c1 = F.building_clean_device(labels, 2)
    f2, c2 = F.building_clean_device(labels, 2)
    parts = [F.building_clean_device(labels[i:j], 2) for i, j in ((0, 5), (5, 64))]
    assert torch.equal(f1, f2) and torch.equal(c1, c2)
    assert torch.equal(torch.cat([p[0] for p in parts]), f1) and torch.equal(torch.cat([p[1] for p in parts]), c1)


def test_guard_bytes_stay_untouched(cuda_device):
    N, H, W, G = 5, 97, 70, 4096
    host = batch(H, W, N)
    planes = _device(host)
    lib, stream = _lib.load(), _lib.current_stream_ptr()
    labels = torch.full((G + N * H * W + G,), -7, dtype=torch.int32, device=cuda_device)
    areas = torch.full((G + N * H * W + G,), -9, dtype=torch.int32, device=cuda_device)
    _lib.check(lib.rsb_label_components(planes.data_ptr(), planes.stride(0), N, H, W, 1, 8, labels[G:].data_ptr(), areas[G:].data_ptr(), stream),
               "rsb_label_components")
    lab, area = labels.cpu().numpy(), areas.cpu().numpy()
    assert (lab[:G] == -7).all() and (lab[G + N * H * W:] == -7).all()
    assert (area[:G] == -9).all() and (area[G + N * H * W:] == -9).all()
    _check_components(host, 1, 8, torch.from_numpy(lab[G:G + N * H * W].reshape(N, H, W)), torch.from_numpy(area[G:G + N * H * W].reshape(N, H, W)))

    out = torch.full((G + N * H * W + G,), 0xAB, dtype=torch.uint8, device=cuda_device)
    counts = torch.full((N + 64,), -7, dtype=torch.int32, device=cuda_device)
    _lib.check(lib.rsb_building_clean(planes.data_ptr(), planes.stride(0), N, H, W, 64, 64, labels[G:].data_ptr(), areas[G:].data_ptr(),
                                      out[G:].data_ptr(), counts[32:].data_ptr(), stream), "rsb_building_clean")
    o, c, lab, area = out.cpu().numpy(), counts.cpu().numpy(), labels.cpu().numpy(), areas.cpu().numpy()
    assert (o[:G] == 0xAB).all() and (o[G + N * H * W:] == 0xAB).all()
    assert (c[:32] == -7).all() and (c[32 + N:] == -7).all()
    assert (lab[:G] == -7).all() and (lab[G + N * H * W:] == -7).all()
    assert (area[:G] == -9).all() and (area[G + N * H * W:] == -9).all()
    for n in range(N):
        want = br.fill(br.drop(host[n], 64), 64)
        assert np.array_equal(o[G + n * H * W:G + (n + 1) * H * W].reshape(H, W), want), n
        assert c[32 + n] == want.sum(), n


def _rect(m, rng, value, lo, hi):
    """a rotated rectangle of `value` with sides in [lo, hi) px"""
    import cv2

    H, W = m.shape
    cy, cx = rng.uniform(0, H), rng.uniform(0, W)
    (a, b), t = rng.uniform(lo, hi, size=2), rng.uniform(0, math.pi)
    c, s = math.cos(t), math.sin(t)
    pts = [(cx + u * c - v * s, cy + u * s + v * c) for u, v in ((-a / 2, -b / 2), (a / 2, -b / 2), (a / 2, b / 2), (-a / 2, b / 2))]
    cv2.fillPoly(m, [np.round(np.array(pts) * 4).astype(np.int32)], int(value), shift=2)


def building_labels(rng, N, H, W):
    """three-class label images: rotated buildings (2) with courtyards of all sizes, parking lots (1), speckle of both"""
    out = np.zeros((N, H, W), np.uint8)
    for n in range(N):
        m = out[n]
        if n % 5 == 4:
            continue  # some empty tiles
        for _ in range(rng.randint(1, 4)):
            _rect(m, rng, 1, 10, 150)
        for _ in range(rng.randint(2, 12)):
            _rect(m, rng, 2, 6, 160)
        for _ in range(rng.randint(0, 8)):
            _rect(m, rng, 0, 3, 30)  # courtyards and cuts
        noise = rng.rand(H, W)
        m[noise < 0.01] = 2
        m[noise > 0.995] = 0
    return out


@pytest.mark.parametrize("shape", [(512, 512), (509, 131), (1, 1)])
def test_building_clean_matches_restatement(cuda_device, shape):
    H, W = shape
    host = building_labels(np.random.RandomState(H + W), 10, H, W)
    filled, counts = F.building_clean_device(_device(host), 2)
    filled, counts = filled.cpu().numpy(), counts.cpu().numpy()
    for n in range(host.shape[0]):
        want = br.clean(host[n], 2)
        assert np.array_equal(filled[n], want), n
        assert counts[n] == want.sum(), n


def _dataset(tmp_path):
    path = tmp_path / "dataset.toml"
    path.write_text("[common]\nclasses = [%s]\ncolors = [%s]\n" % (", ".join("'%s'" % c for c in CLASSES), ", ".join("'%s'" % c for c in COLORS)))
    return str(path)


def _write_masks(root, cases):
    palette = [v for i in range(256) for v in (i, 255 - i, (7 * i) % 256)]
    for tile, labels in cases:
        d = os.path.join(root, str(tile.z), str(tile.x))
        os.makedirs(d, exist_ok=True)
        im = Image.fromarray(labels, mode="P")
        im.putpalette(palette)
        im.save(os.path.join(d, "%d.png" % tile.y))


def _run_features(tmp_path, masks, batch, name="out"):
    from robosat_b200.tools import features as tool

    out = str(tmp_path / ("%s_%d.geojson" % (name, batch)))
    tool.main(argparse.Namespace(masks=masks, type="building", dataset=_dataset(tmp_path), out=out), batch=batch)
    with open(out) as fp:
        return json.load(fp)


def test_tool_matches_cpu_path_in_tile_order(cuda_device, tmp_path):
    host = building_labels(np.random.RandomState(11), 24, 512, 512)
    # x descending with i, so the (z, x, y) order differs from the generation order and from listing order
    cases = [(Tile(70100 - i, 104000 + (i % 3), 18), host[i]) for i in range(len(host))]
    masks = str(tmp_path / "masks")
    _write_masks(masks, cases)
    want = []
    for tile, labels in sorted(cases, key=lambda c: (c[0].z, c[0].x, c[0].y)):
        want.extend(br.cpu_features(tile, labels, 2)[0])
    assert len(want) > 60
    for b in (64, 3):
        got = _run_features(tmp_path, masks, b)
        assert got["type"] == "FeatureCollection"
        assert got["features"] == json.loads(json.dumps(want)), b


def rectangles(tiles, seed):
    """one rotated rectangle of 8-60 m sides per tile, at least 3 m inside it: [(tile, GeoJSON feature)]"""
    rng = np.random.RandomState(seed)
    out = []
    for t in tiles:
        west, south, east, north = F.bounds(t)
        lat0 = 0.5 * (south + north)
        mx, my = 111320.0 * math.cos(math.radians(lat0)), 110574.0  # metres per degree, locally
        width, height = (east - west) * mx, (north - south) * my
        a, b = rng.uniform(8, 60, size=2)
        th = rng.uniform(0, math.pi)
        c, s = math.cos(th), math.sin(th)
        ex, ey = 0.5 * (a * abs(c) + b * abs(s)), 0.5 * (a * abs(s) + b * abs(c))
        cx = rng.uniform(ex + 3, width - ex - 3)
        cy = rng.uniform(ey + 3, height - ey - 3)
        ring = []
        for u, v in ((-a / 2, -b / 2), (a / 2, -b / 2), (a / 2, b / 2), (-a / 2, b / 2)):
            x, y = cx + u * c - v * s, cy + u * s + v * c
            ring.append([west + x / mx, south + y / my])
        ring.append(ring[0])
        out.append((t, {"type": "Feature", "geometry": {"type": "Polygon", "coordinates": [ring]}, "properties": {}}))
    return out


def iou(tile, a, b, size=2048):
    ma, mb = rr.burn(tile, [a], size).astype(bool), rr.burn(tile, [b], size).astype(bool)
    return (ma & mb).sum() / (ma | mb).sum()


def test_rasterized_rectangles_come_back_one_feature_each(cuda_device, tmp_path):
    from robosat_b200.tools import rasterize as rz_tool

    tiles = [Tile(70100 + i, 104000 + j, 18) for i in range(8) for j in range(5)]
    rects = rectangles(tiles, seed=5)
    src = tmp_path / "buildings.geojson"
    src.write_text(json.dumps({"type": "FeatureCollection", "features": [f for _, f in rects]}))
    csv = tmp_path / "tiles.csv"
    csv.write_text("".join("%d,%d,%d\n" % tuple(t) for t in tiles))
    labels = tmp_path / "labels"
    rz_tool.main(argparse.Namespace(features=str(src), tiles=str(csv), out=str(labels), dataset=_dataset(tmp_path), zoom=18, size=512,
                                    class_name="building"))
    got = _run_features(tmp_path, str(labels), 64)["features"]
    assert len(got) == len(rects)
    for (tile, want), feat in zip(rects, got):  # one tile per rectangle, in (z, x, y) order as the tiles
        west, south, east, north = F.bounds(tile)
        lon, lat = np.array(feat["geometry"]["coordinates"][0]).mean(axis=0)
        assert west < lon < east and south < lat < north
        assert iou(tile, want, feat) >= 0.9
