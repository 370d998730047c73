"""rsb_rasterize_polygons and `rs rasterize` on the H100: bit for bit against the numpy restatement (tests/rasterize_reference.py)
on the golden parking masks, every size class, the shapes and ties of GDAL's rule, strided output with guard bytes and foreground
counts, and the tool end to end."""

import argparse
import os

import numpy as np
import pytest
import torch
from PIL import Image

import rasterize_reference as rr
from robosat_b200 import _lib
from robosat_b200 import rasterize as RZ
from robosat_b200.colors import make_palette
from robosat_b200.tiles import Tile

pytestmark = pytest.mark.gpu


def _merc(tile, rings_uv):
    """rings in tile units (u right, v down; the tile is [0, 1]^2) -> Mercator rings"""
    left, bottom, right, top = RZ.xy_bounds(tile)
    return [np.array([(left + u * (right - left), top - v * (top - bottom)) for u, v in ring], dtype=np.float64) for ring in rings_uv]


def _check(tiles, polygons, size):
    out, counts = RZ.burn_device(tiles, polygons, size)
    got, counts = out.cpu().numpy(), counts.cpu().numpy()
    for i, t in enumerate(tiles):
        want = rr.burn_transform(rr.transform(t, size), polygons, size)
        assert np.array_equal(got[i], want), (t, size, int((got[i] != want).sum()))
        assert counts[i] == int(want.sum()), t
    return got


def _launch(polyset, transforms, csr, size, out, image_stride, counts):
    """the C entry with arbitrary transforms (pixel coordinates = c0 + X * c1, r0 + Y * r1)"""
    offsets, ids = csr
    d_off = torch.from_numpy(np.asarray(offsets, np.int32)).cuda()
    d_ids = torch.from_numpy(np.asarray(ids if len(ids) else [0], np.int32)).cuda()
    d_tr = torch.from_numpy(np.asarray(transforms, np.float64)).cuda()
    _lib.check(_lib.load().rsb_rasterize_polygons(polyset.d_vertices.data_ptr(), polyset.d_ring_offsets.data_ptr(), polyset.d_poly_rings.data_ptr(),
                                                  len(polyset), d_off.data_ptr(), d_ids.data_ptr(), d_tr.data_ptr(), len(transforms), size,
                                                  out.data_ptr(), image_stride, counts.data_ptr(), _lib.current_stream_ptr()), "rsb_rasterize_polygons")
    torch.cuda.synchronize()


def _pixel_check(polygons, size, tr=(0.0, 1.0, 0.0, 1.0)):
    """burn polygons given in pixel coordinates under the identity transform; all polygons in one tile"""
    ps = RZ.PolygonSet(polygons, "cuda")
    out = torch.empty((1, size, size), dtype=torch.uint8, device="cuda")
    counts = torch.empty((1,), dtype=torch.int32, device="cuda")
    _launch(ps, [tr], ([0, len(polygons)], list(range(len(polygons)))), size, out, size * size, counts)
    want = rr.burn_transform(tr, polygons, size)
    got = out[0].cpu().numpy()
    assert np.array_equal(got, want), int((got != want).sum())
    assert int(counts[0]) == int(want.sum())
    return got


def test_golden_masks_are_bit_identical(cuda_device):
    g = rr.load_golden()
    feats = g["features"]["features"]
    tiles = [Tile(*t) for t in g["tiles"]]
    for t in tiles:
        got = RZ.burn(t, feats, 512)
        assert got.dtype == np.uint8 and np.array_equal(got, g["masks"][tuple(t)]), t
    polygons = [p["coordinates"] for f in feats for p in RZ.feature_to_mercator(f)]
    out, counts = RZ.burn_device(tiles, polygons, 512)
    for i, t in enumerate(tiles):
        assert np.array_equal(out[i].cpu().numpy(), g["masks"][tuple(t)]), t
        assert int(counts[i]) == int(g["masks"][tuple(t)].sum())
    assert RZ.burn(Tile(70762, 104119, 18), feats, 512).sum() != 0
    assert RZ.burn(Tile(69623, 104946, 18), feats, 512).sum() == 0


def _shapes(tile, rng):
    """convex shapes, a self-intersecting star, a polygon with holes, nested / overlapping / edge-sharing separate polygons,
    polygons past every side, one enclosing the tile, and sub-pixel specks"""
    polys = []
    for _ in range(6):
        cu, cv, r = rng.uniform(0.1, 0.9), rng.uniform(0.1, 0.9), rng.uniform(0.02, 0.3)
        k = rng.randint(3, 9)
        a = np.sort(rng.uniform(0, 2 * np.pi, k))
        polys.append(_merc(tile, [list(zip(cu + r * np.cos(a), cv + r * np.sin(a)))]))
    star = [(0.5 + 0.4 * np.cos(np.pi / 2 + 4 * np.pi * i / 5), 0.5 + 0.4 * np.sin(np.pi / 2 + 4 * np.pi * i / 5)) for i in range(5)]
    polys.append(_merc(tile, [star + [star[0]]]))
    polys.append(_merc(tile, [[(0.05, 0.6), (0.45, 0.6), (0.45, 0.95), (0.05, 0.95)], [(0.1, 0.65), (0.2, 0.65), (0.2, 0.75), (0.1, 0.75)],
                              [(0.3, 0.8), (0.4, 0.8), (0.35, 0.9)]]))
    polys.append(_merc(tile, [[(0.6, 0.6), (0.95, 0.6), (0.95, 0.95), (0.6, 0.95)]]))
    polys.append(_merc(tile, [[(0.7, 0.7), (0.8, 0.7), (0.8, 0.8), (0.7, 0.8)]]))      # nested separate polygon: union, not XOR
    polys.append(_merc(tile, [[(0.55, 0.1), (0.75, 0.1), (0.75, 0.3), (0.55, 0.3)]]))
    polys.append(_merc(tile, [[(0.65, 0.2), (0.85, 0.2), (0.85, 0.4), (0.65, 0.4)]]))   # overlapping
    polys.append(_merc(tile, [[(0.75, 0.3), (0.95, 0.3), (0.95, 0.5), (0.75, 0.5)]]))   # sharing an edge and a corner
    polys.append(_merc(tile, [[(-0.5, 0.45), (1.5, 0.45), (1.5, 0.55), (-0.5, 0.55)]]))  # past the left and right sides
    polys.append(_merc(tile, [[(0.45, -0.5), (0.55, -0.5), (0.55, 1.5), (0.45, 1.5)]]))  # past the top and bottom
    for _ in range(20):
        cu, cv = rng.uniform(0, 1, 2)
        r = rng.uniform(1e-5, 3e-3)
        polys.append(_merc(tile, [[(cu - r, cv), (cu, cv - r), (cu + r, cv + r)]]))       # specks
    return polys


@pytest.mark.parametrize("size", [1, 7, 32, 33, 256, 512, 1000, 1024, 4096])
def test_shapes_at_every_size(cuda_device, size):
    rng = np.random.RandomState(size)
    tile = Tile(140000, 95000, 18)
    polys = _shapes(tile, rng)
    _check([tile, Tile(tile.x + 1, tile.y, 18)], polys, size)
    enclosing = [_merc(tile, [[(-3, -3), (4, -3), (4, 4), (-3, 4)]])]
    got = _check([tile], enclosing, size)
    assert got.all()


def test_random_polygons_over_a_tile_block(cuda_device):
    rng = np.random.RandomState(1)
    base = Tile(70000, 104000, 18)
    tiles = [Tile(base.x + dx, base.y + dy, 18) for dy in range(4) for dx in range(4)]
    polys = []
    for _ in range(300):
        cu, cv = rng.uniform(-0.5, 4.5, 2)
        r = 10 ** rng.uniform(-3, 0)
        k = rng.randint(3, 20)
        a = rng.uniform(0, 2 * np.pi, k)  # unsorted angles: self-intersecting rings
        polys.append(_merc(base, [list(zip(cu + r * np.cos(a), cv + r * np.sin(a)))]))
    _check(tiles, polys, 256)


def test_hundred_thousand_vertex_ring_over_64_tiles(cuda_device):
    rng = np.random.RandomState(2)
    base = Tile(70000, 104000, 18)
    tiles = [Tile(base.x + dx, base.y + dy, 18) for dy in range(8) for dx in range(8)]
    n = 100000
    a = np.linspace(0, 2 * np.pi, n, endpoint=False)
    rad = 3.6 + 0.3 * np.sin(37 * a) + 0.02 * rng.uniform(-1, 1, n)
    polys = [_merc(base, [list(zip(4 + rad * np.cos(a), 4 + rad * np.sin(a)))])]
    got = _check(tiles, polys, 256)
    assert got[27].all() and 0 < got.sum() < got.size


def test_ties_on_pixel_centres_and_boundaries(cuda_device):
    """vertices on pixel centres and half-integers, horizontal and vertical edges on row-centre and pixel-boundary lines"""
    size = 40
    polys = [
        [np.array([(2.5, 2.5), (10.5, 2.5), (10.5, 8.5), (2.5, 8.5)])],      # edges on centre lines
        [np.array([(12.0, 2.0), (20.0, 2.0), (20.0, 8.0), (12.0, 8.0)])],    # edges on pixel boundaries
        [np.array([(22.5, 2.0), (30.0, 2.5), (26.0, 9.5)])],                 # mixed
        [np.array([(2.5, 12.5), (8.5, 18.5), (2.5, 24.5)])],                 # diagonals through centres
        [np.array([(12.0, 12.0), (18.0, 12.0), (18.0, 12.0), (12.0, 12.0)])],  # zero area on a boundary
        [np.array([(22.5, 12.5), (30.5, 12.5), (30.5, 12.5)])],              # degenerate on a centre line
        [np.array([(0.0, 30.0), (40.0, 30.0), (40.0, 40.0), (0.0, 40.0)])],  # flush with three tile sides
        [np.array([(-0.5, 26.5), (40.5, 26.5), (40.5, 27.5), (-0.5, 27.5)])],  # one row exactly, past both sides
        [np.array([(5.5, 32.5), (6.0, 32.5), (6.0, 33.5), (5.5, 33.5)])],    # half a pixel wide
        [np.array([(10.5, 30.0), (10.5, 40.0), (11.5, 40.0), (11.5, 30.0)])],  # vertical edges on centre columns
    ]
    _pixel_check(polys, size)
    for p in polys:
        _pixel_check([p], size)
    # random vertices on the half-integer lattice
    rng = np.random.RandomState(3)
    lat = [[np.array(rng.randint(-4, 2 * size + 4, size=(rng.randint(3, 9), 2)) / 2.0)] for _ in range(60)]
    _pixel_check(lat, size)


def test_empty_polygon_lists(cuda_device):
    tile = Tile(140000, 95000, 18)
    far = _merc(Tile(tile.x + 50, tile.y, 18), [[(0.2, 0.2), (0.8, 0.2), (0.5, 0.8)]])
    got = _check([tile, Tile(tile.x + 1, tile.y, 18)], [far], 64)
    assert not got.any()
    out, counts = RZ.burn_device([tile], [], 64)
    assert not out.cpu().numpy().any() and int(counts[0]) == 0
    out, counts = RZ.burn_device([], [far], 64)
    assert out.shape == (0, 64, 64) and counts.shape == (0,)


def test_strided_output_guard_bytes_and_counts(cuda_device):
    rng = np.random.RandomState(4)
    base = Tile(140000, 95000, 18)
    tiles = [Tile(base.x + i, base.y, 18) for i in range(5)]
    polys = _shapes(base, rng) + [_merc(base, [[(0.5, 0.5), (4.5, 0.2), (3.0, 0.9)]])]
    ps = RZ.PolygonSet(polys, "cuda")
    csr = RZ.bin_polygons(tiles, ps.bboxes)
    for size in (33, 64):
        G, pad = 4096, 37
        stride = size * size + pad
        buf = torch.full((G + len(tiles) * stride + G,), 0xAB, dtype=torch.uint8, device="cuda")
        counts = torch.full((len(tiles) + 64,), -7, dtype=torch.int32, device="cuda")
        _launch(ps, [RZ.tile_transform(t, size) for t in tiles], csr, size, buf[G:], stride, counts[32:])
        b = buf.cpu().numpy()
        c = counts.cpu().numpy()
        assert (b[:G] == 0xAB).all() and (b[G + len(tiles) * stride - pad:] == 0xAB).all()
        assert (c[:32] == -7).all() and (c[32 + len(tiles):] == -7).all()
        for i, t in enumerate(tiles):
            img = b[G + i * stride:G + i * stride + size * size].reshape(size, size)
            want = rr.burn_transform(rr.transform(t, size), polys, size)
            assert np.array_equal(img, want), (size, i)
            assert c[32 + i] == int(want.sum())
            if i + 1 < len(tiles):
                assert (b[G + i * stride + size * size:G + (i + 1) * stride] == 0xAB).all()


def _write_dataset(tmp_path):
    path = tmp_path / "dataset.toml"
    path.write_text("[common]\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n")
    return str(path)


def test_tool_end_to_end(cuda_device, tmp_path, capsys):
    from robosat_b200.tools import rasterize as tool

    rng = np.random.RandomState(5)
    base = Tile(70500, 104100, 18)
    tiles = [Tile(base.x + dx, base.y + dy, 18) for dy in range(3) for dx in range(4)]
    left, bottom, right, top = RZ.xy_bounds(base)
    side = right - left

    def lonlat(u, v):
        X, Y = left + u * side, top - v * side
        return [float(np.degrees(X / RZ.R)), float(np.degrees(2 * np.arctan(np.exp(Y / RZ.R)) - np.pi / 2))]

    feats = []
    for _ in range(40):
        cu, cv, r = rng.uniform(-0.3, 4.3), rng.uniform(-0.3, 3.3), rng.uniform(0.02, 0.6)
        a = np.sort(rng.uniform(0, 2 * np.pi, rng.randint(3, 10)))
        ring = [lonlat(cu + r * np.cos(t), cv + r * np.sin(t)) for t in a]
        feats.append({"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [ring + [ring[0]]]}})
    feats.insert(3, {"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [[lonlat(0, 0), lonlat(1, 1), lonlat(0, 0)]]}})
    feats.insert(5, {"type": "Feature", "properties": {}, "geometry": {"type": "Point", "coordinates": lonlat(0.5, 0.5)}})
    import json

    (tmp_path / "f.geojson").write_text(json.dumps({"type": "FeatureCollection", "features": feats}))
    listed = tiles + [Tile(base.x + 40, base.y, 18), tiles[2]]  # a tile without features, and one listed twice
    (tmp_path / "tiles.csv").write_text("".join("%d,%d,%d\n" % t for t in listed))
    out = tmp_path / "out"
    size = 128
    # pre-existing masks for two tiles: merged with np.maximum
    prev = {}
    for t in (tiles[0], tiles[5]):
        m = np.zeros((size, size), np.uint8)
        m[10:30, 40:100] = 1
        d = out / str(t.z) / str(t.x)
        d.mkdir(parents=True, exist_ok=True)
        im = Image.fromarray(m, mode="P")
        im.putpalette(make_palette("denim", "orange"))
        im.save(str(d / ("%d.png" % t.y)))
        prev[t] = m
    for batch in (64, 5):
        tool.main(argparse.Namespace(features=str(tmp_path / "f.geojson"), tiles=str(tmp_path / "tiles.csv"), out=str(out),
                                     dataset=_write_dataset(tmp_path), zoom=18, size=size), batch=batch)
        err = capsys.readouterr().err
        assert err.splitlines() == ["Warning: invalid feature 3, skipping"]
        polygons, _ = RZ.polygons_from_features(feats)
        for t in dict.fromkeys(listed):
            im = Image.open(str(out / str(t.z) / str(t.x) / ("%d.png" % t.y)))
            assert im.mode == "P"
            assert im.getpalette()[:6] == make_palette("denim", "orange")
            want = rr.burn_transform(rr.transform(t, size), polygons, size)
            if t in prev:
                want = np.maximum(want, prev[t])
            assert np.array_equal(np.array(im), want), t
    assert not np.array(Image.open(str(out / "18" / str(base.x + 40) / ("%d.png" % base.y)))).any()
