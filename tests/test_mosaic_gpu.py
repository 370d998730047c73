"""rsb_mosaic_warp and `rs mosaic` on the H100: output rasters and covered counts bit-identical to the numpy restatement
(tests/mosaic_reference.py) for every CRS, both resamplings, holes, the world's edge, ragged grids and budgets from one chunk per
window to one window; the default grid lays the tiles side by side; gray tiles survive `rs mosaic` then `rs tile`; polygons burned
by `rs rasterize` come back on a UTM grid where they are drawn analytically; and the tool writes what PIL reads."""

import argparse
import math
import os

import numpy as np
import pytest
from PIL import Image

import mosaic_reference as ref
from test_mosaic import smallest_budget
import tiff_writer as tw
from robosat_b200 import mosaic as M
from robosat_b200 import tile as T
from robosat_b200.geotiff import GeoTiff
from robosat_b200.rasterize import CE, PolygonSet, rasterize_device

pytestmark = pytest.mark.gpu

ZOOM, SIZE = 18, 128


def blocks(size, seed):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (size // 8 + 1, size // 8 + 1), dtype=np.uint8)
    return np.repeat(np.repeat(base, 8, 0), 8, 1)[:size, :size].copy()


def write_tiles(root, keys, zoom, size, seed=0, palette=None):
    """gray (or palette) PNG tiles of blocky noise -> ({(x, y): path}, {(x, y): plane})"""
    paths, planes = {}, {}
    for k, (x, y) in enumerate(keys):
        p = blocks(size, seed + k)
        path = os.path.join(root, str(zoom), str(x), "%d.png" % y)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        im = Image.fromarray(p, "L")
        if palette is not None:
            im = im.convert("P")
            im.putpalette(palette)
        im.save(path)
        paths[(x, y)], planes[(x, y)] = path, p
    return paths, planes


def utm_grid(zone, south, lon, lat, W, H, res):
    E, N = T.tm_forward(lon, lat, 6 * zone - 183, fn=1e7 if south else 0.0)
    return M.Grid(W, H, ("utm", zone, south), (float(E), res, 0.0, float(N), 0.0, -res))


def grid_of(kind):
    """grids near (10 E, 48 N) or (-69 E, 33 S), a few hundred pixels a side (ragged against 256-pixel chunks)"""
    px = CE / (2 ** ZOOM * SIZE)
    x0, y0 = 137000, 91000  # a tile of zoom 18 near (8.1 E, 47.9 N)
    left, top = x0 * SIZE * px - CE / 2, CE / 2 - y0 * SIZE * px
    if kind == "3857-native":
        return M.Grid(517, 389, "3857", (left + 37 * px, px, 0.0, top - 21 * px, 0.0, -px))
    if kind == "3857":
        return M.Grid(431, 300, "3857", (left + 10.3, 0.83 * px, 0.0, top - 7.1, 0.0, -0.77 * px))
    lon, lat = T.mercator_to_lonlat(left + 30.0, top - 30.0)
    if kind == "4326":
        return M.Grid(400, 333, "4326", (float(lon), 4e-6, 0.0, float(lat), 0.0, -3e-6))
    if kind == "utm":
        return utm_grid(32, False, float(lon), float(lat), 450, 300, 0.35)
    if kind == "utm-south":
        return utm_grid(19, True, -69.4, -33.1, 300, 280, 0.5)
    if kind == "rotated":
        return M.Grid(300, 280, "3857", (left + 40.0, 0.4, 0.06, top - 10.0, 0.05, -0.4))
    raise ValueError(kind)


def tiles_under(grid, zoom, size, holes=True):
    gx, gy = M.global_coords(grid, zoom, size, np.array([0, grid.width, 0, grid.width]), np.array([0, 0, grid.height, grid.height]))
    keys = [(x, y) for x in range(int(gx.min() // size), int(gx.max() // size) + 1) for y in range(int(gy.min() // size), int(gy.max() // size) + 1)]
    return [k for i, k in enumerate(keys) if not holes or i % 5 != 2]


def check(tmp_path, grid, resampling, zoom=ZOOM, size=SIZE, budget=M.DEFAULT_BUDGET, nodata=0, keys=None):
    keys = keys if keys is not None else tiles_under(grid, zoom, size)
    paths, planes = write_tiles(str(tmp_path / "t"), keys, zoom, size)
    stats = {}
    got, covered = M.mosaic_device(paths, zoom, size, grid, resampling, nodata, budget, stats=stats)
    want, wcov, step = ref.render(planes, grid, zoom, size, resampling, nodata)
    assert stats["step"] == step
    assert covered == wcov and 0 < covered
    assert np.array_equal(got, want), int((got != want).sum())
    return paths, got, covered, stats


@pytest.mark.parametrize("kind", ["3857-native", "3857", "4326", "utm", "utm-south", "rotated"])
@pytest.mark.parametrize("resampling", ["nearest", "bilinear"])
def test_restatement_per_crs(tmp_path, cuda_device, kind, resampling):
    grid = grid_of(kind)
    paths, got, covered, _ = check(tmp_path, grid, resampling, nodata=200)
    assert covered < grid.width * grid.height  # the holes
    again, c2 = M.mosaic_device(paths, ZOOM, SIZE, grid, resampling, 200)
    assert c2 == covered and again.tobytes() == got.tobytes()


@pytest.mark.parametrize("resampling", ["nearest", "bilinear"])
def test_budgets_from_one_chunk_to_one_window(tmp_path, cuda_device, resampling):
    grid = M.Grid(700, 530, "3857", grid_of("3857").geotransform)
    keys = tiles_under(grid, ZOOM, SIZE)
    paths, planes = write_tiles(str(tmp_path / "t"), keys, ZOOM, SIZE)
    want, wcov, _ = ref.render(planes, grid, ZOOM, SIZE, resampling)
    step = M.choose_step(grid, ZOOM, SIZE)
    one = len(M.plan(grid, ZOOM, SIZE, M.tile_array(paths), step))
    for budget in (M.DEFAULT_BUDGET, smallest_budget(grid, ZOOM, SIZE, M.tile_array(paths), step)):
        stats = {}
        got, covered = M.mosaic_device(paths, ZOOM, SIZE, grid, resampling, budget=budget, stats=stats)
        assert covered == wcov and np.array_equal(got, want)
    assert stats["windows"] > one


@pytest.mark.parametrize("resampling", ["nearest", "bilinear"])
def test_world_edge_at_a_low_zoom(tmp_path, cuda_device, resampling):
    zoom, size = 2, 64
    px = CE / (2 ** zoom * size)
    # a 3857 grid that runs off the world's top-left corner, and the tiles of that corner
    grid = M.Grid(150, 130, "3857", (-CE / 2 - 20.5 * px, 0.9 * px, 0.0, CE / 2 + 13.25 * px, 0.0, -0.9 * px))
    _, got, covered, _ = check(tmp_path, grid, resampling, zoom, size, nodata=77, keys=[(0, 0), (1, 0), (0, 1)])
    assert (got[:10, :] == 77).all() and (got[:, :20] == 77).all()


@pytest.mark.parametrize("resampling", ["nearest", "bilinear"])
def test_default_grid_lays_the_tiles_side_by_side(tmp_path, cuda_device, resampling):
    keys = [(1000 + i, 2000 + j) for i in range(3) for j in range(2) if (i, j) != (1, 1)]
    paths, planes = write_tiles(str(tmp_path / "t"), keys, ZOOM, SIZE)
    grid = M.default_grid(paths, ZOOM, SIZE)
    got, covered = M.mosaic_device(paths, ZOOM, SIZE, grid, resampling, 9)
    want = np.full((2 * SIZE, 3 * SIZE), 9, np.uint8)
    for (x, y), p in planes.items():
        want[(y - 2000) * SIZE:(y - 1999) * SIZE, (x - 1000) * SIZE:(x - 999) * SIZE] = p
    assert covered == 5 * SIZE * SIZE and np.array_equal(got, want)


def test_round_trip_through_rs_tile(tmp_path, cuda_device):
    from robosat_b200.tools import mosaic as tool

    keys = [(70000 + i, 45000 + j) for i in range(3) for j in range(3) if (i + j) % 4 != 1]
    paths, planes = write_tiles(str(tmp_path / "t"), keys, ZOOM, SIZE)
    out = str(tmp_path / "m.tif")
    tool.main(argparse.Namespace(zoom=ZOOM, like=None, resampling="nearest", nodata=None, masks=str(tmp_path / "t"), out=out))
    g = GeoTiff(out)
    got = T.tile_device(g, ZOOM, SIZE, "nearest")
    for k, p in planes.items():
        im, count = got[k]
        assert count == SIZE * SIZE
        assert np.array_equal(im, np.repeat(p[..., None], 3, axis=-1)), k


def test_rasterized_polygons_come_back_on_a_utm_grid(tmp_path, cuda_device):
    z, S = 18, 512
    grid = utm_grid(32, False, 9.02, 47.51, 900, 800, 0.3)
    c, a, b, f, d, e = grid.geotransform
    jj, ii = np.mgrid[0:grid.height, 0:grid.width] + 0.5
    lon, lat = T.tm_inverse(c + a * ii, f + e * jj, 9.0)
    rng = np.random.default_rng(5)
    lo0, la0, dlo, dla = lon.min(), lat.max(), lon.max() - lon.min(), lat.max() - lat.min()
    polys = []
    for _ in range(6):
        cx, cy = lo0 + rng.uniform(0.2, 0.8) * dlo, la0 - rng.uniform(0.2, 0.8) * dla
        r = rng.uniform(0.08, 0.15)
        t = np.sort(rng.uniform(0, 2 * np.pi, rng.integers(3, 8)))
        ring = [(cx + r * dlo * math.cos(s), cy + r * dla * math.sin(s)) for s in t]
        polys.append(ring + [ring[0]])
    merc = [[np.stack(T.lonlat_to_mercator(np.asarray(p)[:, 0], np.asarray(p)[:, 1]), axis=1)] for p in polys]
    keys = tiles_under(grid, z, S, holes=False)
    masks, _ = rasterize_device(PolygonSet(merc, cuda_device), [(x, y, z) for x, y in keys], S)
    masks = masks.cpu().numpy()
    paths = {}
    for (x, y), m in zip(keys, masks):
        paths[(x, y)] = str(tmp_path / "l" / str(z) / str(x) / ("%d.png" % y))
        os.makedirs(os.path.dirname(paths[(x, y)]), exist_ok=True)
        im = Image.fromarray(m.astype(np.uint8), "L").convert("P")
        im.putpalette([0, 0, 0, 255, 255, 255])
        im.save(paths[(x, y)], optimize=True)
    got, covered = M.mosaic_device(paths, z, S, grid, "nearest")
    assert covered == grid.width * grid.height
    X, Y = T.lonlat_to_mercator(lon, lat)
    from test_tile_gpu import _inside, _segment_distance

    want = _inside(lon, lat, polys)
    mine = got == 1
    inter, union = int((mine & want).sum()), int((mine | want).sum())
    assert union > 0 and inter / union >= 0.98, inter / union
    rr, cc = np.nonzero(mine != want)
    P = np.stack([X[rr, cc], Y[rr, cc]], axis=1)
    edges = [(m[0][k], m[0][k + 1]) for m in merc for k in range(len(m[0]) - 1)]
    dist = np.min([_segment_distance(P, A, B) for A, B in edges], axis=0)
    tile_px = CE / (2 ** z * S)
    assert dist.max() <= tile_px * 1.0001, (dist.max(), tile_px)


def test_tool_end_to_end(tmp_path, cuda_device, capsys):
    from robosat_b200.tools import mosaic as tool

    grid = grid_of("utm")
    keys = tiles_under(grid, ZOOM, SIZE)
    pal = [0, 0, 0, 255, 0, 0, 0, 255, 0, 0, 0, 255]
    for k, (x, y) in enumerate(keys):  # palettes of 2..4 entries that agree where they overlap, as optimize=True leaves them
        path = str(tmp_path / "m" / str(ZOOM) / str(x) / ("%d.png" % y))
        os.makedirs(os.path.dirname(path), exist_ok=True)
        n = 2 + k % 3
        im = Image.fromarray((blocks(SIZE, k) % n).astype(np.uint8), "P")
        im.putpalette(pal[:3 * n])
        im.save(path)
    like = tw.write_tiff(str(tmp_path / "like.tif"), np.zeros((grid.height, grid.width, 1), np.uint8), geo=tw.geokeys(1, 32632),
                         scale=(grid.geotransform[1], -grid.geotransform[5], 0.0), tiepoint=(0, 0, 0, grid.geotransform[0], grid.geotransform[3], 0))
    out = tmp_path / "o.tif"
    out.write_bytes(b"stale")
    stats = {}
    args = argparse.Namespace(zoom=ZOOM, like=like, resampling="nearest", nodata=None, masks=str(tmp_path / "m"), out=str(out))
    tool.main(args, stats)
    paths = M.scan(str(tmp_path / "m"), ZOOM)
    want, _ = M.mosaic_device(paths, ZOOM, SIZE, grid, "nearest")
    im = Image.open(out)
    assert im.mode == "P" and np.array_equal(np.array(im), want)
    assert im.getpalette()[:12] == pal and not any(im.getpalette()[12:768])
    assert 42113 not in im.tag_v2
    args.nodata, args.resampling = 3, "bilinear"
    tool.main(args)
    im = Image.open(out)
    assert im.tag_v2[42113].strip("\0") == "3" and (np.array(im) == 3).any()
    assert capsys.readouterr().err == ""
    # warnings: a coarse grid, then a grid no tile covers
    coarse = tw.write_tiff(str(tmp_path / "coarse.tif"), np.zeros((40, 40, 1), np.uint8), geo=tw.geokeys(1, 32632),
                           scale=(5.0, 5.0, 0.0), tiepoint=(0, 0, 0, grid.geotransform[0], grid.geotransform[3], 0))
    tool.main(argparse.Namespace(zoom=ZOOM, like=coarse, resampling="nearest", nodata=None, masks=str(tmp_path / "m"), out=str(out)))
    assert capsys.readouterr().err.count("Warning: an output pixel spans") == 1
    far = tw.write_tiff(str(tmp_path / "far.tif"), np.zeros((40, 40, 1), np.uint8), geo=tw.geokeys(1, 32632),
                        scale=(0.3, 0.3, 0.0), tiepoint=(0, 0, 0, 300000.0, 4000000.0, 0))
    tool.main(argparse.Namespace(zoom=ZOOM, like=far, resampling="nearest", nodata=None, masks=str(tmp_path / "m"), out=str(out)))
    assert capsys.readouterr().err.count(M.W_EMPTY) == 1
    # a failed run (a tile that cannot be decoded) leaves no file behind, and the old one stays
    before = out.read_bytes()
    bad = sorted(paths.values())[0]
    with open(bad, "r+b") as fp:
        fp.seek(60)
        fp.write(b"\xff" * 40)
    with pytest.raises(SystemExit, match="Error"):
        tool.main(args)
    assert out.read_bytes() == before
    assert not [n for n in os.listdir(tmp_path) if n.endswith(".tmp")]
