"""Cost of `rs tile --resampling average` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_tile_average.py --out results/h100_tile_average.json [--launches 50 --size 20000 --repeats 2]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query; bench_tile.card)
    kernel    rsb_tile_average alone, and rsb_tile_warp bilinear beside it on the same block of tiles: one launch of 64 (8 x 8) tiles
              of 512^2 at zoom 18 from an RGB EPSG:3857 or UTM source whose pixels are 1/r of a zoom-18 pixel (r = 1, 2, 4, 8, 16), CUDA
              events over `launches` launches after 5 warm-up launches; bytes = the source window the lattice reaches plus the RGB tiles
              written, GB/s and that rate over the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)
    tool      robosat_b200.tools.tile.main --zoom 18 --size 512, average and bilinear alternated `repeats` times, on a seeded `size` x
              `size` RGB GeoTIFF in UTM zone 32 with 0.05 m pixels (about 4 per tile pixel), after a warm-up run of each on a small
              raster: seconds in decode (host threads, overlapped with the device), upload, kernel (CUDA events), PNG encode and write
              (the writer thread), wall clock, tiles/s
"""

import argparse
import json
import os
import struct
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench_tile as BT  # noqa: E402
from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import tile as T  # noqa: E402
from robosat_b200.geotiff import GeoTiff  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402
from robosat_b200.rasterize import CE  # noqa: E402
from robosat_b200.tools import tile as tool  # noqa: E402

ZOOM, S, SIDE = 18, 512, 8
RATIOS = (1, 2, 4, 8, 16)
PIXEL = 0.05  # metres: the tool's raster


def raster_for(kind, r):
    """a raster starting at (BT.LON, BT.LAT) whose pixels are 1/r of a zoom-ZOOM pixel (on the ground, for UTM), wide enough for the block"""
    W = (SIDE + 2) * S * r
    X, Y = T.lonlat_to_mercator(np.float64(BT.LON), np.float64(BT.LAT))
    px = CE / (2 ** ZOOM * S)
    if kind == "3857":
        return BT.Raster("3857", (float(X), px / r, 0.0, float(Y), 0.0, -px / r), W, W)
    E, N = T.tm_forward(BT.LON, BT.LAT, 9.0)
    ground = px * np.cos(np.radians(BT.LAT)) / r
    return BT.Raster(("utm", 32, False), (float(E), ground, 0.0, float(N), 0.0, -ground), W, W)


def kernel_time(kind, r, resampling, launches):
    R = raster_for(kind, r)
    X, Y = T.lonlat_to_mercator(np.float64(BT.LON), np.float64(BT.LAT))
    tile_m = CE / 2 ** ZOOM
    x0, y0 = int((X + CE / 2) / tile_m) + 1, int((CE / 2 - Y) / tile_m) + 1
    tiles = np.array([(x0 + i, y0 + j) for j in range(SIDE) for i in range(SIDE)], np.int64)
    corner = resampling == "average"
    step = T.choose_step(R, ZOOM, S, tiles, corner)
    lg = step.bit_length() - 1
    kx0, ky0 = (x0 * S) >> lg, (y0 * S) >> lg
    nodes = T.lattice(R, ZOOM, S, step, kx0, T.last_node(x0 + SIDE - 1, S, lg, corner), ky0, T.last_node(y0 + SIDE - 1, S, lg, corner), corner)
    row0, rows, col0, cols = T.source_box(nodes, R)
    window = T.Window(y0, list(range(x0, x0 + SIDE)), kx0, ky0, nodes, (row0, rows, col0, cols))
    dev = torch.device("cuda")
    src = torch.randint(0, 256, (rows * cols * 3,), dtype=torch.uint8, device=dev)
    d_nodes = torch.from_numpy(nodes).to(dev)
    d_tiles = torch.from_numpy(tiles).to(dev)
    N = len(tiles)
    out = torch.empty((N, S, S, 3), dtype=torch.uint8, device=dev)
    covered = torch.empty((N,), dtype=torch.int64, device=dev)
    misses = torch.empty((1,), dtype=torch.int64, device=dev)
    lib = _lib.load()

    def launch():
        T.warp(lib, resampling, src.data_ptr(), window, R, d_nodes.data_ptr(), step, d_tiles.data_ptr(), N, S, out.data_ptr(), S * S * 3,
               covered.data_ptr(), misses.data_ptr())

    for _ in range(5):
        launch()
    torch.cuda.synchronize()
    assert int(misses.item()) == 0 and int(covered.sum()) == N * S * S, "the block must lie inside the raster"
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        launch()
    b.record()
    b.synchronize()
    sec = a.elapsed_time(b) / 1e3 / launches
    nbytes = rows * cols * 3 + N * S * S * 3
    del src, out
    torch.cuda.empty_cache()
    return {"crs": kind, "ratio": r, "resampling": resampling, "tiles": N, "step": step, "window": [cols, rows], "launches": launches,
            "us": round(sec * 1e6, 1), "us_per_tile": round(sec * 1e6 / N, 2), "bytes": nbytes, "GB_per_s": round(nbytes / sec / 1e9, 1),
            "share_of_hbm3": round(nbytes / sec / BT.HBM3, 3)}


def write_fine_geotiff(path, size, seed=0):
    """bench_tile's seeded UTM GeoTIFF with PIXEL-metre pixels: the same file with its ModelPixelScale doubles rewritten"""
    BT.write_geotiff(path, size, seed)
    with open(path, "r+b") as fp:
        data = fp.read()
        old = struct.pack("<ddd", 0.2, 0.2, 0.0)
        assert data.count(old) == 1
        fp.seek(data.index(old))
        fp.write(struct.pack("<ddd", PIXEL, PIXEL, 0.0))


def run_tool(path, out, resampling):
    stats = {}
    t0 = time.perf_counter()
    tool.main(argparse.Namespace(zoom=ZOOM, size=S, tiles=None, resampling=resampling, raster=path, out=out), stats)
    wall = time.perf_counter() - t0
    rec = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}
    rec.update(resampling=resampling, wall_s=round(wall, 3), tiles_per_s=round(stats["written"] / wall, 1))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--size", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_average needs a CUDA device")
    _lib.require_device()
    rec = {"card": BT.card(), "kernel": []}
    for kind in ("3857", "utm"):
        for r in RATIOS:
            for resampling in ("average", "bilinear"):
                rec["kernel"].append(kernel_time(kind, r, resampling, args.launches))
                print(json.dumps(rec["kernel"][-1]), file=sys.stderr)
    with tempfile.TemporaryDirectory() as tmp:
        warm = os.path.join(tmp, "warm.tif")
        write_fine_geotiff(warm, 2048, seed=1)
        for resampling in ("average", "bilinear"):
            run_tool(warm, os.path.join(tmp, "warm-" + resampling), resampling)
        big = os.path.join(tmp, "ortho.tif")
        t0 = time.perf_counter()
        write_fine_geotiff(big, args.size)
        gen = time.perf_counter() - t0
        runs = []
        for k in range(args.repeats):
            for resampling in ("average", "bilinear"):
                runs.append(run_tool(big, os.path.join(tmp, "tiles-%s-%d" % (resampling, k)), resampling))
                print(json.dumps(runs[-1]), file=sys.stderr)
        rec["tool"] = dict(raster=args.size, pixel_m=PIXEL, zoom=ZOOM, size=S, file_bytes=os.path.getsize(big), generate_s=round(gen, 1),
                           threads=usable_cores(), coarse_ratio=round(T.coarse_ratio(GeoTiff(big), ZOOM, S), 2), runs=runs)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
