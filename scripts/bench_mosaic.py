"""Cost of `rs mosaic` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_mosaic.py --out results/h100_mosaic.json [--launches 200 --size 20000]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    rsb_mosaic_warp alone: nearest and bilinear x an EPSG:3857 grid at the tiles' own pixel size / EPSG:4326 / UTM, one
              launch over a 4096^2 output window from the zoom-19 512^2 tiles it reaches (all present), CUDA events over `launches`
              launches after 20 warm-up launches; µs per output megapixel, and bytes = the planes of the reached tiles plus the
              output written, GB/s and that rate over the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)
    tool      robosat_b200.tools.mosaic.main --like a `size` x `size` UTM grid of 0.3 m pixels near 5° N from the zoom-18 512^2
              1-bit palette mask PNGs (seeded blobs, PIL optimize=True) that cover it, generated here, after a warm-up run on a small
              grid: seconds of PNG decode (decoder thread, overlapped with the device), upload, warp (CUDA events), deflate and write
              (writer thread), and the wall clock
"""

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import mosaic as M  # noqa: E402
from robosat_b200 import tile as T  # noqa: E402
from robosat_b200.rasterize import CE  # noqa: E402
from robosat_b200.tools import mosaic as tool  # noqa: E402

HBM3 = 3.35e12
ZOOM, S = 19, 512
OUT = 4096


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def grid_for(kind):
    """a 4096^2 grid near (10.2 E, 47.3 N) whose pixels are about one zoom-19 pixel on the ground"""
    px = CE / (2 ** ZOOM * S)
    X, Y = T.lonlat_to_mercator(10.2, 47.3)
    if kind == "3857":
        x0 = round((float(X) + CE / 2) / px)
        y0 = round((CE / 2 - float(Y)) / px)
        return M.Grid(OUT, OUT, "3857", (-CE / 2 + x0 * px, px, 0.0, CE / 2 - y0 * px, 0.0, -px))
    ground = px * np.cos(np.radians(47.3))
    if kind == "4326":
        return M.Grid(OUT, OUT, "4326", (10.2, ground / 75000.0, 0.0, 47.3, 0.0, -ground / 111000.0))
    E, N = T.tm_forward(10.2, 47.3, 9.0)
    return M.Grid(OUT, OUT, ("utm", 32, False), (float(E), ground, 0.0, float(N), 0.0, -ground))


def bench_kernel(kind, resampling, launches):
    grid = grid_for(kind)
    step = M.choose_step(grid, ZOOM, S)
    lg = step.bit_length() - 1
    nodes = M.lattice(grid, ZOOM, S, step, 0, ((OUT - 1) >> lg) + 1, 0, ((OUT - 1) >> lg) + 1)
    tx0, ty0, tx1, ty1 = M.tile_reach(nodes, ZOOM, S)
    tw, th = tx1 - tx0 + 1, ty1 - ty0 + 1
    n = tw * th
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(1)
    planes = torch.randint(0, 256, (n * S * S,), dtype=torch.uint8, device=dev, generator=gen)
    slots = torch.arange(n, dtype=torch.int32, device=dev)
    dnodes = torch.from_numpy(nodes).to(dev)
    out = torch.empty((OUT, OUT), dtype=torch.uint8, device=dev)
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    lib = _lib.load()
    mode = M.RESAMPLING[resampling]

    def launch():
        _lib.check(lib.rsb_mosaic_warp(planes.data_ptr(), S * S, n, slots.data_ptr(), tx0, ty0, tw, th, ZOOM, S, dnodes.data_ptr(), 0, 0,
                                       nodes.shape[1], nodes.shape[0], step, 0, 0, OUT, OUT, mode, 0, out.data_ptr(), OUT, counts[0:1].data_ptr(),
                                       counts[1:2].data_ptr(), _lib.current_stream_ptr()), "rsb_mosaic_warp")

    for _ in range(20):
        launch()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(launches):
        launch()
    end.record()
    torch.cuda.synchronize()
    sec = start.elapsed_time(end) / 1e3 / launches
    assert int(counts[1]) == 0 and int(counts[0]) == OUT * OUT, counts.tolist()
    nbytes = n * S * S + OUT * OUT
    return {"crs": kind, "resampling": resampling, "step": step, "tiles_reached": n, "us_per_launch": round(sec * 1e6, 2),
            "us_per_output_mpx": round(sec * 1e6 / (OUT * OUT / 1e6), 2), "bytes": nbytes, "gb_per_s": round(nbytes / sec / 1e9, 1),
            "share_of_hbm3": round(nbytes / sec / HBM3, 3)}


def write_masks(root, grid, zoom):
    """1-bit palette PNGs of seeded blobs for every tile under the grid -> count"""
    gx, gy = M.global_coords(grid, zoom, 512, np.array([0, grid.width, 0, grid.width]), np.array([0, 0, grid.height, grid.height]))
    keys = [(x, y) for x in range(int(gx.min() // 512), int(gx.max() // 512) + 1) for y in range(int(gy.min() // 512), int(gy.max() // 512) + 1)]
    rng = np.random.default_rng(3)
    for x, y in keys:
        base = rng.random((9, 9)) < 0.3
        m = np.repeat(np.repeat(base, 64, 0), 64, 1)[32:544, 32:544].astype(np.uint8)
        path = os.path.join(root, str(zoom), str(x), "%d.png" % y)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        im = Image.fromarray(m, "P")
        im.putpalette([0, 0, 0, 255, 255, 255])
        im.save(path, optimize=True)
    return len(keys)


def utm_like(path, size, res=0.3):
    import tiff_writer as tw

    E, N = T.tm_forward(9.3, 5.0, 9.0)
    # only the header of a --like raster is read: one pixel of data, with the grid's width and height in the tags
    tw.write_tiff(path, np.zeros((1, 1, 1), np.uint8), geo=tw.geokeys(1, 32632), scale=(res, res, 0.0), tiepoint=(0, 0, 0, float(E), float(N), 0),
                  tags={256: (4, [size]), 257: (4, [size])})
    return M.Grid(size, size, ("utm", 32, False), (float(E), res, 0.0, float(N), 0.0, -res))


def bench_tool(size, workdir):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    like = os.path.join(workdir, "like.tif")
    grid = utm_like(like, size)
    t0 = time.perf_counter()
    n = write_masks(os.path.join(workdir, "masks"), grid, 18)
    gen_s = time.perf_counter() - t0
    small = os.path.join(workdir, "small.tif")
    utm_like(small, 1024)
    out = os.path.join(workdir, "out.tif")
    tool.main(argparse.Namespace(zoom=18, like=small, resampling="nearest", nodata=None, masks=os.path.join(workdir, "masks"), out=out))  # warm-up
    stats = {}
    t0 = time.perf_counter()
    tool.main(argparse.Namespace(zoom=18, like=like, resampling="nearest", nodata=None, masks=os.path.join(workdir, "masks"), out=out), stats)
    wall = time.perf_counter() - t0
    return {"grid": "%d x %d UTM 32N, 0.3 m" % (size, size), "tiles": n, "generate_s": round(gen_s, 1), "step": stats["step"],
            "windows": stats["windows"], "decode_s": round(stats["decode_s"], 3), "upload_s": round(stats["upload_s"], 3),
            "warp_s": round(stats["warp_s"], 3), "deflate_s": round(stats["encode_s"], 3), "write_s": round(stats["write_s"], 3),
            "sink_s": round(stats["sink_s"], 3), "wall_s": round(wall, 3), "file_bytes": os.path.getsize(out),
            "output_mpx_per_s": round(size * size / 1e6 / wall, 1)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=None)
    p.add_argument("--launches", type=int, default=200)
    p.add_argument("--size", type=int, default=20000)
    a = p.parse_args()
    rec = {"card": card(), "kernel": [bench_kernel(k, r, a.launches) for k in ("3857", "4326", "utm") for r in ("nearest", "bilinear")]}
    with tempfile.TemporaryDirectory() as d:
        rec["tool"] = bench_tool(a.size, d)
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fp:
            fp.write(line + "\n")


if __name__ == "__main__":
    main()
