"""Cost of `rs tile` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_tile.py --out results/h100_tile.json [--launches 200 --size 20000]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    rsb_tile_warp alone: nearest and bilinear x EPSG:3857 / 4326 / UTM, one launch of a block of 64 (8 x 8) or 1024
              (32 x 32) tiles of 512^2 at zoom 19 from an RGB source of about the zoom's pixel size, CUDA events over `launches`
              launches after 20 warm-up launches; bytes = the source window the lattice reaches plus the RGB tiles written, GB/s
              and that rate over the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)
    tool      robosat_b200.tools.tile.main at zoom 18 on a seeded `size` x `size` RGB GeoTIFF in UTM zone 32 (0.2 m pixels, 256^2 tiles,
              deflate level 1, predictor 2) generated here, after a warm-up run on a small raster: seconds in decode (host threads,
              overlapped with the device), upload, warp (CUDA events), PNG encode and write (the writer thread), wall clock, tiles/s
"""

import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import tile as T  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402
from robosat_b200.rasterize import CE  # noqa: E402
from robosat_b200.tools import tile as tool  # noqa: E402

HBM3 = 3.35e12
ZOOM, S = 19, 512
TOOL_ZOOM = 18  # 0.2 m UTM pixels are about one zoom-18 pixel on the ground at 47° N
LON, LAT = 10.2, 47.3


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


class Raster:
    def __init__(self, crs, gt, W, H):
        self.crs, self.geotransform, self.width, self.height, self.spp, self.alpha, self.nodata = crs, gt, W, H, 3, False, -1


def raster_for(kind, W=40000):
    """a W x W raster whose top-left corner is at (LON, LAT), with pixels of about the zoom's pixel on the ground"""
    X, Y = T.lonlat_to_mercator(np.float64(LON), np.float64(LAT))
    if kind == "3857":
        return Raster("3857", (float(X), 0.15, 0.0, float(Y), 0.0, -0.15), W, W)
    if kind == "4326":
        return Raster("4326", (LON, 1.35e-6, 0.0, LAT, 0.0, -0.92e-6), W, W)
    E, N = T.tm_forward(LON, LAT, 9.0)
    return Raster(("utm", 32, False), (float(E), 0.1, 0.0, float(N), 0.0, -0.1), W, W)


def kernel_time(kind, resampling, side, launches):
    r = raster_for(kind)
    X, Y = T.lonlat_to_mercator(np.float64(LON), np.float64(LAT))
    tile_m = CE / 2 ** ZOOM
    x0, y0 = int((X + CE / 2) / tile_m) + 1, int((CE / 2 - Y) / tile_m) + 1
    tiles = np.array([(x0 + i, y0 + j) for j in range(side) for i in range(side)], np.int64)
    step = T.choose_step(r, ZOOM, S, tiles)
    lg = step.bit_length() - 1
    kx0, ky0 = (x0 * S) >> lg, (y0 * S) >> lg
    nodes = T.lattice(r, ZOOM, S, step, kx0, (((x0 + side) * S - 1) >> lg) + 1, ky0, (((y0 + side) * S - 1) >> lg) + 1)
    row0, rows, col0, cols = T.source_box(nodes, r)
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
        _lib.check(lib.rsb_tile_warp(src.data_ptr(), cols * 3, row0, col0, rows, cols, r.width, r.height, 3, 0, -1, d_nodes.data_ptr(), kx0, ky0,
                                     nodes.shape[1], nodes.shape[0], step, d_tiles.data_ptr(), N, S, T.RESAMPLING[resampling], out.data_ptr(), S * S * 3,
                                     covered.data_ptr(), misses.data_ptr(), _lib.current_stream_ptr()), "rsb_tile_warp")

    for _ in range(20):
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
    return {"crs": kind, "resampling": resampling, "tiles": N, "step": step, "launches": launches, "us": round(sec * 1e6, 1),
            "us_per_tile": round(sec * 1e6 / N, 2), "bytes": nbytes, "GB_per_s": round(nbytes / sec / 1e9, 1),
            "share_of_hbm3": round(nbytes / sec / HBM3, 3)}


def write_geotiff(path, size, seed=0, chunk=256):
    """a seeded RGB GeoTIFF of size x size in UTM zone 32: blocks of smooth colour plus noise, deflate level 1, predictor 2"""
    rng = np.random.default_rng(seed)
    across = (size + chunk - 1) // chunk
    base = rng.integers(0, 256, (across * 4 + 1, across * 4 + 1, 3), dtype=np.uint8)
    E, N = T.tm_forward(LON, LAT, 9.0)

    def one(k):
        r, c = divmod(k, across)
        g = np.random.default_rng(seed * 1000003 + k)
        blk = np.repeat(np.repeat(base[r * 4:r * 4 + 4, c * 4:c * 4 + 4], chunk // 4, 0), chunk // 4, 1).astype(np.int16)
        px = np.clip(blk + g.integers(-12, 13, blk.shape), 0, 255).astype(np.uint8)
        flat = px.reshape(chunk, -1).astype(np.int16)
        d = flat.copy()
        d[:, 3:] -= flat[:, :-3]
        return zlib.compress((d & 0xff).astype(np.uint8).tobytes(), 1)

    n = across * across
    offsets, counts = [], []
    with open(path, "wb") as fp, ThreadPoolExecutor(usable_cores()) as pool:
        fp.write(b"II" + struct.pack("<HI", 42, 0))
        for b in pool.map(one, range(n)):
            offsets.append(fp.tell())
            counts.append(len(b))
            fp.write(b)
        geo = [1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, 1, 3072, 0, 1, 32632]
        tags = [(256, 4, [size]), (257, 4, [size]), (258, 3, [8, 8, 8]), (259, 3, [8]), (262, 3, [2]), (277, 3, [3]), (284, 3, [1]),
                (317, 3, [2]), (322, 3, [chunk]), (323, 3, [chunk]), (324, 4, offsets), (325, 4, counts), (339, 3, [1, 1, 1]),
                (33550, 12, [0.2, 0.2, 0.0]), (33922, 12, [0, 0, 0, float(E), float(N), 0]), (34735, 3, geo)]
        fmt = {3: "H", 4: "I", 12: "d"}
        entries, blob = [], b""
        blob_at = fp.tell()
        for tag, typ, vals in tags:
            payload = struct.pack("<" + fmt[typ] * len(vals), *vals)
            if len(payload) <= 4:
                value = payload.ljust(4, b"\0")
            else:
                value = struct.pack("<I", blob_at + len(blob))
                blob += payload
            entries.append(struct.pack("<HHI", tag, typ, len(vals)) + value)
        fp.write(blob)
        ifd = fp.tell()
        fp.write(struct.pack("<H", len(entries)) + b"".join(entries) + struct.pack("<I", 0))
        fp.seek(4)
        fp.write(struct.pack("<I", ifd))


def run_tool(path, out):
    stats = {}
    t0 = time.perf_counter()
    tool.main(argparse.Namespace(zoom=TOOL_ZOOM, size=S, tiles=None, resampling="bilinear", raster=path, out=out), stats)
    wall = time.perf_counter() - t0
    return {k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--size", type=int, default=20000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile needs a CUDA device")
    _lib.require_device()
    rec = {"card": card(), "kernel": []}
    for kind in ("3857", "4326", "utm"):
        for resampling in ("nearest", "bilinear"):
            for side in (8, 32):
                rec["kernel"].append(kernel_time(kind, resampling, side, args.launches))
                torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        warm = os.path.join(tmp, "warm.tif")
        write_geotiff(warm, 2048, seed=1)
        run_tool(warm, os.path.join(tmp, "warm"))
        big = os.path.join(tmp, "ortho.tif")
        t0 = time.perf_counter()
        write_geotiff(big, args.size)
        gen = time.perf_counter() - t0
        stats, wall = run_tool(big, os.path.join(tmp, "tiles"))
        rec["tool"] = dict(raster=args.size, file_bytes=os.path.getsize(big), generate_s=round(gen, 1), threads=usable_cores(), wall_s=round(wall, 3),
                           tiles_per_s=round(stats["written"] / wall, 1), **stats)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
