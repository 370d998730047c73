"""Cost of `rs features --type building` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_features_building.py --out results/h100_features_building.json [--tiles 1024 --launches 200]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    the device chain of one batch of 512^2 labels: rsb_morph_binary (the 5 x 5 opening) + rsb_building_clean (label the
              foreground 8-connected, drop specks, label the background 4-connected, fill small holes), at batch 64 and 256, on
              building-like masks (rotated rectangles with courtyards and speckle) and on noise masks (each pixel a building with
              probability 0.5, the worst case for the component count): CUDA events over `launches` launches after 20 warm-up
              launches, us per tile
    tool      end-to-end tiles/s of robosat_b200.tools.features.main --type building over a seeded directory of `tiles` 512^2
              P-mode PNG masks of three classes (about half without buildings), wall clock, after one warm-up run on 64 tiles
    cpu       the CPU path over the same directory with the same thread count: PNG decode, cv2 opening, connectedComponentsWithStats
              for the speck drop and the hole fill, and the same contour / simplify / validity code, all in the pool, features
              gathered in tile order; it must give the tool's features
"""

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import features as F  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402
from robosat_b200.tiles import tiles_from_slippy_map  # noqa: E402
from robosat_b200.tools import features as tool  # noqa: E402

BUILDING = 2
H = F.BuildingHandler


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def _rect(m, rng, value, lo, hi):
    import cv2

    S = m.shape[0]
    cy, cx = rng.uniform(0, S, size=2)
    (a, b), t = rng.uniform(lo, hi, size=2), rng.uniform(0, math.pi)
    c, s = math.cos(t), math.sin(t)
    pts = [(cx + u * c - v * s, cy + u * s + v * c) for u, v in ((-a / 2, -b / 2), (a / 2, -b / 2), (a / 2, b / 2), (-a / 2, b / 2))]
    cv2.fillPoly(m, [np.round(np.array(pts) * 4).astype(np.int32)], int(value), shift=2)


def building_mask(rng, S=512):
    m = np.zeros((S, S), np.uint8)
    for _ in range(rng.randint(1, 4)):
        _rect(m, rng, 1, 10, 150)  # parking
    for _ in range(rng.randint(4, 30)):
        _rect(m, rng, BUILDING, 20, 120)
    for _ in range(rng.randint(0, 10)):
        _rect(m, rng, 0, 3, 20)  # courtyards and cuts
    noise = rng.rand(S, S)
    m[noise < 0.005] = BUILDING
    m[noise > 0.997] = 0
    return m


def noise_mask(rng, S=512):
    return np.where(rng.rand(S, S) < 0.5, BUILDING, 0).astype(np.uint8)


def kernel_time(kind, batch, launches, S=512):
    rng = np.random.RandomState(batch)
    make = building_mask if kind == "buildings" else noise_mask
    labels = torch.from_numpy(np.stack([make(rng, S) for _ in range(batch)])).cuda()
    ops = (_lib.MorphOp * 2)(*[F._op_struct(o) for o in F.building_open(H.kernel_size_denoise)])
    opened = torch.empty_like(labels)
    out = torch.empty_like(labels)
    counts = torch.empty(batch, dtype=torch.int32, device=labels.device)
    work = torch.empty((batch, S, S), dtype=torch.int32, device=labels.device)
    stats = torch.empty_like(work)
    lib, stream = _lib.load(), _lib.current_stream_ptr()

    def launch():
        _lib.check(lib.rsb_morph_binary(labels.data_ptr(), S * S, batch, S, S, BUILDING, ops, 2, opened.data_ptr(), counts.data_ptr(), stream), "morph")
        _lib.check(lib.rsb_building_clean(opened.data_ptr(), S * S, batch, S, S, H.min_area, H.min_hole_area, work.data_ptr(), stats.data_ptr(),
                                          out.data_ptr(), counts.data_ptr(), stream), "building_clean")

    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        launch()
    end.record()
    end.synchronize()
    return {"masks": kind, "batch": batch, "launches": launches, "us_per_tile": round(start.elapsed_time(end) * 1e3 / launches / batch, 4)}


def write_masks(root, n, seed=7):
    rng = np.random.RandomState(seed)
    palette = [0, 0, 0, 255, 128, 0, 60, 60, 60]
    for i in range(n):
        x, y = 70000 + i // 32, 104000 + i % 32
        m = building_mask(rng) if rng.rand() < 0.5 else np.where(rng.rand(512, 512) < 0.3, 1, 0).astype(np.uint8)
        os.makedirs(os.path.join(root, "18", str(x)), exist_ok=True)
        im = Image.fromarray(m, mode="P")
        im.putpalette(palette)
        im.save(os.path.join(root, "18", str(x), "%d.png" % y), optimize=True)


def run_tool(masks, dataset, out):
    t0 = time.perf_counter()
    tool.main(argparse.Namespace(masks=masks, type="building", dataset=dataset, out=out))
    return time.perf_counter() - t0


def cpu_clean(mask):
    """the building rule's steps 1-4 with OpenCV"""
    import cv2

    e = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (H.kernel_size_denoise, H.kernel_size_denoise))
    o = cv2.morphologyEx(mask, cv2.MORPH_OPEN, e)
    n, lab, st, _ = cv2.connectedComponentsWithStats(o, connectivity=8)
    keep = st[:, cv2.CC_STAT_AREA] >= H.min_area
    keep[0] = False
    d = keep[lab].astype(np.uint8)
    n, lab, st, _ = cv2.connectedComponentsWithStats(1 - d, connectivity=4)
    border = np.zeros(n, bool)
    border[np.concatenate([lab[0], lab[-1], lab[:, 0], lab[:, -1]])] = True
    hole = ~border & (st[:, cv2.CC_STAT_AREA] < H.min_hole_area)
    hole[0] = False  # label 0 is d's foreground
    return (d | hole[lab]).astype(np.uint8)


def cpu_path(masks, workers):
    tiles = sorted(tiles_from_slippy_map(masks), key=lambda tp: (tp[0].z, tp[0].x, tp[0].y))

    def one(tp):
        mask = (np.array(Image.open(tp[1]).convert("P"), dtype=np.uint8) == BUILDING).astype(np.uint8)
        return F.polygons_from_filled(tp[0], cpu_clean(mask), H.simplify_epsilon)

    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=workers) as pool:
        feats = [f for fs, _ in pool.map(one, tiles) for f in fs]
    return time.perf_counter() - t0, feats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--tiles", type=int, default=1024)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_features_building needs a CUDA device")
    _lib.require_device()
    rec = {"card": card(), "kernel": [kernel_time(k, b, args.launches) for k in ("buildings", "noise") for b in (64, 256)]}
    workers = min(32, usable_cores())
    with tempfile.TemporaryDirectory() as tmp:
        dataset = os.path.join(tmp, "dataset.toml")
        with open(dataset, "w") as fp:
            fp.write("[common]\nclasses = ['background', 'parking', 'building']\ncolors = ['denim', 'orange', 'dark']\n")
        warm, masks = os.path.join(tmp, "warm"), os.path.join(tmp, "masks")
        write_masks(warm, 64, seed=1)
        write_masks(masks, args.tiles)
        run_tool(warm, dataset, os.path.join(tmp, "warm.geojson"))
        t_gpu = run_tool(masks, dataset, os.path.join(tmp, "out.geojson"))
        with open(os.path.join(tmp, "out.geojson")) as fp:
            gpu_feats = json.load(fp)["features"]
        t_cpu, cpu_feats = cpu_path(masks, workers)
    rec["tool"] = {"tiles": args.tiles, "threads": workers, "seconds": round(t_gpu, 3), "tiles_per_s": round(args.tiles / t_gpu, 1),
                   "features": len(gpu_feats)}
    rec["cpu"] = {"tiles": args.tiles, "threads": workers, "seconds": round(t_cpu, 3), "tiles_per_s": round(args.tiles / t_cpu, 1),
                  "features": len(cpu_feats)}
    assert gpu_feats == json.loads(json.dumps(cpu_feats)), "the tool and the CPU path disagree"
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
