"""Cost of `rs features --type road` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_features_road.py --out results/h100_features_road.json [--tiles 1024 --launches 50]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    on halo'd 640^2 planes (512^2 tiles plus a 64 px halo) of seeded roads 8-40 px wide, at batch 64 and 256, CUDA events
              over `launches` launches after 5 warm-up launches, us per tile: rsb_road_thin alone, and the whole device chain of
              `road_device` (rsb_building_clean, thinning, degrees, pruning, degrees, rsb_label_components, chain count, the one
              synchronisation for the totals, chain write and the copy back); plus the thinning iteration counts seen
    tool      end-to-end tiles/s of robosat_b200.tools.features.main --type road over a seeded 32 x 32 block of 512^2 P-mode PNG
              masks of three classes (roads crossing tile borders, building speckle), wall clock, after one warm-up run
    cpu       the numpy restatement (tests/road_reference.py: scipy labels, numpy Zhang-Suen, Python graph walks) plus the same host
              line code, on the same thread count over the first `cpu_tiles` tiles: a CPU restatement of this project's rule, not
              the reference (which has no road handler); it must give the tool's features for those tiles
"""

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from robosat_b200 import features as F  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402
from robosat_b200.tiles import Tile  # noqa: E402
from robosat_b200.tools import features as tool  # noqa: E402

ROAD = 2
S = 512
X0, Y0 = 70000, 104000


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def roads(rng, H, W, n):
    """n seeded polylines 8-40 px wide on an H x W canvas of class indices: background 0, building speckle 1, roads 2"""
    import cv2

    m = np.zeros((H, W), np.uint8)
    m[rng.rand(H, W) < 0.01] = 1
    for _ in range(n):
        pts = np.cumsum(rng.uniform(-150, 150, size=(8, 2)), axis=0) + rng.uniform(0, (W, H), size=2)
        cv2.polylines(m, [np.round(pts).astype(np.int32)], False, ROAD, thickness=int(rng.randint(8, 41)))
    return m


def halo_planes(N, seed):
    rng = np.random.RandomState(seed)
    h = F.RoadHandler.halo
    return np.stack([(roads(rng, S + 2 * h, S + 2 * h, 5) == ROAD).astype(np.uint8) for _ in range(N)])


def timed(fn, launches):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / launches


def kernel(batch, launches):
    planes = torch.from_numpy(halo_planes(batch, batch)).cuda()
    H = F.RoadHandler
    _, its = F.road_thin_device(planes)
    its = its.cpu().numpy()
    thin_us = timed(lambda: F.road_thin_device(planes), launches)
    chain_us = timed(lambda: F.road_device(planes, H.min_area, H.min_hole_area, H.min_length), launches)
    return {"batch": batch, "launches": launches, "thin_us_per_tile": round(thin_us / batch, 3), "chain_us_per_tile": round(chain_us / batch, 3),
            "iterations_min": int(its.min()), "iterations_max": int(its.max())}


def write_masks(root, side, seed=7):
    rng = np.random.RandomState(seed)
    big = roads(rng, side * S, side * S, side * side // 2)
    palette = [v for i in range(256) for v in (i, 255 - i, (7 * i) % 256)]
    masks = {}
    for i in range(side):
        d = os.path.join(root, "18", str(X0 + i))
        os.makedirs(d, exist_ok=True)
        for j in range(side):
            m = big[j * S:(j + 1) * S, i * S:(i + 1) * S].copy()
            masks[(X0 + i, Y0 + j)] = m
            im = Image.fromarray(m, mode="P")
            im.putpalette(palette)
            im.save(os.path.join(d, "%d.png" % (Y0 + j)))
    return masks


def run_tool(masks, dataset, out):
    tool.main(argparse.Namespace(masks=masks, type="road", dataset=dataset, out=out))
    with open(out) as fp:
        return json.load(fp)["features"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--tiles", type=int, default=1024)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--cpu_tiles", type=int, default=64)
    args = ap.parse_args()
    import road_reference as rr

    rec = {"card": card(), "kernel": [kernel(b, args.launches) for b in (64, 256)]}
    side = int(round(args.tiles ** 0.5))
    threads = min(32, usable_cores())
    with tempfile.TemporaryDirectory() as tmp:
        ds = os.path.join(tmp, "dataset.toml")
        with open(ds, "w") as fp:
            fp.write("[common]\nclasses = ['background', 'building', 'road']\ncolors = ['denim', 'dark', 'orange']\n")
        masks = write_masks(os.path.join(tmp, "masks"), side)
        run_tool(os.path.join(tmp, "masks"), ds, os.path.join(tmp, "warm.geojson"))
        t = time.perf_counter()
        feats = run_tool(os.path.join(tmp, "masks"), ds, os.path.join(tmp, "out.geojson"))
        sec = time.perf_counter() - t
        rec["tool"] = {"tiles": side * side, "threads": threads, "seconds": round(sec, 3), "tiles_per_s": round(side * side / sec, 1),
                       "features": len(feats)}

        keys = sorted(masks)[:args.cpu_tiles]

        def one(k):
            return rr.cpu_features(Tile(k[0], k[1], 18), rr.halo(masks, k, ROAD), (S, S))

        t = time.perf_counter()
        with ThreadPoolExecutor(max_workers=threads) as pool:
            cpu = [f for fs in pool.map(one, keys) for f in fs]
        sec = time.perf_counter() - t
        rec["cpu"] = {"kind": "numpy restatement of the rule (not the reference)", "tiles": len(keys), "threads": threads, "seconds": round(sec, 3),
                      "tiles_per_s": round(len(keys) / sec, 2), "features": len(cpu)}
        assert feats[:len(cpu)] == json.loads(json.dumps(cpu)), "the tool and the restatement disagree"
    line = json.dumps(rec)
    print(line)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
