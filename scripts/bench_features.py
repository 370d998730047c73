"""Cost of `rs features --type parking` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_features.py --out results/h100_features.json [--tiles 1024 --launches 200]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    rsb_morph_binary alone, the parking chain (erode, dilate, dilate, erode with the 20 x 20 ellipse) on 512^2 labels, at
              batch 64 and 256: CUDA events over `launches` launches after 20 warm-up launches; us per tile, and GB/s against the
              512 KB per tile the kernel must move (256 KB of labels in, 256 KB of mask out)
    tool      end-to-end tiles/s of robosat_b200.tools.features.main over a seeded directory of `tiles` 512^2 P-mode PNG masks
              (about half empty, the rest fields of discs and rectangles), wall clock, after one warm-up run on 64 tiles
    cpu       the reference-equivalent CPU path over the same directory with the same thread count: PNG decode, cv2 open + close
              and the same contour / simplify / validity code, all in the pool, features gathered in tile order
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

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import features as F  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402
from robosat_b200.tiles import tiles_from_slippy_map  # noqa: E402
from robosat_b200.tools import features as tool  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def blob_mask(rng, S=512):
    m = np.zeros((S, S), np.uint8)
    yy, xx = np.mgrid[:S, :S]
    for _ in range(rng.randint(2, 12)):
        cy, cx = rng.randint(0, S, size=2)
        if rng.rand() < 0.5:
            r = rng.randint(10, 60)
            m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 1
        else:
            m[cy:cy + rng.randint(10, 120), cx:cx + rng.randint(10, 120)] = 1
    m[rng.rand(S, S) < 0.002] = 1  # specks the opening removes
    return m


def kernel_time(batch, launches, S=512):
    rng = np.random.RandomState(batch)
    labels = torch.from_numpy(np.stack([blob_mask(rng, S) for _ in range(batch)])).cuda()
    ops = (_lib.MorphOp * 4)(*[F._op_struct(o) for o in F.parking_chain()])
    out = torch.empty_like(labels)
    counts = torch.empty(batch, dtype=torch.int32, device=labels.device)
    lib, stream = _lib.load(), _lib.current_stream_ptr()

    def launch():
        _lib.check(lib.rsb_morph_binary(labels.data_ptr(), S * S, batch, S, S, 1, ops, 4, out.data_ptr(), counts.data_ptr(), stream), "morph")

    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        launch()
    end.record()
    end.synchronize()
    us_tile = start.elapsed_time(end) * 1e3 / launches / batch
    return {"batch": batch, "launches": launches, "us_per_tile": round(us_tile, 4), "GBps": round(2 * S * S / us_tile / 1e3, 1)}


def write_masks(root, n, seed=7):
    rng = np.random.RandomState(seed)
    for i in range(n):
        x, y = 70000 + i // 32, 104000 + i % 32
        m = blob_mask(rng) if rng.rand() < 0.5 else np.zeros((512, 512), np.uint8)
        os.makedirs(os.path.join(root, "18", str(x)), exist_ok=True)
        im = Image.fromarray(m, mode="P")
        im.putpalette([0, 0, 0, 255, 255, 255])
        im.save(os.path.join(root, "18", str(x), "%d.png" % y), optimize=True)


def run_tool(masks, dataset, out):
    t0 = time.perf_counter()
    tool.main(argparse.Namespace(masks=masks, type="parking", dataset=dataset, out=out))
    return time.perf_counter() - t0


def cpu_path(masks, workers):
    import cv2

    e = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (20, 20))
    tiles = sorted(tiles_from_slippy_map(masks), key=lambda tp: (tp[0].z, tp[0].x, tp[0].y))

    def one(tp):
        mask = (np.array(Image.open(tp[1]).convert("P"), dtype=np.uint8) == 1).astype(np.uint8)
        grown = cv2.morphologyEx(cv2.morphologyEx(mask, cv2.MORPH_OPEN, e), cv2.MORPH_CLOSE, e)
        return F.polygons_from_grown(tp[0], grown)

    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=workers) as pool:
        feats = [f for fs, _ in pool.map(one, tiles) for f in fs]
    return time.perf_counter() - t0, len(feats)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--tiles", type=int, default=1024)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_features needs a CUDA device")
    _lib.require_device()
    rec = {"card": card(), "kernel": [kernel_time(b, args.launches) for b in (64, 256)]}
    workers = min(32, usable_cores())
    with tempfile.TemporaryDirectory() as tmp:
        dataset = os.path.join(tmp, "dataset.toml")
        with open(dataset, "w") as fp:
            fp.write("[common]\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n")
        warm, masks = os.path.join(tmp, "warm"), os.path.join(tmp, "masks")
        write_masks(warm, 64, seed=1)
        write_masks(masks, args.tiles)
        run_tool(warm, dataset, os.path.join(tmp, "warm.geojson"))
        t_gpu = run_tool(masks, dataset, os.path.join(tmp, "out.geojson"))
        with open(os.path.join(tmp, "out.geojson")) as fp:
            n_gpu = len(json.load(fp)["features"])
        t_cpu, n_cpu = cpu_path(masks, workers)
    rec["tool"] = {"tiles": args.tiles, "threads": workers, "seconds": round(t_gpu, 3), "tiles_per_s": round(args.tiles / t_gpu, 1), "features": n_gpu}
    rec["cpu"] = {"tiles": args.tiles, "threads": workers, "seconds": round(t_cpu, 3), "tiles_per_s": round(args.tiles / t_cpu, 1), "features": n_cpu}
    assert n_gpu == n_cpu, (n_gpu, n_cpu)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
