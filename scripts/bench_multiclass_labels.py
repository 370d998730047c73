"""Cost of the multi-class label tools on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_multiclass_labels.py --out results/h100_multiclass_labels.json [--launches 200 --tool-block 16]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    counts    rsb_compare_class_counts against rsb_compare_count on the same batch of 64 tiles at 512², M = 1 and 4 masks,
              C = 3 and 32 classes: CUDA events over `launches` launches after 20 warm-up launches, us per launch and bytes read
              (label + masks) over kernel time. Two seeded plane sets: "label-like" (rectangles of classes on background, the
              masks the label with rectangles added and removed) and "noise" (every pixel a uniform class, one run per pixel).
    rasterize robosat_b200.tools.rasterize.main --class building on the buildings workload of scripts/bench_rasterize.py over a
              `tool-block` x `tool-block` block of z18 tiles at 512² (GeoJSON and CSV in a temporary directory), wall clock after
              one warm-up run, in tiles/s: into an empty directory, and again into the full directory (every tile merged with its
              existing label), with the host share of each step including the time spent reading the existing labels.
"""

import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench_rasterize as BR  # noqa: E402
from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import compare as C  # noqa: E402
from robosat_b200.tools import rasterize as tool  # noqa: E402

N = 64
SIZE = 512


def label_like(rng, n, planes, classes):
    """uint8 [n, planes, SIZE * SIZE]: plane 0 about 40 rectangles of classes 1..C-1 on background; the others copies of it
    with 8 rectangles painted over (a class or background)"""
    out = np.zeros((n, planes, SIZE, SIZE), np.uint8)
    for i in range(n):
        base = np.zeros((SIZE, SIZE), np.uint8)
        for _ in range(40):
            y, x = rng.randint(0, SIZE, 2)
            h, w = rng.randint(4, 80, 2)
            base[y:y + h, x:x + w] = rng.randint(1, classes)
        for p in range(planes):
            out[i, p] = base
            if p:
                for _ in range(8):
                    y, x = rng.randint(0, SIZE, 2)
                    h, w = rng.randint(4, 60, 2)
                    out[i, p, y:y + h, x:x + w] = rng.randint(0, classes)
    return out.reshape(n, planes, -1)


def noise(rng, n, planes, classes):
    return rng.randint(0, classes, size=(n, planes, SIZE * SIZE)).astype(np.uint8)


def time_launches(fn, launches):
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / launches


def count_run(planes, M, classes, launches):
    hw = SIZE * SIZE
    d = torch.from_numpy(planes).cuda()
    masks, labels = d[:, 1:].contiguous(), d[:, 0].contiguous()
    counts = torch.empty((N, M, 4), dtype=torch.int64, device="cuda")
    hists = tuple(torch.empty(s, dtype=torch.int64, device="cuda") for s in ((N, classes), (N, M, classes), (N, M, classes), (N, 1 + M)))
    bytes_read = N * (1 + M) * hw
    rec = {"M": M, "C": classes, "tiles": N, "launches": launches, "bytes_read": bytes_read}
    for name, fn in (("compare_count", lambda: C.count_device(masks, labels, hw, counts)),
                     ("compare_class_counts", lambda: C.class_counts_device(masks, labels, hw, classes, hists))):
        ms = time_launches(fn, launches)
        rec[name] = {"us_per_launch": round(ms * 1e3, 2), "GB_per_s": round(bytes_read / (ms * 1e-3) / 1e9, 1)}
    rec["class_over_count"] = round(rec["compare_class_counts"]["us_per_launch"] / rec["compare_count"]["us_per_launch"], 2)
    return rec


def run_tool(features, csv, dataset, out):
    stats = {}
    t0 = time.perf_counter()
    tool.main(argparse.Namespace(features=features, tiles=csv, out=out, dataset=dataset, zoom=18, size=SIZE, class_name="building"), stats=stats)
    return time.perf_counter() - t0, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--tool-block", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_multiclass_labels needs a CUDA device")
    _lib.require_device()
    rec = {"card": BR.card(), "size": SIZE, "counts": {}}
    rng = np.random.RandomState(0)
    for kind, make in (("label-like", label_like), ("noise", noise)):
        runs = []
        for classes in (3, 32):
            planes = make(rng, N, 5, classes)
            runs += [count_run(np.ascontiguousarray(planes[:, :1 + M]), M, classes, args.launches) for M in (1, 4)]
        rec["counts"][kind] = runs
    tiles = BR.block_tiles(args.tool_block)
    polys = BR.buildings(args.tool_block, seed=2)
    with tempfile.TemporaryDirectory() as tmp:
        features, csv, dataset = BR.write_inputs(tmp, polys, tiles)
        with open(dataset, "w") as fp:
            fp.write("[common]\nclasses = ['background', 'parking', 'building']\ncolors = ['denim', 'orange', 'dark']\n")
        run_tool(features, csv, dataset, os.path.join(tmp, "warm"))
        out = os.path.join(tmp, "out")
        rec["rasterize"] = {"workload": "buildings", "tiles": len(tiles), "polygons": len(polys)}
        for case in ("empty_directory", "full_directory"):
            dt, stats = run_tool(features, csv, dataset, out)
            rec["rasterize"][case] = {"seconds": round(dt, 3), "tiles_per_s": round(len(tiles) / dt, 1),
                                      "host_share_s": {k: round(v, 3) for k, v in stats.items()}}
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
