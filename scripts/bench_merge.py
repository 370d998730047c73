"""Cost of `rs merge` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_merge.py --out results/h100_merge.json [--repeats 3]

Seeded synthetic workloads (tests/merge_reference.py, tests/cover_reference.py, the golden parking features):
    parking    100 shifted copies of the golden parking features, d = 2
    fragments  300 seeded convex lots straddling 2 x 2 or 3 x 3 z18 tiles, cut at the tile borders by `rs rasterize` and
               `rs features --type parking`, d = 1
    buildings  20 000 star-shaped buildings at zoom 19, d = 1
    landuse    3 noisy rings of 10^4, 3 x 10^4 and 10^5 vertices, 3-4 z18 tiles across, d = 2, so the grids hold millions of cells

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    per workload: rsb_dedupe_intersects (on EPSG:3395), rsb_merge_near, rsb_merge_components, rsb_merge_fill and
              rsb_merge_close, CUDA events around each launch inside `merge_device`, summed over batches; mean of `repeats` runs
              after one warm-up
    device    `merge_device` on parsed features (host set-up of pairs and grids, the kernels, the copies back), wall clock, mean of
              `repeats`
    tool      robosat_b200.tools.merge.main per workload (GeoJSON in a temporary directory), one run, split into
              parse, device, tracing and write (the device path was warmed up by the kernel runs)
The reference (shapely / GEOS, rtree, pyproj) is not installed here and was not timed.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import cover_reference as cr  # noqa: E402
import merge_reference as ref  # noqa: E402
import rasterize_reference as rr  # noqa: E402
from robosat_b200 import merge as MG  # noqa: E402
from robosat_b200.tools import merge as tool  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def shifted(features, dlon, dlat):
    def ring(r):
        return [[p[0] + dlon, p[1] + dlat] for p in r]

    return [{"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [ring(r) for r in f["geometry"]["coordinates"]]}}
            for f in features]


def workloads():
    golden = rr.load_golden()["features"]["features"]
    parking = [f for k in range(100) for f in shifted(golden, 0.01 * (k % 10), 0.01 * (k // 10))]
    source, tiles = ref.straddling(300, 1)
    return {
        "parking": (parking, 2),
        "fragments": (ref.fragments(source, tiles), 1),
        "buildings": (cr.buildings(20000, 19, 0), 1),
        "landuse": (cr.landuse([10000, 30000, 100000], 18, 2, sizes=(3, 4)), 2),
    }


KERNELS = ("intersects_ms", "near_ms", "components_ms", "fill_ms", "close_ms")


def run(features, d, repeats):
    shapes, _ = MG.parse(features)
    MG.merge_device(shapes, d)  # warm-up
    rec = {k: 0.0 for k in KERNELS}
    wall = 0.0
    for _ in range(repeats):
        stats = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, comps = MG.merge_device(shapes, d, stats=stats)
        wall += time.perf_counter() - t0
        for k in KERNELS:
            rec[k] += stats.get(k, 0.0) / repeats
    rec = {k: round(v, 4) for k, v in rec.items()}
    rec.update(features=len(shapes), vertices=int(len(shapes.next)), candidate_pairs=stats["pairs"], linked=stats["linked"],
               components=stats["components"], cells=stats.get("cells", 0), batches=stats["batches"], merge_device_ms=round(1e3 * wall / repeats, 3))
    return rec


def run_tool(features, d):
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "in.geojson")
        with open(src, "w") as fp:
            json.dump({"type": "FeatureCollection", "features": features}, fp)
        args = argparse.Namespace(features=src, threshold=d, out=os.path.join(tmp, "out.geojson"))
        stats = {}
        t0 = time.perf_counter()
        tool.main(args, stats)
        total = time.perf_counter() - t0
    keys = ("parse_s", "device_s", "trace_s", "write_s")
    return dict({k: round(stats[k], 4) for k in keys}, total_s=round(total, 4), input=stats["input"], merged=stats["merged"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    rec = {"card": card(), "kernel": {}, "tool": {}}
    for name, (features, d) in workloads().items():
        rec["kernel"][name] = dict(run(features, d, args.repeats), threshold=d)
        rec["tool"][name] = run_tool(features, d)
        print(name, rec["kernel"][name], rec["tool"][name], file=sys.stderr, flush=True)
    rec["note"] = "the reference (shapely / GEOS, rtree, pyproj) is not installed here and was not timed"
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as fp:
            fp.write(line + "\n")


if __name__ == "__main__":
    main()
