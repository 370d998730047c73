"""Cost of `rs dedupe` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_dedupe.py --out results/h100_dedupe.json [--repeats 5]

Seeded synthetic workloads (tests/dedupe_reference.py, tests/cover_reference.py):
    parking    400 shifted copies of the golden parking features as predictions; OSM is a jittered, shifted copy with 30 % of
               the features removed
    buildings  20 000 star-shaped polygons of 8-20 vertices at zoom 19 against a shifted copy with 30 % removed plus
               3 000 unrelated buildings
    landuse    3 separate noisy rings of 2 x 10^4, 5 x 10^4 and 10^5 vertices as OSM, each under 700 building-sized predictions, plus 30
               squares on each ring's boundary
    shared_border  a 10^5-gon disc split into two OSM polygons of ~7 x 10^4 vertices along a zigzag border of 2 x 10^4 points,
               with 500 squares on the border, so each prediction has both huge polygons in S(P)

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    per workload: rsb_dedupe_intersects and rsb_dedupe_areas, CUDA events around each launch inside `decide`, summed
              over its batches; mean of `repeats` runs after one warm-up
    device    `decide` on parsed collections (candidate pairs on the host, both kernels, copies back), wall clock, mean of `repeats`
    tool      robosat_b200.tools.dedupe.main on the buildings workload (GeoJSON in a temporary directory), after one warm-up run,
              split into parse + project, device and write
The reference (shapely, rtree, pyproj) is not installed here and was not timed.
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
import dedupe_reference as ref  # noqa: E402
import rasterize_reference as rr  # noqa: E402
from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import dedupe as DD  # noqa: E402
from robosat_b200.cover import tile  # noqa: E402
from robosat_b200.tools import dedupe as tool  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def parking():
    golden = rr.load_golden()["features"]["features"]
    predicted = []
    for k in range(200):
        du, dv = 0.004 * (k % 20), 0.003 * (k // 20)
        for f in golden:
            rings = [[[p[0] + du, p[1] + dv] for p in r] for r in f["geometry"]["coordinates"]]
            predicted.append({"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": rings}})
    return predicted, ref.perturbed(predicted, seed=51, jitter=2e-6, shift=2e-5, drop=0.3)


def buildings():
    predicted = cr.buildings(20_000, 19, seed=52, span=256)
    return predicted, ref.perturbed(predicted, seed=53, jitter=0.0, shift=3e-5, drop=0.3) + cr.buildings(3000, 19, seed=54, span=256)


def landuse():
    osm = [cr.landuse([k], 18, seed=55 + i, origin=(70000 + 2000 * i, 104000))[0] for i, k in enumerate((20_000, 50_000, 100_000))]
    predicted = []
    for i, f in enumerate(osm):
        cx, cy = tile(*np.concatenate(ref.rings_ll(f)).mean(0), 19)
        predicted += cr.buildings(700, 19, seed=56 + i, origin=(cx - 300, cy - 300), span=600)
        predicted += ref.boundary_squares(f, 30, 2e-4, seed=60 + i)
    return predicted, osm


def shared_border():
    a, b, _, border = ref.split_disc(100_000, 20_000)
    idx = np.random.default_rng(61).choice(len(border), 500, replace=False)
    return ref.squares_at(border[idx], 3e-4), [a, b]


def device_run(predicted, osm, repeats):
    ps, _ = DD.parse(predicted, False)
    qs, _ = DD.parse(osm, True)
    passthrough = [False] * len(predicted)
    DD.decide(ps, qs, 0.5, passthrough)
    runs = []
    for _ in range(repeats):
        stats = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        keep, _ = DD.decide(ps, qs, 0.5, passthrough, stats=stats)
        runs.append((time.perf_counter() - t0, stats))
    s = runs[-1][1]
    return {"predicted": len(ps), "osm": len(qs), "predicted_vertices": int(len(ps.xy.vertices)), "osm_vertices": int(len(qs.xy.vertices)),
            "candidate_pairs": s["pairs"], "intersecting_predictions": s["intersecting"], "edge_items": s["items"], "batches": s["batches"],
            "kept": int(keep.sum()), "intersects_ms": round(float(np.mean([r[1]["intersects_ms"] for r in runs])), 4),
            "areas_ms": round(float(np.mean([r[1]["areas_ms"] for r in runs])), 4),
            "decide_ms": round(1e3 * float(np.mean([r[0] for r in runs])), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    _lib.require_device()
    rec = {"card": card()}
    loads = {"parking": parking(), "buildings": buildings(), "landuse": landuse(), "shared_border": shared_border()}
    rec["kernel"] = {name: device_run(p, o, args.repeats) for name, (p, o) in loads.items()}

    with tempfile.TemporaryDirectory() as tmp:
        p, o = loads["buildings"]
        paths = [os.path.join(tmp, n) for n in ("osm.geojson", "predicted.geojson", "out.geojson")]
        for path, feats in zip(paths, (o, p)):
            with open(path, "w") as f:
                json.dump({"type": "FeatureCollection", "features": feats}, f)
        ns = argparse.Namespace(osm=paths[0], predicted=paths[1], out=paths[2], threshold=0.5)
        tool.main(ns)
        stats = {}
        t0 = time.perf_counter()
        tool.main(ns, stats=stats)
        secs = time.perf_counter() - t0
    rec["tool"] = {"workload": "buildings", "seconds": round(secs, 3), "split": {k: (round(v, 4) if isinstance(v, float) else v) for k, v in stats.items()}}
    rec["reference"] = "not measured: shapely, rtree and pyproj are not installed"
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
