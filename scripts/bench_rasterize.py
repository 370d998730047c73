"""Cost of `rs rasterize` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_rasterize.py --out results/h100_rasterize.json [--launches 200 --tool-block 16]

Seeded synthetic workloads on a 64 x 64 block of z18 tiles at 512²:
    buildings  about 150 polygons of 8-20 vertices per tile (614 400 polygons)
    landuse    4 rings of 100 000 vertices, each covering most of the block

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    rsb_rasterize_polygons alone per workload, at batch 64 and 1024 tiles: CUDA events over `launches` launches after 20
              warm-up launches; us per tile. The polygons are uploaded and binned once, outside the timed window.
    tool      robosat_b200.tools.rasterize.main end to end on the buildings workload over a `tool-block` x `tool-block` sub-block
              (GeoJSON and CSV written to a temporary directory), wall clock after one warm-up run, in tiles/s, with the host share:
              parse + project + bin, device + D2H, merge with existing files, PNG
    cpu       rasterio.features.rasterize on the same tiles when rasterio imports; otherwise "not measured"
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

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import rasterize as RZ  # noqa: E402
from robosat_b200.tiles import Tile  # noqa: E402
from robosat_b200.tools import rasterize as tool  # noqa: E402

BASE = Tile(70000, 104000, 18)
BLOCK = 64
SIZE = 512


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def block_tiles(n):
    return [Tile(BASE.x + dx, BASE.y + dy, 18) for dy in range(n) for dx in range(n)]


def to_merc(u, v):
    """tile units from BASE's top-left corner -> Mercator"""
    left, bottom, right, top = RZ.xy_bounds(BASE)
    side = right - left
    return np.stack([left + u * side, top - v * side], axis=-1)


def buildings(n, per_tile=150, seed=0):
    rng = np.random.RandomState(seed)
    polys = []
    for _ in range(n * n * per_tile):
        k = rng.randint(8, 21)
        cu, cv = rng.uniform(0, n, 2)
        r = rng.uniform(0.005, 0.04)  # 2.5 - 20 px at 512² per tile
        a = np.sort(rng.uniform(0, 2 * np.pi, k))
        rad = r * rng.uniform(0.6, 1.0, k)
        ring = to_merc(cu + rad * np.cos(a), cv + rad * np.sin(a))
        polys.append([np.vstack([ring, ring[:1]])])
    return polys


def landuse(n, count=4, vertices=100000, seed=1):
    rng = np.random.RandomState(seed)
    polys = []
    for i in range(count):
        a = np.linspace(0, 2 * np.pi, vertices, endpoint=False)
        cu, cv = n / 2 + rng.uniform(-2, 2), n / 2 + rng.uniform(-2, 2)
        rad = n * (0.3 + 0.05 * i) * (1 + 0.1 * np.sin((13 + i) * a)) + rng.uniform(-0.01, 0.01, vertices)
        polys.append([to_merc(cu + rad * np.cos(a), cv + rad * np.sin(a))])
    return polys


def kernel_time(polyset, tiles, launches):
    csr = RZ.bin_polygons(tiles, polyset.bboxes)
    out = torch.empty((len(tiles), SIZE, SIZE), dtype=torch.uint8, device="cuda")
    for _ in range(20):
        RZ.rasterize_device(polyset, tiles, SIZE, csr=csr, out=out)
    torch.cuda.synchronize()
    # the launches alone: pre-upload the per-batch arrays once, as the loop would reuse them
    offsets, ids = csr
    d_off = torch.from_numpy(offsets).cuda()
    d_ids = torch.from_numpy(ids if len(ids) else np.zeros(1, np.int32)).cuda()
    d_tr = torch.from_numpy(np.asarray([RZ.tile_transform(t, SIZE) for t in tiles])).cuda()
    counts = torch.empty(len(tiles), dtype=torch.int32, device="cuda")
    lib, stream = _lib.load(), _lib.current_stream_ptr()

    def launch():
        _lib.check(lib.rsb_rasterize_polygons(polyset.d_vertices.data_ptr(), polyset.d_ring_offsets.data_ptr(), polyset.d_poly_rings.data_ptr(),
                                              len(polyset), d_off.data_ptr(), d_ids.data_ptr(), d_tr.data_ptr(), len(tiles), SIZE, out.data_ptr(),
                                              SIZE * SIZE, counts.data_ptr(), stream), "rsb_rasterize_polygons")

    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        launch()
    end.record()
    end.synchronize()
    ms = start.elapsed_time(end) / launches
    fg = int(counts.sum())
    return {"batch": len(tiles), "launches": launches, "pairs": int(offsets[-1]), "us_per_tile": round(ms * 1e3 / len(tiles), 3),
            "ms_per_launch": round(ms, 3), "fg_fraction": round(fg / (len(tiles) * SIZE * SIZE), 4)}


def write_inputs(tmp, polys, tiles):
    def lonlat(ring):
        return np.stack([np.degrees(ring[:, 0] / RZ.R), np.degrees(2 * np.arctan(np.exp(ring[:, 1] / RZ.R)) - np.pi / 2)], axis=1).tolist()

    fc = {"type": "FeatureCollection",
          "features": [{"type": "Feature", "properties": {}, "geometry": {"type": "Polygon", "coordinates": [lonlat(r) for r in p]}} for p in polys]}
    features = os.path.join(tmp, "features.geojson")
    with open(features, "w") as fp:
        json.dump(fc, fp)
    csv = os.path.join(tmp, "tiles.csv")
    with open(csv, "w") as fp:
        fp.write("".join("%d,%d,%d\n" % t for t in tiles))
    dataset = os.path.join(tmp, "dataset.toml")
    with open(dataset, "w") as fp:
        fp.write("[common]\nclasses = ['background', 'building']\ncolors = ['denim', 'orange']\n")
    return features, csv, dataset


def run_tool(features, csv, dataset, out):
    stats = {}
    t0 = time.perf_counter()
    tool.main(argparse.Namespace(features=features, tiles=csv, out=out, dataset=dataset, zoom=18, size=SIZE), stats=stats)
    return time.perf_counter() - t0, stats


def cpu_reference(polys, tiles):
    try:
        from rasterio.features import rasterize
        from rasterio.transform import from_bounds
    except ImportError as exc:
        return {"status": "not measured: rasterio is not installed (%s)" % exc}
    ps = RZ.PolygonSet(polys)
    offsets, ids = RZ.bin_polygons(tiles, ps.bboxes)
    t0 = time.perf_counter()
    for i, t in enumerate(tiles):
        shapes = [({"type": "Polygon", "coordinates": [r.tolist() for r in polys[p]]}, 1) for p in ids[offsets[i]:offsets[i + 1]]]
        if shapes:
            rasterize(shapes, out_shape=(SIZE, SIZE), transform=from_bounds(*RZ.xy_bounds(t), SIZE, SIZE))
    dt = time.perf_counter() - t0
    return {"tiles": len(tiles), "seconds": round(dt, 3), "tiles_per_s": round(len(tiles) / dt, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--tool-block", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rasterize needs a CUDA device")
    _lib.require_device()
    rec = {"card": card(), "size": SIZE, "block": [BLOCK, BLOCK], "kernel": {}}
    tiles = block_tiles(BLOCK)
    work = {"buildings": buildings(BLOCK), "landuse": landuse(BLOCK)}
    for name, polys in work.items():
        ps = RZ.PolygonSet(polys, "cuda")
        rec["kernel"][name] = {"polygons": len(polys), "vertices": len(ps.vertices),
                               "runs": [kernel_time(ps, tiles[:b], args.launches) for b in (64, 1024)]}
    sub = [t for t in tiles if t.x - BASE.x < args.tool_block and t.y - BASE.y < args.tool_block]
    sub_polys = buildings(args.tool_block, seed=2)
    with tempfile.TemporaryDirectory() as tmp:
        features, csv, dataset = write_inputs(tmp, sub_polys, sub)
        run_tool(features, csv, dataset, os.path.join(tmp, "warm"))
        dt, stats = run_tool(features, csv, dataset, os.path.join(tmp, "out"))
    rec["tool"] = {"workload": "buildings", "tiles": len(sub), "polygons": len(sub_polys), "seconds": round(dt, 3),
                   "tiles_per_s": round(len(sub) / dt, 1), "host_share_s": {k: round(v, 3) for k, v in stats.items()}}
    rec["cpu"] = cpu_reference(sub_polys, sub)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
