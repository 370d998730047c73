"""Cost of `rs compare` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_compare.py --out results/h100_compare.json [--tiles 512 --launches 100]

Records, read in the same run:
    card      name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    kernel    rsb_compare_count and rsb_compare_compose alone on a batch of 64 512^2 tiles with 1 and 3 masks (labels given,
              composite written to pinned host memory): CUDA events over `launches` launches after 10 warm-up launches, us per tile
              and GB/s against the bytes each kernel must move
    tool      robosat_b200.compare.compare_device end to end over a seeded directory of `tiles` 512^2 tiles (RGB PNG images, 1-bit
              palette labels and masks as `rs rasterize` / `rs masks` write them, a third of the tiles outside the coverage range)
              with --csv, after one warm-up run on 32 tiles: wall seconds, tiles/s, and the tool's own split into decode / device /
              encode / wait seconds and kernel milliseconds. The tool is expected to be bound by the host PNG codec, not by the kernels.
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
from robosat_b200 import compare as C  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402

S = 512


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def blobs(rng, p):
    """a 1-bit mask of discs covering about a share p of the tile"""
    m = np.zeros((S, S), np.uint8)
    yy, xx = np.mgrid[:S, :S]
    while m.mean() < p:
        cy, cx, r = rng.randint(0, S), rng.randint(0, S), rng.randint(10, 60)
        m[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = 1
    return m


def write_tiles(root, n, masks, rng):
    yy, xx = np.mgrid[:S, :S]
    for i in range(n):
        x, y = 1000 + i // 32, 2000 + i % 32
        rgb = np.stack([(xx + 3 * i) % 256, (yy + 5 * i) % 256, (xx + yy) % 256], -1) + rng.randint(0, 16, size=(S, S, 3))
        for kind, arr, pal in [("images", rgb.astype(np.uint8), None), ("labels", blobs(rng, rng.uniform(0, 0.3)), [0, 0, 0, 250, 0, 0])] + \
                              [("masks%d" % m, blobs(rng, rng.uniform(0, 0.45)), [80, 102, 127, 249, 136, 108]) for m in range(masks)]:
            path = os.path.join(root, kind, "18", str(x), "%d.png" % y)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            im = Image.fromarray(arr, "RGB" if pal is None else "P")
            if pal is not None:
                im.putpalette(pal)
            im.save(path, optimize=pal is not None)


def kernel_times(M, launches, N=64):
    rng = np.random.RandomState(M)
    pitch = C.pitch_of(S * S)
    planes = torch.from_numpy((rng.rand(N, 1 + M, pitch) < 0.3).astype(np.uint8)).cuda()
    masks, labels = planes[:, 1:].contiguous(), planes[:, 0].contiguous()
    images = torch.from_numpy(rng.randint(0, 256, size=(N, S * S * 3)).astype(np.uint8)).cuda()
    pal = torch.from_numpy(rng.randint(0, 1 << 24, size=(N, 1 + M, 256)).astype(np.int32)).cuda()
    out = torch.empty((N, C.out_stride_of((S, S), 1 + M)), dtype=torch.uint8, pin_memory=True)
    counts = torch.empty((N, M, 4), dtype=torch.int64, device="cuda")
    rec = {"masks": M, "batch": N}
    for name, fn in (("count", lambda: C.count_device(masks, labels, S * S, counts)), ("compose", lambda: C.compose_device(images, planes, pal, (S, S), out))):
        for _ in range(10):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        b.synchronize()
        rec[name + "_us_per_tile"] = round(a.elapsed_time(b) * 1000 / launches / N, 3)
    # bytes each kernel must move: count reads the label and every mask once (the label's re-reads per mask hit L2); compose
    # writes the composite, to pinned host memory over PCIe
    rec["count_GBps"] = round((1 + M) * S * S / (rec["count_us_per_tile"] * 1e3), 1)
    rec["compose_GBps_written"] = round(S * S * (2 + M) * 3 / (rec["compose_us_per_tile"] * 1e3), 1)
    return rec


def run(root, M, out, tiles=None):
    st = {}
    t0 = time.perf_counter()
    C.compare_device(os.path.join(root, "images"), os.path.join(root, "labels"), [os.path.join(root, "masks%d" % m) for m in range(M)], out,
                     0.05, 0.4, csv=out + ".csv", stats=st)
    return time.perf_counter() - t0, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_compare.json"))
    ap.add_argument("--tiles", type=int, default=512)
    ap.add_argument("--launches", type=int, default=100)
    args = ap.parse_args()
    _lib.require_device()
    rec = {"card": card(), "threads": usable_cores(), "kernel": [kernel_times(M, args.launches) for M in (1, 3)], "tool": []}
    rng = np.random.RandomState(0)
    with tempfile.TemporaryDirectory() as tmp:
        warm = os.path.join(tmp, "warm")
        write_tiles(warm, 32, 3, rng)
        data = os.path.join(tmp, "data")
        write_tiles(data, args.tiles, 3, rng)
        for M in (1, 3):
            run(warm, M, os.path.join(tmp, "warm_out%d" % M))
            seconds, st = run(data, M, os.path.join(tmp, "out%d" % M))
            rec["tool"].append({"masks": M, "tiles": args.tiles, "seconds": round(seconds, 3), "tiles_per_s": round(args.tiles / seconds, 1),
                                "kept": st["kept"], "decode_s": round(st["decode_s"], 3), "device_s": round(st["device_s"], 3),
                                "encode_s": round(st["encode_s"], 3), "wait_s": round(st["wait_s"], 3), "kernel_ms": round(st["kernel_ms"], 3)})
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
