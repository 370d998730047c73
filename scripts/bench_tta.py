"""Cost of test-time augmentation on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_tta.py --out results/h100_tta.json [--steps K --warmup W]

Records, read in the same run:
    card          name, power limit, current and maximum SM clocks (nvidia-smi, read-only query)
    predict       device-resident tiles/s of TilePredictor (graph replay, submit_device / collect with `depth` batches in flight,
                  inputs already in the slots' device buffers, the uint8 bins copied back), batch 32, 512 + 2 x 32 overlap,
                  strict and fast x tta none / flip / d4; CUDA events around K batches after W warm-up batches
    serve         SegmentEngine 512^2 batch-1 request latency (graph replay incl. H2D of the pixels and D2H of the mask, ending in a
                  stream synchronise), strict, tta none / flip / d4: median and p90 of 200 requests after 20 warm-up requests
    head          rsb_head_tta_accumulate alone (CUDA events over 200 launches): the d4 predict pass (B = 32 tiles, one view per
                  launch, accumulating) and the d4 serve pass (B = 1, 8 views, overwriting); bytes it must move (logits of the
                  crop read once per view, int64 sums read and/or written once) against the 3.35 TB/s HBM3 data-sheet figure
"""

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from robosat_b200 import _lib, synth, tta  # noqa: E402
from robosat_b200.predictor import TilePredictor  # noqa: E402
from robosat_b200.serve import SegmentEngine  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def predict_rate(sd, precision, mode, steps, warmup, batch=32, tile=512, overlap=32):
    dev = torch.device("cuda")
    size = tile + 2 * overlap
    pred = TilePredictor(sd, 2, batch, size, overlap=overlap, device=dev, precision=precision, use_graph=True, tta=mode)
    assert pred.graph_error is None, pred.graph_error
    tiles = synth.make_tiles_u8(batch, size, seed=5).to(dev)
    for slot in pred._slots:
        slot["d_in"].copy_(tiles)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    in_flight = 0
    for i in range(warmup + steps):
        if i == warmup:
            while in_flight:
                pred.collect()
                in_flight -= 1
            torch.cuda.synchronize()
            start.record()
        pred.submit_device()
        in_flight += 1
        if in_flight == pred.depth:
            pred.collect()
            in_flight -= 1
    end.record()
    while in_flight:
        pred.collect()
        in_flight -= 1
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / steps
    rec = {"tiles_per_s": batch * 1e3 / ms, "ms_per_batch": ms, "engine_tiles": pred.engine.N,
           "passes": pred.tta.passes if pred.tta else 1, "launches_per_batch": pred.num_launches()}
    del pred
    torch.cuda.empty_cache()
    return rec


def serve_latency(sd, mode, size=512, reps=200, warmup=20):
    eng = SegmentEngine(sd, 2, size, size, device=torch.device("cuda"), use_graph=True, precision="strict", tta=mode)
    assert eng.graph is not None, eng.graph_error
    eng.h_in.copy_(synth.make_tiles_u8(1, size, seed=6))
    for _ in range(warmup):
        eng.run()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        eng.run()  # replay + stream synchronise
        times.append((time.perf_counter() - t0) * 1e3)
    times.sort()
    rec = {"median_ms": statistics.median(times), "p90_ms": times[int(0.9 * len(times))], "engine_tiles": eng.engine.N}
    del eng
    torch.cuda.empty_cache()
    return rec


def head_time(B, views, S, overlap, accumulate, C=2, launches=200):
    dev = torch.device("cuda")
    lib = _lib.load()
    logits = torch.randn((views * B, C, S, S), device=dev)
    OS = S - 2 * overlap
    acc = torch.zeros((B, C, OS, OS), dtype=torch.int64, device=dev)
    ops = (ctypes.c_int32 * views)(*range(views))
    stream = _lib.current_stream_ptr()

    def launch():
        _lib.check(lib.rsb_head_tta_accumulate(logits.data_ptr(), acc.data_ptr(), ops, views, B, C, S, S, overlap, accumulate, stream), "accumulate")

    for _ in range(10):
        launch()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        launch()
    end.record()
    torch.cuda.synchronize()
    us = start.elapsed_time(end) * 1e3 / launches
    logit_bytes = views * B * C * OS * OS * 4
    acc_bytes = B * C * OS * OS * 8 * (2 if accumulate else 1)
    total = logit_bytes + acc_bytes
    return {"B": B, "views": views, "size": S, "overlap": overlap, "accumulate": accumulate, "us_per_launch": us,
            "bytes_per_launch": total, "bytes_per_view": total / views, "tb_per_s": total / (us * 1e-6) / 1e12,
            "frac_of_hbm_datasheet": total / (us * 1e-6) / 1e12 / HBM_TBS}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="JSON file to write the record to")
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    _lib.require_device()
    sd = synth.make_state_dict(2, seed=0)
    rec = {"what": "test-time augmentation cost (scripts/bench_tta.py)", "card": card(), "steps": args.steps, "warmup": args.warmup,
           "predict": {}, "serve": {}, "head": {}}
    for precision in ("strict", "fast"):
        for mode in tta.MODES:
            rec["predict"]["%s/%s" % (precision, mode)] = predict_rate(sd, precision, mode, args.steps, args.warmup)
    for mode in tta.MODES:
        rec["serve"][mode] = serve_latency(sd, mode)
    rec["head"]["predict_d4_pass"] = head_time(32, 1, 576, 32, 1)
    rec["head"]["serve_d4"] = head_time(1, 8, 512, 0, 0)
    p = rec["predict"]
    for precision in ("strict", "fast"):
        d4 = p["%s/d4" % precision]
        none = p["%s/none" % precision]
        d4["cost_vs_none"] = none["tiles_per_s"] / d4["tiles_per_s"]
        d4["head_share"] = rec["head"]["predict_d4_pass"]["us_per_launch"] * d4["passes"] * 1e-3 / d4["ms_per_batch"]
    rec["card_after"] = card()
    line = json.dumps(rec)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
