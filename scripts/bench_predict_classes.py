"""Cost of `rs predict` / `rs masks --dataset` for models of more than two classes on one GPU: prints ONE JSON line and writes the
same record to --out.

    python scripts/bench_predict_classes.py --out results/h100_predict_classes.json [--tiles 512]

Records, read in the same run:
    card          name, power limit, current and maximum SM clocks (nvidia-smi, read-only query), before and after
    head          the predict head alone (CUDA events over 200 launches after 10), B = 32, 576^2 logits, overlap 32: C = 2 through
                  rsb_head_quantize (the binary kernel), C = 3 and 6 through rsb_head_quantize_classes; bytes it must move (the
                  cropped logits read once, the bins written once) against the 3.35 TB/s HBM3 data-sheet figure
    predictor     TilePredictor device-resident tiles/s (graph replay, `depth` batches in flight, bins copied back), batch 32,
                  512 + 2 x 32 overlap, strict, C = 2 against C = 6
    rs_predict    run_shard (the `rs predict` loop, device stitch, library PNG encoder) over --tiles seeded 512^2 PNG tiles at z18,
                  C = 6, after one warm-up run over the same tiles; its stage stats (wall_s, gpu_wait_s, png_cpu_s, ...)
    rs_masks      `rs masks --dataset` (K = 2 roots of C = 6 class directories from the two predict runs, weighted) wall time
"""

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from robosat_b200 import _lib, synth  # noqa: E402
from robosat_b200.predictor import TilePredictor  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet
CLASSES6 = ["background", "parking", "building", "road", "water", "trees"]
COLORS6 = ["denim", "orange", "red", "dark", "blue", "green"]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.CalledProcessError, ValueError) as exc:
        return {"name": torch.cuda.get_device_name(), "error": str(exc)}


def head_time(C, B=32, S=576, overlap=32, launches=200):
    dev = torch.device("cuda")
    lib = _lib.load()
    logits = torch.randn((B, C, S, S), device=dev) * 4
    OS = S - 2 * overlap
    planes = 1 if C == 2 else C
    quant = torch.empty((B, planes, OS, OS), dtype=torch.uint8, device=dev)
    stream = _lib.current_stream_ptr()

    def launch():
        if C == 2:
            _lib.check(lib.rsb_head_quantize(logits.data_ptr(), quant.data_ptr(), None, B, S, S, overlap, stream), "head_quantize")
        else:
            _lib.check(lib.rsb_head_quantize_classes(logits.data_ptr(), quant.data_ptr(), None, B, C, S, S, overlap, stream), "head_quantize_classes")

    for _ in range(10):
        launch()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        launch()
    end.record()
    torch.cuda.synchronize()
    us = start.elapsed_time(end) * 1e3 / launches
    total = B * C * OS * OS * 4 + B * planes * OS * OS
    return {"kernel": "rsb_head_quantize" if C == 2 else "rsb_head_quantize_classes", "C": C, "B": B, "size": S, "overlap": overlap,
            "us_per_launch": us, "bytes_per_launch": total, "tb_per_s": total / (us * 1e-6) / 1e12,
            "frac_of_hbm_datasheet": total / (us * 1e-6) / 1e12 / HBM_TBS, "uncropped_logit_bytes": B * C * S * S * 4}


def predictor_rate(C, steps, warmup, batch=32, tile=512, overlap=32):
    dev = torch.device("cuda")
    size = tile + 2 * overlap
    pred = TilePredictor(synth.make_state_dict(C, seed=0), C, batch, size, overlap=overlap, device=dev, precision="strict", use_graph=True)
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
    rec = {"C": C, "tiles_per_s": batch * 1e3 / ms, "ms_per_batch": ms, "d2h_bytes_per_batch": pred.d2h_bytes}
    del pred
    torch.cuda.empty_cache()
    return rec


def tools(work, ntiles, batch=32):
    from robosat_b200.tools import masks
    from robosat_b200.tools.predict import run_shard

    tiles_dir = os.path.join(work, "tiles")
    nx = 16
    written = synth.write_slippy_tiles(tiles_dir, 18, range(70000, 70000 + nx), range(100000, 100000 + (ntiles + nx - 1) // nx), size=512)
    dataset = os.path.join(work, "dataset.toml")
    with open(dataset, "w") as f:
        f.write("[common]\ndataset = '%s'\nclasses = %s\ncolors = %s\n" % (work, json.dumps(CLASSES6), json.dumps(COLORS6)))
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = []
    for seed, name in ((1, "probs_warm"), (0, "probs")):
        args = argparse.Namespace(batch_size=batch, overlap=32, tile_size=512, workers=0, tiles=tiles_dir, probs=os.path.join(work, name),
                                  dataset=dataset)
        st = run_shard(0, 1, args, dev, synth.make_state_dict(6, seed=seed), 6, stats={})
        runs.append({k: v for k, v in st.items() if isinstance(v, (int, float))})
    rec = {"tiles": written, "warm_up_run": runs[0], "timed_run": runs[1], "tiles_per_s": written / runs[1]["wall_s"]}
    out = os.path.join(work, "masks")
    t0 = time.perf_counter()
    masks.main(argparse.Namespace(masks=out, probs=[os.path.join(work, "probs_warm"), os.path.join(work, "probs")], weights=[0.4, 0.6],
                                  dataset=dataset))
    wall = time.perf_counter() - t0
    return rec, {"K": 2, "C": 6, "tiles": written, "wall_s": wall, "tiles_per_s": written / wall}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="JSON file to write the record to")
    ap.add_argument("--tiles", type=int, default=512)
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    _lib.require_device()
    os.environ.setdefault("RSB_QUIET", "1")
    rec = {"what": "rs predict / rs masks for C > 2 classes (scripts/bench_predict_classes.py)", "card": card(), "steps": args.steps,
           "warmup": args.warmup}
    rec["head"] = {"C%d" % C: head_time(C) for C in (2, 3, 6)}
    rec["predictor"] = {"C%d" % C: predictor_rate(C, args.steps, args.warmup) for C in (2, 6)}
    work = tempfile.mkdtemp(prefix="rsb_predict_classes_")
    try:
        rec["rs_predict"], rec["rs_masks"] = tools(work, args.tiles)
    finally:
        shutil.rmtree(work, ignore_errors=True)
    rec["card_after"] = card()
    line = json.dumps(rec)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
