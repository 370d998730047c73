"""`rs segment` against the four-tool pipeline it replaces, on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_segment.py --out results/h100_segment.json [--size 20000]

Input: the seeded `size` x `size` RGB GeoTIFF in UTM zone 32 of scripts/bench_tile.py (0.2 m pixels, deflate, predictor 2), zoom 18,
tiles of 512² with a 32-pixel overlap, batches of 32, seeded weights of a two-class model, strict precision. After a warm-up of both
on a small raster, the two are timed alternately, twice each, in this one process:
    fused     robosat_b200.tools.segment.main
    pipeline  tools.tile.main -> tools.predict.main -> tools.masks.main -> tools.mosaic.main --like, through PNG directories in a
              temporary directory
Records: the card's name and power limit, wall seconds of each run, the fused tool's stage split (decode on a host thread; warp,
predict = stitch + network + head + vote, and mosaic warp from CUDA events; encode and write on the writer thread), the stage
that bounds it, and whether the two outputs have equal pixels and equal tags in the same run.
"""

import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from bench_tile import card, write_geotiff  # noqa: E402
from robosat_b200 import synth  # noqa: E402
from robosat_b200.tools import masks, mosaic, predict, segment, tile  # noqa: E402

ZOOM, S, OVERLAP, BATCH = 18, 512, 32, 32
TAGS = (256, 257, 258, 262, 320, 33550, 33922, 34264, 34735, 42113)
STAGES = ("decode_s", "warp_s", "predict_s", "mosaic_s", "encode_s", "write_s")


def fused(d, raster, out):
    stats = {}
    t0 = time.perf_counter()
    segment.main(argparse.Namespace(zoom=ZOOM, size=S, overlap=OVERLAP, batch_size=BATCH, tiles=None, resampling="bilinear", output="masks", tta="none",
                                    nodata=None, model=os.path.join(d, "model.toml"), dataset=os.path.join(d, "dataset.toml"),
                                    checkpoint=os.path.join(d, "ckpt.pth"), raster=raster, out=out), stats)
    return time.perf_counter() - t0, stats


def pipeline(d, raster, out):
    work = os.path.join(d, "pipeline")
    shutil.rmtree(work, ignore_errors=True)
    t = {}
    t0 = time.perf_counter()
    tile.main(argparse.Namespace(zoom=ZOOM, size=S, tiles=None, resampling="bilinear", raster=raster, out=os.path.join(work, "images")))
    t["tile_s"] = time.perf_counter() - t0
    t1 = time.perf_counter()
    predict.main(argparse.Namespace(batch_size=BATCH, checkpoint=os.path.join(d, "ckpt.pth"), overlap=OVERLAP, tile_size=S, workers=0,
                                    tiles=os.path.join(work, "images"), probs=os.path.join(work, "probs"), model=os.path.join(d, "model.toml"),
                                    dataset=os.path.join(d, "dataset.toml"), tta="none"))
    t["predict_s"] = time.perf_counter() - t1
    t1 = time.perf_counter()
    masks.main(argparse.Namespace(masks=os.path.join(work, "masks"), probs=[os.path.join(work, "probs")], weights=None, dataset=None))
    t["masks_s"] = time.perf_counter() - t1
    t1 = time.perf_counter()
    mosaic.main(argparse.Namespace(zoom=ZOOM, like=raster, resampling="nearest", nodata=None, masks=os.path.join(work, "masks"), out=out))
    t["mosaic_s"] = time.perf_counter() - t1
    return time.perf_counter() - t0, {k: round(v, 3) for k, v in t.items()}


def read(path):
    Image.MAX_IMAGE_PIXELS = None  # a 20 000² output is no decompression bomb
    im = Image.open(path)
    return np.array(im), {t: im.tag_v2.get(t) for t in TAGS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--size", type=int, default=20000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_segment: no CUDA device")
    os.environ.update(RSB_GPUS="1", RSB_QUIET="1")
    os.environ.pop("RSB_PRECISION", None)  # strict
    rec = {"card": card(), "zoom": ZOOM, "size": S, "overlap": OVERLAP, "batch": BATCH, "raster": args.size, "precision": "strict"}
    with tempfile.TemporaryDirectory() as d:
        torch.save({"epoch": 1, "state_dict": synth.make_state_dict(2, seed=0), "optimizer": {}}, os.path.join(d, "ckpt.pth"))
        with open(os.path.join(d, "model.toml"), "w") as fp:
            fp.write("[common]\ncuda = true\nbatch_size = 2\nimage_size = 512\ncheckpoint = '%s'\n" % d)
        with open(os.path.join(d, "dataset.toml"), "w") as fp:
            fp.write("[common]\ndataset = '%s'\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n" % d)
        small, big = os.path.join(d, "small.tif"), os.path.join(d, "ortho.tif")
        write_geotiff(small, 2048, seed=1)
        write_geotiff(big, args.size, seed=0)
        fused(d, small, os.path.join(d, "warm_f.tif"))
        pipeline(d, small, os.path.join(d, "warm_p.tif"))
        runs = []
        for i in range(2):
            wall, stats = fused(d, big, os.path.join(d, "fused.tif"))
            runs.append({"tool": "segment", "wall_s": round(wall, 3), "stats": {k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}})
            print("fused %d: %.2f s" % (i, wall), file=sys.stderr)
            wall, split = pipeline(d, big, os.path.join(d, "pipeline.tif"))
            runs.append({"tool": "pipeline", "wall_s": round(wall, 3), "split": split})
            print("pipeline %d: %.2f s" % (i, wall), file=sys.stderr)
        got, tags_g = read(os.path.join(d, "fused.tif"))
        want, tags_w = read(os.path.join(d, "pipeline.tif"))
        rec["equal_pixels"] = bool(got.shape == want.shape and np.array_equal(got, want))
        rec["differing_pixels"] = int((got != want).sum()) if got.shape == want.shape else None
        rec["equal_tags"] = tags_g == tags_w
    rec["runs"] = runs
    best = min((r for r in runs if r["tool"] == "segment"), key=lambda r: r["wall_s"])
    rec["segment_wall_s"] = best["wall_s"]
    rec["pipeline_wall_s"] = min(r["wall_s"] for r in runs if r["tool"] == "pipeline")
    rec["stage_split_s"] = {k: best["stats"][k] for k in STAGES}
    rec["bound_by"] = max(STAGES, key=lambda k: best["stats"][k])
    rec["tiles_per_s"] = round(best["stats"]["existing"] / best["wall_s"], 1)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
