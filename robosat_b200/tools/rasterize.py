"""`rs rasterize` (robosat/tools/rasterize.py): label masks from GeoJSON polygons.

Same flags, warnings and output files. The Polygon features are projected and uploaded to the device once, binned to the tiles
of the CSV by their bounding boxes, and burned in batches of tiles by one `rsb_rasterize_polygons` launch each
(`robosat_b200.rasterize`). Every tile of the CSV is written, in CSV order; a tile listed twice is written once. An existing
mask file is merged with np.maximum, as in the reference, and the PNGs of a batch are written by the library's encoder threads
(`tools/predict.py:_save_batch`)."""

import argparse
import json
import os
import sys

import numpy as np
from PIL import Image

from robosat_b200.colors import make_palette
from robosat_b200.config import load_config
from robosat_b200.hostinfo import usable_cores
from robosat_b200.tiles import tiles_from_csv


def add_parser(subparser):
    parser = subparser.add_parser("rasterize", help="rasterize features to label masks", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("features", type=str, help="path to GeoJSON features file")
    parser.add_argument("tiles", type=str, help="path to .csv tiles file")
    parser.add_argument("out", type=str, help="directory to write converted images")
    parser.add_argument("--dataset", type=str, required=True, help="path to dataset configuration file")
    parser.add_argument("--zoom", type=int, required=True, help="zoom level of tiles")
    parser.add_argument("--size", type=int, default=512, help="size of rasterized image tiles in pixels")
    parser.set_defaults(func=main)


def _merge_existing(root, tiles, masks):
    """np.maximum with the masks already on disk (rasterize.py:131-133), in place"""
    for i, t in enumerate(tiles):
        path = os.path.join(root, str(t.z), str(t.x), "{}.png".format(t.y))
        if os.path.exists(path):
            masks[i] = np.maximum(masks[i], np.array(Image.open(path)))


def main(args, batch=64, stats=None):
    """`stats` (a dict), when given, receives the seconds spent per host step and on the device."""
    import time

    import torch

    from robosat_b200 import _lib
    from robosat_b200 import rasterize as RZ
    from robosat_b200.tools.predict import _save_batch

    dataset = load_config(args.dataset)
    classes = dataset["common"]["classes"]
    colors = dataset["common"]["colors"]
    assert len(classes) == len(colors), "classes and colors coincide"
    assert len(colors) == 2, "only binary models supported right now"
    palette = make_palette(colors[0], colors[1])
    tiles = list(tiles_from_csv(args.tiles))
    assert all(tile.z == args.zoom for tile in tiles)  # we can only rasterize all tiles at a single zoom
    if not 1 <= args.size <= _lib.RSB_RASTER_MAX_SIZE:
        sys.exit("Error: --size must be in 1..%d" % _lib.RSB_RASTER_MAX_SIZE)
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    device = torch.device("cuda")
    os.makedirs(args.out, exist_ok=True)
    stats = stats if stats is not None else {}

    t0 = time.perf_counter()
    with open(args.features) as f:
        fc = json.load(f)
    polygons, warnings = RZ.polygons_from_features(fc["features"])
    for w in warnings:
        print(w, file=sys.stderr)
    tiles = list(dict.fromkeys(tiles))
    polyset = RZ.PolygonSet(polygons, device)
    offsets, ids = RZ.bin_polygons(tiles, polyset.bboxes)
    stats["parse_project_bin_s"] = time.perf_counter() - t0

    size = args.size
    host = torch.empty((batch, size, size), dtype=torch.uint8, pin_memory=True)
    out = torch.empty((batch, size, size), dtype=torch.uint8, device=device)
    threads = min(32, usable_cores())
    for s in range(0, len(tiles), batch):
        chunk = tiles[s:s + batch]
        n = len(chunk)
        t1 = time.perf_counter()
        lo, hi = offsets[s], offsets[s + n]
        csr = (offsets[s:s + n + 1] - lo, ids[lo:hi])
        RZ.rasterize_device(polyset, chunk, size, csr=csr, out=out[:n])
        host[:n].copy_(out[:n])  # synchronous: the batch is on the host after this
        t2 = time.perf_counter()
        masks = host[:n].numpy()
        _merge_existing(args.out, chunk, masks)
        t3 = time.perf_counter()
        _save_batch(args.out, palette, [(t.x, t.y, t.z) for t in chunk], masks, threads)
        t4 = time.perf_counter()
        stats["device_and_d2h_s"] = stats.get("device_and_d2h_s", 0.0) + (t2 - t1)
        stats["merge_s"] = stats.get("merge_s", 0.0) + (t3 - t2)
        stats["png_s"] = stats.get("png_s", 0.0) + (t4 - t3)
