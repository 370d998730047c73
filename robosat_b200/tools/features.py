"""`rs features` (robosat/tools/features.py): simplified GeoJSON features from segmentation masks.

Same flags and output. Masks are decoded in a thread pool, batches of same-size tiles go to the device for the morphology
(`robosat_b200.features.ParkingHandler.apply_batch`), and the contour step of non-empty tiles runs in the same pool. Tiles are
processed in (z, x, y) order, so features come out in that order rather than in directory-listing order."""

import argparse
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from PIL import Image

from robosat_b200.config import load_config
from robosat_b200.features import ParkingHandler
from robosat_b200.hostinfo import usable_cores
from robosat_b200.tiles import tiles_from_slippy_map

handlers = {"parking": ParkingHandler}


def add_parser(subparser):
    parser = subparser.add_parser("features", help="extracts simplified GeoJSON features from segmentation masks",
                                  formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("masks", type=str, help="slippy map directory with segmentation masks")
    parser.add_argument("--type", type=str, required=True, choices=handlers.keys(), help="type of feature to extract")
    parser.add_argument("--dataset", type=str, required=True, help="path to dataset configuration file")
    parser.add_argument("out", type=str, help="path to GeoJSON file to store features in")
    parser.set_defaults(func=main)


def _load(path):
    return np.array(Image.open(path).convert("P"), dtype=np.uint8)  # features.py:46


def _batches(tiles, shapes, batch):
    """Runs of at most `batch` consecutive tiles of one shape."""
    start = 0
    for i in range(1, len(tiles) + 1):
        if i == len(tiles) or i - start == batch or shapes[i] != shapes[start]:
            yield start, i
            start = i


def main(args, batch=64):
    import torch

    from robosat_b200 import _lib

    dataset = load_config(args.dataset)
    labels = dataset["common"]["classes"]
    assert set(labels).issuperset(set(handlers.keys())), "handlers have a class label"
    index = labels.index(args.type)
    try:
        import cv2  # noqa: F401
    except ImportError as exc:
        sys.exit("Error: rs features needs OpenCV (cv2) for contour tracing (%s)" % exc)
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    device = torch.device("cuda")

    handler = handlers[args.type]()
    tiles = sorted(tiles_from_slippy_map(args.masks), key=lambda tp: (int(tp[0].z), int(tp[0].x), int(tp[0].y)))
    for tile, _ in tiles:
        handler.check_zoom(tile)

    with ThreadPoolExecutor(max_workers=min(32, usable_cores())) as pool:
        step = 4 * batch  # decode ahead in chunks; a chunk splits into same-shape batches
        for c in range(0, len(tiles), step):
            chunk = tiles[c:c + step]
            arrays = list(pool.map(_load, [p for _, p in chunk]))
            shapes = [a.shape for a in arrays]
            for i, j in _batches(chunk, shapes, batch):
                host = torch.from_numpy(np.stack(arrays[i:j]))
                handler.apply_batch([t for t, _ in chunk[i:j]], host.to(device), index, pool=pool)
    handler.save(args.out)
