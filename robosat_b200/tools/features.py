"""`rs features` (robosat/tools/features.py): simplified GeoJSON features from segmentation masks.

Same flags and output, plus `--type building` (this project's rule, `robosat_b200.features.BuildingHandler`). Masks are decoded
in a thread pool, batches of same-size tiles go to the device for the mask cleanup (the handler's `apply_batch`), and the contour
step of non-empty tiles runs in the same pool. Tiles are processed in (z, x, y) order, so features come out in that order rather
than in directory-listing order. `--type` must be one of the dataset's classes.

`--type road` (`robosat_b200.features.RoadHandler`) needs each tile's 8 neighbours: every mask is decoded once and kept while a
later batch can still need it, and each batch's halo'd binary planes are built on the host in pinned memory."""

import argparse
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from PIL import Image

from robosat_b200.config import load_config
from robosat_b200.features import BuildingHandler, ParkingHandler, RoadHandler, halo_plane
from robosat_b200.hostinfo import usable_cores
from robosat_b200.tiles import tiles_from_slippy_map

handlers = {"parking": ParkingHandler, "building": BuildingHandler, "road": RoadHandler}


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
    if args.type not in labels:
        sys.exit("Error: rs features --type %s needs a class %r in the dataset's classes %s" % (args.type, args.type, labels))
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

    if args.type == "road":
        _roads(handler, tiles, index, device, batch)
        handler.save(args.out)
        return

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


def _roads(handler, tiles, index, device, batch):
    """Batches of `batch` consecutive tiles of one shape, each with the halo of its neighbours' masks (missing ones background)"""
    import torch

    paths = {(int(t.z), int(t.x), int(t.y)): p for t, p in tiles}
    cache = {}
    h = handler.halo
    pinned = {}
    with ThreadPoolExecutor(max_workers=min(32, usable_cores())) as pool:
        for b in range(0, len(tiles), batch):
            chunk = [t for t, _ in tiles[b:b + batch]]
            z0, x0 = int(chunk[0].z), int(chunk[0].x)
            for key in [k for k in cache if (k[0], k[1]) < (z0, x0 - 1)]:
                del cache[key]  # every later tile's neighbours are at (z0, x0 - 1) or after
            need = {(int(t.z), int(t.x) + dx, int(t.y) + dy) for t in chunk for dx in (-1, 0, 1) for dy in (-1, 0, 1)}
            need = sorted(k for k in need if k in paths and k not in cache)
            cache.update(zip(need, pool.map(lambda k: _load(paths[k]), need)))
            for i, j in _batches(chunk, [cache[(int(t.z), int(t.x), int(t.y))].shape for t in chunk], batch):
                H, W = cache[(int(chunk[i].z), int(chunk[i].x), int(chunk[i].y))].shape
                if H < h or W < h:
                    sys.exit("Error: rs features --type road needs masks of at least %d px, not %d x %d" % (h, H, W))
                if (H, W) not in pinned:
                    pinned[(H, W)] = torch.empty((batch, H + 2 * h, W + 2 * h), dtype=torch.uint8).pin_memory()
                host = pinned[(H, W)][:j - i]
                planes = host.numpy()

                def fill(k):
                    t = chunk[i + k]
                    z, x, y = int(t.z), int(t.x), int(t.y)
                    neighbours = {}
                    for dy in (-1, 0, 1):
                        for dx in (-1, 0, 1):
                            m = cache.get((z, x + dx, y + dy))
                            if m is not None and m.shape != (H, W):
                                sys.exit("Error: rs features --type road: mask %s is %d x %d, its neighbour %s is %d x %d" % (
                                    paths[(z, x, y)], H, W, paths[(z, x + dx, y + dy)], m.shape[0], m.shape[1]))
                            neighbours[(dy, dx)] = m
                    halo_plane(cache[(z, x, y)], neighbours, index, h, planes[k])

                list(pool.map(fill, range(j - i)))
                handler.apply_batch(chunk[i:j], host.to(device, non_blocking=True), pool=pool)
