"""`rs rasterize` (robosat/tools/rasterize.py): label masks from GeoJSON polygons.

Same flags, warnings and output files. The Polygon features are projected and uploaded to the device once, binned to the tiles
of the CSV by their bounding boxes, and burned in batches of tiles by one `rsb_rasterize_polygons` launch each
(`robosat_b200.rasterize`). Every tile of the CSV is written, in CSV order; a tile listed twice is written once. An existing
mask file is merged with np.maximum, as in the reference, and the PNGs of a batch are written by the library's encoder threads
(`tools/predict.py:_save_batch`).

`--class NAME` makes labels for a dataset of more than two classes: the features file is burned as class c =
classes.index(NAME), so a pixel the fill sets gets c and every other pixel 0, and the tile is merged with the label file
already in the output directory by np.maximum. Run the tool once per class into one directory. Where classes overlap the
higher class index wins whatever the order of the runs, and repeating a run changes nothing, so a run that stopped can be
started again: order the dataset's classes by priority. The PNGs carry the palette of all C colours. Existing label files
must be palette PNGs of 1, 2, 4 or 8 bits or 8-bit gray PNGs of --size x --size (checked for every file from its header
before anything is written) with values below C; they are read by the library's decoder threads (`compare.decode_indexed`)
and merged on the device. For two classes and NAME = classes[1] the files are the ones a run without --class writes."""

import argparse
import json
import os
import struct
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
    parser.add_argument("--class", dest="class_name", type=str, default=None,
                        help="burn the features as this dataset class (not the first) and merge with existing labels by maximum, "
                             "so the higher class index wins where classes overlap: list the dataset's classes by priority "
                             "and run once per class into one directory")
    parser.set_defaults(func=main)


def _merge_existing(root, tiles, masks):
    """np.maximum with the masks already on disk (rasterize.py:131-133), in place"""
    for i, t in enumerate(tiles):
        path = os.path.join(root, str(t.z), str(t.x), "{}.png".format(t.y))
        if os.path.exists(path):
            masks[i] = np.maximum(masks[i], np.array(Image.open(path)))


def class_value(classes, colors, name):
    """The index the features of class `name` are burned with; exits naming the problem unless the dataset has as many colours as
    classes, 2 <= C <= 256 classes, and `name` is one of them other than the first (burning background under a maximum changes
    nothing)."""
    if len(classes) != len(colors):
        sys.exit("Error: the dataset has %d classes and %d colors; --class needs one color per class" % (len(classes), len(colors)))
    if not 2 <= len(classes) <= 256:
        sys.exit("Error: the dataset has %d classes; --class supports 2..256" % len(classes))
    if name not in classes:
        sys.exit("Error: --class %r is not one of the dataset's classes %s" % (name, list(classes)))
    value = list(classes).index(name)
    if value == 0:
        sys.exit("Error: --class %r is the background class; burning it under the maximum rule changes nothing" % name)
    return value


def label_path(root, tile):
    return os.path.join(root, str(tile.z), str(tile.x), "{}.png".format(tile.y))


def check_existing_labels(root, tiles, size):
    """[bool] per tile: whether its label file exists. Exits naming the first existing file that is not a non-interlaced palette
    PNG of 1, 2, 4 or 8 bits or 8-bit gray PNG of size x size, from its header alone: the formats whose index plane the library's
    decoder reads as np.array(Image.open(path)) does. RGB and the rest would need a conversion that changes values."""
    from robosat_b200.compare import PNG_SIGNATURE

    exists = []
    for t in tiles:
        path = label_path(root, t)
        if not os.path.exists(path):
            exists.append(False)
            continue
        with open(path, "rb") as fp:
            head = fp.read(29)
        if len(head) < 29 or head[:8] != PNG_SIGNATURE or head[12:16] != b"IHDR":
            sys.exit("Error: existing label %s is not a PNG file" % path)
        w, h = struct.unpack(">II", head[16:24])
        depth, ctype, interlace = head[24], head[25], head[28]
        if not ((ctype == 3 and depth in (1, 2, 4, 8)) or (ctype == 0 and depth == 8)) or interlace != 0:
            sys.exit("Error: existing label %s is a PNG of colour type %d, %d bits%s; --class merges palette PNGs of 1, 2, 4 or 8 bits "
                     "and 8-bit gray PNGs" % (path, ctype, depth, ", interlaced" if interlace else ""))
        if (w, h) != (size, size):
            sys.exit("Error: existing label %s is %dx%d, --size is %d" % (path, w, h, size))
        exists.append(True)
    return exists


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
    name = getattr(args, "class_name", None)
    if name is None:
        assert len(classes) == len(colors), "classes and colors coincide"
        assert len(colors) == 2, "only binary models supported right now"
        palette = make_palette(colors[0], colors[1])
    else:
        value = class_value(classes, colors, name)
        palette = make_palette(*colors)
    tiles = list(tiles_from_csv(args.tiles))
    assert all(tile.z == args.zoom for tile in tiles)  # we can only rasterize all tiles at a single zoom
    if not 1 <= args.size <= _lib.RSB_RASTER_MAX_SIZE:
        sys.exit("Error: --size must be in 1..%d" % _lib.RSB_RASTER_MAX_SIZE)
    if name is not None:
        tiles = list(dict.fromkeys(tiles))
        existing = check_existing_labels(args.out, tiles, args.size)
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
    if name is not None:
        _class_batches(args.out, tiles, polyset, offsets, ids, size, value, len(classes), existing, palette, batch, stats)
        return
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


def _class_batches(root, tiles, polyset, offsets, ids, size, value, num_classes, existing, palette, batch, stats):
    """The --class loop: per batch, the fill times `value`, then one torch.maximum with the batch's existing labels (read by the
    library's decoder threads into pinned memory and uploaded) before the copy to the host. A label holding a value >= C exits
    naming the file before the batch is written."""
    import time

    import torch

    from robosat_b200 import _lib
    from robosat_b200 import rasterize as RZ
    from robosat_b200.compare import decode_indexed
    from robosat_b200.tools.predict import _save_batch

    device = polyset.device
    host = torch.empty((batch, size, size), dtype=torch.uint8, pin_memory=True)
    prev_host = torch.empty((batch, size, size), dtype=torch.uint8, pin_memory=True)
    out = torch.empty((batch, size, size), dtype=torch.uint8, device=device)
    prev = torch.empty((batch, size, size), dtype=torch.uint8, device=device)
    threads = min(32, usable_cores())
    prev_np = prev_host.numpy()
    no_palettes = np.empty((batch, 256, 3), np.uint8)
    stats.setdefault("read_labels_s", 0.0)
    for s in range(0, len(tiles), batch):
        chunk = tiles[s:s + batch]
        n = len(chunk)
        t0 = time.perf_counter()
        have = [i for i in range(n) if existing[s + i]]
        if have:
            for i in range(n):
                if not existing[s + i]:
                    prev_np[i] = 0
            try:
                decode_indexed([label_path(root, chunk[i]) for i in have], [prev_np[i].reshape(-1) for i in have], no_palettes, (size, size),
                               threads, native_only=True)
            except _lib.RsbError as e:
                sys.exit("Error: reading the existing labels: %s" % e)
        t1 = time.perf_counter()
        lo, hi = offsets[s], offsets[s + n]
        csr = (offsets[s:s + n + 1] - lo, ids[lo:hi])
        RZ.rasterize_device(polyset, chunk, size, csr=csr, out=out[:n])
        out[:n].mul_(value)
        if have:
            prev[:n].copy_(prev_host[:n], non_blocking=True)
            highest = prev[:n].view(n, -1).amax(dim=1)
            torch.maximum(out[:n], prev[:n], out=out[:n])
        host[:n].copy_(out[:n])  # synchronous: the batch is on the host after this
        if have:
            highest = highest.cpu().numpy()
            bad = np.flatnonzero(highest >= num_classes)
            if len(bad):
                i = int(bad[0])
                sys.exit("Error: existing label %s holds the value %d, but the dataset has the %d classes 0..%d"
                         % (label_path(root, chunk[i]), int(highest[i]), num_classes, num_classes - 1))
        t2 = time.perf_counter()
        _save_batch(root, palette, [(t.x, t.y, t.z) for t in chunk], host[:n].numpy(), threads)
        t3 = time.perf_counter()
        stats["read_labels_s"] += t1 - t0
        stats["device_and_d2h_s"] = stats.get("device_and_d2h_s", 0.0) + (t2 - t1)
        stats["png_s"] = stats.get("png_s", 0.0) + (t3 - t2)
