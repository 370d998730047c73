"""`rs tile`: slippy-map tiles `{out}/{z}/{x}/{y}.png` (8-bit RGB, --size² pixels) cut from a GeoTIFF, with the reprojection and the
resampling on the GPU (`robosat_b200.tile`, the rule in DESIGN.md §8). The layout is the one `rs download` writes and
`tiles_from_slippy_map` reads, so users with their own imagery (drone orthomosaics, aerial surveys) can feed `rs predict` and
`rs train` without GDAL. Existing files are overwritten. The reference has no such tool."""

import argparse
import os
import sys


def add_parser(subparser):
    parser = subparser.add_parser("tile", help="cuts a GeoTIFF into slippy-map image tiles", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--zoom", type=int, required=True, help="zoom level of tiles")
    parser.add_argument("--size", type=int, default=512, help="size of image tiles in pixels")
    parser.add_argument("--tiles", type=str, default=None, help="only the tiles of this `rs cover` csv file")
    parser.add_argument("--resampling", choices=["nearest", "bilinear", "average"], default="bilinear", help="resampling method")
    parser.add_argument("raster", type=str, help="path to the GeoTIFF")
    parser.add_argument("out", type=str, help="directory to write the tiles to")
    parser.set_defaults(func=main)


def read_tiles(path, zoom):
    """the (x, y) of a tiles csv; exits naming the first row whose zoom is not `zoom`"""
    from robosat_b200.tiles import tiles_from_csv

    tiles = []
    for i, t in enumerate(tiles_from_csv(path), 1):
        if t.z != zoom:
            sys.exit("Error: %s row %d is tile (%d, %d, %d), not at --zoom %d" % (path, i, t.x, t.y, t.z, zoom))
        tiles.append((t.x, t.y))
    return tiles


def main(args, stats=None):
    """`stats` (a dict), when given, receives tile.run's counts and seconds plus the total"""
    import ctypes
    import time

    import torch

    from robosat_b200 import _lib
    from robosat_b200 import tile as T
    from robosat_b200.compare import PNG_LEVEL
    from robosat_b200.geotiff import GeoTiff
    from robosat_b200.hostinfo import usable_cores

    if not 0 <= args.zoom <= _lib.RSB_COVER_MAX_ZOOM:
        sys.exit("Error: --zoom must be in 0..%d" % _lib.RSB_COVER_MAX_ZOOM)
    if not 1 <= args.size <= _lib.RSB_TILE_MAX_SIZE:
        sys.exit("Error: --size must be in 1..%d" % _lib.RSB_TILE_MAX_SIZE)
    listed = read_tiles(args.tiles, args.zoom) if args.tiles else None
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    t0 = time.perf_counter()
    try:
        raster = GeoTiff(args.raster)
    except (_lib.RsbError, OSError) as e:
        sys.exit("Error: %s" % e)
    ratio = T.coarse_ratio(raster, args.zoom, args.size)
    if ratio > 2 and args.resampling != "average":
        print(T.W_COARSE.format(args.zoom, ratio), file=sys.stderr)
    threads = usable_cores()

    def write(xy, images, counts):
        paths = [os.path.join(args.out, str(args.zoom), str(x), "%d.png" % y) for x, y in xy.tolist()]
        cpaths = (ctypes.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
        _lib.check(_lib.load().rsb_png_write_rgb8_batch(cpaths, len(paths), images.ctypes.data, images.strides[0], args.size, args.size, PNG_LEVEL,
                                                        threads, 1), "rsb_png_write_rgb8_batch")

    stats = stats if stats is not None else {}
    try:
        T.run(raster, args.zoom, args.size, args.resampling, listed, write, stats=stats, threads=threads)
    except _lib.RsbError as e:
        sys.exit("Error: %s" % e)
    if listed is not None:
        missing = len(set(listed)) - stats["written"]
        if missing:
            print("Warning: %d of the %d listed tiles have no pixel inside the raster and were not written" % (missing, len(set(listed))),
                  file=sys.stderr)
    stats["total_s"] = time.perf_counter() - t0
