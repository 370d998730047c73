"""`rs tile`: slippy-map tiles `{out}/{z}/{x}/{y}.png` (8-bit RGB, --size² pixels) cut from a GeoTIFF, with the reprojection and the
resampling on the GPU (`robosat_b200.tile`, the rule in DESIGN.md §8). The layout is the one `rs download` writes and
`tiles_from_slippy_map` reads, so users with their own imagery (drone orthomosaics, aerial surveys) can feed `rs predict` and
`rs train` without GDAL. Existing files are overwritten. The reference has no such tool.

With --bands, --scale or --stretch the raster is read under the band rule (DESIGN.md §8): 8- or 16-bit, any number of bands,
chunky or band-interleaved, 1 or 3 bands selected and mapped linearly from LO..HI to 0..255 on the GPU; --stretch takes LO and HI
from percentiles of the whole raster (counted on the GPU) and prints them as a --scale to reuse, e.g. for `rs segment`."""

import argparse
import os
import re
import sys


def add_parser(subparser):
    parser = subparser.add_parser("tile", help="cuts a GeoTIFF into slippy-map image tiles", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--zoom", type=int, required=True, help="zoom level of tiles")
    parser.add_argument("--size", type=int, default=512, help="size of image tiles in pixels")
    parser.add_argument("--tiles", type=str, default=None, help="only the tiles of this `rs cover` csv file")
    parser.add_argument("--resampling", choices=["nearest", "bilinear", "average"], default="bilinear", help="resampling method")
    add_band_options(parser)
    parser.add_argument("raster", type=str, help="path to the GeoTIFF")
    parser.add_argument("out", type=str, help="directory to write the tiles to")
    parser.set_defaults(func=main)


def add_band_options(parser):
    parser.add_argument("--bands", type=str, default=None, help="1-based bands to read, 1 (gray) or 3 (R,G,B), e.g. 3,2,1; default 1,2,3 of an RGB "
                        "raster or the band of a gray one. Any of --bands, --scale, --stretch reads 8- or 16-bit rasters of any band count")
    parser.add_argument("--scale", type=str, default=None, help="LO,HI for every band, or LO,HI,LO,HI,LO,HI per band: raw samples LO..HI map to "
                        "0..255 (default for 8-bit rasters: 0,255; 16-bit rasters need --scale or --stretch)")
    parser.add_argument("--stretch", type=str, default=None, help="P_LO,P_HI: --scale from these percentiles (at most two decimals) of each band "
                        "over the valid pixels of the whole raster; the scale is printed for reuse")


def _ints(text, what):
    try:
        return [int(v) for v in text.split(",")]
    except ValueError:
        sys.exit("Error: %s %r is not a list of integers" % (what, text))


def _basis_points(text):
    """a percent with at most two decimals -> hundredths of a percent, or None"""
    m = re.fullmatch(r"\s*(\d{1,3})(?:\.(\d{1,2}))?\s*", text)
    return None if m is None else int(m.group(1)) * 100 + int((m.group(2) or "0").ljust(2, "0"))


def band_options(args):
    """None when none of --bands, --scale, --stretch is given (the plain rule); else (bands, scale pairs, stretch (q_lo, q_hi) in
    hundredths of a percent), each None when not given. Exits naming a malformed value, before any file or device is touched."""
    bands, scale, stretch = (getattr(args, name, None) for name in ("bands", "scale", "stretch"))
    if bands is None and scale is None and stretch is None:
        return None
    if scale is not None and stretch is not None:
        sys.exit("Error: --scale and --stretch are exclusive: --stretch computes the scale")
    if bands is not None:
        bands = _ints(bands, "--bands")
        if len(bands) not in (1, 3):
            sys.exit("Error: --bands takes 1 band (gray) or 3 (R,G,B), not %d" % len(bands))
        if min(bands) < 1:
            sys.exit("Error: --bands are 1-based, not %s" % args.bands)
    if scale is not None:
        values = _ints(scale, "--scale")
        if len(values) not in (2, 6):
            sys.exit("Error: --scale takes LO,HI or three pairs LO,HI,LO,HI,LO,HI, not %d values" % len(values))
        scale = [tuple(values[i:i + 2]) for i in range(0, len(values), 2)]
    if stretch is not None:
        q = [_basis_points(v) for v in stretch.split(",")]
        if len(q) != 2 or None in q or not 0 <= q[0] < q[1] <= 10000:
            sys.exit("Error: --stretch takes P_LO,P_HI, percents with at most two decimals, 0 <= P_LO < P_HI <= 100, not %r" % stretch)
        stretch = tuple(q)
    return bands, scale, stretch


def open_band_raster(path, opts):
    """the geotiff.BandTiff of `path` under band_options `opts`, its --scale set; exits naming what the band rule refuses"""
    from robosat_b200 import _lib
    from robosat_b200.geotiff import open_bands

    bands, scale, stretch = opts
    try:
        raster = open_bands(path, bands)
        if scale is not None:
            raster.set_scale(scale)
    except (_lib.RsbError, OSError) as e:
        sys.exit("Error: %s" % e)
    if raster.scale is None and stretch is None:
        sys.exit("Error: %s: %d-bit samples need --scale LO,HI or --stretch P_LO,P_HI" % (path, raster.bits))
    return raster


def apply_stretch(raster, opts, stats, threads):
    """for --stretch: count the raster's band histograms on the device, set the percentile scale and print it as a --scale line on
    stderr"""
    from robosat_b200 import _lib
    from robosat_b200 import tile as T

    if opts[2] is None:
        return
    q_lo, q_hi = opts[2]
    try:
        raster.set_scale(T.stretch_scale(T.band_stats(raster, threads=threads, stats=stats), q_lo, q_hi))
    except _lib.RsbError as e:
        sys.exit("Error: %s: %s" % (raster.path, e))
    pct = ",".join(("%d.%02d" % divmod(q, 100)).rstrip("0").rstrip(".") for q in (q_lo, q_hi))
    print("--stretch %s of bands %s: --scale %s" % (pct, ",".join(str(b + 1) for b in raster.bands), ",".join("%d,%d" % p for p in raster.scale)),
          file=sys.stderr)


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
    """`stats` (a dict), when given, receives tile.run's counts and seconds, the --stretch pass's (stats_s) and the total"""
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
    opts = band_options(args)
    listed = read_tiles(args.tiles, args.zoom) if args.tiles else None
    raster = open_band_raster(args.raster, opts) if opts else None
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    t0 = time.perf_counter()
    stats = stats if stats is not None else {}
    threads = usable_cores()
    if raster is None:
        try:
            raster = GeoTiff(args.raster)
        except (_lib.RsbError, OSError) as e:
            sys.exit("Error: %s" % e)
    else:
        apply_stretch(raster, opts, stats, threads)
    ratio = T.coarse_ratio(raster, args.zoom, args.size)
    if ratio > 2 and args.resampling != "average":
        print(T.W_COARSE.format(args.zoom, ratio), file=sys.stderr)

    def write(xy, images, counts):
        paths = [os.path.join(args.out, str(args.zoom), str(x), "%d.png" % y) for x, y in xy.tolist()]
        cpaths = (ctypes.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
        _lib.check(_lib.load().rsb_png_write_rgb8_batch(cpaths, len(paths), images.ctypes.data, images.strides[0], args.size, args.size, PNG_LEVEL,
                                                        threads, 1), "rsb_png_write_rgb8_batch")

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
