"""`rs mosaic`: the mask, probability or label tiles `{masks}/{z}/{x}/{y}.png` of one zoom back into one GeoTIFF, with the
reprojection and the resampling on the GPU (`robosat_b200.mosaic`, the rule in DESIGN.md §8). The output is pixel-aligned with
`--like` (an existing GeoTIFF, e.g. the orthomosaic `rs tile` cut) or, by default, the EPSG:3857 grid of the tiles themselves, so a
segmentation can go back into GIS software without GDAL. An existing file is overwritten; a failed run leaves none. The reference
has no such tool."""

import argparse
import sys


def add_parser(subparser):
    parser = subparser.add_parser("mosaic", help="merges slippy-map mask tiles into one GeoTIFF", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--zoom", type=int, required=True, help="zoom level of the tiles")
    parser.add_argument("--like", type=str, default=None, help="GeoTIFF whose grid (CRS, geotransform, size) the output takes; "
                        "default: EPSG:3857 at the zoom's pixel size over the tiles")
    parser.add_argument("--resampling", choices=["nearest", "bilinear"], default="nearest",
                        help="nearest for masks and labels (class indices); bilinear only for probability bins")
    parser.add_argument("--nodata", type=int, default=None, help="value of pixels no tile covers (0..255), written as GDAL_NODATA; "
                        "default: 0 and no nodata tag")
    parser.add_argument("masks", type=str, help="slippy-map directory of palette or gray PNG tiles")
    parser.add_argument("out", type=str, help="path of the GeoTIFF to write")
    parser.set_defaults(func=main)


def main(args, stats=None, budget=None):
    """`stats` (a dict), when given, receives mosaic.run's counts and seconds, the encode and write seconds and the total"""
    import time

    import torch

    from robosat_b200 import _lib
    from robosat_b200 import mosaic as M
    from robosat_b200.compare import PNG_LEVEL
    from robosat_b200.geotiff import read_grid

    t0 = time.perf_counter()
    if args.nodata is not None and not 0 <= args.nodata <= 255:
        sys.exit("Error: --nodata must be in 0..255, not %d" % args.nodata)
    if not 0 <= args.zoom <= _lib.RSB_COVER_MAX_ZOOM:
        sys.exit("Error: --zoom must be in 0..%d" % _lib.RSB_COVER_MAX_ZOOM)
    tiles = M.scan(args.masks, args.zoom)
    if not tiles:
        sys.exit("Error: no tiles at zoom %d in %s" % (args.zoom, args.masks))
    try:
        size, palette = M.check_tiles(tiles)
    except (M.MosaicError, OSError) as e:
        sys.exit("Error: %s" % e)
    if size > _lib.RSB_TILE_MAX_SIZE:
        sys.exit("Error: tiles of %d pixels; rs mosaic reads tiles of up to %d" % (size, _lib.RSB_TILE_MAX_SIZE))
    if args.like:
        try:
            grid = M.Grid(*read_grid(args.like))
        except (_lib.RsbError, OSError) as e:
            sys.exit("Error: --like %s" % e)
    else:
        grid = M.default_grid(tiles, args.zoom, size)
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    ratio = M.coarse_ratio(grid, args.zoom, size)
    if ratio > 2:
        print(M.W_COARSE.format(ratio, args.zoom), file=sys.stderr)
    stats = stats if stats is not None else {}
    writer = M.TiffWriter(args.out, grid, palette, args.nodata, level=PNG_LEVEL)
    try:
        M.run(tiles, args.zoom, size, grid, args.resampling, args.nodata or 0, writer.write, budget or M.DEFAULT_BUDGET, stats=stats)
        writer.close()
    except BaseException as e:
        writer.abort()
        if isinstance(e, _lib.RsbError):
            sys.exit("Error: %s" % e)
        raise
    if stats["covered"] == 0:
        print(M.W_EMPTY, file=sys.stderr)
    stats.update(encode_s=writer.encode_s, write_s=writer.write_s, total_s=time.perf_counter() - t0, width=grid.width, height=grid.height,
                 tiles=len(tiles))
