"""`rs segment`: an orthomosaic GeoTIFF in, one 1-band GeoTIFF of masks (or foreground probability bins) on the raster's own grid out.
Its pixels are those of `rs tile → rs predict → rs masks → rs mosaic --like` run with the same settings (DESIGN.md §8), but the tiles,
the network's bins and the masks never leave the GPU (`robosat_b200.segment`): no PNG is written or read. One device; RSB_GPUS is
not read. An existing file is overwritten; a failed run leaves none. The reference has no such tool. --bands, --scale and --stretch read
the raster under the band rule, as `rs tile` does."""

import argparse
import os
import sys

from robosat_b200.tools.tile import add_band_options


def add_parser(subparser):
    parser = subparser.add_parser("segment", help="segments a GeoTIFF into a mask GeoTIFF on the same grid",
                                  formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--zoom", type=int, required=True, help="zoom level of the tiles the network sees")
    parser.add_argument("--size", type=int, default=512, help="size of the tiles in pixels")
    parser.add_argument("--overlap", type=int, default=32, help="tile pixel overlap to predict on")
    parser.add_argument("--batch_size", type=int, default=32, help="tiles per batch")
    parser.add_argument("--tiles", type=str, default=None, help="only the tiles of this `rs cover` csv file")
    parser.add_argument("--resampling", choices=["nearest", "bilinear", "average"], default="bilinear", help="resampling of the image tiles")
    parser.add_argument("--output", choices=["masks", "probs"], default="masks",
                        help="masks: class indices (as rs masks writes them); probs: foreground probability bins (two classes only)")
    parser.add_argument("--tta", type=str, default="none", choices=["none", "flip", "d4"],
                        help="test-time augmentation: mean probability over flipped (flip) or all 8 dihedral (d4) views of each tile")
    parser.add_argument("--nodata", type=int, default=None, help="value of pixels no tile covers (0..255), written as GDAL_NODATA; "
                        "default: 0 and no nodata tag")
    parser.add_argument("--model", type=str, required=True, help="path to model configuration file")
    parser.add_argument("--dataset", type=str, required=True, help="path to dataset configuration file")
    parser.add_argument("--checkpoint", type=str, required=True, help="model checkpoint to load")
    add_band_options(parser)
    parser.add_argument("raster", type=str, help="path to the GeoTIFF")
    parser.add_argument("out", type=str, help="path of the GeoTIFF to write")
    parser.set_defaults(func=main)


def main(args, stats=None, budget=None):
    """`stats` (a dict), when given, receives segment.run's counts and seconds, the --stretch pass's (stats_s), the encode and write
    seconds and the total"""
    import time

    import torch

    from robosat_b200 import _lib
    from robosat_b200 import mosaic as M
    from robosat_b200 import segment as SEG
    from robosat_b200 import tile as T
    from robosat_b200.colors import continuous_palette_for_color, make_palette
    from robosat_b200.compare import PNG_LEVEL
    from robosat_b200.config import load_config
    from robosat_b200.geotiff import GeoTiff, read_grid
    from robosat_b200.hostinfo import usable_cores
    from robosat_b200.predictor import TilePredictor
    from robosat_b200.tools.predict import check_class_names, load_state_dict
    from robosat_b200.tools.tile import apply_stretch, band_options, open_band_raster, read_tiles

    t0 = time.perf_counter()
    if not 0 <= args.zoom <= _lib.RSB_COVER_MAX_ZOOM:
        sys.exit("Error: --zoom must be in 0..%d" % _lib.RSB_COVER_MAX_ZOOM)
    if not 1 <= args.size <= _lib.RSB_TILE_MAX_SIZE:
        sys.exit("Error: --size must be in 1..%d" % _lib.RSB_TILE_MAX_SIZE)
    if not 0 <= args.overlap <= args.size:
        sys.exit("Error: --overlap must be in 0..--size")
    if (args.size + 2 * args.overlap) % 64:
        sys.exit("Error: --size + 2 --overlap must be a multiple of 64 (the network's input), not %d" % (args.size + 2 * args.overlap))
    if args.batch_size < 1:
        sys.exit("Error: --batch_size must be at least 1")
    if args.nodata is not None and not 0 <= args.nodata <= 255:
        sys.exit("Error: --nodata must be in 0..255, not %d" % args.nodata)
    common = load_config(args.dataset)["common"]
    classes = common["classes"]
    if len(classes) > 2:
        if args.output == "probs":
            sys.exit("Error: --output probs writes one band of foreground probabilities, for two-class models only; the dataset has %d classes"
                     % len(classes))
        try:
            check_class_names(classes)
        except ValueError as exc:
            sys.exit("Error: dataset %s: %s" % (args.dataset, exc))
    if not load_config(args.model)["common"]["cuda"]:
        sys.exit("Error: robosat_b200 runs on CUDA devices only; set cuda = true in the model configuration")
    opts = band_options(args)
    listed = read_tiles(args.tiles, args.zoom) if args.tiles else None
    raster = open_band_raster(args.raster, opts) if opts else None
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    stats = stats if stats is not None else {}
    try:
        raster = raster or GeoTiff(args.raster)
        grid = M.Grid(*read_grid(args.raster))
    except (_lib.RsbError, OSError) as e:
        sys.exit("Error: %s" % e)
    if opts:
        apply_stretch(raster, opts, stats, usable_cores())
    ratio = T.coarse_ratio(raster, args.zoom, args.size)
    if ratio > 2 and args.resampling != "average":
        print(T.W_COARSE.format(args.zoom, ratio), file=sys.stderr)
    ratio = M.coarse_ratio(grid, args.zoom, args.size)
    if ratio > 2:
        print(M.W_COARSE.format(ratio, args.zoom), file=sys.stderr)
    try:
        plan = SEG.plan(raster, grid, args.zoom, args.size, args.batch_size, listed, budget or SEG.DEFAULT_BUDGET, args.resampling)
    except _lib.RsbError as e:
        sys.exit("Error: %s" % e)
    if not len(plan.tiles):
        sys.exit("Error: no tile at zoom %d has a pixel inside %s" % (args.zoom, args.raster))

    if args.output == "probs":
        flat = continuous_palette_for_color("pink", 256)  # rs predict's palette
    elif len(classes) > 2:
        flat = make_palette(*common["colors"])  # rs masks --dataset
    else:
        flat = make_palette("denim", "orange")  # rs masks
    torch.cuda.set_device(0)
    device = torch.device("cuda", 0)
    predictor = TilePredictor(load_state_dict(args.checkpoint), len(classes), args.batch_size, args.size + 2 * args.overlap, overlap=args.overlap,
                              device=device, use_graph=os.environ.get("RSB_PREDICT_GRAPH", "1") == "1",
                              depth=int(os.environ.get("RSB_PREDICT_DEPTH", "3")), tta=args.tta)
    threads = usable_cores()
    writer = M.TiffWriter(args.out, grid, SEG.output_palette(flat), args.nodata, level=PNG_LEVEL, threads=threads)
    try:
        existing = SEG.run(raster, plan, predictor, args.resampling, args.output, args.nodata or 0, writer.write, device, stats, threads)
        if not existing:
            raise _lib.RsbError("no tile at zoom %d has a pixel inside %s" % (args.zoom, args.raster))
        writer.close()
    except BaseException as e:
        writer.abort()
        if isinstance(e, _lib.RsbError):
            sys.exit("Error: %s" % e)
        raise
    if listed is not None:
        missing = len(set(listed)) - existing
        if missing:
            print("Warning: %d of the %d listed tiles have no pixel inside the raster and were not segmented" % (missing, len(set(listed))),
                  file=sys.stderr)
    if stats["covered"] == 0:
        print(M.W_EMPTY, file=sys.stderr)
    stats.update(encode_s=writer.encode_s, write_s=writer.write_s, total_s=time.perf_counter() - t0, width=grid.width, height=grid.height)
