"""`rs compare` (robosat/tools/compare.py): side-by-side images image | label | mask ... of the tiles whose mask coverage lies in
[--minimum, --maximum], for reviewing what a model got wrong.

Same positional arguments, flags and defaults. The coverage filter and the composites run on the device
(`robosat_b200.compare.compare_device`). One flag is added: `--csv PATH` writes one row per (tile, mask), in (z, x, y) order and
kept or not, with the mask's coverage and its tp / fp / fn / tn pixel counts and foreground IoU against the label (foreground:
index != 0, the filter's notion of "not background"; `mask` is the mask directory's position in the arguments, from 0; `fg_iou`
is empty when tp + fp + fn = 0). Unlike the reference, a missing file or a size mismatch stops the tool before it writes
anything."""

import argparse
import sys


def add_parser(subparser):
    parser = subparser.add_parser("compare", help="compare images, labels and masks side by side", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("out", type=str, help="directory to save visualizations to")
    parser.add_argument("images", type=str, help="directory to read slippy map images from")
    parser.add_argument("labels", type=str, help="directory to read slippy map labels from")
    parser.add_argument("masks", type=str, nargs="+", help="slippy map directories to read masks from")
    parser.add_argument("--minimum", type=float, default=0.0, help="minimum percentage of mask not background")
    parser.add_argument("--maximum", type=float, default=1.0, help="maximum percentage of mask not background")
    parser.add_argument("--csv", type=str, default=None, help="CSV file to write per-tile, per-mask agreement with the label to")
    parser.set_defaults(func=main)


def main(args, stats=None):
    """`stats` (a dict), when given, receives what `compare_device` reports: decode / device / encode seconds, kernel
    milliseconds, tiles, kept and written."""
    import torch

    from robosat_b200 import _lib
    from robosat_b200.compare import CompareError, compare_device

    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    try:
        compare_device(args.images, args.labels, args.masks, args.out, args.minimum, args.maximum, csv=args.csv, stats=stats)
    except CompareError as e:
        sys.exit("Error: %s" % e)
