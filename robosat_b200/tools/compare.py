"""`rs compare` (robosat/tools/compare.py): side-by-side images image | label | mask ... of the tiles whose mask coverage lies in
[--minimum, --maximum], for reviewing what a model got wrong.

Same positional arguments, flags and defaults. The coverage filter and the composites run on the device
(`robosat_b200.compare.compare_device`). One flag is added: `--csv PATH` writes one row per (tile, mask), in (z, x, y) order and
kept or not, with the mask's coverage and its tp / fp / fn / tn pixel counts and foreground IoU against the label (foreground:
index != 0, the filter's notion of "not background"; `mask` is the mask directory's position in the arguments, from 0; `fg_iou`
is empty when tp + fp + fn = 0). Unlike the reference, a missing file or a size mismatch stops the tool before it writes
anything.

`--dataset PATH` (with `--csv`) scores every class of the dataset instead: the CSV then has the columns z, x, y, mask, class,
coverage, tp, fp, fn, tn, iou, one row per (tile, mask, class) with the classes in dataset order and `class` the class name;
tp counts the pixels where label == mask == class, fp = mask pixels of the class - tp, fn = label pixels of the class - tp,
iou = tp / (tp + fp + fn), empty when that is 0. `coverage` stays the non-background share, so the rows join with the CSV
without `--dataset`. For a two-class dataset the class-1 row equals the `fg_iou` row only when the planes hold only 0 and 1
(`fg_iou` counts every non-zero index as foreground). A label or mask value outside the dataset's classes stops the tool
naming the tile and the file. The coverage filter and the images do not change."""

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
    parser.add_argument("--dataset", type=str, default=None,
                        help="dataset configuration file: with --csv, write one row per (tile, mask, class) with per-class tp / fp / fn / tn / iou")
    parser.set_defaults(func=main)


def dataset_classes(args):
    """The checked class names of `--dataset`, or None without it; exits naming the problem: --dataset without --csv, fewer than
    2 or more than 256 classes, or a class name `rs predict` would refuse (tools/predict.check_class_names)."""
    from robosat_b200 import _lib
    from robosat_b200.config import load_config
    from robosat_b200.tools.predict import check_class_names

    path = getattr(args, "dataset", None)
    if path is None:
        return None
    if not args.csv:
        sys.exit("Error: --dataset needs --csv: the per-class counts are written to the CSV")
    classes = load_config(path)["common"]["classes"]
    if not 2 <= len(classes) <= _lib.RSB_COMPARE_MAX_CLASSES:
        sys.exit("Error: the dataset has %d classes, --dataset supports 2..%d" % (len(classes), _lib.RSB_COMPARE_MAX_CLASSES))
    try:
        return check_class_names(classes)
    except ValueError as e:
        sys.exit("Error: dataset %s: %s" % (path, e))


def main(args, stats=None):
    """`stats` (a dict), when given, receives what `compare_device` reports: decode / device / encode seconds, kernel
    milliseconds, tiles, kept and written."""
    import torch

    from robosat_b200 import _lib
    from robosat_b200.compare import CompareError, compare_device

    classes = dataset_classes(args)
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    try:
        compare_device(args.images, args.labels, args.masks, args.out, args.minimum, args.maximum, csv=args.csv, stats=stats, classes=classes)
    except CompareError as e:
        sys.exit("Error: %s" % e)
