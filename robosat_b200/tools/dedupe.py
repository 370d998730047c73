"""`rs dedupe` (robosat/tools/dedupe.py): the predicted features that OpenStreetMap does not already map, as GeoJSON.

Same flags and output layout. The overlap test and the areas run on the device (`robosat_b200.dedupe`, whose `dedupe` is the
same computation as a function); shapely, rtree, pyproj and geojson are not needed. Kept features keep their order and geometry,
with rings closed and coordinates written as floats, and lose their properties, as the reference's
`geojson.Feature(geometry=mapping(shape))` does. Warnings go to stderr."""

import argparse
import json
import sys


def add_parser(subparser):
    parser = subparser.add_parser("dedupe", help="deduplicates features against OpenStreetMap", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("osm", type=str, help="ground truth GeoJSON feature collection from OpenStreetMap")
    parser.add_argument("predicted", type=str, help="predicted GeoJSON feature collection to deduplicate")
    parser.add_argument("--threshold", type=float, required=True, help="maximum allowed IoU to keep predictions, between 0.0 and 1.0")
    parser.add_argument("out", type=str, help="path to GeoJSON to save deduplicated features to")
    parser.set_defaults(func=main)


def write(path, features, keep):
    """the kept features as a FeatureCollection in the reference's layout (`dedupe.kept_features`) -> how many were written"""
    from robosat_b200 import dedupe as DD

    kept = DD.kept_features(features, keep)
    with open(path, "w") as fp:
        json.dump({"type": "FeatureCollection", "features": kept}, fp)
    return len(kept)


def main(args, stats=None):
    """`stats` (a dict), when given, receives the seconds spent parsing and projecting, on the device (candidate pairs, both
    kernels and the copies back) and writing the file, plus the counts and kernel times of `dedupe.decide`."""
    import time

    import torch

    from robosat_b200 import _lib
    from robosat_b200 import dedupe as DD

    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    stats = stats if stats is not None else {}

    t0 = time.perf_counter()
    with open(args.osm) as fp:
        osm = json.load(fp)["features"]
    with open(args.predicted) as fp:
        predicted = json.load(fp)["features"]
    qs, osm_warnings = DD.parse(osm, True)
    ps, warnings = DD.parse(predicted, False)
    for w in osm_warnings + warnings:
        print(w, file=sys.stderr)
    t1 = time.perf_counter()
    keep, _ = DD.decide(ps, qs, args.threshold, [not DD.is_areal(f) for f in predicted], stats=stats)
    t2 = time.perf_counter()
    kept = write(args.out, predicted, keep)
    t3 = time.perf_counter()
    stats.update(parse_project_s=t1 - t0, device_s=t2 - t1, write_s=t3 - t2, predicted=len(predicted), osm=len(osm), kept=kept)
