"""`rs merge` (robosat/tools/merge.py): merge adjacent GeoJSON features, such as the fragments of one parking lot that
`rs features` writes on both sides of a tile border.

Same flags. The adjacency test, the components and the closing run on the device (`robosat_b200.merge`, whose `merge` is the
same computation as a function); shapely, rtree, pyproj and geojson are not needed. Each component is written as
`{"type": "Feature", "geometry": Polygon or MultiPolygon, "properties": {"area": m²}}` in component order. Warnings go to
stderr."""

import argparse
import json
import sys


def add_parser(subparser):
    parser = subparser.add_parser("merge", help="merged adjacent GeoJSON features", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("features", type=str, help="GeoJSON file to read features from")
    parser.add_argument("--threshold", type=int, required=True, help="minimum distance to adjacent features, in m")
    parser.add_argument("out", type=str, help="path to GeoJSON to save merged features to")
    parser.set_defaults(func=main)


def main(args, stats=None):
    """`stats` (a dict), when given, receives the seconds spent parsing and projecting, on the device (pairs, components, fill,
    closing and the copies back), tracing and writing, plus the counts and kernel times of `merge.merge_device`."""
    import time

    import torch

    from robosat_b200 import _lib
    from robosat_b200 import merge as MG

    if args.threshold <= 0:
        sys.exit("Error: --threshold must be a positive number of metres")
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    stats = stats if stats is not None else {}

    t0 = time.perf_counter()
    with open(args.features) as fp:
        features = json.load(fp)["features"]
    shapes, warnings = MG.parse(features)
    for w in warnings:
        print(w, file=sys.stderr)
    t1 = time.perf_counter()
    merged, warnings = MG.merge_shapes(shapes, args.threshold, stats=stats)
    for w in warnings:
        print(w, file=sys.stderr)
    t2 = time.perf_counter()
    with open(args.out, "w") as fp:
        json.dump({"type": "FeatureCollection", "features": merged}, fp)
    t3 = time.perf_counter()
    stats.update(parse_s=t1 - t0, write_s=t3 - t2, merged=len(merged), input=len(features))
