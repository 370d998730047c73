"""`rs extract` (robosat/tools/extract.py): parking-lot or building polygons from an OpenStreetMap `.osm.pbf` file, as GeoJSON.

Same flags and output layout as the reference's FeatureStorage: the features go, `--batch` per file, into files named
`{base}-{uuid4 hex}{ext}` after `os.path.splitext(out)`, each a `{"type": "FeatureCollection", "features": [...]}`; an empty result
writes no file. The DenseNodes decode, the node-location join and the validity check run on the device (`robosat_b200.extract`);
osmium, shapely and geojson are not needed. `--type road` is not ported: its buffer is GEOS's. Warnings go to stderr."""

import argparse
import json
import os
import sys
import uuid

TYPES = ("parking", "building", "road")


def add_parser(subparser):
    parser = subparser.add_parser("extract", help="extracts GeoJSON features from OpenStreetMap", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--type", type=str, required=True, choices=TYPES, help="type of feature to extract")
    parser.add_argument("--batch", type=int, default=100000, help="number of features to save per file")
    parser.add_argument("map", type=str, help="path to .osm.pbf base map")
    parser.add_argument("out", type=str, help="path to GeoJSON file to store features in")
    parser.set_defaults(func=main)


def save(features, out, batch):
    """FeatureStorage.add / flush: `batch` features per file -> the paths written, in order"""
    base, ext = os.path.splitext(out)
    paths = []
    for i in range(0, len(features), batch):
        path = "{}-{}{}".format(base, uuid.uuid4().hex, ext)
        with open(path, "w") as fp:
            json.dump({"type": "FeatureCollection", "features": features[i: i + batch]}, fp)
        paths.append(path)
    return paths


def main(args, stats=None):
    """`stats` (a dict), when given, receives `extract.extract_device`'s stage times and counts and the seconds spent writing."""
    import time

    if args.type == "road":
        sys.exit("Error: --type road is not ported: its polygons are GEOS buffers of the road lines, which this project does not restate")
    if args.batch <= 0:
        sys.exit("Error: --batch must be a positive number of features")
    import torch

    from robosat_b200 import _lib
    from robosat_b200 import extract as EX

    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    features, warnings = EX.extract_device(args.map, args.type, stats=stats)
    for w in warnings:
        print(w, file=sys.stderr)
    t0 = time.perf_counter()
    save(features, args.out, args.batch)
    if stats is not None:
        stats["write_s"] = time.perf_counter() - t0
