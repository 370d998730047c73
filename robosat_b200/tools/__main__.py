"""`python -m robosat_b200.tools {train,predict,serve,masks,weights,features,rasterize,cover,dedupe,merge,extract,compare,tile,mosaic,segment} ...` --
the `rs` sub-commands on the hot path (dispatch as in robosat/tools/__main__.py:22-59; the other sub-commands stay with the reference package)."""

import argparse

from robosat_b200.tools import compare, cover, dedupe, extract, features, masks, merge, mosaic, predict, rasterize, segment, serve, tile, train, weights


def add_parsers():
    parser = argparse.ArgumentParser(prog="./rs")
    subparser = parser.add_subparsers(title="robosat tools", metavar="")
    train.add_parser(subparser)
    predict.add_parser(subparser)
    serve.add_parser(subparser)
    masks.add_parser(subparser)
    weights.add_parser(subparser)
    features.add_parser(subparser)
    rasterize.add_parser(subparser)
    cover.add_parser(subparser)
    dedupe.add_parser(subparser)
    merge.add_parser(subparser)
    extract.add_parser(subparser)
    compare.add_parser(subparser)
    tile.add_parser(subparser)
    mosaic.add_parser(subparser)
    segment.add_parser(subparser)
    subparser.required = True
    return parser.parse_args()


def main():
    args = add_parsers()
    args.func(args)


if __name__ == "__main__":
    main()
