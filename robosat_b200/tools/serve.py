"""`rs serve` (robosat/tools/serve.py:76-128): on-demand tile server whose per-request model call is the H100 graph-replay
path (`robosat_b200.serve.Predictor.segment`). Same flags and endpoints; the HTTP shell needs `flask` and `requests`, which
this package does not vendor -- without them the command exits with the reference's style of error message."""

import argparse
import io
import os
import sys

from robosat_b200.config import load_config


def add_parser(subparser):
    parser = subparser.add_parser("serve", help="serves predicted masks with on-demand tileserver", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--model", type=str, required=True, help="path to model configuration file")
    parser.add_argument("--dataset", type=str, required=True, help="path to dataset configuration file")
    parser.add_argument("--url", type=str, help="endpoint with {z}/{x}/{y} variables to fetch image tiles from")
    parser.add_argument("--checkpoint", type=str, required=True, help="model checkpoint to load")
    parser.add_argument("--tile_size", type=int, default=512, help="tile size for slippy map tiles")
    parser.add_argument("--host", type=str, default="127.0.0.1", help="host to serve on")
    parser.add_argument("--port", type=int, default=5000, help="port to serve on")
    parser.add_argument("--tta", type=str, default="none", choices=["none", "flip", "d4"],
                        help="test-time augmentation: argmax of the mean probability over flipped (flip) or all 8 dihedral (d4) views")
    parser.set_defaults(func=main)


def make_app(predictor, url_template, token, size, session=None):
    """The reference's two routes (serve.py:46-75) around `predictor.segment`."""
    from flask import Flask, abort, render_template, send_file
    from PIL import Image

    # the page template ships with this package (robosat_b200/tools/templates/map.html); the tile route does not need it
    app = Flask(__name__, template_folder=os.path.join(os.path.dirname(os.path.abspath(__file__)), "templates"))

    @app.route("/")
    def index():
        return render_template("map.html", token=token, size=size)

    @app.route("/<int:z>/<int:x>/<int:y>.png")
    def tile(z, x, y):
        if z != 18:  # serve.py:55-56
            abort(404)
        res = session.get(url_template.format(x=x, y=y, z=z))
        if res.status_code != 200:
            abort(500)
        mask = predictor.segment(Image.open(io.BytesIO(res.content)))
        output = io.BytesIO()
        mask.save(output, format="png", optimize=True)
        output.seek(0)
        return send_file(output, mimetype="image/png")

    @app.after_request
    def after_request(response):
        response.headers["Access-Control-Allow-Origin"] = "*"
        return response

    return app


def main(args):
    import torch

    from robosat_b200.serve import Predictor

    model = load_config(args.model)
    dataset = load_config(args.dataset)
    if model["common"]["cuda"] and not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    token = os.getenv("MAPBOX_ACCESS_TOKEN")
    if not token:
        sys.exit("Error: map token needed visualizing results; export MAPBOX_ACCESS_TOKEN")
    try:
        import flask  # noqa: F401
        import requests
    except ImportError as exc:
        sys.exit("Error: rs serve needs flask and requests for its HTTP shell (%s)" % exc)
    predictor = Predictor(args.checkpoint, model, dataset, tta=args.tta)
    app = make_app(predictor, args.url, token, args.tile_size, session=requests.Session())
    app.run(host=args.host, port=args.port, threaded=False)
