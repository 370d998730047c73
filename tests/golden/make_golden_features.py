"""Golden fixture for `rs features --type parking` from the REAL reference (run in the build container only):

    python tests/golden/make_golden_features.py

Imports the unmodified `robosat.features.parking` / `robosat.features.core` (/root/reference) with three stub modules:
`mercantile.bounds` returns (0, 0, 1, 1), so every ring is the normalised (px / H, 1 - py / W) exactly; `geojson`'s Polygon,
Feature and FeatureCollection are plain dicts; `shapely.geometry.shape(...)` reports every polygon valid. This pins the
morphology, contours, simplification, hierarchy walk and ring order to the reference's own code; only the validity filter and
the real tile bounds are restated in robosat_b200/features.py.

Writes tests/golden/features.npz (per case: `labels<i>`, `class<i>` and the reference's grown mask `grown<i>`) and
tests/golden/features.json (per case: name, tile, shape, the rings of every feature and the warnings printed). The GPU box has no
/root/reference: tests read only these two files.
"""

import contextlib
import io
import json
import os
import sys
import types
from collections import namedtuple

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"

mercantile = types.ModuleType("mercantile")
mercantile.Tile = namedtuple("Tile", ["x", "y", "z"])
mercantile.bounds = lambda tile: (0.0, 0.0, 1.0, 1.0)
geojson = types.ModuleType("geojson")
geojson.Polygon = lambda rings: {"type": "Polygon", "coordinates": rings}
geojson.Feature = lambda geometry: {"type": "Feature", "geometry": geometry, "properties": {}}
geojson.FeatureCollection = lambda features: {"type": "FeatureCollection", "features": features}
shapely = types.ModuleType("shapely")
shapely.geometry = types.ModuleType("shapely.geometry")
shapely.geometry.shape = lambda geometry: types.SimpleNamespace(is_valid=True)
sys.modules.update({"mercantile": mercantile, "geojson": geojson, "shapely": shapely, "shapely.geometry": shapely.geometry})
sys.path.insert(0, REF)

from robosat.features import core  # noqa: E402
from robosat.features.parking import ParkingHandler  # noqa: E402


def _blobs(rng, H, W, n, rmin, rmax):
    m = np.zeros((H, W), np.uint8)
    yy, xx = np.mgrid[:H, :W]
    for _ in range(n):
        cy, cx = rng.randint(0, H), rng.randint(0, W)
        if rng.rand() < 0.5:
            r = rng.randint(rmin, rmax)
            m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 1
        else:
            h, w = rng.randint(rmin, 2 * rmax), rng.randint(rmin, 2 * rmax)
            m[cy:cy + h, cx:cx + w] = 1
    return m


def cases():
    rng = np.random.RandomState(0)
    root = os.path.join(REF, "tests", "fixtures", "parking", "labels")
    out = []
    for z in sorted(os.listdir(root)):
        for x in sorted(os.listdir(os.path.join(root, z))):
            for name in sorted(os.listdir(os.path.join(root, z, x))):
                labels = np.array(Image.open(os.path.join(root, z, x, name)).convert("P"), dtype=np.uint8)
                out.append(("fixture_%s_%s" % (x, name.split(".")[0]), labels, 1))
    out.append(("zeros", np.zeros((512, 512), np.uint8), 1))
    out.append(("ones", np.ones((512, 512), np.uint8), 1))
    holes = np.zeros((512, 512), np.uint8)
    holes[30:480, 20:500] = 1
    for i in range(4):
        for j in range(3):
            holes[60 + 110 * j:60 + 110 * j + 50 + 5 * i, 50 + 110 * i:50 + 110 * i + 45 + 4 * j] = 0
    out.append(("twelve_holes", holes, 1))
    nest = np.zeros((512, 512), np.uint8)
    for k, v in enumerate((1, 0, 1, 0)):
        nest[16 + 60 * k:496 - 60 * k, 16 + 60 * k:496 - 60 * k] = v
    out.append(("nesting_depth_3", nest, 1))
    sliver = np.zeros((1024, 1024), np.uint8)
    sliver[500:521, 5:1019] = 1
    out.append(("sliver", sliver, 1))
    specks = _blobs(rng, 512, 512, 6, 40, 80)
    specks[rng.rand(512, 512) < 0.01] = 1          # specks the opening removes
    specks[200:300, 100:240] = 1
    specks[200:300, 246:400] = 1                    # a 6 px gap the closing bridges
    specks[380:440, 300:400] = 0
    specks[400:420, 320:326] = 1
    out.append(("specks_and_gaps", specks, 1))
    edges = np.zeros((512, 512), np.uint8)
    for cy, cx in ((0, 0), (0, 511), (511, 0), (511, 511), (0, 256), (511, 256), (256, 0), (256, 511)):
        edges[max(cy - 60, 0):cy + 60, max(cx - 60, 0):cx + 60] = 1
    out.append(("edges_and_corners", edges, 1))
    rect = _blobs(rng, 300, 500, 14, 20, 60)
    rect[:, 270:] = 0  # the reference scales px by the row count (core.py:49): columns past H would fail its range assert
    out.append(("rect_300x500", rect, 1))
    six = np.kron(rng.randint(0, 6, size=(8, 8)), np.ones((64, 64), np.int64)).astype(np.uint8)
    six[rng.rand(512, 512) < 0.02] = 3
    out.append(("six_classes", six, 3))
    out.append(("blobs_512", _blobs(rng, 512, 512, 30, 10, 50), 1))
    out.append(("blobs_1024", _blobs(rng, 1024, 1024, 80, 10, 70), 1))
    return out


def main():
    arrays, meta = {}, []
    for i, (name, labels, cls) in enumerate(cases()):
        mask = (labels == cls).astype(np.uint8)  # robosat/tools/features.py:47
        grown = core.grow(core.denoise(mask, ParkingHandler.kernel_size_denoise), ParkingHandler.kernel_size_grow)
        tile = mercantile.Tile(70000 + i, 104000 + i, 18)
        handler = ParkingHandler()
        err = io.StringIO()
        with contextlib.redirect_stderr(err):
            handler.apply(tile, mask)
        rings = [[[list(map(float, pt)) for pt in ring] for ring in f["geometry"]["coordinates"]] for f in handler.features]
        meta.append({"name": name, "tile": list(tile), "shape": list(labels.shape), "rings": rings,
                     "warnings": err.getvalue().splitlines()})
        arrays["labels%d" % i], arrays["class%d" % i], arrays["grown%d" % i] = labels, np.array(cls), grown
        print("%-22s fg %7d -> grown %7d, %d features, %d warnings" % (name, mask.sum(), grown.sum(), len(rings), len(meta[-1]["warnings"])))
    np.savez_compressed(os.path.join(HERE, "features.npz"), **arrays)
    with open(os.path.join(HERE, "features.json"), "w") as fp:
        json.dump(meta, fp)


if __name__ == "__main__":
    main()
