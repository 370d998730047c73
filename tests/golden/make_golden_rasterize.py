"""Golden fixture for `rs rasterize` from the reference's parking fixtures (run in the build container only):

    python tests/golden/make_golden_rasterize.py

Copies, as data only, `tests/fixtures/parking/features.geojson` (2 polygons), `tiles.csv` (4 tiles at z18) and the 4 label
masks `labels/18/x/y.png` (512², GDAL's rasterization of those polygons) of the reference checkout at /root/reference into
tests/golden/rasterize.json (features, tiles, labelled tiles) and tests/golden/rasterize.npz (`mask_x_y_z`, uint8 {0, 1}).
The GPU box has no /root/reference: tests read only these two files.
"""

import csv
import json
import os

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/tests/fixtures/parking"


def main():
    with open(os.path.join(SRC, "features.geojson")) as fp:
        features = json.load(fp)
    with open(os.path.join(SRC, "tiles.csv")) as fp:
        tiles = [[int(v) for v in row] for row in csv.reader(fp) if row]
    arrays, labelled = {}, []
    root = os.path.join(SRC, "labels")
    for z in sorted(os.listdir(root)):
        for x in sorted(os.listdir(os.path.join(root, z))):
            for name in sorted(os.listdir(os.path.join(root, z, x))):
                y = int(name.split(".")[0])
                im = Image.open(os.path.join(root, z, x, name))
                assert im.mode == "P", im.mode
                mask = np.array(im, dtype=np.uint8)
                assert set(np.unique(mask)) <= {0, 1}
                arrays["mask_%d_%d_%d" % (int(x), y, int(z))] = mask
                labelled.append([int(x), y, int(z)])
                print("%s/%s/%d: %d foreground pixels" % (z, x, y, int(mask.sum())))
    np.savez_compressed(os.path.join(HERE, "rasterize.npz"), **arrays)
    with open(os.path.join(HERE, "rasterize.json"), "w") as fp:
        json.dump({"features": features, "tiles": tiles, "labelled": labelled}, fp)


if __name__ == "__main__":
    main()
