"""Regenerate tests/golden/jpeg.npz: seeded JPEG streams encoded by PIL (libjpeg-turbo) and PIL's decodes of them, so the numpy
restatement (tests/jpeg_reference.py) is pinned to libjpeg-turbo on machines whose Pillow differs.

    python tests/golden/make_golden_jpeg.py
"""

import io
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import jpeg_tiff_writer as jw  # noqa: E402

CASES = [  # (H, W, spp, photometric, encode settings)
    (1, 1, 3, 6, dict(quality=75, subsampling=2)),
    (7, 13, 3, 6, dict(quality=90, subsampling=2, restart_marker_blocks=1)),
    (17, 33, 3, 6, dict(quality=50, subsampling=1, optimize=True)),
    (150, 200, 3, 6, dict(quality=75, subsampling=2, restart_marker_blocks=7)),
    (257, 255, 3, 6, dict(quality=95, subsampling=2, restart_marker_rows=1)),
    (64, 48, 3, 6, dict(quality=10, subsampling=0)),
    (33, 29, 3, 2, dict(quality=85)),
    (45, 37, 1, 1, dict(quality=60, restart_marker_blocks=5)),
    (4, 4, 3, 6, dict(quality=100, subsampling=2)),
    (5, 3, 3, 6, dict(quality=80, subsampling=1)),
]


def main():
    out = {}
    for i, (H, W, spp, photometric, kw) in enumerate(CASES):
        s = jw.encode(jw.image(H, W, spp, seed=i), photometric, **kw)
        px = np.asarray(Image.open(io.BytesIO(s)))
        out["stream_%d" % i] = np.frombuffer(s, np.uint8)
        out["pixels_%d" % i] = px.reshape(H, W, spp)
        out["layout_%d" % i] = np.array([spp, photometric], np.int64)
    np.savez_compressed(os.path.join(HERE, "jpeg.npz"), **out)


if __name__ == "__main__":
    main()
