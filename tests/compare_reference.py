"""numpy restatement of `rs compare` (robosat/tools/compare.py), the rule the device path is checked against.

Decoding is PIL's, as in the reference: the image is `convert("RGB")`, the label and masks `convert("P")`. A P plane is expanded
through its own palette, entries past the palette black (what `paste` does when it converts P to RGB). Coverage of a mask is
`np.sum(mask != 0) / np.prod(image.size)` in float64; a tile is kept when any mask's coverage p has minimum <= p <= maximum.
"""

import io
import os

import numpy as np
from PIL import Image


def open_any(src):
    return Image.open(io.BytesIO(src) if isinstance(src, (bytes, bytearray)) else src)


def load_rgb(src):
    return np.asarray(open_any(src).convert("RGB"), dtype=np.uint8)


def load_indexed(src):
    """-> (index plane uint8 [H, W], colour table uint8 [256, 3])"""
    im = open_any(src).convert("P")
    lut = np.zeros((256, 3), np.uint8)
    pal = np.asarray(im.getpalette() or [], np.uint8)[:768]
    lut.reshape(-1)[:len(pal)] = pal
    return np.asarray(im, dtype=np.uint8), lut


def coverage(mask):
    return np.sum(mask != 0) / np.prod((mask.shape[1], mask.shape[0]))


def confusion(mask, label):
    """(tp, fp, fn, tn) of mask against label, foreground = index != 0"""
    m, l = mask != 0, label != 0
    return int(np.sum(m & l)), int(np.sum(m & ~l)), int(np.sum(~m & l)), int(np.sum(~m & ~l))


def keep(coverages, minimum, maximum):
    return any(minimum <= p <= maximum for p in coverages)


def compose(image, planes, luts):
    """image | lut_0[plane_0] | lut_1[plane_1] | ... as uint8 [H, (1 + P) * W, 3]"""
    return np.concatenate([image] + [lut[p] for p, lut in zip(planes, luts)], axis=1)


def compare(images, labels, masks, minimum, maximum, tiles):
    """tiles: [(z, x, y, image path)] -> ({"z/x/y.png": composite} of the kept tiles, [CSV row values] of every (tile, mask))"""
    out, rows = {}, []
    for z, x, y, path in tiles:
        image = load_rgb(path)
        label, label_lut = load_indexed(os.path.join(labels, str(z), str(x), "%d.png" % y))
        planes = [load_indexed(os.path.join(d, str(z), str(x), "%d.png" % y)) for d in masks]
        covs = [coverage(p) for p, _ in planes]
        for m, ((p, _), cov) in enumerate(zip(planes, covs)):
            tp, fp, fn, tn = confusion(p, label)
            rows.append([z, x, y, m, float(cov), tp, fp, fn, tn, tp / (tp + fp + fn) if tp + fp + fn else None])
        if keep(covs, minimum, maximum):
            out["%d/%d/%d.png" % (z, x, y)] = compose(image, [label] + [p for p, _ in planes], [label_lut] + [lut for _, lut in planes])
    return out, rows


def materialize(golden, root):
    """write the input files of tests/golden/compare.npz under `root`"""
    for key in golden.files:
        if key.startswith("file:"):
            path = os.path.join(root, key[len("file:"):])
            os.makedirs(os.path.dirname(path), exist_ok=True)
            with open(path, "wb") as fp:
                fp.write(golden[key].tobytes())


def golden_tiles(root, images):
    """[(z, x, y, path)] of an image directory in (z, x, y) order"""
    found = []
    for z in os.listdir(os.path.join(root, images)):
        for x in os.listdir(os.path.join(root, images, z)):
            for name in os.listdir(os.path.join(root, images, z, x)):
                found.append((int(z), int(x), int(os.path.splitext(name)[0]), os.path.join(root, images, z, x, name)))
    return sorted(found)
