"""Golden fixture for `rs compare` from the REAL reference (run in the build container only):

    python tests/golden/make_golden_compare.py

Writes seeded tiles plus two of the reference's parking fixtures, runs the unmodified `robosat.tools.compare.main`
(/root/reference/robosat/tools/compare.py) on them with several mask sets and thresholds, and stores in tests/golden/compare.npz:
every input file's bytes ("file:<path>"), each case's arguments and the files it wrote ("case<i>:args", JSON), and each written
file's decoded pixels ("case<i>:<path>"; for the 512 x 512 parking tiles their SHA-256 instead, "case<i>:sha256:<path>").

The inputs pin the decoding cases the port must reproduce:
  images: RGB, RGBA (alpha dropped), gray, palette PNG, JPEG and WebP;
  labels: 1-bit palette PNGs as PIL writes them with optimize=True, and an 8-bit one;
  masks: the `rs masks` palette (1-bit), a PLTE shorter than the largest index, a tRNS chunk, an L-mode mask, an RGB mask
  (PIL's quantiser), a 4-bit palette and 8-bit 256-entry palettes;
  thresholds that drop tiles, with one coverage exactly equal to --minimum and another exactly equal to --maximum.
The GPU box has no /root/reference: tests read only the npz.
"""

import argparse
import hashlib
import io
import json
import os
import struct
import sys
import tempfile
import types
import zlib
from collections import namedtuple

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
shim = types.ModuleType("mercantile")
shim.Tile = namedtuple("Tile", ["x", "y", "z"])
sys.modules["mercantile"] = shim
sys.path.insert(0, "/root/reference")

from robosat.colors import continuous_palette_for_color, make_palette  # noqa: E402
from robosat.tools import compare as ref_compare  # noqa: E402

PARKING = "/root/reference/tests/fixtures/parking"
PARKING_TILES = [("18", "70761", "104120"), ("18", "70762", "104119")]
SIZE = 64


def raw_png(a, ctype, plte=None, trns=None):
    """8-bit PNG written chunk by chunk, so that palettes PIL would pad or remap can be stored as they are"""
    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d))

    h, w = a.shape[:2]
    raw = b"".join(b"\0" + a[y].tobytes() for y in range(h))
    s = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, ctype, 0, 0, 0))
    if plte is not None:
        s += chunk(b"PLTE", bytes(plte))
    if trns is not None:
        s += chunk(b"tRNS", bytes(trns))
    return s + chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b"")


def pil_bytes(im, fmt="PNG", **kw):
    b = io.BytesIO()
    im.save(b, format=fmt, **kw)
    return b.getvalue()


def p_image(a, palette):
    im = Image.fromarray(a.astype(np.uint8), mode="P")
    im.putpalette(palette)
    return im


def exact(rng, shape, k, values=(1,)):
    """uint8 plane with exactly k non-zero pixels drawn from `values`"""
    a = np.zeros(int(np.prod(shape)), np.uint8)
    idx = rng.permutation(a.size)[:k]
    a[idx] = rng.choice(np.asarray(values, np.uint8), size=k)
    return a.reshape(shape)


def smooth_rgb(rng, h, w, channels=3):
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 4 + c * 40 + yy * 2) % 256 for c in range(channels)], axis=-1)
    return np.clip(base + rng.randint(-2, 3, size=base.shape), 0, 255).astype(np.uint8)


def seeded_files(rng):
    """{relative path: bytes} of the seeded tiles"""
    files = {}
    mask_pal = make_palette("denim", "orange")
    label_pal = [0, 0, 0, 250, 0, 0]
    cont = continuous_palette_for_color("pink", 256)
    hw = SIZE * SIZE
    # (x, y, size, image kind, m0 non-zero count)
    tiles = [(10, 20, (SIZE, SIZE), "rgb", hw // 4), (10, 21, (SIZE, SIZE), "rgba", 3 * hw // 4), (10, 22, (SIZE, SIZE), "gray", 4 * hw // 5),
             (11, 20, (SIZE, SIZE), "jpeg", hw // 10), (11, 23, (SIZE, SIZE), "palette", 0), (12, 5, (47, 61), "rgb", 1400),
             (12, 6, (SIZE, SIZE), "rgb", 3 * hw // 10)]
    for i, (x, y, (h, w), kind, k0) in enumerate(tiles):
        name = "18/%d/%d" % (x, y)
        if kind == "rgb":
            files["images/%s.png" % name] = pil_bytes(Image.fromarray(smooth_rgb(rng, h, w), "RGB"))
        elif kind == "rgba":
            files["images/%s.png" % name] = pil_bytes(Image.fromarray(smooth_rgb(rng, h, w, 4), "RGBA"))
        elif kind == "gray":
            files["images/%s.png" % name] = pil_bytes(Image.fromarray(smooth_rgb(rng, h, w)[..., 0], "L"))
        elif kind == "jpeg":
            files["images/%s.jpg" % name] = pil_bytes(Image.fromarray(smooth_rgb(rng, h, w), "RGB"), "JPEG", quality=90)
        else:
            files["images/%s.png" % name] = pil_bytes(p_image(rng.randint(0, 256, size=(h, w)), cont), optimize=True)
        # labels: 1-bit palette as `rs rasterize` writes them, one 8-bit label with a 3-entry palette
        lab = exact(rng, (h, w), rng.randint(0, h * w // 2))
        if i == 6:
            files["labels/%s.png" % name] = raw_png(lab * rng.randint(1, 3, size=lab.shape).astype(np.uint8), 3, plte=[0, 0, 0, 9, 200, 30, 250, 0, 0])
        else:
            files["labels/%s.png" % name] = pil_bytes(p_image(lab, label_pal), optimize=True)
        # m0: the `rs masks` palette, exact coverages
        files["m0/%s.png" % name] = pil_bytes(p_image(exact(rng, (h, w), k0), mask_pal), optimize=True)
        # m1: one decoding case per tile
        m1 = exact(rng, (h, w), rng.randint(0, h * w), values=(1, 2, 3))
        if i == 0:  # PLTE of 2 entries, indices up to 3
            files["m1/%s.png" % name] = raw_png(m1, 3, plte=[0, 0, 0, 255, 128, 0])
        elif i == 1:  # tRNS
            files["m1/%s.png" % name] = raw_png(m1, 3, plte=[5, 5, 5, 40, 80, 120, 200, 10, 10, 0, 255, 0], trns=[0, 128])
        elif i == 2:  # L mode
            files["m1/%s.png" % name] = pil_bytes(Image.fromarray(m1 * 60, "L"))
        elif i == 3:  # RGB: PIL's convert("P") quantises it
            files["m1/%s.png" % name] = pil_bytes(Image.fromarray(smooth_rgb(rng, h, w) * (m1[..., None] > 0), "RGB"))
        elif i == 4:
            files["m1/%s.png" % name] = pil_bytes(p_image(m1 > 0, mask_pal), optimize=True)
        elif i == 5:  # 10-entry palette: PIL writes 4 bits per pixel
            files["m1/%s.png" % name] = pil_bytes(p_image(rng.randint(0, 10, size=(h, w)) * (m1 > 0), cont[:30]), optimize=True)
        else:
            files["m1/%s.png" % name] = pil_bytes(p_image(m1 * 80, cont), optimize=True)
        # m2: 8-bit, 256-entry palette
        files["m2/%s.png" % name] = pil_bytes(p_image(exact(rng, (h, w), rng.randint(0, h * w), values=range(1, 256)), cont))
    return files


def parking_files():
    files = {}
    for z, x, y in PARKING_TILES:
        for kind, ext in (("images", "webp"), ("labels", "png")):
            with open(os.path.join(PARKING, kind, z, x, "%s.%s" % (y, ext)), "rb") as fp:
                files["parking/%s/%s/%s/%s.%s" % (kind, z, x, y, ext)] = fp.read()
        # the labels are also the masks: a perfect prediction
        files["parking/masks/%s/%s/%s.png" % (z, x, y)] = files["parking/labels/%s/%s/%s.png" % (z, x, y)]
    return files


# (images, labels, masks, minimum, maximum): coverages of m0 are 0.25, 0.75, 0.8, 0.1, 0, ~0.49 and 0.3
CASES = [
    ("images", "labels", ["m0"], 0.25, 0.75),
    ("images", "labels", ["m0", "m1", "m2"], 0.4, 0.5),
    ("images", "labels", ["m2", "m1"], 0.0, 1.0),
    ("parking/images", "parking/labels", ["parking/masks"], 0.22, 1.0),
]


def main():
    rng = np.random.RandomState(0)
    files = seeded_files(rng)
    files.update(parking_files())
    out = {"file:" + k: np.frombuffer(v, np.uint8) for k, v in files.items()}
    with tempfile.TemporaryDirectory() as tmp:
        for rel, data in files.items():
            os.makedirs(os.path.dirname(os.path.join(tmp, rel)), exist_ok=True)
            with open(os.path.join(tmp, rel), "wb") as fp:
                fp.write(data)
        for ci, (images, labels, masks, lo, hi) in enumerate(CASES):
            dest = os.path.join(tmp, "out%d" % ci)
            ref_compare.main(argparse.Namespace(out=dest, images=os.path.join(tmp, images), labels=os.path.join(tmp, labels),
                                                masks=[os.path.join(tmp, m) for m in masks], minimum=lo, maximum=hi))
            written = sorted(os.path.relpath(os.path.join(d, f), dest) for d, _, fs in os.walk(dest) for f in fs)
            out["case%d:args" % ci] = np.array(json.dumps({"images": images, "labels": labels, "masks": masks, "minimum": lo, "maximum": hi,
                                                           "written": written}))
            for rel in written:
                px = np.asarray(Image.open(os.path.join(dest, rel)))
                if images.startswith("parking"):
                    out["case%d:sha256:%s" % (ci, rel)] = np.array(hashlib.sha256(px.tobytes()).hexdigest() + " %s" % (px.shape,))
                else:
                    out["case%d:%s" % (ci, rel)] = px
            print("case %d: %d of %d tiles written" % (ci, len(written), sum(1 for k in files if k.startswith(images + "/"))))
    np.savez_compressed(os.path.join(HERE, "compare.npz"), **out)
    print("wrote compare.npz: %d arrays, %d bytes" % (len(out), os.path.getsize(os.path.join(HERE, "compare.npz"))))


if __name__ == "__main__":
    main()
