"""`rs compare` on the CPU: the flags, the numpy restatement against the reference's own output (tests/golden/compare.npz), the
indexed PNG reader against PIL, the RGB PNG writer, the checks that run before anything is written, and the CSV format."""

import argparse
import ctypes
import collections
import hashlib
import io
import json
import os
import struct
import sys
import zlib

import numpy as np
import pytest
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import compare_reference as R  # noqa: E402

from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import compare as C  # noqa: E402
from robosat_b200.tools import compare as tool  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "compare.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def cases(golden):
    i = 0
    while "case%d:args" % i in golden.files:
        yield i, json.loads(str(golden["case%d:args" % i]))
        i += 1


def test_parser_matches_the_reference():
    parser = argparse.ArgumentParser()
    tool.add_parser(parser.add_subparsers())
    sub = parser._subparsers._group_actions[0].choices["compare"]
    acts = {a.dest: a for a in sub._actions}
    for dest, help_ in (("out", "directory to save visualizations to"), ("images", "directory to read slippy map images from"),
                        ("labels", "directory to read slippy map labels from"), ("masks", "slippy map directories to read masks from")):
        assert acts[dest].help == help_ and not acts[dest].option_strings
    assert acts["masks"].nargs == "+"
    assert [a.dest for a in sub._actions if not a.option_strings] == ["out", "images", "labels", "masks"]
    assert acts["minimum"].default == 0.0 and acts["minimum"].type is float and acts["minimum"].help == "minimum percentage of mask not background"
    assert acts["maximum"].default == 1.0 and acts["maximum"].type is float and acts["maximum"].help == "maximum percentage of mask not background"
    assert acts["csv"].default is None
    args = sub.parse_args(["o", "i", "l", "m1", "m2", "--minimum", "0.1"])
    assert args.masks == ["m1", "m2"] and args.minimum == 0.1 and args.maximum == 1.0 and args.csv is None


def test_restatement_reproduces_the_reference(golden, tmp_path):
    R.materialize(golden, str(tmp_path))
    checked = 0
    for ci, a in cases(golden):
        root = str(tmp_path)
        got, rows = R.compare(os.path.join(root, a["images"]), os.path.join(root, a["labels"]),
                              [os.path.join(root, m) for m in a["masks"]], a["minimum"], a["maximum"], R.golden_tiles(root, a["images"]))
        assert sorted(got) == a["written"], ci
        for rel, px in got.items():
            if "case%d:%s" % (ci, rel) in golden.files:
                assert np.array_equal(px, golden["case%d:%s" % (ci, rel)]), (ci, rel)
            else:
                assert str(golden["case%d:sha256:%s" % (ci, rel)]) == hashlib.sha256(px.tobytes()).hexdigest() + " %s" % (px.shape,), (ci, rel)
            checked += 1
    assert checked >= 10


def test_golden_pins_the_threshold_edges(golden):
    """one kept tile's coverage equals --minimum exactly and another's equals --maximum (case 0)"""
    a = dict(cases(golden))[0]
    covs = []
    for key in golden.files:
        if key.startswith("file:m0/"):
            plane, _ = R.load_indexed(golden[key].tobytes())
            covs.append(R.coverage(plane))
    assert a["minimum"] in covs and a["maximum"] in covs
    assert len(a["written"]) < len(covs)


def decode_indexed(data, w, h):
    plane = np.zeros((h, w), np.uint8)
    pal = np.zeros((256, 3), np.uint8)
    entries = ctypes.c_int32()
    rc = _lib.load().rsb_png_decode_indexed(data, len(data), plane.ctypes.data, pal.ctypes.data, ctypes.byref(entries), w, h)
    return rc, plane, pal, entries.value


def test_indexed_decoder_matches_pil_on_the_fixtures(golden):
    n = 0
    for key in golden.files:
        if not key.startswith("file:") or not key.endswith(".png") or key.startswith("file:images/") or "/images/" in key:
            continue
        data = golden[key].tobytes()
        im = Image.open(io.BytesIO(data))
        w, h = im.size
        rc, plane, pal, entries = decode_indexed(data, w, h)
        ref_plane, ref_lut = R.load_indexed(data)
        if im.mode in ("P", "L"):
            assert rc == 0, (key, _lib.last_error())
            assert np.array_equal(plane, ref_plane) and np.array_equal(pal, ref_lut), key
            assert entries == (256 if im.mode == "L" else len(im.getpalette()) // 3)
            n += 1
        else:
            assert rc == _lib.RSB_E_UNSUPPORTED, key  # the RGB mask goes to PIL
    assert n >= 20


def _filtered(rows, filters, bpp):
    """PNG scanlines of `rows` (uint8 arrays), row y filtered with filters[y % len(filters)] (0-4)"""
    out, prev = [], np.zeros(len(rows[0]), np.int32)
    for y, row in enumerate(rows):
        ft = filters[y % len(filters)]
        r = row.astype(np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), r[:-bpp]])
        upleft = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]])
        if ft == 0:
            f = r
        elif ft == 1:
            f = r - left
        elif ft == 2:
            f = r - prev
        elif ft == 3:
            f = r - (left + prev) // 2
        else:
            p = left + prev - upleft
            pa, pb, pc = abs(p - left), abs(p - prev), abs(p - upleft)
            f = r - np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, prev, upleft))
        out.append(bytes([ft]) + (f & 255).astype(np.uint8).tobytes())
        prev = r
    return b"".join(out)


def _png(plane, depth, ctype, plte, filters):
    h, w = plane.shape
    rows = []
    for y in range(h):
        if depth == 8:
            rows.append(plane[y])
        else:
            per = 8 // depth
            padded = np.zeros(-(-w // per) * per, np.uint8)
            padded[:w] = plane[y]
            packed = np.zeros(len(padded) // per, np.uint8)
            for k in range(per):
                packed |= padded[k::per] << (8 - depth * (k + 1))
            rows.append(packed)
    raw = _filtered(rows, filters, 1)

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d))

    s = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, 0))
    if plte is not None:
        s += chunk(b"PLTE", bytes(plte))
    return s + chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b"")


@pytest.mark.parametrize("depth", [1, 2, 4, 8])
def test_indexed_decoder_matches_pil_on_seeded_pngs(depth):
    rng = np.random.RandomState(depth)
    for entries in sorted({1, 2, 3, 1 << depth, min(256, (1 << depth) + 5), 256} - {0}):
        for w, h in ((1, 1), (37, 23), (64, 5)):
            plane = rng.randint(0, 1 << depth, size=(h, w)).astype(np.uint8)
            plte = rng.randint(0, 256, size=3 * entries).astype(np.uint8).tolist()
            data = _png(plane, depth, 3, plte, [0, 1, 2, 3, 4])
            rc, got, pal, n = decode_indexed(data, w, h)
            ref_plane, ref_lut = R.load_indexed(data)
            assert rc == 0, _lib.last_error()
            assert np.array_equal(got, plane) and np.array_equal(got, ref_plane), (depth, entries, w, h)
            assert np.array_equal(pal, ref_lut) and n == entries
    if depth == 8:  # gray: index = value, the gray ramp
        plane = rng.randint(0, 256, size=(23, 37)).astype(np.uint8)
        data = _png(plane, 8, 0, None, [4, 3, 2, 1, 0])
        rc, got, pal, n = decode_indexed(data, 37, 23)
        ref_plane, ref_lut = R.load_indexed(data)
        assert rc == 0 and np.array_equal(got, ref_plane) and np.array_equal(pal, ref_lut) and n == 256


def test_indexed_decoder_rejects_what_it_does_not_handle():
    rgb = np.zeros((4, 4, 3), np.uint8)
    buf = io.BytesIO()
    Image.fromarray(rgb).save(buf, format="PNG")
    assert decode_indexed(buf.getvalue(), 4, 4)[0] == _lib.RSB_E_UNSUPPORTED
    buf = io.BytesIO()
    Image.fromarray(rgb).save(buf, format="JPEG")
    assert decode_indexed(buf.getvalue(), 4, 4)[0] == _lib.RSB_E_UNSUPPORTED
    data = _png(np.zeros((4, 4), np.uint8), 8, 3, [1, 2, 3], [0])
    assert decode_indexed(data, 5, 4)[0] == -1 and "expected 5x4" in _lib.last_error()


@pytest.mark.parametrize("w,h", [(1, 1), (61, 47), (192, 64)])
def test_rgb_encoder_round_trips_through_pil(w, h, tmp_path):
    rng = np.random.RandomState(w)
    smooth = np.stack(np.meshgrid(np.arange(w), np.arange(h)), -1).sum(-1)[..., None] * np.array([1, 2, 3])
    for pixels in ((smooth % 256).astype(np.uint8), rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)):
        cap = pixels.size + h + 4096 + pixels.size // 512
        buf = np.empty(cap, np.uint8)
        n = _lib.load().rsb_png_encode_rgb8(pixels.ctypes.data, w, h, 6, buf.ctypes.data, cap)
        assert n > 0, _lib.last_error()
        im = Image.open(io.BytesIO(buf[:n].tobytes()))
        assert im.mode == "RGB" and np.array_equal(np.asarray(im), pixels)
    batch = np.ascontiguousarray(np.stack([pixels, pixels[::-1]]))
    paths = [str(tmp_path / "18" / "3" / "4.png"), str(tmp_path / "18" / "5" / "6.png")]
    C.write_composites(paths, batch.reshape(2, -1), (w, h), 1, 2)
    for p, px in zip(paths, batch):
        assert np.array_equal(np.asarray(Image.open(p)), px)


def _tiles(root, sizes):
    for name, (w, h) in sizes.items():
        os.makedirs(os.path.join(root, os.path.dirname(name)), exist_ok=True)
        Image.fromarray(np.zeros((h, w), np.uint8), "P").save(os.path.join(root, name))


def test_checks_fail_before_anything_is_written(tmp_path):
    root = str(tmp_path)
    _tiles(root, {"img/18/1/1.png": (8, 8), "img/18/1/2.png": (8, 8), "lab/18/1/1.png": (8, 8), "lab/18/1/2.png": (8, 8),
                  "m/18/1/1.png": (8, 8), "m/18/1/2.png": (8, 6)})
    out = os.path.join(root, "out")
    with pytest.raises(C.CompareError, match=r"tile 18/1/2: .*m/18/1/2.png is 8x6, the image .* is 8x8"):
        C.compare_device(os.path.join(root, "img"), os.path.join(root, "lab"), [os.path.join(root, "m")], out)
    assert not os.path.exists(out)
    os.remove(os.path.join(root, "lab/18/1/2.png"))
    with pytest.raises(C.CompareError, match=r"tile 18/1/2: .*lab/18/1/2.png does not exist"):
        C.compare_device(os.path.join(root, "img"), os.path.join(root, "lab"), [os.path.join(root, "m")], out, csv=os.path.join(root, "a.csv"))
    assert not os.path.exists(out) and not os.path.exists(os.path.join(root, "a.csv"))


def test_csv_format(tmp_path):
    Tile = collections.namedtuple("Tile", ["x", "y", "z"])
    batch = [C.Job(Tile(3, 4, 18), "", "", ["", ""], (4, 4))]
    counts = np.array([[[2, 1, 3, 10], [0, 0, 5, 11]]], np.int64)
    rows = C.csv_rows(batch, counts, (counts[..., 0] + counts[..., 1]) / np.int64(16))
    path = str(tmp_path / "c.csv")
    C.write_csv(path, rows + C.csv_rows(batch, np.zeros((1, 2, 4), np.int64), np.zeros((1, 2))))
    lines = open(path).read().splitlines()
    assert lines[0] == "z,x,y,mask,coverage,tp,fp,fn,tn,fg_iou"
    assert lines[1] == "18,3,4,0,0.1875,2,1,3,10,0.3333333333333333"
    assert lines[2] == "18,3,4,1,0.0,0,0,5,11,0.0"
    assert lines[3] == "18,3,4,0,0.0,0,0,0,0,"  # tp + fp + fn = 0: no IoU


def test_batches_follow_size_and_budget():
    Tile = collections.namedtuple("Tile", ["x", "y", "z"])
    jobs = [C.Job(Tile(i, 0, 18), "", "", [""], s) for i, s in enumerate([(8, 8)] * 5 + [(9, 8)] * 2 + [(8, 8)])]
    per = C.tile_bytes((8, 8), 1, False)
    assert [len(b) for b in C.batches(jobs, 1, False, 2 * per)] == [2, 2, 1, 1, 1, 1]  # a 9 x 8 tile needs more than per
    assert [len(b) for b in C.batches(jobs, 1, False, 1)] == [1] * 8
    assert [len(b) for b in C.batches(jobs, 1, False, 1 << 30)] == [5, 2, 1]
