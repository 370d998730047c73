"""rsb_morph_binary and `rs features` on the H100: bit-identical to the numpy restatement / OpenCV, foreground counts, guard bytes,
the golden grown masks, and the tool end to end against the CPU path."""

import argparse
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import features_reference as fr
from robosat_b200 import _lib
from robosat_b200 import features as F
from robosat_b200.tiles import Tile

pytestmark = pytest.mark.gpu


def _labels(rng, N, H, W, classes=3, pad=37):
    """uint8 labels [N][H][W] on the device with an image stride of H*W + pad, and the host copy"""
    host = rng.randint(0, classes, size=(N, H, W)).astype(np.uint8)
    buf = torch.full((N * (H * W + pad) + pad,), 255, dtype=torch.uint8)
    buf.as_strided((N, H, W), (H * W + pad, W, 1)).copy_(torch.from_numpy(host))
    return buf.cuda().as_strided((N, H, W), (H * W + pad, W, 1)), host


def _check(host, cls, ops, got, counts, ref=fr.morph_ref):
    got, counts = got.cpu().numpy(), counts.cpu().numpy()
    for n in range(host.shape[0]):
        want = ref((host[n] == cls).astype(np.uint8), ops)
        assert np.array_equal(got[n], want), n
        assert counts[n] == np.count_nonzero(want), n


@pytest.mark.parametrize("shape", ["rect", "ellipse", "cross"])
@pytest.mark.parametrize("k", [1, 2, 3, 5, 20, 21, 64])
@pytest.mark.parametrize("dilate", [False, True])
def test_single_op_matches_restatement(cuda_device, shape, k, dilate):
    rng = np.random.RandomState(k * 2 + dilate)
    labels, host = _labels(rng, 2, 64, 70)
    ops = [fr.op(shape, k, dilate)]
    out, counts = F.morph_device(labels, 1, ops)
    _check(host, 1, ops, out, counts)


@pytest.mark.parametrize("hw", [(1, 1), (7, 33), (33, 7), (64, 70), (300, 500), (512, 512), (1024, 1024)])
@pytest.mark.parametrize("N", [1, 300])
@pytest.mark.parametrize("k", [3, 20])
def test_open_close_chain_matches_opencv(cuda_device, hw, N, k):
    H, W = hw
    if N == 300 and H * W > 512 * 512:
        N = 40
    rng = np.random.RandomState(H + W + N + k)
    # blocky multi-class labels with speckle, so the chain has real structure to remove and fill
    host = np.kron(rng.randint(0, 4, size=(N, (H + 15) // 16, (W + 15) // 16)), np.ones((1, 16, 16), np.int64))[:, :H, :W].astype(np.uint8)
    host[rng.rand(N, H, W) < 0.05] = 2
    pad = 129
    buf = torch.full((N * (H * W + pad),), 7, dtype=torch.uint8)
    buf.as_strided((N, H, W), (H * W + pad, W, 1)).copy_(torch.from_numpy(host))
    labels = buf.cuda().as_strided((N, H, W), (H * W + pad, W, 1))
    ops = [fr.op("ellipse", k, False), fr.op("ellipse", k, True), fr.op("ellipse", k, True), fr.op("ellipse", k, False)]
    out, counts = F.morph_device(labels, 2, ops)
    _check(host, 2, ops, out, counts, ref=fr.cv_ref if H * W > 64 * 70 else fr.morph_ref)


def test_mixed_chain_with_off_centre_anchors(cuda_device):
    rng = np.random.RandomState(5)
    labels, host = _labels(rng, 3, 97, 130, classes=2)
    ops = [fr.op("rect", 5, False, anchor=(0, 4)), fr.op("cross", 3, True), fr.op("ellipse", 21, True, anchor=(3, 17)),
           fr.op("ellipse", 2, False)]
    out, counts = F.morph_device(labels, 1, ops)
    _check(host, 1, ops, out, counts)
    for nops in (1, 2, 3):
        out, counts = F.morph_device(labels, 1, ops[:nops])
        _check(host, 1, ops[:nops], out, counts)


def test_guard_bytes_stay_untouched(cuda_device):
    rng = np.random.RandomState(9)
    N, H, W, G = 5, 33, 45, 4096
    labels, host = _labels(rng, N, H, W)
    out = torch.full((G + N * H * W + G,), 0xAB, dtype=torch.uint8, device=cuda_device)
    counts = torch.full((N + 64,), -7, dtype=torch.int32, device=cuda_device)
    ops = F.parking_chain(7, 9)
    arr = (_lib.MorphOp * 4)(*[F._op_struct(o) for o in ops])
    _lib.check(_lib.load().rsb_morph_binary(labels.data_ptr(), labels.stride(0), N, H, W, 1, arr, 4, out[G:].data_ptr(), counts[32:].data_ptr(),
                                            _lib.current_stream_ptr()), "rsb_morph_binary")
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert (o[:G] == 0xAB).all() and (o[G + N * H * W:] == 0xAB).all()
    c = counts.cpu().numpy()
    assert (c[:32] == -7).all() and (c[32 + N:] == -7).all()
    _check(host, 1, ops, torch.from_numpy(o[G:G + N * H * W].reshape(N, H, W)), torch.from_numpy(c[32:32 + N]))


def test_golden_grown_masks_are_bit_identical(cuda_device):
    for case in fr.load_golden():
        labels = torch.from_numpy(case["labels"][None].copy()).to(cuda_device)
        out, counts = F.morph_device(labels, case["class"], F.parking_chain())
        assert np.array_equal(out[0].cpu().numpy(), case["grown"]), case["name"]
        assert int(counts[0]) == int(case["grown"].sum()), case["name"]


def _write_dataset(tmp_path):
    path = tmp_path / "dataset.toml"
    path.write_text("[common]\nclasses = ['background', 'parking', 'a', 'b', 'c', 'd']\ncolors = ['denim', 'orange']\n")
    return str(path)


def _write_masks(root, cases):
    palette = [v for i in range(256) for v in (i, 255 - i, (7 * i) % 256)]
    for tile, labels in cases:
        d = os.path.join(root, str(tile.z), str(tile.x))
        os.makedirs(d, exist_ok=True)
        im = Image.fromarray(labels, mode="P")
        im.putpalette(palette)
        im.save(os.path.join(d, "%d.png" % tile.y))


def _run(tmp_path, masks, batch):
    from robosat_b200.tools import features as tool

    out = str(tmp_path / ("out_%d.geojson" % batch))
    tool.main(argparse.Namespace(masks=masks, type="parking", dataset=_write_dataset(tmp_path), out=out), batch=batch)
    with open(out) as fp:
        return json.load(fp)


def test_tool_matches_cpu_path_in_tile_order(cuda_device, tmp_path):
    golden = fr.load_golden()
    cases = []
    for i, case in enumerate(golden):
        # class 1 is parking: remap the 6-class case's selected class onto it
        labels = case["labels"] if case["class"] == 1 else np.where(case["labels"] == case["class"], 1, (case["labels"] == 1) * 2).astype(np.uint8)
        # x descending with i, so the (z, x, y) order differs from the golden's order and from listing order
        cases.append((Tile(70100 - i, 104000 + (i % 3), 18), labels))
    masks = str(tmp_path / "masks")
    _write_masks(masks, cases)
    want = []
    for tile, labels in sorted(cases, key=lambda c: (c[0].z, c[0].x, c[0].y)):
        want.extend(fr.cpu_features(tile, labels, 1)[0])
    assert len(want) > 30
    for batch in (64, 3):
        got = _run(tmp_path, masks, batch)
        assert got["type"] == "FeatureCollection"
        assert got["features"] == json.loads(json.dumps(want)), batch


def test_tool_empty_inputs(cuda_device, tmp_path):
    empty = tmp_path / "empty"
    empty.mkdir()
    assert _run(tmp_path, str(empty), 64) == {"type": "FeatureCollection", "features": []}
    zeros = str(tmp_path / "zeros")
    _write_masks(zeros, [(Tile(5 + i, 9, 18), np.zeros((256, 256), np.uint8)) for i in range(5)])
    assert _run(tmp_path, zeros, 2) == {"type": "FeatureCollection", "features": []}
