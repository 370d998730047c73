"""Test-time augmentation on the H100: the head kernels against their numpy restatement (tests/tta_reference.py), exactly; the
network chain (`TilePredictor`, `SegmentEngine`, `rs predict --tta`) against the oracle averaged over the same views."""

import argparse
import ctypes
import os

import numpy as np
import pytest
import torch
from PIL import Image

import tta_reference as ref
from oracle import unet_oracle
from robosat_b200 import _lib, synth, tta
from robosat_b200.datasets import BufferedSlippyMapDirectory
from robosat_b200.transforms import ImageToUint8Tensor

pytestmark = pytest.mark.gpu

ANCHORS = np.linspace(0, 1, 256)


def _softmax_dev(logits_d):
    """device probabilities from rsb_softmax_nchw, whose expf / sum / division are the head's"""
    N, C, H, W = logits_d.shape
    probs = torch.empty_like(logits_d)
    _lib.check(_lib.load().rsb_softmax_nchw(logits_d.data_ptr(), probs.data_ptr(), N, C, H * W, _lib.current_stream_ptr()), "softmax")
    return probs


def _accumulate(logits_d, acc, ops, B, C, H, W, o, accumulate=0):
    arr = (ctypes.c_int32 * len(ops))(*ops)
    _lib.check(_lib.load().rsb_head_tta_accumulate(logits_d.data_ptr(), acc.data_ptr(), arr, len(ops), B, C, H, W, o, accumulate,
                                                   _lib.current_stream_ptr()), "rsb_head_tta_accumulate")


def _tta_quantize(acc, B, views):
    OH, OW = acc.shape[2], acc.shape[3]
    q = torch.empty((B, OH, OW), dtype=torch.uint8, device=acc.device)
    _lib.check(_lib.load().rsb_head_tta_quantize(acc.data_ptr(), q.data_ptr(), B, OH * OW, views, _lib.current_stream_ptr()), "tta_quantize")
    return q


def _tta_argmax(acc, B, C):
    OH, OW = acc.shape[2], acc.shape[3]
    m = torch.empty((B, OH, OW), dtype=torch.uint8, device=acc.device)
    _lib.check(_lib.load().rsb_head_tta_argmax(acc.data_ptr(), m.data_ptr(), B, C, OH * OW, _lib.current_stream_ptr()), "tta_argmax")
    return m


def _spatial(a, op):
    """ref.view on the two trailing (spatial) axes of [..., H, W]"""
    return np.ascontiguousarray(np.moveaxis(ref.view(np.moveaxis(a, (-2, -1), (0, 1)), op), (0, 1), (-2, -1)))


@pytest.mark.parametrize("C", [2, 3, 6, 20])  # 32x32, 16x16 and 8x8 staging windows
def test_head_matches_numpy(C, cuda_device):
    B, S, o, ops = 2, 96, 16, tuple(range(8))
    g = torch.Generator().manual_seed(C)
    logits = torch.randn((8 * B, C, S, S), generator=g) * 4
    d = logits.to(cuda_device)
    probs = _softmax_dev(d).cpu().numpy()
    assert np.abs(probs - ref.softmax(logits.numpy())).max() < 1e-6
    acc = torch.full((B, C, S - 2 * o, S - 2 * o), 12345, dtype=torch.int64, device=cuda_device)  # accumulate=0 overwrites
    _accumulate(d, acc, ops, B, C, S, S, o)
    want = ref.accumulate(probs, ops, B, o)
    assert np.array_equal(acc.cpu().numpy(), want)
    assert np.array_equal(_tta_argmax(acc, B, C).cpu().numpy(), ref.argmax(want))
    if C == 2:
        assert np.array_equal(_tta_quantize(acc, B, 8).cpu().numpy(), ref.quantize(want, 8))


def test_head_flip_on_a_rectangle(cuda_device):
    B, C, H, W, o, ops = 2, 3, 64, 96, 8, (0, 1)
    logits = torch.randn((2 * B, C, H, W), generator=torch.Generator().manual_seed(5)) * 4
    d = logits.to(cuda_device)
    probs = _softmax_dev(d).cpu().numpy()
    acc = torch.empty((B, C, H - 2 * o, W - 2 * o), dtype=torch.int64, device=cuda_device)
    _accumulate(d, acc, ops, B, C, H, W, o)
    assert np.array_equal(acc.cpu().numpy(), ref.accumulate(probs, ops, B, o))
    assert _lib.load().rsb_head_tta_accumulate(d.data_ptr(), acc.data_ptr(), (ctypes.c_int32 * 1)(2), 1, B, C, H, W, o, 0,
                                               _lib.current_stream_ptr()) == -1  # a quarter turn of a rectangle is refused


def test_identity_view_reproduces_head_quantize(cuda_device):
    B, S, o = 2, 96, 16
    logits = torch.randn((B, 2, S, S), generator=torch.Generator().manual_seed(1)) * 6
    logits[0, 0, 20:30, 20:60] = 80.0
    logits[0, 1, 40:50, 20:60] = 80.0
    logits[1, 0, 20:30, 20:60] = -80.0
    logits[1, 1, 40:50, 20:60] = -80.0
    logits[1, :, 60:70, 20:60] = 80.0  # exact ties: p = 0.5
    d = logits.to(cuda_device)
    lib = _lib.load()
    plain = torch.empty((B, S - 2 * o, S - 2 * o), dtype=torch.uint8, device=cuda_device)
    _lib.check(lib.rsb_head_quantize(d.data_ptr(), plain.data_ptr(), None, B, S, S, o, _lib.current_stream_ptr()), "head_quantize")
    acc = torch.empty((B, 2, S - 2 * o, S - 2 * o), dtype=torch.int64, device=cuda_device)
    _accumulate(d, acc, (0,), B, 2, S, S, o)
    assert torch.equal(_tta_quantize(acc, B, 1), plain)


def test_head_is_exactly_equivariant_and_pass_split_free(cuda_device):
    B, C, S, o = 2, 2, 96, 16
    logits = torch.randn((8 * B, C, S, S), generator=torch.Generator().manual_seed(3)) * 4
    d = logits.to(cuda_device)
    OS = S - 2 * o
    acc = torch.empty((B, C, OS, OS), dtype=torch.int64, device=cuda_device)
    _accumulate(d, acc, tuple(range(8)), B, C, S, S, o)
    base = acc.cpu().numpy()
    base_bins = _tta_quantize(acc, B, 8).cpu().numpy()
    for r in range(8):
        # view v of the tile turned by r is view compose(v, r) of the tile: the same logits, arriving in another order
        order = [ref.compose(v, r) for v in range(8)]
        permuted = torch.cat([d[w * B:(w + 1) * B] for w in order]).contiguous()
        _accumulate(permuted, acc, tuple(range(8)), B, C, S, S, o)
        assert np.array_equal(acc.cpu().numpy(), _spatial(base, r)), r
        assert np.array_equal(_tta_quantize(acc, B, 8).cpu().numpy(), _spatial(base_bins, r)), r
    for P in (1, 2, 4, 8):
        per = 8 // P
        for p in range(P):
            _accumulate(d[p * per * B:(p + 1) * per * B], acc, tuple(range(p * per, (p + 1) * per)), B, C, S, S, o, 1 if p else 0)
        assert np.array_equal(acc.cpu().numpy(), base), P


# ------------------------------------------------------------------------------------------------ network level


def _oracle_mean_probs(sd, tile_u8, ops):
    """float64 mean over `ops` of the oracle's softmax of each view, mapped back to the tile: [C, H, W]"""
    total = 0.0
    for op in ops:
        v = torch.from_numpy(np.ascontiguousarray(ref.view(tile_u8, op)))[None]
        p = unet_oracle.predict_probs(sd, synth.normalize_tiles(v)).numpy()[0].astype(np.float64)
        total = total + np.moveaxis(ref.unview(np.moveaxis(p, 0, -1), op), -1, 0)
    return total / len(ops)


def _bins_vs_oracle(got, want):
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    return int(diff.max()), int((diff > 0).sum()), int(((got >= 129) != (want >= 129)).sum()), diff.size


@pytest.mark.parametrize("mode", ["d4", "flip"])
def test_tile_predictor_matches_oracle(mode, cuda_device):
    from robosat_b200.predictor import TilePredictor

    sd = synth.make_state_dict(2, seed=0)
    S, o = 128, 16
    tiles = synth.make_tiles_u8(2, S, seed=11)
    ops = tta.views(mode)
    want = np.stack([np.digitize(_oracle_mean_probs(sd, tiles[i].numpy(), ops)[1, o:S - o, o:S - o], ANCHORS).astype(np.uint8) for i in range(2)])
    for batch in (2, 1):
        pred = TilePredictor(sd, 2, batch, S, overlap=o, device=cuda_device, precision="strict", tta=mode)
        got = np.concatenate([pred.predict_u8(tiles[i:i + batch]).numpy().copy() for i in range(0, 2, batch)])
        worst, ndiff, flips, total = _bins_vs_oracle(got, want)
        print("TilePredictor(tta=%s) batch %d vs oracle: worst bin difference %d, pixels whose bin differs %d / %d, argmax flips %d" % (
            mode, batch, worst, ndiff, total, flips))
        assert worst <= 1 and ndiff <= 0.02 * total
        assert flips <= max(2, 8 * total // 131072)


def test_tile_predictor_graph_replay_equals_kernel_by_kernel(cuda_device, monkeypatch):
    from robosat_b200.predictor import TilePredictor

    monkeypatch.setattr(tta, "ENGINE_CAP", 4)  # 2 tiles x 8 views in 4 passes of 4
    sd = synth.make_state_dict(2, seed=0)
    tiles = [synth.make_tiles_u8(2, 128, seed=60 + i) for i in range(5)]
    outs = {}
    for use_graph in (False, True):
        pred = TilePredictor(sd, 2, 2, 128, overlap=16, device=cuda_device, use_graph=use_graph, tta="d4")
        assert pred.tta.passes == 4 and pred.engine.N == 4
        if use_graph:
            assert pred.graph_error is None, pred.graph_error
        res = []
        for i, t in enumerate(tiles):
            pred.submit(t)
            if i >= 1:
                res.append(pred.collect().clone())
        res.append(pred.collect().clone())
        outs[use_graph] = res
    for a, b in zip(outs[False], outs[True]):
        assert torch.equal(a, b)
    assert not all(torch.equal(outs[True][0], r) for r in outs[True][1:])  # different inputs, different bins


def _slippy_dir(tmp_path):
    tiles_dir = tmp_path / "tiles"
    u8 = synth.make_tiles_u8(5, 256, seed=9).numpy()
    coords = [(100, 200), (101, 200), (100, 201), (101, 201), (103, 205)]
    for (x, y), arr in zip(coords, u8):
        os.makedirs(tiles_dir / "17" / str(x), exist_ok=True)
        Image.fromarray(arr).save(tiles_dir / "17" / str(x) / ("%d.png" % y))
    sd = synth.make_state_dict(2, seed=0)
    ckpt = tmp_path / "checkpoint-00001-of-00001.pth"
    torch.save({"epoch": 1, "state_dict": sd, "optimizer": {}}, ckpt)
    (tmp_path / "model.toml").write_text("[common]\ncuda = true\nbatch_size = 2\nimage_size = 256\ncheckpoint = '%s'\n[opt]\nepochs = 1\nlr = 0.0001\nloss = 'Lovasz'\n" % tmp_path)
    (tmp_path / "dataset.toml").write_text("[common]\ndataset = '%s'\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n" % tmp_path)
    return tiles_dir, coords, sd


def test_rs_predict_tta_end_to_end(tmp_path, cuda_device, monkeypatch):
    from robosat_b200.tools import predict

    tiles_dir, coords, sd = _slippy_dir(tmp_path)
    monkeypatch.setenv("RSB_GPUS", "1")
    monkeypatch.setenv("RSB_QUIET", "1")
    base = dict(batch_size=2, checkpoint=str(tmp_path / "checkpoint-00001-of-00001.pth"), overlap=32, tile_size=256, workers=0,
                tiles=str(tiles_dir), model=str(tmp_path / "model.toml"), dataset=str(tmp_path / "dataset.toml"))

    def png(root, x, y):
        return root / "17" / str(x) / ("%d.png" % y)

    # --tta none writes the same files as a caller whose Namespace predates the flag
    predict.main(argparse.Namespace(probs=str(tmp_path / "plain"), **base))
    predict.main(argparse.Namespace(probs=str(tmp_path / "none"), tta="none", **base))
    for (x, y) in coords:
        assert png(tmp_path / "plain", x, y).read_bytes() == png(tmp_path / "none", x, y).read_bytes(), (x, y)

    predict.main(argparse.Namespace(probs=str(tmp_path / "d4"), tta="d4", **base))
    monkeypatch.setenv("RSB_HOST_STITCH", "1")
    predict.main(argparse.Namespace(probs=str(tmp_path / "d4_host"), tta="d4", **base))
    monkeypatch.delenv("RSB_HOST_STITCH")
    for (x, y) in coords:
        assert png(tmp_path / "d4", x, y).read_bytes() == png(tmp_path / "d4_host", x, y).read_bytes(), (x, y)

    directory = BufferedSlippyMapDirectory(str(tiles_dir), transform=ImageToUint8Tensor(), size=256, overlap=32)
    worst, ndiff, flips, total, changed = 0, 0, 0, 0, 0
    for i in range(len(directory)):
        image, xyz = directory[i]
        x, y, z = (int(v) for v in xyz)
        got = np.array(Image.open(png(tmp_path / "d4", x, y)))
        want = np.digitize(directory.unbuffer(_oracle_mean_probs(sd, image.numpy(), tta.views("d4")))[1], ANCHORS).astype(np.uint8)
        w, n, f, t = _bins_vs_oracle(got, want)
        worst, ndiff, flips, total = max(worst, w), ndiff + n, flips + f, total + t
        changed += int((got != np.array(Image.open(png(tmp_path / "plain", x, y)))).sum())
    print("rs predict --tta d4 vs oracle: worst bin difference %d, pixels whose bin differs %d / %d, argmax flips %d; %d pixels differ from --tta none" % (
        worst, ndiff, total, flips, changed))
    assert worst <= 1 and ndiff <= 0.02 * total
    assert flips <= max(2, 8 * total // 131072)
    assert changed > 0


def test_segment_engine_tta(cuda_device):
    from robosat_b200.serve import SegmentEngine

    C, S = 3, 128
    sd = synth.make_state_dict(C, seed=0)
    tiles = synth.make_tiles_u8(2, S, seed=7).numpy()
    graph = SegmentEngine(sd, C, S, S, device=cuda_device, use_graph=True, precision="strict", tta="d4")
    eager = SegmentEngine(sd, C, S, S, device=cuda_device, use_graph=False, precision="strict", tta="d4")
    assert graph.graph is not None, graph.graph_error
    assert graph.engine.N == 8 and graph.tta.passes == 1
    for i in (0, 1, 0):
        got = graph.segment_u8(tiles[i])
        assert np.array_equal(got, eager.segment_u8(tiles[i]))
        mean = _oracle_mean_probs(sd, tiles[i], tta.views("d4"))
        top2 = np.sort(mean, axis=0)[-2:]
        diff = got != mean.argmax(axis=0)
        print("SegmentEngine(tta=d4) vs oracle mean: %d argmax flips, largest top-2 margin among them %.2e" % (
            int(diff.sum()), float((top2[1] - top2[0])[diff].max()) if diff.any() else 0.0))
        assert diff.mean() < 5e-3
        assert ((top2[1] - top2[0])[diff] < 2e-3).all()

    with pytest.raises(ValueError):
        SegmentEngine(sd, C, 128, 192, device=cuda_device, tta="d4")
    rect = synth.make_tiles_u8(1, 192, seed=8).numpy()[0, :128]
    flip = SegmentEngine(sd, C, 128, 192, device=cuda_device, precision="strict", tta="flip")
    got = flip.segment_u8(rect)
    mean = _oracle_mean_probs(sd, rect, tta.views("flip"))
    top2 = np.sort(mean, axis=0)[-2:]
    diff = got != mean.argmax(axis=0)
    assert got.shape == (128, 192) and diff.mean() < 5e-3 and ((top2[1] - top2[0])[diff] < 2e-3).all()


def test_predictor_tta_contract(cuda_device):
    from robosat_b200.serve import Predictor

    sd = synth.make_state_dict(2, seed=0)
    model = {"common": {"cuda": True}}
    dataset = {"common": {"classes": ["background", "parking"], "colors": ["denim", "orange"]}}
    chk = {"epoch": 1, "state_dict": sd, "optimizer": {}}
    with pytest.raises(ValueError):
        Predictor(chk, model, dataset, tta="d8")
    img = Image.fromarray(synth.make_tiles_u8(1, 128, seed=3)[0].numpy())
    out = Predictor(chk, model, dataset, tta="d4").segment(img)
    assert out.mode == "P" and out.size == (128, 128) and set(np.unique(np.asarray(out))) <= {0, 1}


def test_network_equivariance_report(cuda_device):
    """d4 bins of a turned tile against the turned bins of the tile: equal up to the network's own batch-position effects"""
    from robosat_b200.predictor import TilePredictor

    sd = synth.make_state_dict(2, seed=0)
    S, o = 128, 16
    tile = synth.make_tiles_u8(1, S, seed=21)
    pred = TilePredictor(sd, 2, 1, S, overlap=o, device=cuda_device, precision="strict", tta="d4")
    base = pred.predict_u8(tile).numpy().copy()[0]
    worst, differ = 0, 0
    for r in range(1, 8):
        turned = torch.from_numpy(np.ascontiguousarray(ref.view(tile[0].numpy(), r)))[None]
        got = pred.predict_u8(turned).numpy().copy()[0]
        d = np.abs(got.astype(np.int32) - ref.view(base, r).astype(np.int32))
        worst, differ = max(worst, int(d.max())), differ + int((d > 0).sum())
    print("network-level d4 equivariance over 7 turns: worst bin difference %d, %d / %d pixels differ" % (worst, differ, 7 * base.size))
    assert worst <= 1
