"""`rs predict` and `rs masks --dataset` for models of more than two classes on the H100: the head, TTA-quantize and soft-vote kernels
against the numpy restatement (tests/multiclass_reference.py), `TilePredictor` at C = 6 against the oracle, and the tools end to
end (predict -> masks -> features)."""

import argparse
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import multiclass_reference as ref
import tta_reference
from oracle import unet_oracle
from robosat_b200 import _lib, colors, synth, tta
from robosat_b200.datasets import BufferedSlippyMapDirectory
from robosat_b200.transforms import ImageToUint8Tensor

pytestmark = pytest.mark.gpu

RSB_E_INVALID = -1


def _head(logits_d, overlap, probs=True):
    N, C, H, W = logits_d.shape
    shape = (N, C, H - 2 * overlap, W - 2 * overlap)
    q = torch.full(shape, 77, dtype=torch.uint8, device=logits_d.device)
    p = torch.full(shape, -1.0, dtype=torch.float32, device=logits_d.device) if probs else None
    _lib.check(_lib.load().rsb_head_quantize_classes(logits_d.data_ptr(), q.data_ptr(), p.data_ptr() if probs else None, N, C, H, W, overlap,
                                                     _lib.current_stream_ptr()), "rsb_head_quantize_classes")
    return q, p


@pytest.mark.parametrize("C", [2, 3, 6, 20])
@pytest.mark.parametrize("overlap", [0, 8, 32])
@pytest.mark.parametrize("N,H,W", [(2, 96, 100), (3, 81, 101)])  # cropped width a multiple of 4 (word stores) and not
def test_head_matches_softmax_and_digitize(C, overlap, N, H, W, cuda_device):
    g = torch.Generator().manual_seed(1000 * C + overlap + W)
    logits = torch.randn((N, C, H, W), generator=g) * 4
    logits[0, C - 1, overlap + 3, overlap + 5] = 100.0  # saturated: p = 1 -> bin 256 wraps to 0
    logits[0, :C - 1, overlap + 3, overlap + 5] = -100.0
    q, p = _head(logits.to(cuda_device), overlap)
    q, p = q.cpu().numpy(), p.cpu().numpy()
    want_p = ref.crop(torch.softmax(logits, 1).numpy(), overlap)
    assert np.abs(p - want_p).max() <= 2e-7
    want_q = ref.digitize(want_p)
    diff = np.abs(q.astype(np.int32) - want_q.astype(np.int32))
    diff = np.minimum(diff, 256 - diff)  # a wrap 255 <-> 0 (p within an ulp of 1) is one bin
    print("C %d overlap %d %dx%d: bins differ on %d / %d pixels" % (C, overlap, H, W, int((diff > 0).sum()), diff.size))
    assert diff.max() <= 1 and (diff > 0).sum() < 1e-3 * diff.size
    assert np.array_equal(q, ref.digitize(p))  # the device's own probabilities, digitized on the host: exact
    assert q[0, C - 1, 3, 5] == 0 and p[0, C - 1, 3, 5] == 1.0
    if C == 2:
        binary = torch.empty((N, H - 2 * overlap, W - 2 * overlap), dtype=torch.uint8, device=cuda_device)
        d = logits.to(cuda_device)
        _lib.check(_lib.load().rsb_head_quantize(d.data_ptr(), binary.data_ptr(), None, N, H, W, overlap, _lib.current_stream_ptr()), "head_quantize")
        assert np.array_equal(q[:, 1], binary.cpu().numpy())


def test_head_rejects_bad_arguments(cuda_device):
    lib = _lib.load()
    d = torch.zeros((1, 3, 32, 32), device=cuda_device)
    q = torch.empty((1, 3, 32, 32), dtype=torch.uint8, device=cuda_device)
    s = _lib.current_stream_ptr()
    assert lib.rsb_head_quantize_classes(d.data_ptr(), q.data_ptr(), None, 1, 3, 32, 32, 0, s) == 0
    for args in [(None, q.data_ptr(), None, 1, 3, 32, 32, 0), (d.data_ptr(), None, None, 1, 3, 32, 32, 0),
                 (d.data_ptr(), q.data_ptr(), None, 0, 3, 32, 32, 0), (d.data_ptr(), q.data_ptr(), None, 1, 1, 32, 32, 0),
                 (d.data_ptr(), q.data_ptr(), None, 1, 256, 32, 32, 0), (d.data_ptr(), q.data_ptr(), None, 1, 3, 32, 32, 16),
                 (d.data_ptr(), q.data_ptr(), None, 1, 3, 64, 32, 16), (d.data_ptr(), q.data_ptr(), None, 1, 3, 32, 32, -1)]:
        assert lib.rsb_head_quantize_classes(*args, s) == RSB_E_INVALID, args
    acc = torch.zeros((1, 3, 16), dtype=torch.int64, device=cuda_device)
    assert lib.rsb_head_tta_quantize_classes(acc.data_ptr(), q.data_ptr(), 1, 1, 16, 1, s) == RSB_E_INVALID
    assert lib.rsb_head_tta_quantize_classes(acc.data_ptr(), q.data_ptr(), 1, 3, 16, 0, s) == RSB_E_INVALID
    assert lib.rsb_softvote_classes(q.data_ptr(), None, q.data_ptr(), 1, 1, 16, s) == RSB_E_INVALID
    assert lib.rsb_softvote_classes(q.data_ptr(), None, q.data_ptr(), 0, 3, 16, s) == RSB_E_INVALID


@pytest.mark.parametrize("C", [2, 3, 6, 20])
def test_tta_quantize_matches_mean_per_class(C, cuda_device):
    B, S, o, ops = 2, 64, 8, tuple(range(8))
    logits = torch.randn((8 * B, C, S, S), generator=torch.Generator().manual_seed(C)) * 4
    d = logits.to(cuda_device)
    probs = torch.empty_like(d)
    lib, s = _lib.load(), _lib.current_stream_ptr()
    _lib.check(lib.rsb_softmax_nchw(d.data_ptr(), probs.data_ptr(), 8 * B, C, S * S, s), "softmax")
    OS = S - 2 * o
    acc = torch.empty((B, C, OS, OS), dtype=torch.int64, device=cuda_device)
    _lib.check(lib.rsb_head_tta_accumulate(d.data_ptr(), acc.data_ptr(), (ctypes.c_int32 * 8)(*ops), 8, B, C, S, S, o, 0, s), "accumulate")
    want_acc = tta_reference.accumulate(probs.cpu().numpy(), ops, B, o)
    assert np.array_equal(acc.cpu().numpy(), want_acc)
    q = torch.empty((B, C, OS, OS), dtype=torch.uint8, device=cuda_device)
    _lib.check(lib.rsb_head_tta_quantize_classes(acc.data_ptr(), q.data_ptr(), B, C, OS * OS, 8, s), "tta_quantize_classes")
    assert np.array_equal(q.cpu().numpy(), ref.digitize(tta_reference.mean(want_acc, 8)))
    if C == 2:
        binary = torch.empty((B, OS, OS), dtype=torch.uint8, device=cuda_device)
        _lib.check(lib.rsb_head_tta_quantize(acc.data_ptr(), binary.data_ptr(), B, OS * OS, 8, s), "tta_quantize")
        assert torch.equal(q[:, 1], binary)


def _softvote(q, w, cuda_device):
    from robosat_b200.tools import masks

    return masks.softvote_classes_device(torch.from_numpy(np.ascontiguousarray(q)).to(cuda_device), w).cpu().numpy()


@pytest.mark.parametrize("K", [1, 2, 3])
@pytest.mark.parametrize("C", [3, 6])
@pytest.mark.parametrize("weighted", [False, True])
def test_softvote_classes_bit_identical(K, C, weighted, cuda_device):
    rng = np.random.RandomState(10 * K + C)
    w = [0.1, 0.7, 0.2][:K] if weighted else None
    q = rng.randint(0, 256, size=(K, C, 37, 41)).astype(np.uint8)  # n = 1517, not a multiple of the block
    q[:, :, 0, :4] = 0
    q[:, 1, 0, 0] = 128  # class 1 alone
    q[:, 0, 0, 1] = q[:, 2, 0, 1] = 200  # tie of classes 0 and 2: class 0
    q[:, 1, 0, 2] = q[:, C - 1, 0, 2] = 255  # tie at the pinned anchor 1.0: class 1
    if K >= 2:  # ties between different sums: anchors 100 + 155 on either side
        q[0, 0, 1, :], q[1, 0, 1, :], q[0, 1, 1, :], q[1, 1, 1, :] = 100, 155, 155, 100
        q[2:, :2, 1, :] = 50  # a third model adds the same to both classes
        q[:, 2:, 1, :] = 0
    got = _softvote(q, w, cuda_device)
    want = ref.softvote(q, w)
    assert np.array_equal(got, want), (K, C, w)
    assert got[0, 0] == 1 and got[0, 1] == 0 and got[0, 2] == 1
    if K >= 2 and w is None:
        assert (got[1] == 0).all()


# ------------------------------------------------------------------------------------------------ network level


def _oracle_bins(sd, tiles_u8, ops, overlap):
    """np.digitize bins of every class of the oracle's mean softmax over `ops`: uint8 [N, C, h, w]"""
    out = []
    for tile in tiles_u8:
        total = 0.0
        for op in ops:
            v = torch.from_numpy(np.ascontiguousarray(tta_reference.view(tile, op)))[None]
            p = unet_oracle.predict_probs(sd, synth.normalize_tiles(v)).numpy()[0].astype(np.float64)
            total = total + np.moveaxis(tta_reference.unview(np.moveaxis(p, 0, -1), op), -1, 0)
        out.append(ref.digitize(ref.crop(total / len(ops), overlap)))
    return np.stack(out)


@pytest.mark.parametrize("mode", ["none", "flip", "d4"])
def test_tile_predictor_six_classes_matches_oracle(mode, cuda_device):
    from robosat_b200.predictor import TilePredictor

    sd = synth.make_state_dict(6, seed=2)
    S, o = 128, 16
    tiles = synth.make_tiles_u8(2, S, seed=21)
    want = _oracle_bins(sd, tiles.numpy(), tta.views(mode), o)
    pred = TilePredictor(sd, 6, 2, S, overlap=o, device=cuda_device, precision="strict", use_graph=True, tta=mode)
    assert pred.graph_error is None, pred.graph_error
    assert pred.d2h_bytes == 2 * 6 * (S - 2 * o) ** 2
    got = pred.predict_u8(tiles).numpy()
    assert got.shape == (2, 6, S - 2 * o, S - 2 * o)
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    print("TilePredictor C=6 tta=%s vs oracle: worst bin difference %d, pixels whose bin differs %d / %d" % (
        mode, int(diff.max()), int((diff > 0).sum()), diff.size))
    assert diff.max() <= 1 and (diff > 0).sum() <= 0.02 * diff.size


def test_tile_predictor_six_classes_graph_replay_equals_kernel_by_kernel(cuda_device):
    from robosat_b200.predictor import TilePredictor

    sd = synth.make_state_dict(6, seed=2)
    tiles = [synth.make_tiles_u8(2, 128, seed=50 + i) for i in range(5)]
    for mode in ("none", "flip"):
        outs = {}
        for use_graph in (False, True):
            pred = TilePredictor(sd, 6, 2, 128, overlap=16, device=cuda_device, use_graph=use_graph, tta=mode)
            if use_graph:
                assert pred.graph_error is None and all("graph" in s for s in pred._slots), pred.graph_error
            res = []
            for i, t in enumerate(tiles):
                pred.submit(t)
                if i >= 1:
                    res.append(pred.collect().clone())
            res.append(pred.collect().clone())
            outs[use_graph] = res
        for a, b in zip(outs[False], outs[True]):
            assert a.shape == (2, 6, 96, 96) and torch.equal(a, b), mode


# ------------------------------------------------------------------------------------------------ tools end to end

CLASSES = ["background", "parking", "building"]
COLORS = ["denim", "orange", "red"]


def _setup(tmp_path, seeds=(0, 1)):
    tiles_dir = tmp_path / "tiles"
    u8 = synth.make_tiles_u8(5, 256, seed=9).numpy()
    coords = [(100, 200), (101, 200), (100, 201), (101, 201), (103, 205)]  # a 2x2 block with neighbours + one isolated tile
    for (x, y), arr in zip(coords, u8):
        os.makedirs(tiles_dir / "18" / str(x), exist_ok=True)
        Image.fromarray(arr).save(tiles_dir / "18" / str(x) / ("%d.png" % y))
    ckpts = {}
    for seed in seeds:
        ckpts[seed] = tmp_path / ("checkpoint-%d.pth" % seed)
        torch.save({"epoch": 1, "state_dict": synth.make_state_dict(3, seed=seed), "optimizer": {}}, ckpts[seed])
    (tmp_path / "model.toml").write_text("[common]\ncuda = true\nbatch_size = 2\nimage_size = 256\ncheckpoint = '%s'\n[opt]\nepochs = 1\nlr = 0.0001\nloss = 'Lovasz'\n" % tmp_path)
    (tmp_path / "dataset.toml").write_text("[common]\ndataset = '%s'\nclasses = %s\ncolors = %s\n" % (tmp_path, json.dumps(CLASSES), json.dumps(COLORS)))
    return tiles_dir, coords, ckpts


def _read_planes(root, coords):
    return {(x, y): np.stack([np.array(Image.open(os.path.join(root, name, "18", str(x), "%d.png" % y))) for name in CLASSES]) for x, y in coords}


def test_rs_predict_masks_features_three_classes(tmp_path, cuda_device, monkeypatch):
    from robosat_b200.tools import features, masks, predict

    tiles_dir, coords, ckpts = _setup(tmp_path)
    monkeypatch.setenv("RSB_GPUS", "1")
    base = dict(batch_size=2, overlap=32, tile_size=256, workers=0, tiles=str(tiles_dir), model=str(tmp_path / "model.toml"),
                dataset=str(tmp_path / "dataset.toml"))
    runs = {}
    for stitch in ("device", "host"):
        for encoder in ("native", "pil"):
            out = tmp_path / ("probs_%s_%s" % (stitch, encoder))
            monkeypatch.setattr(predict, "NATIVE_PNG", encoder == "native")
            if stitch == "host":
                monkeypatch.setenv("RSB_HOST_STITCH", "1")
            predict.main(argparse.Namespace(checkpoint=str(ckpts[0]), probs=str(out), **base))
            monkeypatch.delenv("RSB_HOST_STITCH", raising=False)
            assert sorted(os.listdir(out)) == sorted(CLASSES)  # one directory per class, no probs/<z>
            runs[(stitch, encoder)] = _read_planes(out, coords)
    monkeypatch.setattr(predict, "NATIVE_PNG", True)
    first = runs[("device", "native")]
    for key, planes in runs.items():
        for xy in coords:
            assert np.array_equal(planes[xy], first[xy]), (key, xy)

    # against the reference pipeline restated on the CPU, per class
    sd = synth.make_state_dict(3, seed=0)
    directory = BufferedSlippyMapDirectory(str(tiles_dir), transform=ImageToUint8Tensor(), size=256, overlap=32)
    pink = colors.continuous_palette_for_color("pink", 256)
    worst, ndiff, total = 0, 0, 0
    for i in range(len(directory)):
        image, xyz = directory[i]
        x, y, z = (int(v) for v in xyz)
        for name in CLASSES:
            im = Image.open(tmp_path / "probs_device_native" / name / str(z) / str(x) / ("%d.png" % y))
            assert im.mode == "P" and im.size == (256, 256) and im.getpalette()[:768] == pink
        with torch.no_grad():
            probs = unet_oracle.predict_probs(sd, synth.normalize_tiles(image.unsqueeze(0))).numpy()[0]
        want = ref.digitize(directory.unbuffer(probs))
        d = np.abs(first[(x, y)].astype(np.int32) - want.astype(np.int32))
        worst, ndiff, total = max(worst, int(d.max())), ndiff + int((d > 0).sum()), total + d.size
    print("rs predict C=3 vs reference pipeline: worst bin difference %d, pixels whose bin differs %d / %d" % (worst, ndiff, total))
    # As for the binary tool (tests/test_predict_tool_gpu.py): strict precision moves a probability by ~1e-5, so a bin can differ
    # only where the reference sits that close to a bin edge, by one bin (1.6e-3 of the pixels here on an H100)
    assert worst <= 1 and ndiff <= 0.02 * total

    # a second model, then the weighted multi-class vote over both runs
    second = tmp_path / "probs_seed1"
    predict.main(argparse.Namespace(checkpoint=str(ckpts[1]), probs=str(second), **base))
    other = _read_planes(second, coords)
    out = tmp_path / "masks"
    masks.main(argparse.Namespace(masks=str(out), probs=[str(tmp_path / "probs_device_native"), str(second)], weights=[0.4, 0.6],
                                  dataset=str(tmp_path / "dataset.toml")))
    seen = set()
    for xy in coords:
        im = Image.open(out / "18" / str(xy[0]) / ("%d.png" % xy[1]))
        assert im.mode == "P" and im.getpalette()[:9] == colors.make_palette(*COLORS)
        got = np.array(im)
        assert np.array_equal(got, ref.softvote(np.stack([first[xy], other[xy]]), [0.4, 0.6])), xy
        seen.update(np.unique(got).tolist())
    print("rs masks --dataset: classes present", sorted(seen))

    # a root without a class directory is refused by name
    broken = tmp_path / "broken"
    os.makedirs(broken / "background")
    with pytest.raises(SystemExit, match="no directory for class 'parking'"):
        masks.main(argparse.Namespace(masks=str(tmp_path / "m2"), probs=[str(broken)], weights=None, dataset=str(tmp_path / "dataset.toml")))

    # rs features finds `parking` in the dataset's class list and reads the multi-class masks
    geojson = tmp_path / "parking.geojson"
    features.main(argparse.Namespace(masks=str(out), type="parking", dataset=str(tmp_path / "dataset.toml"), out=str(geojson)))
    with open(geojson) as fp:
        collection = json.load(fp)
    assert collection["type"] == "FeatureCollection" and isinstance(collection["features"], list)
    for f in collection["features"]:
        assert f["type"] == "Feature" and f["geometry"]["type"] in ("Polygon", "MultiPolygon")
