"""`rs compare` on the H100: the count and compose kernels against the numpy restatement (tests/compare_reference.py), counts
across batchings, and the tool end to end against the reference's own output (tests/golden/compare.npz)."""

import csv
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import compare_reference as R  # noqa: E402

from robosat_b200 import compare as C  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "compare.npz")


def seeded(rng, N, M, w, h):
    """N tiles of M masks: planes with densities from empty to full, labels, images, palettes"""
    hw = w * h
    dens = rng.choice([0.0, 0.001, 0.3, 0.5, 0.97, 1.0], size=(N, 1 + M))
    planes = np.where(rng.rand(N, 1 + M, hw) < dens[..., None], rng.randint(1, 256, size=(N, 1 + M, hw)), 0).astype(np.uint8)
    images = rng.randint(0, 256, size=(N, h, w, 3)).astype(np.uint8)
    luts = rng.randint(0, 256, size=(N, 1 + M, 256, 3)).astype(np.uint8)
    return planes, images, luts


def run_kernels(planes, images, luts, w, h, with_labels=True):
    N, P, hw = planes.shape
    M = P - 1
    pitch = C.pitch_of(hw)
    padded = np.full((N, P, pitch), 0xA5, np.uint8)  # padding bytes past W * H must not count
    padded[..., :hw] = planes
    d = torch.from_numpy(padded).cuda()
    d_masks = d[:, 1:].contiguous()
    d_labels = d[:, 0].contiguous() if with_labels else None
    counts = C.count_device(d_masks, d_labels, hw).cpu().numpy()
    out = torch.empty((N, C.out_stride_of((w, h), P)), dtype=torch.uint8, pin_memory=True)
    pal = torch.from_numpy(C.pack_palettes(luts).view(np.int32)).cuda()
    C.compose_device(torch.from_numpy(images.reshape(N, -1)).cuda(), d, pal, (w, h), out)
    torch.cuda.synchronize()
    comp = out.numpy()[:, :h * w * (1 + P) * 3].reshape(N, h, w * (1 + P), 3)
    return counts, comp


@pytest.mark.parametrize("M,w,h,N", [(1, 512, 512, 3), (2, 256, 256, 5), (3, 509, 509, 2), (4, 509, 131, 3), (2, 512, 512, 1), (1, 1, 1, 2)])
def test_kernels_match_the_restatement(M, w, h, N):
    rng = np.random.RandomState(M * 1000 + w + N)
    planes, images, luts = seeded(rng, N, M, w, h)
    counts, comp = run_kernels(planes, images, luts, w, h)
    for n in range(N):
        for m in range(M):
            assert tuple(counts[n, m]) == R.confusion(planes[n, 1 + m], planes[n, 0]), (n, m)
        want = R.compose(images[n], [p.reshape(h, w) for p in planes[n]], list(luts[n]))
        assert np.array_equal(comp[n], want), n
    no_label, _ = run_kernels(planes, images, luts, w, h, with_labels=False)
    nz = (planes[:, 1:] != 0).sum(-1)
    assert np.array_equal(no_label[..., 0], 0 * nz) and np.array_equal(no_label[..., 1], nz) and np.array_equal(no_label[..., 2], 0 * nz)
    assert np.array_equal(no_label[..., 3], w * h - nz)


def test_compose_writes_device_memory_too():
    rng = np.random.RandomState(7)
    planes, images, luts = seeded(rng, 2, 2, 61, 47)
    pitch = C.pitch_of(61 * 47)
    d = torch.zeros((2, 3, pitch), dtype=torch.uint8, device="cuda")
    d[..., :61 * 47] = torch.from_numpy(planes).cuda()
    out = torch.zeros((2, C.out_stride_of((61, 47), 3)), dtype=torch.uint8, device="cuda")
    pal = torch.from_numpy(C.pack_palettes(luts).view(np.int32)).cuda()
    C.compose_device(torch.from_numpy(images.reshape(2, -1)).cuda(), d, pal, (61, 47), out)
    got = out.cpu().numpy()[:, :47 * 61 * 4 * 3].reshape(2, 47, 61 * 4, 3)
    for n in range(2):
        assert np.array_equal(got[n], R.compose(images[n], [p.reshape(47, 61) for p in planes[n]], list(luts[n])))


def test_counts_do_not_depend_on_the_batching():
    rng = np.random.RandomState(3)
    planes, images, luts = seeded(rng, 6, 3, 509, 509)
    whole, _ = run_kernels(planes, images, luts, 509, 509)
    parts = np.concatenate([run_kernels(planes[i:i + k], images[i:i + k], luts[i:i + k], 509, 509)[0] for i, k in ((0, 1), (1, 3), (4, 2))])
    assert np.array_equal(whole, parts)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def check_case(golden, ci, a, root, out, rows):
    written = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)
    assert written == a["written"], ci
    for rel in written:
        px = np.asarray(Image.open(os.path.join(out, rel)))
        if "case%d:%s" % (ci, rel) in golden.files:
            assert np.array_equal(px, golden["case%d:%s" % (ci, rel)]), (ci, rel)
        else:
            assert str(golden["case%d:sha256:%s" % (ci, rel)]) == hashlib.sha256(px.tobytes()).hexdigest() + " %s" % (px.shape,), (ci, rel)
    _, want = R.compare(os.path.join(root, a["images"]), os.path.join(root, a["labels"]), [os.path.join(root, m) for m in a["masks"]],
                        a["minimum"], a["maximum"], R.golden_tiles(root, a["images"]))
    got = list(csv.reader(open(rows)))
    assert got[0] == C.CSV_COLUMNS and len(got) == len(want) + 1
    for g, w in zip(got[1:], want):
        assert [int(v) for v in g[:4]] == w[:4] and float(g[4]) == w[4] and [int(v) for v in g[5:9]] == w[5:9], (g, w)
        assert (g[9] == "" and w[9] is None) or float(g[9]) == w[9], (g, w)


def run_cases(golden, tmp_path, budget=C.DEFAULT_BUDGET, only=None):
    root = str(tmp_path)
    R.materialize(golden, root)
    i = 0
    while "case%d:args" % i in golden.files:
        a = json.loads(str(golden["case%d:args" % i]))
        if only is None or i in only:
            out, rows = os.path.join(root, "out%d" % i), os.path.join(root, "rows%d.csv" % i)
            st = {}
            C.compare_device(os.path.join(root, a["images"]), os.path.join(root, a["labels"]), [os.path.join(root, m) for m in a["masks"]], out,
                             a["minimum"], a["maximum"], csv=rows, budget=budget, stats=st)
            assert st["kept"] == st["written"] == len(a["written"])
            check_case(golden, i, a, root, out, rows)
        i += 1


def test_tool_reproduces_the_reference(golden, tmp_path):
    run_cases(golden, tmp_path)


def test_tool_in_small_batches(golden, tmp_path):
    run_cases(golden, tmp_path, budget=2 * C.tile_bytes((64, 64), 3, True), only=(1, 2))


def test_pil_paths(golden, tmp_path, monkeypatch):
    """every file through PIL (decode and encode): the same pixels"""
    monkeypatch.setattr(C, "NATIVE_DECODE", False)
    monkeypatch.setattr(C, "NATIVE_ENCODE", False)
    run_cases(golden, tmp_path, only=(2,))


def test_cli_without_csv(golden, tmp_path):
    import argparse

    from robosat_b200.tools import compare as tool

    root = str(tmp_path)
    R.materialize(golden, root)
    a = json.loads(str(golden["case0:args"]))
    out = os.path.join(root, "out")
    st = {}
    tool.main(argparse.Namespace(out=out, images=os.path.join(root, a["images"]), labels=os.path.join(root, a["labels"]),
                                 masks=[os.path.join(root, m) for m in a["masks"]], minimum=a["minimum"], maximum=a["maximum"], csv=None), stats=st)
    written = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)
    assert written == a["written"] and st["tiles"] == 7
    for rel in written:
        assert np.array_equal(np.asarray(Image.open(os.path.join(out, rel))), golden["case0:%s" % rel])
