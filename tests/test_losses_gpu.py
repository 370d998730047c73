"""GPU parity of the loss / metric / optimiser kernels against the committed reference fixtures and the oracle."""

import os

import numpy as np
import pytest
import torch

from oracle import losses_oracle
from robosat_b200 import _lib, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _lovasz(logits, targets, dev, want_grad=True):
    lib = _lib.load()
    N, C, H, W = logits.shape
    x = logits.to(dev).contiguous()
    t = targets.to(dev).contiguous()
    nbytes = lib.rsb_lovasz_workspace_bytes(N, C, H * W)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    grad = torch.full_like(x, float("nan")) if want_grad else None
    _lib.check(lib.rsb_lovasz(x.data_ptr(), t.data_ptr(), loss.data_ptr(), grad.data_ptr() if want_grad else None, ws.data_ptr(), nbytes,
                              N, C, H * W, _lib.current_stream_ptr()), "rsb_lovasz")
    torch.cuda.synchronize()
    return loss.item(), (grad.cpu() if want_grad else None)


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_lovasz_matches_reference_fixture(tag, cuda_device):
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    logits = torch.from_numpy(gold["lovasz_%s_logits" % tag])
    targets = torch.from_numpy(gold["lovasz_%s_targets" % tag])
    loss, grad = _lovasz(logits, targets, cuda_device)
    ref = float(gold["lovasz_%s_loss" % tag])
    assert abs(loss - ref) <= 2e-6 * abs(ref), (loss, ref)
    # integer-exact cumulative sums + identical fp32 Jaccard arithmetic: the gradient is bit-identical
    assert np.array_equal(grad.numpy(), gold["lovasz_%s_grad" % tag])


def test_lovasz_full_size_against_oracle(cuda_device):
    """BASELINE config 3 shape per image (2 x 512 x 512), N = 4: P is 128 whole sort tiles. Fixture b (P = 1536) is less than one
    tile; several tiles with a ragged last one, N that is not a power of two and equal errors are in tests/test_losses_edges_gpu.py."""
    g = torch.Generator().manual_seed(5)
    logits = torch.randn((4, 2, 512, 512), generator=g) * 3
    targets = synth.make_masks(4, 512, 2, seed=9)
    loss, grad = _lovasz(logits, targets, cuda_device)
    ref_loss, ref_grad = losses_oracle.lovasz_loss(logits, targets, with_grad=True)
    assert abs(loss - float(ref_loss)) <= 5e-6 * abs(float(ref_loss))
    assert torch.equal(grad, ref_grad)
    # size-independent properties: sum of gradient magnitudes telescopes to N^-1 * sum_n J_last-ish bound; grad is zero where e <= 0
    e = 1 - (2 * torch.nn.functional.one_hot(targets, 2).permute(0, 3, 1, 2).float() - 1) * logits
    assert torch.all(grad[e <= 0] == 0)


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_cross_entropy_metrics_match_reference_fixture(tag, cuda_device):
    lib = _lib.load()
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    logits = torch.from_numpy(gold["lovasz_%s_logits" % tag]).to(cuda_device)
    targets = torch.from_numpy(gold["lovasz_%s_targets" % tag]).to(cuda_device)
    w = torch.from_numpy(gold["ce_%s_weight" % tag]).to(cuda_device)
    N, C, H, W = logits.shape
    loss = torch.zeros(1, dtype=torch.float32, device=cuda_device)
    grad = torch.empty_like(logits)
    scratch = torch.empty(2, dtype=torch.float64, device=cuda_device)
    _lib.check(lib.rsb_cross_entropy(logits.data_ptr(), targets.data_ptr(), w.data_ptr(), loss.data_ptr(), grad.data_ptr(), scratch.data_ptr(),
                                     N, C, H * W, _lib.current_stream_ptr()), "ce")
    counts = torch.zeros(4, dtype=torch.int64, device=cuda_device)
    _lib.check(lib.rsb_metrics_count(logits.data_ptr(), targets.data_ptr(), counts.data_ptr(), N, C, H * W, _lib.current_stream_ptr()), "metrics")
    torch.cuda.synchronize()
    ref = float(gold["ce_%s_loss" % tag])
    assert abs(loss.item() - ref) <= 5e-6 * abs(ref)
    np.testing.assert_allclose(grad.cpu().numpy(), gold["ce_%s_grad" % tag], rtol=2e-4, atol=1e-9)
    assert counts.cpu().tolist() == gold["metrics_%s" % tag].tolist()  # integer work: exact


def test_adam_matches_reference_fixture(cuda_device):
    lib = _lib.load()
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    p = torch.from_numpy(gold["adam_p0"]).to(cuda_device)
    m = torch.zeros_like(p)
    v = torch.zeros_like(p)
    for s in range(3):
        g = torch.from_numpy(gold["adam_grads"][s]).to(cuda_device)
        _lib.check(lib.rsb_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), 1e-4, 0.9, 0.999, 1e-8, s + 1,
                                     _lib.current_stream_ptr()), "adam")
        torch.cuda.synchronize()
        np.testing.assert_allclose(p.cpu().numpy(), gold["adam_p%d" % (s + 1)], rtol=3e-7, atol=1e-9)


def test_guarded_adam_skips_non_finite_steps_and_equals_plain_adam_otherwise(cuda_device):
    """rsb_adam_step_guarded: equal to rsb_adam_step (to the last bit of each value) while gradients are finite; a step with an inf / NaN gradient leaves
    parameters and moments untouched, is counted, and later bias corrections use the number of steps actually taken (what
    torch.optim.Adam behind a GradScaler does)."""
    lib = _lib.load()
    gold = np.load(os.path.join(GOLD, "losses.npz"))
    st = _lib.current_stream_ptr()
    p = torch.from_numpy(gold["adam_p0"]).to(cuda_device)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    state = torch.zeros(4, dtype=torch.int32, device=cuda_device)
    grads = [torch.from_numpy(gold["adam_grads"][s]).to(cuda_device) for s in range(3)]
    bad = grads[1].clone()
    bad[7] = float("inf")
    seq = [grads[0], bad, grads[1], grads[2]]  # host step counter 1, 2, 3, 4; effective steps 1, -, 2, 3
    expect = ["adam_p1", "adam_p1", "adam_p2", "adam_p3"]
    for i, (g, key) in enumerate(zip(seq, expect)):
        _lib.check(lib.rsb_adam_step_guarded(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), 1e-4, 0.9, 0.999, 1e-8, i + 1,
                                             state.data_ptr(), st), "adam_guarded")
        torch.cuda.synchronize()
        np.testing.assert_allclose(p.cpu().numpy(), gold[key], rtol=3e-7, atol=1e-9)
        assert state.cpu().tolist() == [0, 1 if i >= 1 else 0, 1 if i == 1 else 0, i + 1]
    assert torch.isfinite(m).all() and torch.isfinite(v).all()


def test_loss_scaler_halves_on_overflow(cuda_device):
    from robosat_b200.optim import Adam, LossScaler

    w = torch.nn.Parameter(torch.ones(1024, device=cuda_device))

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = w
            self.loss_scale = 4096.0
            self._train_engines = {}

    net = Net()
    opt = Adam(net.parameters(), lr=1e-2)
    scaler = LossScaler(net, opt, init_scale=4096.0, growth_interval=3)
    before = w.detach().clone()
    opt.zero_grad()
    w.grad.fill_(float("nan"))
    opt.step()
    scaler.update()
    torch.cuda.synchronize()
    assert torch.equal(w.detach(), before) and opt.skipped_steps() == 1
    for _ in range(5):  # clean steps: the (one step late) reading first halves the scale, then grows it again after 3 clean steps
        opt.zero_grad()
        w.grad.fill_(0.5)
        opt.step()
        scaler.update()
        torch.cuda.synchronize()
    assert scaler.overflows == 1 and net.loss_scale in (2048.0, 4096.0)
    assert not torch.equal(w.detach(), before)


def test_head_quantize_matches_numpy_digitize(cuda_device):
    """predict.py:87-103 on identical logits: bins may differ by one only where expf rounding moves p across an anchor."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(2)
    logits = torch.randn((2, 2, 64, 96), generator=g) * 4
    o = 8
    q = torch.zeros((2, 64 - 2 * o, 96 - 2 * o), dtype=torch.uint8, device=cuda_device)
    pf = torch.zeros((2, 64 - 2 * o, 96 - 2 * o), dtype=torch.float32, device=cuda_device)
    logits_d = logits.to(cuda_device)
    _lib.check(lib.rsb_head_quantize(logits_d.data_ptr(), q.data_ptr(), pf.data_ptr(), 2, 64, 96, o, _lib.current_stream_ptr()), "head")
    torch.cuda.synchronize()
    probs = torch.softmax(logits, dim=1).numpy()[:, 1, o:-o, o:-o]
    ref = np.digitize(probs, np.linspace(0, 1, 256)).astype(np.uint8)
    got = q.cpu().numpy()
    np.testing.assert_allclose(pf.cpu().numpy(), probs, rtol=0, atol=2e-7)
    diff = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    assert diff.max() <= 1 and (diff > 0).mean() < 1e-3
    # digitising the device's own probabilities on the host is exact: the binning itself is bit-identical to numpy
    assert np.array_equal(np.digitize(pf.cpu().numpy(), np.linspace(0, 1, 256)).astype(np.uint8), got)
    # saturated probability 1.0 wraps to bin 0 exactly like .astype(np.uint8) on 256
    sat = torch.tensor([[[[-200.0]], [[200.0]]]])
    q1 = torch.zeros((1, 1, 1), dtype=torch.uint8, device=cuda_device)
    sat_d = sat.to(cuda_device)
    _lib.check(lib.rsb_head_quantize(sat_d.data_ptr(), q1.data_ptr(), None, 1, 1, 1, 0, _lib.current_stream_ptr()), "head")
    torch.cuda.synchronize()
    assert int(q1.item()) == int(np.digitize(np.float32(1.0), np.linspace(0, 1, 256)).astype(np.uint8))


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_focal_and_miou_match_reference_fixture(tag, cuda_device):
    """FocalLoss2d (losses.py:49-50) and mIoULoss2d (losses.py:71-83, both branches of its max()) through the module API."""
    from robosat_b200.losses import FocalLoss2d, mIoULoss2d

    gold = np.load(os.path.join(GOLD, "losses.npz"))
    targets = torch.from_numpy(gold["lovasz_%s_targets" % tag]).to(cuda_device)
    w = torch.from_numpy(gold["ce_%s_weight" % tag])
    logits = torch.from_numpy(gold["lovasz_%s_logits" % tag]).to(cuda_device).requires_grad_(True)
    loss = FocalLoss2d(gamma=2, weight=w).to(cuda_device)(logits, targets)
    loss.backward()
    ref = float(gold["focal_%s_loss" % tag])
    assert abs(loss.item() - ref) <= 1e-5 * abs(ref)
    np.testing.assert_allclose(logits.grad.cpu().numpy(), gold["focal_%s_grad" % tag], rtol=1e-3, atol=2e-9)
    branches = set()
    for sub, scale in (("", 1.0), ("_sharp", 4.0), ("_aligned", None)):
        base = torch.from_numpy(gold["lovasz_%s_logits" % tag]) * scale if scale is not None else torch.from_numpy(gold["miou_aligned_%s_logits" % tag])
        lg = base.to(cuda_device).requires_grad_(True)
        loss = mIoULoss2d(weight=w).to(cuda_device)(lg, targets)
        loss.backward()
        ref = float(gold["miou%s_%s_loss" % (sub, tag)])
        assert abs(loss.item() - ref) <= 1e-5 * abs(ref)
        np.testing.assert_allclose(lg.grad.cpu().numpy(), gold["miou%s_%s_grad" % (sub, tag)], rtol=2e-3, atol=2e-9)
        branches.add(abs(ref - float(losses_oracle.cross_entropy_loss(lg.detach().cpu(), targets.cpu(), w))) < 1e-5 * abs(ref))
    print("mIoU loss branches exercised for", tag, branches)
    if tag in "ac":
        assert branches == {True, False}  # both the cross-entropy and the soft-IoU branch of max() occur
