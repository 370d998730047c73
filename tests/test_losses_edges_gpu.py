"""The loss, metric and optimiser kernels (robosat_b200/csrc/rsb_loss.cu) and rsb_sort_unique_u64 at the shapes and values where
such kernels go wrong, against oracle/losses_oracle.py, numpy or a closed form. The inputs come from tests/loss_cases.py;
tests/test_losses_edges.py shows without a GPU that each of them tells a right implementation from a wrong one.

Every raw call writes into buffers that are pre-filled with NaN (an element the kernel does not write is seen) and lie between
4 KiB bands of a sentinel byte that must come back untouched (a write outside the declared size is seen).

What is compared how:
  Lovasz    loss within 5e-6 relative (only the final dot product is accumulated differently: double), gradient bit-identical.
  metrics   integers, exact.
  cross entropy / focal / mIoU
            against the float64 restatements with the tolerance of test_train_lockstep_gpu._grad_check, imported from there:
            |err| <= 1e-4 |ref| + 1e-5 * scale, where 1e-4 covers the fp32 expf / logf / powf of the kernels against float64 and scale
            is the largest gradient magnitude a pixel can have, max(weight) / sum of the pixels' weights (for mIoU also the largest
            reference gradient). Losses: 1e-5 relative + 1e-7, as there.
            Defined by the reference as undefined (the float64 restatement itself is not finite, so no numbers are compared; the
            kernel must be non-finite in the same places): cross entropy and focal when every class weight is 0 (0 / 0), mIoU when a
            class is absent from an image and its softmax is exactly 0 on every pixel there (intersection 0 / union 0).
  Adam      against losses_oracle.adam_step element for element, at 3e-7 relative like tests/test_losses_gpu.py: nvcc contracts
            m + (1 - b1) * (g - m) and v * b2 + (1 - b2) * g * g into fused multiply-adds, numpy rounds each operation, so the last
            bit differs. A skipped step is compared bit for bit (int32 views).
"""

import numpy as np
import pytest
import torch

import loss_cases as LC
from oracle import losses_oracle
from robosat_b200 import _lib
from test_train_lockstep_gpu import _grad_check

pytestmark = pytest.mark.gpu

GUARD = 4096
SENTINEL = 0xA5


class Banded:
    """`numel` elements of `dtype` on the device between two GUARD-byte bands of SENTINEL; floats start as NaN, integers as `fill`."""

    def __init__(self, numel, dtype, dev, fill=0, nbytes=None):
        item = torch.empty((), dtype=dtype).element_size()
        self.nbytes = numel * item if nbytes is None else nbytes
        self.raw = torch.full((2 * GUARD + self.nbytes,), SENTINEL, dtype=torch.uint8, device=dev)
        self.t = self.raw[GUARD:GUARD + numel * item].view(dtype)
        assert self.ptr() % 256 == 0
        self.t.fill_(float("nan") if dtype.is_floating_point else fill)

    def ptr(self):
        return self.raw.data_ptr() + GUARD

    def check(self, what):
        assert bool((self.raw[:GUARD] == SENTINEL).all()), "%s: bytes before the buffer were written" % what
        assert bool((self.raw[GUARD + self.nbytes:] == SENTINEL).all()), "%s: bytes after the buffer were written" % what


def _banded_copy(x, dev):
    b = Banded(x.numel(), x.dtype, dev)
    b.t.copy_(x.reshape(-1))
    return b


# --------------------------------------------------------------------------------------------------
# Lovasz
# --------------------------------------------------------------------------------------------------
def _lovasz_raw(logits, targets, dev, want_grad=True):
    lib = _lib.load()
    N, C, H, W = logits.shape
    x, t = logits.to(dev).contiguous(), targets.to(dev).contiguous()
    nbytes = lib.rsb_lovasz_workspace_bytes(N, C, H * W)
    ws = Banded(0, torch.uint8, dev, nbytes=nbytes)
    loss = Banded(1, torch.float32, dev)
    grad = Banded(x.numel(), torch.float32, dev)
    _lib.check(lib.rsb_lovasz(x.data_ptr(), t.data_ptr(), loss.ptr(), grad.ptr() if want_grad else None, ws.ptr(), nbytes,
                              N, C, H * W, _lib.current_stream_ptr()), "rsb_lovasz")
    torch.cuda.synchronize()
    for b, what in ((ws, "workspace"), (loss, "loss"), (grad, "gradient")):
        b.check("rsb_lovasz %s" % what)
    if not want_grad:
        assert bool(torch.isnan(grad.t).all()), "grad = NULL, yet something wrote a gradient"
    return float(loss.t.item()), grad.t.view(logits.shape).cpu()


def _lovasz_check(name, logits, targets, dev):
    loss, grad = _lovasz_raw(logits, targets, dev)
    ref_loss, ref_grad = losses_oracle.lovasz_loss(logits, targets, with_grad=True)
    assert not torch.isnan(grad).any(), "%s: %d gradient elements were not written" % (name, int(torch.isnan(grad).sum()))
    if not torch.equal(grad, ref_grad):
        bad = grad != ref_grad
        per_image = bad.reshape(bad.shape[0], -1).sum(1).tolist()
        first = bad.reshape(-1).nonzero()[0].item()
        raise AssertionError("%s: %d gradient elements differ (per image %s), first at flat index %d: %r != %r"
                             % (name, int(bad.sum()), per_image, first, grad.reshape(-1)[first].item(), ref_grad.reshape(-1)[first].item()))
    assert abs(loss - float(ref_loss)) <= 5e-6 * abs(float(ref_loss)), (name, loss, float(ref_loss))
    return loss, grad


@pytest.mark.parametrize("shape", LC.LOVASZ_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_lovasz_shapes(shape, cuda_device):
    """under one sort tile, several tiles with a ragged last one, an exact tile, P = 2, C = 1, odd H*W; N = 1, 2, 3, 5, 7 (the
    gradient is scaled by fp32(1 / N), which is not a division by N unless N is a power of two)"""
    logits, targets = LC.lovasz_gaussian(shape, 21)
    loss, _ = _lovasz_check("gaussian %s" % (shape,), logits, targets, cuda_device)
    loss_only, _ = _lovasz_raw(logits, targets, cuda_device, want_grad=False)
    assert loss_only == loss


@pytest.mark.parametrize("shape", LC.RAGGED_MULTI_TILE, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", list(LC.LOVASZ_TIE_CASES))
def test_lovasz_equal_errors_keep_index_order(name, shape, cuda_device):
    """the order of equal errors decides the gradient: fp16-rounded logits, five logit values (a fifth of the errors exactly 0), all
    errors equal, errors that differ in one byte of the sort key only (each of the four radix passes alone), a run of 5000 equal
    errors across tile boundaries"""
    logits, targets = LC.LOVASZ_TIE_CASES[name](shape, 5)
    _, grad = _lovasz_check("%s %s" % (name, shape), logits, targets, cuda_device)
    e = LC.errors(logits, targets)
    assert torch.all(grad[e <= 0] == 0)  # an error of exactly 0 (logit exactly +-1) or below gets no gradient
    if name == "all_equal":
        assert torch.equal(grad, LC.lovasz_index_order_grad(targets, shape[1]))


@pytest.mark.parametrize("name,build", [("x 1e4", lambda s: LC.lovasz_scaled(s, 23, 1e4)), ("x 1e-30", lambda s: LC.lovasz_scaled(s, 23, 1e-30)),
                                        ("subnormal", lambda s: LC.lovasz_subnormal(s, 23))], ids=["1e4", "1e-30", "subnormal"])
def test_lovasz_magnitudes(name, build, cuda_device):
    """large errors of both signs; logits so small that every error is exactly 1. A subnormal error cannot occur: 1 - x is 0 or at
    least 2^-24 in fp32."""
    for shape in LC.RAGGED_MULTI_TILE:
        logits, targets = build(shape)
        _lovasz_check("%s %s" % (name, shape), logits, targets, cuda_device)


def test_lovasz_refuses_2_pow_24_elements_without_launching(cuda_device):
    lib = _lib.load()
    N, C, HW = 1, 2, 1 << 23
    nbytes = lib.rsb_lovasz_workspace_bytes(N, C, HW)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=cuda_device)
    x = torch.zeros(16, device=cuda_device)  # never read: the call has to fail on the host
    t = torch.zeros(16, dtype=torch.int64, device=cuda_device)
    loss = Banded(1, torch.float32, cuda_device)
    with pytest.raises(_lib.RsbError, match=r"below 2\^24"):
        _lib.check(lib.rsb_lovasz(x.data_ptr(), t.data_ptr(), loss.ptr(), None, ws.data_ptr(), nbytes, N, C, HW, _lib.current_stream_ptr()), "rsb_lovasz")
    torch.cuda.synchronize()
    assert bool(torch.isnan(loss.t).all())
    loss.check("refused rsb_lovasz")


def test_lovasz_module_scales_the_saved_gradient(cuda_device):
    from robosat_b200.losses import LovaszLoss2d

    logits, targets = LC.lovasz_fp16_rounded((3, 6, 96, 160), 5)
    lg = logits.to(cuda_device).requires_grad_(True)
    loss = LovaszLoss2d()(lg, targets.to(cuda_device))
    (loss * 2).backward()
    ref_loss, ref_grad = losses_oracle.lovasz_loss(logits, targets, with_grad=True)
    assert abs(loss.item() - float(ref_loss)) <= 5e-6 * abs(float(ref_loss))
    assert torch.equal(lg.grad.cpu(), ref_grad * 2)


# --------------------------------------------------------------------------------------------------
# cross entropy, focal, mIoU
# --------------------------------------------------------------------------------------------------
def _softmax_loss_raw(kind, logits, targets, weight, dev, gamma=2.0, want_grad=True):
    lib = _lib.load()
    N, C, H, W = logits.shape
    x, t = logits.to(dev).contiguous(), targets.to(dev).contiguous()
    w = weight.float().to(dev).contiguous() if weight is not None else None
    wp = w.data_ptr() if w is not None else None
    loss = Banded(1, torch.float32, dev)
    grad = Banded(x.numel(), torch.float32, dev)
    gp = grad.ptr() if want_grad else None
    st = _lib.current_stream_ptr()
    if kind == "miou":
        doubles = lib.rsb_miou_scratch_doubles(N, C)
        assert doubles == 4 + 2 * N * C
        scratch = Banded(doubles, torch.float64, dev)
        rc = lib.rsb_miou(x.data_ptr(), t.data_ptr(), wp, loss.ptr(), gp, scratch.ptr(), N, C, H * W, st)
    else:
        scratch = Banded(2, torch.float64, dev)
        if kind == "ce":
            rc = lib.rsb_cross_entropy(x.data_ptr(), t.data_ptr(), wp, loss.ptr(), gp, scratch.ptr(), N, C, H * W, st)
        else:
            rc = lib.rsb_focal(x.data_ptr(), t.data_ptr(), wp, float(gamma), loss.ptr(), gp, scratch.ptr(), N, C, H * W, st)
    _lib.check(rc, "rsb_" + kind)
    torch.cuda.synchronize()
    for b, what in ((loss, "loss"), (grad, "gradient"), (scratch, "scratch")):
        b.check("rsb_%s %s" % (kind, what))
    if not want_grad:
        assert bool(torch.isnan(grad.t).all())
    return float(loss.t.item()), grad.t.view(logits.shape).cpu()


def _oracle(kind, logits, targets, weight, gamma):
    if kind == "ce":
        return losses_oracle.cross_entropy_loss(logits, targets, weight, with_grad=True)
    if kind == "focal":  # the closed form: autograd of losses_oracle.focal_loss is not finite for gamma < 1 on saturated pixels
        return LC.focal_reference(logits, targets, weight, gamma)
    return losses_oracle.miou_loss(logits, targets, weight, with_grad=True)


def _grad_scale(targets, weight, C):
    w = weight.double() if weight is not None else torch.ones(C, dtype=torch.float64)
    total = w[targets].sum()
    return float(w.max() / total) if total > 0 else 0.0


def _softmax_loss_check(name, kind, logits, targets, weight, dev, gamma=2.0, undefined=False):
    loss, grad = _softmax_loss_raw(kind, logits, targets, weight, dev, gamma)
    loss_only, _ = _softmax_loss_raw(kind, logits, targets, weight, dev, gamma, want_grad=False)  # the one-block finish launch
    assert loss_only == loss or (np.isnan(loss_only) and np.isnan(loss)), (name, loss_only, loss)
    ref_loss, ref_grad = _oracle(kind, logits, targets, weight, gamma)
    assert np.isfinite(float(ref_loss)) != undefined, (name, float(ref_loss))
    if undefined:
        assert not np.isfinite(loss), (name, loss)
        assert bool((~torch.isfinite(grad))[~torch.isfinite(ref_grad)].all()), name
        return
    assert abs(loss - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)) + 1e-7, (name, loss, float(ref_loss))
    assert torch.isfinite(ref_grad).all(), name  # a NaN in the reference would compare as "in tolerance"
    scale = _grad_scale(targets, weight, logits.shape[1])
    _grad_check(name, grad, ref_grad, scale if kind != "miou" else max(scale, float(ref_grad.abs().max())))


_SOFTMAX_CASES = LC.softmax_edge_cases()


@pytest.mark.parametrize("case", _SOFTMAX_CASES, ids=[c["name"].replace(" ", "_") for c in _SOFTMAX_CASES])
def test_softmax_losses_at_the_edges(case, cuda_device):
    """expf underflowing to subnormals and to 0 on and off the target, |logits| of 1e4, a class absent from an image, a class of
    weight 0, C = 1 and 64, H*W = 1 and odd; focal with gamma 0.5, 2 and 5 (gamma < 1 on a saturated pixel used to give
    inf * 0 = NaN in the gradient: the regression test of that fix is every case here whose softmax reaches 1 at the target)"""
    x, t, w = case["logits"], case["targets"], case["weight"]
    for kind, gamma in (("ce", None), ("focal", 0.5), ("focal", 2.0), ("focal", 5.0), ("miou", None)):
        name = "%s gamma=%s: %s" % (kind, gamma, case["name"])
        _softmax_loss_check(name, kind, x, t, w, cuda_device, gamma, undefined=kind in case["undefined"])


def test_miou_refuses_65_classes(cuda_device):
    lib = _lib.load()
    x = torch.zeros((1, 65, 2, 2), device=cuda_device)
    t = torch.zeros((1, 2, 2), dtype=torch.int64, device=cuda_device)
    loss = Banded(1, torch.float32, cuda_device)
    scratch = torch.zeros(lib.rsb_miou_scratch_doubles(1, 65), dtype=torch.float64, device=cuda_device)
    with pytest.raises(_lib.RsbError, match="miou"):
        _lib.check(lib.rsb_miou(x.data_ptr(), t.data_ptr(), None, loss.ptr(), None, scratch.data_ptr(), 1, 65, 4, _lib.current_stream_ptr()), "rsb_miou")
    torch.cuda.synchronize()
    assert bool(torch.isnan(loss.t).all())
    assert lib.rsb_miou_scratch_doubles(0, 2) == 0 and lib.rsb_miou_scratch_doubles(2, 0) == 0


def test_softmax_loss_modules_at_an_edge(cuda_device):
    from robosat_b200.losses import CrossEntropyLoss2d, FocalLoss2d, mIoULoss2d

    case = _SOFTMAX_CASES[0]
    x, t, w = case["logits"], case["targets"], case["weight"]
    for kind, gamma, mod in (("ce", None, CrossEntropyLoss2d(weight=w)), ("focal", 0.5, FocalLoss2d(gamma=0.5, weight=w)), ("miou", None, mIoULoss2d(weight=w))):
        lg = x.to(cuda_device).requires_grad_(True)
        loss = mod.to(cuda_device)(lg, t.to(cuda_device))
        (loss * 0.5).backward()
        raw_loss, raw_grad = _softmax_loss_raw(kind, x, t, w, cuda_device, gamma)
        assert loss.item() == raw_loss and torch.equal(lg.grad.cpu(), raw_grad * 0.5), kind


def test_labels_outside_the_classes_are_left_out(cuda_device):
    """A label outside [0, C) contributes to no sum and gets a zero gradient: the result is the float64 reference on the image
    without those pixels (whole columns here, so that what is left is still an image)."""
    N, C, H, W = 3, 3, 12, 20
    g = torch.Generator().manual_seed(70)
    logits = torch.randn((N, C, H, W), generator=g) * 2
    targets = LC.targets_random(N, C, H, W, 71)
    weight = torch.tensor([0.7, 1.0, 1.6])
    keep = torch.ones(W, dtype=torch.bool)
    for col, label in ((2, -1), (7, C), (8, 255), (19, -(1 << 40))):
        targets[:, :, col] = label
        keep[col] = False
    kept_x, kept_t = logits[:, :, :, keep].contiguous(), targets[:, :, keep].contiguous()
    for kind, gamma in (("ce", None), ("focal", 2.0), ("miou", None)):
        loss, grad = _softmax_loss_raw(kind, logits, targets, weight, cuda_device, gamma)
        ref_loss, ref_grad = _oracle(kind, kept_x, kept_t, weight, gamma)
        assert abs(loss - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)) + 1e-7, (kind, loss, float(ref_loss))
        assert torch.all(grad[:, :, :, ~keep] == 0), kind
        scale = _grad_scale(kept_t, weight, C)
        _grad_check(kind, grad[:, :, :, keep], ref_grad, scale if kind != "miou" else max(scale, float(ref_grad.abs().max())))


# --------------------------------------------------------------------------------------------------
# metrics
# --------------------------------------------------------------------------------------------------
def test_metrics_first_maximum_wins(cuda_device):
    """argmax ties on a large share of the pixels (fp16-rounded logits, five logit values, +0.0 against -0.0) and targets >= 2,
    where predicted / actual is counted in no cell"""
    lib = _lib.load()
    for name, logits, targets in LC.metrics_tie_cases():
        N, C, H, W = logits.shape
        x, t = logits.to(cuda_device), targets.to(cuda_device)
        counts = Banded(4, torch.int64, cuda_device, fill=0)
        _lib.check(lib.rsb_metrics_count(x.data_ptr(), t.data_ptr(), counts.ptr(), N, C, H * W, _lib.current_stream_ptr()), "rsb_metrics_count")
        torch.cuda.synchronize()
        counts.check("rsb_metrics_count")
        assert tuple(counts.t.cpu().tolist()) == tuple(losses_oracle.metrics_counts(logits, targets)), name


# --------------------------------------------------------------------------------------------------
# Adam
# --------------------------------------------------------------------------------------------------
# The entry points take lr, the betas and eps as C floats, and form 1 - beta from the float they receive: 1 - 0.999f is
# 0.00099998712, not torch's 1 - 0.999 = 0.001 (1.3e-5 less; in the parameters the bias correction, formed from the same float,
# cancels it to below 1e-9). The reference below is therefore evaluated at the betas the kernel really gets.
LR, EPS = 1e-4, 1e-8
B1, B2 = float(np.float32(0.9)), float(np.float32(0.999))


def _close(name, got, ref, extra=0.0):
    """|err| <= 3e-7 |ref| + 1e-9 + extra (elementwise)"""
    got, ref = got.cpu().numpy().astype(np.float64), np.asarray(ref, dtype=np.float64)
    bad = ~(np.abs(got - ref) <= 3e-7 * np.abs(ref) + 1e-9 + extra)  # NaN counts as bad
    assert not bad.any(), "%s: %d of %d elements out of tolerance, first at %d: %r != %r" % (name, bad.sum(), bad.size, bad.argmax(), got[bad][0], ref[bad][0])


def _adam_bands(p, dev):
    return _banded_copy(torch.from_numpy(p), dev), _banded_copy(torch.zeros(p.size), dev), _banded_copy(torch.zeros(p.size), dev)


@pytest.mark.parametrize("n", LC.ADAM_SIZES)
def test_adam_sizes(n, cuda_device):
    """below one block, around a block, exactly one sweep of the capped grid, one element more, several sweeps with a ragged end;
    steps 1, 2 and 100 000 (bias corrections saturated); a tenth of the elements have gradient 0 and second moment 0"""
    lib = _lib.load()
    p0, grads = LC.adam_inputs(n, 31)
    P, M, V = _adam_bands(p0, cuda_device)
    rp, rm, rv = p0, np.zeros_like(p0), np.zeros_like(p0)
    slack = np.zeros(n)  # exp_avg is a sum that can cancel: a rounding error of the operands' size stays, decaying by beta1 per step
    for g, step in zip(grads, (1, 2, 100_000)):
        G = _banded_copy(torch.from_numpy(g), cuda_device)
        _lib.check(lib.rsb_adam_step(P.ptr(), G.ptr(), M.ptr(), V.ptr(), n, LR, B1, B2, EPS, step, _lib.current_stream_ptr()), "rsb_adam_step")
        torch.cuda.synchronize()
        rm_old = rm
        rp, rm, rv = losses_oracle.adam_step(rp, g, rm, rv, lr=LR, step=step, b1=B1, b2=B2, eps=EPS)
        what = "n=%d step=%d" % (n, step)
        slack = B1 * slack + 3e-7 * (np.abs(rm_old) + np.abs(g))
        _close(what + " exp_avg", M.t, rm, extra=slack)
        _close(what + " exp_avg_sq", V.t, rv)
        _close(what + " param", P.t, rp)
        for b in (P, G, M, V):
            b.check(what)
        zero = torch.from_numpy(g == 0).to(cuda_device)
        assert bool((V.t[zero] == 0).all()) and torch.equal(P.t[zero], torch.from_numpy(p0).to(cuda_device)[zero])


def _guarded(P, G, M, V, n, step, state, lib):
    _lib.check(lib.rsb_adam_step_guarded(P.data_ptr(), G.data_ptr(), M.data_ptr(), V.data_ptr(), n, LR, B1, B2, EPS, step, state.ptr(),
                                         _lib.current_stream_ptr()), "rsb_adam_step_guarded")
    torch.cuda.synchronize()


def _bits(t):
    return t.view(torch.int32).clone()


_N_GUARDED = 3_000_001  # n / 4 exceeds one sweep of the grid, so the 16-byte loop iterates; n % 4 = 1, so the last element is in the tail
_POSITIONS = {"first": 0, "last": _N_GUARDED - 1, "second sweep of the scalar loop": LC.GRID_SWEEP + 5, "second sweep of the 16-byte loop": 4 * LC.GRID_SWEEP + 5}


@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("value", [float("inf"), float("-inf"), float("nan")], ids=["+inf", "-inf", "nan"])
def test_guarded_adam_finds_one_non_finite_element_anywhere(value, aligned, cuda_device):
    """one non-finite gradient element at index 0, n - 1 and in the second sweep of either loop of grad_finite_kernel, in arenas that
    are 16-byte aligned (float4 loop + scalar tail) or not (scalar loop only). Sequence per position: good, bad, bad, good. A skipped
    step leaves parameters and both moments bitwise unchanged, and the good step after it uses the count of steps really taken."""
    lib = _lib.load()
    n, dev = _N_GUARDED, cuda_device
    p0, grads = LC.adam_inputs(n, 33)
    off = 0 if aligned else 1  # arenas that start one float after a 16-byte boundary
    for where, pos in _POSITIONS.items():
        bands = [_banded_copy(torch.from_numpy(a), dev) for a in (np.concatenate([np.zeros(off, np.float32), p0]), np.zeros(n + off, np.float32), np.zeros(n + off, np.float32))]
        P, M, V = (b.t[off:] for b in bands)
        state = Banded(4, torch.int32, dev, fill=0)
        good = [torch.from_numpy(np.concatenate([np.zeros(off, np.float32), g])).to(dev)[off:] for g in grads[:2]]
        bad = torch.cat([torch.zeros(off, device=dev), good[1]])[off:]  # a clone would be aligned again
        bad[pos] = value
        assert (P.data_ptr() % 16 == 0) == aligned and (bad.data_ptr() % 16 == 0) == aligned
        rp, rm, rv = losses_oracle.adam_step(p0, grads[0], np.zeros_like(p0), np.zeros_like(p0), lr=LR, step=1, b1=B1, b2=B2, eps=EPS)
        rm_old, g_taken = np.zeros_like(p0), grads[0]
        expect_state = [[0, 0, 0, 1], [0, 1, 1, 2], [0, 2, 1, 3], [0, 2, 0, 4]]
        for i, g in enumerate((good[0], bad, bad, good[1])):
            before = [_bits(a) for a in (P, M, V)]
            _guarded(P, g, M, V, n, i + 1, state, lib)
            what = "%s at %s (%d), call %d" % (value, where, pos, i + 1)
            assert state.t.cpu().tolist() == expect_state[i], what
            if i in (1, 2):
                for a, b, label in zip((P, M, V), before, ("param", "exp_avg", "exp_avg_sq")):
                    assert torch.equal(_bits(a), b), "%s: %s changed in a skipped step" % (what, label)
            else:
                if i == 3:  # host step 4, two skipped: the second step really taken
                    rm_old, g_taken = rm, grads[1]
                    rp, rm, rv = losses_oracle.adam_step(rp, grads[1], rm, rv, lr=LR, step=2, b1=B1, b2=B2, eps=EPS)
                _close(what + " param", P, rp)
                _close(what + " exp_avg_sq", V, rv)
                _close(what + " exp_avg", M, rm, extra=3e-7 * (np.abs(g_taken) + np.abs(rm_old)))
            for b in bands + [state]:
                b.check(what)


def test_guarded_adam_equals_plain_adam_on_finite_gradients(cuda_device):
    """While no step is skipped the guarded kernel computes what the plain one does, to rounding: the compiler contracts the two
    kernels' updates into fused multiply-adds differently, so exp_avg_sq and a few parameters differ in the last bit. Compared at
    the 3e-7 of the other Adam checks."""
    lib = _lib.load()
    n = LC.GRID_SWEEP + 257
    p0, grads = LC.adam_inputs(n, 35)
    plain, guarded = _adam_bands(p0, cuda_device), _adam_bands(p0, cuda_device)
    state = Banded(4, torch.int32, cuda_device, fill=0)
    slack = np.zeros(n)
    for s, g in enumerate(grads):
        G = torch.from_numpy(g).to(cuda_device)
        m_old = plain[1].t.cpu().numpy()
        _lib.check(lib.rsb_adam_step(plain[0].ptr(), G.data_ptr(), plain[1].ptr(), plain[2].ptr(), n, LR, B1, B2, EPS, s + 1, _lib.current_stream_ptr()), "rsb_adam_step")
        _guarded(guarded[0].t, G, guarded[1].t, guarded[2].t, n, s + 1, state, lib)
        slack = B1 * slack + 3e-7 * (np.abs(m_old) + np.abs(g))
        for a, b, label, extra in zip(plain, guarded, ("param", "exp_avg", "exp_avg_sq"), (0.0, slack, 0.0)):
            _close("step %d %s" % (s + 1, label), b.t, a.t.cpu().numpy(), extra=extra)
            a.check("plain step %d" % (s + 1))
            b.check("guarded step %d" % (s + 1))
        assert state.t.cpu().tolist() == [0, 0, 0, s + 1]


# --------------------------------------------------------------------------------------------------
# rsb_sort_unique_u64
# --------------------------------------------------------------------------------------------------
def test_sort_unique_edges(cuda_device):
    """The contract (include/rsb200.h): the keys are below 2^key_bits, of which ceil(key_bits / 8) bytes are sorted; key_bits = 64
    sorts the whole word as unsigned, so int64 keys with the top bit set come after the others. Keys above 2^key_bits are the
    caller's error, which the function cannot see; every case asserts that it is inside the contract before it calls. n = 0, whole
    tiles, all keys equal, sorted unique input, key_bits 0, 1, 63 and 64. Only keys[0 .. unique_count) is defined afterwards."""
    lib = _lib.load()
    for name, keys, bits in LC.sort_unique_cases():
        assert LC.in_contract(keys, bits), name
        n = keys.size
        K = Banded(n, torch.int64, cuda_device, fill=-1)
        K.t.copy_(torch.from_numpy(keys.view(np.int64)))
        nbytes = lib.rsb_sort_unique_workspace_bytes(n)
        ws = Banded(0, torch.uint8, cuda_device, nbytes=nbytes)
        count = Banded(1, torch.int64, cuda_device, fill=-1)
        _lib.check(lib.rsb_sort_unique_u64(K.ptr(), n, bits, ws.ptr() if n else None, nbytes, count.ptr(), _lib.current_stream_ptr()), "rsb_sort_unique_u64")
        torch.cuda.synchronize()
        ref = np.unique(keys)
        u = int(count.t.item())
        assert u == ref.size, (name, u, ref.size)
        assert np.array_equal(K.t[:u].cpu().numpy().view(np.uint64), ref), name
        for b, what in ((K, "keys"), (ws, "workspace"), (count, "count")):
            b.check("%s %s" % (name, what))
