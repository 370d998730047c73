"""Every kernel launch of the training step against a float64 replay of the same op on the kernel's own inputs
(tests/lockstep.py; bounds derived in its docstring), the split-K weight-gradient kernel at shapes where its tiling is ragged,
and the loss kernels at training batch sizes against float64."""

import ctypes

import numpy as np
import pytest
import torch

import emulate
import lockstep
from oracle import losses_oracle
from robosat_b200 import _lib, synth, train_engine
from robosat_b200.engine import _src_dense, make_conv_desc

pytestmark = pytest.mark.gpu


# --------------------------------------------------------------------------------------------------
# the whole training step in lockstep
# --------------------------------------------------------------------------------------------------
def _lockstep(cuda_device, C, B, H, W, dlogits_from_ce, chained=True, deterministic=True):
    _, dut, twin = lockstep.make_pair(C, B, H, W, 1024.0, cuda_device)
    x = synth.normalize_tiles(synth.make_tiles_u8(B, max(H, W), seed=1))[:, :, :H, :W].contiguous()
    if dlogits_from_ce:
        # the cross-entropy gradient of the network's own logits on synthetic masks: realistic magnitudes (~1 / pixels)
        with torch.no_grad():
            ref = torch.randn((B, C, H, W), generator=torch.Generator().manual_seed(2))
        masks = synth.make_masks(B, max(H, W), C, seed=3)[:, :H, :W].contiguous()
        lib = _lib.load()
        ld, md = ref.to(cuda_device), masks.to(cuda_device)
        loss = torch.zeros(1, device=cuda_device)
        dl = torch.empty_like(ld)
        scratch = torch.empty(2, dtype=torch.float64, device=cuda_device)
        _lib.check(lib.rsb_cross_entropy(ld.data_ptr(), md.data_ptr(), None, loss.data_ptr(), dl.data_ptr(), scratch.data_ptr(), B, C, H * W,
                                         _lib.current_stream_ptr()), "rsb_cross_entropy")
        torch.cuda.synchronize()
        dlogits = dl.cpu()
    else:
        dlogits = torch.randn((B, C, H, W), generator=torch.Generator().manual_seed(3)) * 1e-3
    ex = lockstep.GpuExecutor(dut, chained_bn=chained, repeat_wgrad=deterministic)
    ls = lockstep.Lockstep(ex, twin)
    ls.run(x, dlogits, dut_x=x.to(cuda_device), dut_dlogits=dlogits.to(cuda_device))
    print("\n%d x %d x %d x %d, %d classes:\n%s" % (B, 3, H, W, C, ls.table()))
    assert len(ls.checked["fwd"]) == len(dut.fwd_ops) and len(ls.checked["bwd"]) == len(dut.bwd_ops)
    return dut, ls


def test_train_step_lockstep_128(cuda_device):
    dut, ls = _lockstep(cuda_device, 2, 2, 128, 128, dlogits_from_ce=True)
    assert lockstep.n_ops(dut) == 413
    lib = _lib.load()
    plans = dut.__dict__.get("_wgrad_plans", [])
    assert len(plans) == 60 and any(lib.rsb_wgrad_plan_scratch_bytes(p) > 0 for p in plans), \
        "no weight-gradient plan used the deterministic split-K scratch: its reduction would be unchecked"


def test_train_step_lockstep_rectangular_six_classes(cuda_device):
    _lockstep(cuda_device, 6, 3, 64, 128, dlogits_from_ce=False)


def test_train_step_lockstep_unchained_paths(cuda_device, monkeypatch):
    """the non-default paths: BatchNorm statistics re-read z, separate (memset) BatchNorm launches, fp32-atomic split-K"""
    monkeypatch.setattr(train_engine, "CONV_STATS", False)
    monkeypatch.setattr(train_engine, "BN_CHAINED", False)
    monkeypatch.setenv("RSB_WGRAD_DETERMINISTIC", "0")
    dut, _ = _lockstep(cuda_device, 2, 2, 64, 64, dlogits_from_ce=False, chained=False, deterministic=False)
    assert all(u.stats is None for u in dut.units.values()) and dut.__dict__.get("_wgrad_scratch") is None


# --------------------------------------------------------------------------------------------------
# weight gradients: split-K with and without the deterministic scratch, ragged tilings
# --------------------------------------------------------------------------------------------------
def _wgrad_cases(dev):
    """(name, desc, dy tensor, dy element offset, keep-alive) for engine layers and synthetic ragged shapes"""
    params = {k[7:]: v.to(dev) for k, v in synth.make_state_dict(2, seed=0).items()}
    eng = train_engine.UNetTrainEngine(params, 2, 2, 128, 128, device=dev)
    eng.forward(synth.normalize_tiles(synth.make_tiles_u8(2, 128, seed=1)).to(dev))  # real activations as the A operands
    torch.cuda.synchronize()
    g = torch.Generator().manual_seed(7)
    cases = []
    for name in ("stem", "resnet.layer1.0.conv1", "resnet.layer1.0.conv2", "resnet.layer2.0.conv2", "dec3", "dec4", "dec5"):
        u = eng.units[name]
        dy = (torch.randn(tuple(u.out.shape), generator=g) * 0.5).half().to(dev)
        cases.append((name, u.desc, dy, u.out_offset, (eng,)))
    # synthetic 1x1 / 3x3 convolutions: 5 and 3 K blocks (the last group of 4 ragged), ragged Wt / Ht, Cout below one 128 block
    for (N, H, W, Cin, cout, taps) in ((3, 20, 36, 320, 64, 1), (2, 28, 44, 192, 32, 1), (3, 18, 26, 64, 64, 3)):
        x = (torch.randn((N, H, W, Cin), generator=g)).half().to(dev)
        out = torch.zeros((N, H, W, cout), dtype=torch.float16, device=dev)
        segs = [(0, kh - 1, kw - 1, Cin // 64) for kh in range(taps) for kw in range(taps)] if taps == 3 else [(0, 0, 0, Cin // 64)]
        K = 64 * sum(s[3] for s in segs)
        w = torch.zeros((cout, K), dtype=torch.float16, device=dev)
        d = make_conv_desc([_src_dense(x, N, H, W, Cin)], segs, w, None, cout, 1, (W, H, N), out, (cout, W * cout, H * W * cout), relu=False)
        dy = (torch.randn((N, H, W, cout), generator=g) * 0.5).half().to(dev)
        cases.append(("synthetic N%d %dx%d Cin%d Cout%d %dx%d" % (N, H, W, Cin, cout, taps, taps), d, dy, 0, (x, out, w)))
    return cases


def _host_copy(d, keep):
    """the descriptor re-pointed at host copies of its sources and of dy, for the float64 replay"""
    hd = type(d).from_buffer_copy(d)
    host = []
    for i in range(d.nsrc):
        s = d.srcs[i]
        t = next(t for t in _all_tensors(keep) if t.data_ptr() <= s.ptr < t.data_ptr() + t.numel() * t.element_size())
        h = t.cpu()
        host.append(h)
        hd.srcs[i].ptr = h.data_ptr() + (s.ptr - t.data_ptr())
    return hd, host


def _all_tensors(keep):
    out = []
    for k in keep:
        if isinstance(k, torch.Tensor):
            out.append(k)
        else:
            out += [t for t in k._keep] + list(k.params.values())
    return out


def _check_wgrad(name, got, ref, tol):
    err = np.abs(got.double().cpu().numpy().reshape(ref.shape) - ref)
    err[np.isnan(err)] = np.inf
    worst = float(np.divide(err, tol, out=np.where(err > 0, np.inf, 0.0), where=tol > 0).max())
    assert (err <= tol).all(), "%s: %d elements out of tolerance, worst err/tol %.3g" % (name, int((err > tol).sum()), worst)
    return worst


def test_wgrad_split_k_paths_match_float64(cuda_device):
    lib, st = _lib.load(), _lib.current_stream_ptr()
    cases = _wgrad_cases(cuda_device)
    refs, plans, outs = [], [], []
    kblocks = set()
    for name, d, dy, off, keep in cases:
        hd, host = _host_copy(d, keep)
        dyh = dy.cpu()
        ref, mag = emulate.run_wgrad(hd, dyh.data_ptr() + 2 * off, None, f64=True)
        P = d.Nt * d.Ht * d.Wt
        refs.append((ref, 2.0 ** -23 * (P / 16 + P / 64 + 17) * mag))  # the bound of tests/lockstep.py
        dw = torch.full((ref.size,), float("nan"), dtype=torch.float32, device=cuda_device)
        plan = ctypes.c_void_p()
        _lib.check(lib.rsb_wgrad_plan_create(ctypes.byref(d), dy.data_ptr() + 2 * off, dw.data_ptr(), ctypes.byref(plan)), "wgrad_plan[%s]" % name)
        need = int(lib.rsb_wgrad_plan_scratch_bytes(plan))
        assert need > 0, "%s: a single-slice plan would not exercise split-K" % name
        plans.append(plan)
        outs.append(dw)
        kblocks.add(sum(d.segs[j].cblocks for j in range(d.nseg)) % 4)
        del host
    assert kblocks >= {1, 2, 3}, kblocks  # ragged last K group of every size
    worst = {}
    try:
        for (name, d, dy, off, keep), plan, dw, (ref, tol) in zip(cases, plans, outs, refs):
            need = int(lib.rsb_wgrad_plan_scratch_bytes(plan))
            # 1. fp32-atomic split-K (no scratch)
            _lib.check(lib.rsb_wgrad_run(plan, st), "wgrad_run")
            torch.cuda.synchronize()
            worst[name + " atomics"] = _check_wgrad(name + " atomics", dw, ref, tol)
            # 2. deterministic split-K: twice, bit-identical
            scratch = torch.empty(need // 4 + 4, dtype=torch.float32, device=cuda_device)
            _lib.check(lib.rsb_wgrad_plan_set_scratch(plan, scratch.data_ptr(), need), "set_scratch")
            runs = []
            for _ in range(2):
                dw.fill_(float("nan"))
                _lib.check(lib.rsb_wgrad_run(plan, st), "wgrad_run")
                torch.cuda.synchronize()
                runs.append(dw.clone())
            assert torch.equal(runs[0], runs[1]), name
            worst[name + " scratch"] = _check_wgrad(name + " scratch", dw, ref, tol)
            # rejected scratches: too small, not 16-byte aligned
            assert lib.rsb_wgrad_plan_set_scratch(plan, scratch.data_ptr(), need - 16) != 0
            assert lib.rsb_wgrad_plan_set_scratch(plan, scratch.data_ptr() + 4, need) != 0
        # 3. every plan on ONE shared scratch, launched back to back, then checked
        big = max(int(lib.rsb_wgrad_plan_scratch_bytes(p)) for p in plans)
        shared = torch.empty(big // 4, dtype=torch.float32, device=cuda_device)
        for plan, dw in zip(plans, outs):
            _lib.check(lib.rsb_wgrad_plan_set_scratch(plan, shared.data_ptr(), big), "set_scratch")
            dw.fill_(float("nan"))
        for plan in plans:
            _lib.check(lib.rsb_wgrad_run(plan, st), "wgrad_run")
        torch.cuda.synchronize()
        for (name, *_), dw, (ref, tol) in zip(cases, outs, refs):
            worst[name + " shared"] = _check_wgrad(name + " shared", dw, ref, tol)
    finally:
        for p in plans:
            lib.rsb_wgrad_plan_destroy(p)
    for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:8]:
        print("wgrad worst err/tol %-52s %.3g" % (k, v))


# --------------------------------------------------------------------------------------------------
# losses at training scale
# --------------------------------------------------------------------------------------------------
def _loss_inputs(N, C, S, seed, aligned=False):
    g = torch.Generator().manual_seed(seed)
    targets = synth.make_masks(N, S, C, seed=seed + 1)
    if aligned:  # confident and mostly right: the soft-IoU term exceeds the cross entropy
        logits = 2.0 * (torch.nn.functional.one_hot(targets, C).permute(0, 3, 1, 2).float() * 2 - 1) + 0.5 * torch.randn((N, C, S, S), generator=g)
    else:
        logits = torch.randn((N, C, S, S), generator=g) * 3
    # saturated pixels, where the fp32 softmax is exactly 1 / 0: rows 0-3 at the target class, rows 4-5 at another class
    # (those cost -log p = 120 each, so only the unaligned inputs get them: they would make cross entropy the larger mIoU term)
    for rows, shift in ((slice(0, 4), 0),) + (() if aligned else ((slice(4, 6), 1),)):
        hot = torch.nn.functional.one_hot((targets[:, rows, :] + shift) % C, C).permute(0, 3, 1, 2).bool()
        logits[:, :, rows, :] = torch.where(hot, 60.0, -60.0)
    return logits.contiguous(), targets  # the one-hot arithmetic leaves channels-last strides


def _grad_check(name, got, ref, scale):
    """elementwise: |err| <= 1e-4 |ref| + 1e-5 * (largest gradient magnitude of that pixel's weight)"""
    err = (got.double() - ref.double()).abs()
    tol = 1e-4 * ref.double().abs() + 1e-5 * scale
    bad = err > tol
    assert torch.isfinite(got).all(), "%s: non-finite gradient" % name
    assert not bad.any(), "%s: %d elements out of tolerance, worst err %.3g" % (name, int(bad.sum()), float(err.max()))


@pytest.mark.parametrize("N,C,S", [(16, 2, 512), (8, 6, 256)])
@pytest.mark.parametrize("weighted", [False, True])
def test_losses_at_training_scale_match_float64(N, C, S, weighted, cuda_device):
    from robosat_b200.losses import CrossEntropyLoss2d, FocalLoss2d, mIoULoss2d

    lib = _lib.load()
    w = (torch.rand(C, generator=torch.Generator().manual_seed(9)) + 0.5) if weighted else None
    branches = set()
    for aligned in (False, True):
        logits, targets = _loss_inputs(N, C, S, 11 + C, aligned)
        td = targets.to(cuda_device)
        wsum = (w[targets] if w is not None else torch.ones(targets.shape)).sum().double()
        scale = float(((w.max() if w is not None else 1.0)) / wsum)
        for label, mod, oracle in (("ce", CrossEntropyLoss2d(weight=w), lambda l: losses_oracle.cross_entropy_loss(l, targets, w, with_grad=True)),
                                   ("focal", FocalLoss2d(gamma=2, weight=w), lambda l: losses_oracle.focal_loss(l, targets, w, gamma=2, with_grad=True)),
                                   ("miou", mIoULoss2d(weight=w), lambda l: losses_oracle.miou_loss(l, targets, w, with_grad=True))):
            lg = logits.to(cuda_device).requires_grad_(True)
            loss = mod.to(cuda_device)(lg, td)
            loss.backward()
            ref_loss, ref_grad = oracle(logits)
            assert abs(loss.item() - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)) + 1e-7, (label, loss.item(), float(ref_loss))
            gscale = scale if label != "miou" else max(scale, float(ref_grad.abs().max()))
            _grad_check("%s N%d C%d %d^2 weighted=%s aligned=%s" % (label, N, C, S, weighted, aligned), lg.grad.cpu(), ref_grad, gscale)
            if label == "miou":
                ce = float(losses_oracle.cross_entropy_loss(logits, targets, w))
                branches.add("ce" if abs(float(ref_loss) - ce) <= 1e-6 * abs(ce) else "iou")
        counts = torch.zeros(4, dtype=torch.int64, device=cuda_device)
        ld = logits.to(cuda_device)
        _lib.check(lib.rsb_metrics_count(ld.data_ptr(), td.data_ptr(), counts.data_ptr(), N, C, S * S, _lib.current_stream_ptr()), "metrics")
        torch.cuda.synchronize()
        assert tuple(counts.cpu().tolist()) == losses_oracle.metrics_counts(logits, targets)
    assert branches == {"ce", "iou"}, branches


def test_focal_gamma_zero_is_finite_on_saturated_pixels(cuda_device):
    """gamma = 0 is plain cross entropy. On a pixel whose softmax is exactly 1 the derivative of the penalty,
    gamma * (1 - p)^(gamma - 1), must count as zero (torch's pow backward does so for exponent 0), not 0 * inf = NaN,
    which would make the guarded Adam skip every step without an error."""
    from robosat_b200.losses import FocalLoss2d

    logits = torch.tensor([[[[60.0, -1.0, 0.5]], [[-60.0, 1.0, 0.25]]]])  # pixel 0: p_t == 1 exactly in fp32
    targets = torch.tensor([[[0, 1, 0]]])
    lg = logits.to(cuda_device).requires_grad_(True)
    FocalLoss2d(gamma=0)(lg, targets.to(cuda_device)).backward()
    ref_loss, ref_grad = losses_oracle.focal_loss(logits, targets, gamma=0, with_grad=True)
    assert torch.isfinite(lg.grad).all(), lg.grad
    assert torch.allclose(lg.grad.cpu(), ref_grad, rtol=1e-5, atol=1e-7)
