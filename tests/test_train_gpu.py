"""GPU parity of the training path: helper kernels vs torch, the wgmma weight-gradient kernel vs its CPU emulation,
and the whole UNetTrainEngine (train-mode forward + backward) vs (a) the fp32 oracle forward and (b) autograd through the
mask-frozen fp32 network (tests/linearized.py).

Tolerances: activations / activation gradients are fp16, so single kernels agree to fp16 rounding of their outputs;
whole-network gradients are compared in relative L2 per parameter tensor (<= 6e-2, median <= 3e-2: ~100 chained fp16
roundings, batch statistics over as few as 8 pixels in layer4 at this test size)."""

import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_cases
import emulate
import linearized
from oracle import unet_oracle
from robosat_b200 import _lib, synth
from robosat_b200.train_engine import UNetTrainEngine

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a - b).pow(2).sum().sqrt() / b.pow(2).sum().sqrt().clamp_min(1e-30)).item()


def test_batchnorm_chained_train_kernels(cuda_device):
    lib, st = _lib.load(), _lib.current_stream_ptr()
    g = torch.Generator().manual_seed(0)
    for (M, C) in [(2 * 16 * 16, 64), (3 * 8 * 8, 2048), (5 * 7 * 9, 256), (4 * 96 * 96, 128)]:  # last: > 1000 blocks
        z = (torch.randn((M, C), generator=g) * 1.5 + 0.3).half()
        res = torch.randn((M, C), generator=g).half()
        gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
        rm, rv = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
        # torch reference on the same fp16 values
        zt = z.float().t().reshape(1, C, M, 1).clone().requires_grad_(True)
        gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        rm_ref, rv_ref = rm.clone(), rv.clone()
        y_ref = F.relu(F.batch_norm(zt, rm_ref, rv_ref, gt, bt, training=True, momentum=0.1, eps=1e-5) + res.float().t().reshape(1, C, M, 1))
        dy = torch.randn((M, C), generator=g).half()
        y_ref.backward(dy.float().t().reshape(1, C, M, 1))
        d = cuda_device
        zd, resd, dyd = z.to(d), res.to(d), dy.to(d)
        gd, bd, rmd, rvd = gamma.to(d), beta.to(d), rm.to(d), rv.to(d)
        nb = torch.zeros((), dtype=torch.int64, device=d)
        sums = torch.zeros(20 * C, dtype=torch.float64, device=d)  # zeroed once: every kernel below leaves it zeroed again
        mean, invstd, scale, shift = (torch.zeros(C, device=d) for _ in range(4))
        y = torch.zeros((M, C), dtype=torch.float16, device=d)
        # the statistics input a convolution epilogue writes: [rows][2][C] fp32 column sums / sums of squares of 32-row blocks
        rows = -(-M // 32)
        zb = torch.zeros((rows * 32, C), dtype=torch.float64)
        zb[:M] = z.double()
        zb = zb.reshape(rows, 32, C)
        partials = torch.stack((zb.sum(1), (zb * zb).sum(1)), 1).float().contiguous().to(d)
        _lib.check(lib.rsb_bn_partials_finalize(partials.data_ptr(), rows, sums.data_ptr(), gd.data_ptr(), bd.data_ptr(), rmd.data_ptr(),
                                                rvd.data_ptr(), nb.data_ptr(), mean.data_ptr(), invstd.data_ptr(), scale.data_ptr(),
                                                shift.data_ptr(), M, C, 1e-5, 0.1, st), "partials_finalize")
        _lib.check(lib.rsb_bn_apply_chained(zd.data_ptr(), scale.data_ptr(), shift.data_ptr(), resd.data_ptr(), y.data_ptr(), M, C, 1, st), "apply")
        dz, gout = torch.zeros_like(y), torch.zeros_like(y)
        dg, db = torch.zeros(C, device=d), torch.zeros(C, device=d)
        _lib.check(lib.rsb_bn_backward_chained(dyd.data_ptr(), y.data_ptr(), zd.data_ptr(), mean.data_ptr(), invstd.data_ptr(), gd.data_ptr(), None,
                                               None, sums.data_ptr(), dz.data_ptr(), gout.data_ptr(), dg.data_ptr(), db.data_ptr(), 0.5, M, C, st),
                   "bwd")
        torch.cuda.synchronize()
        yr = y_ref.detach().reshape(C, M).t()
        assert (y.float().cpu() - yr).abs().max().item() <= 4e-3 * max(1.0, yr.abs().max().item() / 4)
        assert torch.allclose(rmd.cpu(), rm_ref, atol=1e-5) and torch.allclose(rvd.cpu(), rv_ref, rtol=1e-4, atol=1e-5) and int(nb.item()) == 1
        assert _rel(dz.float().cpu(), zt.grad.reshape(C, M).t()) < 3e-3
        assert _rel(dg.cpu() * 2, gt.grad) < 2e-3 and _rel(db.cpu() * 2, bt.grad) < 2e-3
        mask = (yr > 0).float()
        assert _rel(gout.float().cpu(), dy.float() * mask) < 1e-3
        # plain relu(bn(z)) (no identity branch): the mask re-derived from z gives the same bits as the mask read from y
        y2 = torch.zeros_like(y)
        _lib.check(lib.rsb_bn_apply_chained(zd.data_ptr(), scale.data_ptr(), shift.data_ptr(), None, y2.data_ptr(), M, C, 1, st), "apply")
        outs = []
        for use_z in (False, True):
            dz2, go2 = torch.zeros_like(y), torch.zeros_like(y)
            dg2, db2 = torch.zeros(C, device=d), torch.zeros(C, device=d)
            _lib.check(lib.rsb_bn_backward_chained(dyd.data_ptr(), None if use_z else y2.data_ptr(), zd.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
                                                   gd.data_ptr(), scale.data_ptr() if use_z else None, shift.data_ptr() if use_z else None,
                                                   sums.data_ptr(), dz2.data_ptr(), go2.data_ptr(), dg2.data_ptr(), db2.data_ptr(), 1.0, M, C, st), "bwd")
            torch.cuda.synchronize()
            outs.append((dz2.clone(), go2.clone(), dg2.clone(), db2.clone()))
        assert torch.equal(outs[0][1], outs[1][1])  # the masked gradient: identical masks
        assert torch.allclose(outs[0][0].float(), outs[1][0].float(), atol=2e-3, rtol=2e-3)  # dz: fp64 atomics may reorder the sums' last bits
        assert torch.allclose(outs[0][2], outs[1][2], rtol=1e-5, atol=1e-6) and torch.allclose(outs[0][3], outs[1][3], rtol=1e-5, atol=1e-6)


def test_relu_maxpool_final_pack_unpack_kernels(cuda_device):
    lib, st, d = _lib.load(), _lib.current_stream_ptr(), cuda_device
    g = torch.Generator().manual_seed(1)
    # relu backward with fan-in
    a, b, y = (torch.randn((4096,), generator=g).half() for _ in range(3))
    out = torch.zeros(4096, dtype=torch.float16, device=d)
    ad, bd_, yd = a.to(d), b.to(d), y.to(d)  # keep the device copies alive until the kernel has run
    _lib.check(lib.rsb_relu_backward(ad.data_ptr(), bd_.data_ptr(), yd.data_ptr(), out.data_ptr(), 4096, st), "relu_bwd")
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), ((a.float() + b.float()) * (y.float() > 0)).half())
    # max-pool backward (both pools of the network)
    for (N, H, W, C, k, s, p) in [(2, 16, 16, 64, 3, 2, 1), (2, 4, 4, 128, 2, 2, 0), (3, 10, 14, 8, 3, 2, 1)]:
        # post-ReLU inputs: many exact ties (zeros) -> the first maximum of a window must take the gradient, as in ATen
        x = torch.relu(torch.randn((N, C, H, W), generator=g)).half().float().requires_grad_(True)
        yy = F.max_pool2d(x, k, s, p)
        dy = torch.randn(yy.shape, generator=g).half()
        yy.backward(dy.float())
        xd = x.detach().permute(0, 2, 3, 1).contiguous().half().to(d)
        dyd = dy.permute(0, 2, 3, 1).contiguous().to(d)
        scratch = torch.zeros(dyd.numel(), dtype=torch.uint8, device=d)
        got = []
        for ws in (None, scratch.data_ptr()):  # single-pass kernel, and the two-pass (argmax scratch) one the engine uses
            dx = torch.zeros_like(xd)
            _lib.check(lib.rsb_maxpool_backward(xd.data_ptr(), dyd.data_ptr(), dx.data_ptr(), ws, N, H, W, C, k, s, p, st), "maxpool_bwd")
            torch.cuda.synchronize()
            assert (dx.float().cpu().permute(0, 3, 1, 2) - x.grad).abs().max().item() <= 2e-3
            got.append(dx.clone())
        assert torch.equal(got[0], got[1])
    # final 1x1 forward / backward
    N, H, W, C = 2, 16, 24, 6
    y5 = torch.randn((N, H, W, 32), generator=g).half()
    w = (torch.randn((C, 32), generator=g) * 0.3).requires_grad_(True)
    bb = (torch.randn(C, generator=g) * 0.1).requires_grad_(True)
    y5t = y5.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    ref = F.conv2d(y5t, w.reshape(C, 32, 1, 1), bb)
    dl = torch.randn(ref.shape, generator=g) * 1e-2
    ref.backward(dl)
    logits = torch.zeros((N, C, H, W), device=d)
    y5d, wd, bd = y5.to(d), w.detach().to(d), bb.detach().to(d)
    _lib.check(lib.rsb_final_forward(y5d.data_ptr(), wd.data_ptr(), bd.data_ptr(), logits.data_ptr(), N, H * W, C, st), "final_fwd")
    dy5 = torch.zeros_like(y5d)
    acc = torch.zeros(C * 32 + 8, dtype=torch.float64, device=d)
    dw, dbv = torch.zeros((C, 32), device=d), torch.zeros(C, device=d)
    dld = dl.to(d)
    _lib.check(lib.rsb_final_backward(dld.data_ptr(), y5d.data_ptr(), wd.data_ptr(), dy5.data_ptr(), acc.data_ptr(), dw.data_ptr(), dbv.data_ptr(), 256.0,
                                      N, H * W, C, st), "final_bwd")
    torch.cuda.synchronize()
    assert torch.allclose(logits.cpu(), ref.detach(), atol=1e-4)
    assert _rel(dy5.float().cpu() / 256.0, y5t.grad.permute(0, 2, 3, 1)) < 2e-3
    assert _rel(dw.cpu(), w.grad) < 1e-4 and _rel(dbv.cpu(), bb.grad) < 1e-5
    # pack / unpack with the upsample-phase map (sums of up to 4 taps)
    from robosat_b200.train_engine import invert_unpack_map, map_up_fwd
    from robosat_b200.engine import pack_upsample_phases

    wt = torch.randn((8, 64, 3, 3), generator=g)
    m = torch.from_numpy(map_up_fwd(tuple(wt.shape))).to(d)
    dst = torch.zeros(m.shape[0], dtype=torch.float16, device=d)
    wtd = wt.to(d)
    _lib.check(lib.rsb_pack_weights(wtd.data_ptr(), m.data_ptr(), dst.data_ptr(), m.shape[0], st), "pack")
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu().reshape(32, 256), pack_upsample_phases(wt).half())
    gp = torch.randn(m.shape[0], generator=g)
    grad = torch.zeros_like(wt).to(d)
    gpd = gp.to(d)
    dst_idx, inv4 = invert_unpack_map(m)
    _lib.check(lib.rsb_unpack_grads_gather(gpd.data_ptr(), dst_idx.data_ptr(), inv4.data_ptr(), grad.data_ptr(), dst_idx.numel(), 0.5, st), "unpack")
    torch.cuda.synchronize()
    wref = wt.clone().requires_grad_(True)
    (pack_upsample_phases(wref).reshape(-1) * gp * 0.5).sum().backward()
    assert torch.allclose(grad.cpu(), wref.grad, atol=1e-5)
    # single-source layouts: the 1-index kernel equals the 4-index one (and the whole-engine re-pack equals the per-layout one)
    from robosat_b200.train_engine import map_conv_fwd

    wc = torch.randn((64, 128, 3, 3), generator=g).to(d)
    m4 = torch.from_numpy(map_conv_fwd(tuple(wc.shape))).to(d)
    assert bool((m4[:, 1:] < 0).all()) and m4.shape[0] % 8 == 0
    m1 = m4[:, 0].contiguous()
    m1[5], m4[5, 0] = -1, -1  # a hole packs as zero
    d4, d1 = (torch.full((m4.shape[0],), 7.0, dtype=torch.float16, device=d) for _ in range(2))
    _lib.check(lib.rsb_pack_weights(wc.data_ptr(), m4.data_ptr(), d4.data_ptr(), m4.shape[0], st), "pack")
    _lib.check(lib.rsb_pack_weights1(wc.data_ptr(), m1.data_ptr(), d1.data_ptr(), m1.shape[0], st), "pack1")
    torch.cuda.synchronize()
    assert torch.equal(d1, d4) and float(d1[5]) == 0.0
    assert lib.rsb_pack_weights1(wc.data_ptr(), m1.data_ptr(), d1.data_ptr(), 12, st) == -1  # not a multiple of 8


@pytest.mark.parametrize("i", range(len(conv_cases.default_cases(None)) - 2))  # head cases have no packed fp16 output
def test_wgrad_split_k_scratch_matches_cpu_emulation(i, cuda_device):
    lib, st = _lib.load(), _lib.current_stream_ptr()
    case = conv_cases.default_cases(cuda_device)[i]()
    cpu = conv_cases.default_cases("cpu")[i]()
    d = case.desc
    g = torch.Generator().manual_seed(100 + i)
    dy = (torch.randn(tuple(case.out.shape), generator=g) * 0.5).half()
    K = 64 * sum(d.segs[j].cblocks for j in range(d.nseg))
    dw = torch.zeros(d.phases * d.Cout * K, dtype=torch.float32, device=cuda_device)
    dyd = dy.to(cuda_device)
    plan = ctypes.c_void_p()
    _lib.check(lib.rsb_wgrad_plan_create(ctypes.byref(d), dyd.data_ptr(), dw.data_ptr(), ctypes.byref(plan)), "wgrad_plan")
    need = int(lib.rsb_wgrad_plan_scratch_bytes(plan))  # split-K plans keep their per-slice partials there
    scratch = torch.empty(need // 4 + 4, dtype=torch.float32, device=cuda_device)
    _lib.check(lib.rsb_wgrad_plan_set_scratch(plan, scratch.data_ptr(), need), "wgrad_set_scratch")
    for _ in range(2):  # the second run overwrites dw, it does not add to it
        _lib.check(lib.rsb_wgrad_run(plan, st), "wgrad_run")
    torch.cuda.synchronize()
    ref = torch.zeros(d.phases * d.Cout * K, dtype=torch.float32)
    emulate.run_wgrad(cpu.desc, dy.data_ptr(), ref)
    lib.rsb_wgrad_plan_destroy(plan)
    assert _rel(dw.cpu(), ref) < 2e-3, case.name
    assert (dw.cpu() - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-3


def _engine_pair(C, B, S, device, loss_scale=1024.0):
    sd0 = {k[7:]: v.clone() for k, v in synth.make_state_dict(C, seed=0).items()}
    x = synth.normalize_tiles(synth.make_tiles_u8(B, S, seed=1))
    params = {k: v.clone().to(device) for k, v in sd0.items()}
    eng = UNetTrainEngine(params, C, B, S, S, device=device, loss_scale=loss_scale)
    return sd0, x, params, eng


def test_train_forward_matches_oracle_train_mode(cuda_device):
    sd0, x, params, eng = _engine_pair(2, 2, 128, cuda_device)
    logits = eng.forward(x.to(cuda_device)).float().cpu()
    sd = {k: v.clone() for k, v in sd0.items()}
    with torch.no_grad():
        ref, feats = unet_oracle.unet_forward_train(sd, x, return_features=True)
    assert _rel(logits, ref) < 5e-3
    for name in ("stem", "enc1", "enc2", "enc3", "enc4", "dec1", "dec3", "dec5"):
        t, (n, h, w, c) = eng.feats[name]
        assert _rel(t.float().cpu().reshape(n, h, w, c).permute(0, 3, 1, 2), feats[name]) < 2e-2, name
    # running statistics follow torch's momentum / unbiased-variance update
    for k in ("resnet.bn1", "resnet.layer2.0.downsample.1", "resnet.layer4.2.bn3"):
        assert torch.allclose(params[k + ".running_mean"].cpu(), sd[k + ".running_mean"], atol=3e-3)
        assert _rel(params[k + ".running_var"].cpu(), sd[k + ".running_var"]) < 1e-2
        assert int(params[k + ".num_batches_tracked"].item()) == int(sd0[k + ".num_batches_tracked"].item()) + 1


@pytest.mark.parametrize("classes,size", [(2, 128), (6, 64)])
def test_train_backward_matches_mask_frozen_autograd(classes, size, cuda_device):
    sd0, x, params, eng = _engine_pair(classes, 2, size, cuda_device)
    g = torch.Generator().manual_seed(3)
    dlogits = torch.randn((2, classes, size, size), generator=g) * 1e-3
    eng.forward(x.to(cuda_device))
    grads = eng.backward(dlogits.to(cuda_device))
    torch.cuda.synchronize()
    sd = {k: v.clone() for k, v in sd0.items()}
    for k, v in sd.items():
        if v.dtype == torch.float32 and "running" not in k:
            v.requires_grad_(True)
    lo = linearized.forward(eng, sd, x)
    (lo * dlogits).sum().backward()
    rels = {}
    for k, v in sd.items():
        if v.requires_grad and not k.startswith("resnet.fc"):
            rels[k] = _rel(grads[k].cpu(), v.grad)
    worst = sorted(rels.items(), key=lambda kv: -kv[1])[:5]
    print("worst parameter-gradient rel-L2:", worst, "median", float(np.median(list(rels.values()))))
    assert len(rels) == 168  # every trainable tensor except the unused resnet.fc (SURVEY.md A11)
    assert worst[0][1] < 6e-2 and np.median(list(rels.values())) < 3e-2


def test_unet_module_train_step_with_lovasz_and_adam(cuda_device):
    """The `rs train` inner loop (train.py:172-194) on the H100 path: net.train(); outputs = net(images);
    loss = LovaszLoss2d()(outputs, masks); loss.backward(); optimizer.step() -- loss matches the fp32 oracle at step 0,
    gradients reach every parameter, BN buffers move, the loss goes down on a fixed batch, checkpoint layout is kept."""
    from oracle import losses_oracle
    from robosat_b200.losses import LovaszLoss2d
    from robosat_b200.metrics import Metrics
    from robosat_b200.optim import Adam
    from robosat_b200.unet import UNet

    sd = synth.make_state_dict(2, seed=0)
    net = torch.nn.DataParallel(UNet(2, pretrained=False), device_ids=[0]).to(cuda_device)
    net.load_state_dict(sd)
    opt = Adam(net.parameters(), lr=1e-3)
    opt.mark_used([not n.startswith("module.resnet.fc.") for n, _ in net.named_parameters()])
    crit = LovaszLoss2d().to(cuda_device)
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 128, seed=1)).to(cuda_device)
    masks = synth.make_masks(2, 128, 2, seed=3).to(cuda_device)
    with torch.no_grad():
        ref_logits = unet_oracle.unet_forward_train({k: v.clone() for k, v in sd.items()}, x.cpu())
    ref_loss = float(losses_oracle.lovasz_loss(ref_logits, masks.cpu()))
    net.train()
    losses = []
    metrics = Metrics(range(2))
    rm0 = net.module.resnet.bn1.running_mean.clone()
    for step in range(4):
        opt.zero_grad()
        out = net(x)
        loss = crit(out, masks)
        loss.backward()
        if step == 0:
            gnorm = {n: float(p.grad.abs().sum()) for n, p in net.named_parameters()}
            assert all(v > 0 for n, v in gnorm.items() if not n.startswith("module.resnet.fc.")), [n for n, v in gnorm.items() if v == 0][:5]
            assert all(gnorm[n] == 0 for n in gnorm if n.startswith("module.resnet.fc."))
        opt.step()
        losses.append(loss.item())
        metrics.add_batch(masks, out.detach())
    print("lovasz losses", losses, "oracle step-0", ref_loss)
    assert abs(losses[0] - ref_loss) <= 5e-3 * abs(ref_loss)
    assert losses[-1] < losses[0]
    assert not torch.equal(net.module.resnet.bn1.running_mean, rm0)
    assert 0.0 <= metrics.get_miou() <= 1.0
    ckpt = {"epoch": 1, "state_dict": net.state_dict(), "optimizer": opt.state_dict()}
    assert list(ckpt["state_dict"].keys()) == list(sd.keys()) and len(ckpt["optimizer"]["state"]) == 168
    # eval after training uses freshly folded weights (plans invalidated by train())
    net.eval()
    with torch.no_grad():
        ev = net(x)
    ref_eval = unet_oracle.unet_forward({k: v.detach().cpu() for k, v in net.state_dict().items()}, x.cpu())
    assert _rel(ev.float().cpu(), ref_eval) < 1e-2


def test_fused_grad_accumulation_matches_autograd_accumulate(cuda_device):
    """loss.backward() with the one-kernel accumulation (rsb_multi_axpy into existing .grad tensors) == handing every
    gradient to autograd's AccumulateGrad; a second backward without zero_grad() adds, as torch does."""
    from robosat_b200.losses import CrossEntropyLoss2d
    from robosat_b200.unet import UNet

    net = UNet(2, pretrained=False).to(cuda_device)
    net.load_state_dict({k[7:]: v for k, v in synth.make_state_dict(2, seed=0).items()})
    net.train()
    crit = CrossEntropyLoss2d().to(cuda_device)
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 64, seed=4)).to(cuda_device)
    masks = synth.make_masks(2, 64, 2, seed=5).to(cuda_device)
    used = [(n, p) for n, p in net.named_parameters() if not n.startswith("resnet.fc.")]

    def run(fused, times):
        net.fused_grad_accumulation = fused
        for _, p in net.named_parameters():
            p.grad = torch.zeros_like(p)
        for _ in range(times):
            crit(net(x), masks).backward()
        torch.cuda.synchronize()
        return {n: p.grad.clone() for n, p in used}

    ref, one, two = run(False, 1), run(True, 1), run(True, 2)
    for n, _ in used:
        scale = ref[n].abs().max().item() + 1e-12
        assert (one[n] - ref[n]).abs().max().item() <= 1e-4 * scale, n      # split-K fp32 atomics: order-dependent last bits
        assert (two[n] - 2 * ref[n]).abs().max().item() <= 2e-4 * scale, n
    # parameters without a .grad tensor still get theirs through autograd
    net.fused_grad_accumulation = True
    for _, p in net.named_parameters():
        p.grad = None
    crit(net(x), masks).backward()
    assert all(p.grad is not None for _, p in used)
    assert (dict(net.named_parameters())["final.weight"].grad - ref["final.weight"]).abs().max().item() <= 1e-4 * ref["final.weight"].abs().max().item()


def test_train_backward_vs_plain_fp32_autograd(cuda_device):
    """The honest number next to the mask-frozen check above: parameter gradients of ONE step against plain fp32 autograd of the
    oracle (train-mode BatchNorm, its own ReLU masks and max-pool arg-maxes). The fp16 forward flips a small fraction of masks
    relative to an fp32 run and every flip changes gradient elements by O(1), so this is looser by construction -- it is the
    error any reduced-precision forward (fp16 / bf16 / TF32 autocast) shows against an fp32 run. Printed and bounded."""
    C, B, S = 2, 2, 128
    sd0, x, params, eng = _engine_pair(C, B, S, cuda_device)
    g = torch.Generator().manual_seed(3)
    dlogits = torch.randn((B, C, S, S), generator=g) * 1e-3
    eng.forward(x.to(cuda_device))
    grads = eng.backward(dlogits.to(cuda_device))
    torch.cuda.synchronize()
    sd = {k: v.clone() for k, v in sd0.items()}
    for k, v in sd.items():
        if v.dtype == torch.float32 and "running" not in k:
            v.requires_grad_(True)
    lo = unet_oracle.unet_forward_train(sd, x)
    (lo * dlogits).sum().backward()
    rels, dots, n1, n2 = {}, 0.0, 0.0, 0.0
    for k, v in sd.items():
        if v.requires_grad and not k.startswith("resnet.fc"):
            a, b = grads[k].cpu().double(), v.grad.double()
            rels[k] = _rel(a, b)
            dots += float((a * b).sum())
            n1 += float((a * a).sum())
            n2 += float((b * b).sum())
    cosine = dots / (n1 ** 0.5 * n2 ** 0.5)
    vals = sorted(rels.values())
    worst = sorted(rels.items(), key=lambda kv: -kv[1])[:3]
    print("gradient vs plain fp32 autograd: median rel-L2 %.3f, 90th pct %.3f, worst %s, cosine of the full gradient %.5f" % (
        vals[len(vals) // 2], vals[int(0.9 * len(vals))], worst, cosine))
    assert len(rels) == 168
    assert cosine >= 0.97 and vals[len(vals) // 2] <= 0.2 and vals[-1] <= 0.8


def test_config5_six_class_train_step_256_and_plan_for_batch8_1024(cuda_device):
    """BASELINE config 5 (6 classes, 3x1024x1024, batch 8 per GPU): a 6-class train step at 256^2 against the oracle's loss, and
    the batch-8 1024^2 training plan builds, fits and runs forward + backward (finite gradients everywhere)."""
    from oracle import losses_oracle
    from robosat_b200.losses import LovaszLoss2d
    from robosat_b200.optim import Adam
    from robosat_b200.unet import UNet

    sd = synth.make_state_dict(6, seed=0)
    net = torch.nn.DataParallel(UNet(6, pretrained=False), device_ids=[0]).to(cuda_device)
    net.load_state_dict(sd)
    opt = Adam(net.parameters(), lr=1e-4)
    opt.mark_used([not n.startswith("module.resnet.fc.") for n, _ in net.named_parameters()])
    crit = LovaszLoss2d().to(cuda_device)
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 256, seed=1))
    masks = synth.make_masks(2, 256, 6, seed=3)
    net.train()
    opt.zero_grad()
    loss = crit(net(x.to(cuda_device)), masks.to(cuda_device))
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    with torch.no_grad():
        ref_logits = unet_oracle.unet_forward_train({k: v.clone() for k, v in sd.items()}, x)
    ref_loss = float(losses_oracle.lovasz_loss(ref_logits, masks))
    print("6-class 256^2 Lovasz loss %.5f (oracle %.5f), skipped steps %d" % (loss.item(), ref_loss, opt.skipped_steps()))
    assert abs(loss.item() - ref_loss) <= 5e-3 * abs(ref_loss) and opt.skipped_steps() == 0
    del net, opt
    torch.cuda.empty_cache()
    params = {k[7:]: v.clone().to(cuda_device) for k, v in sd.items()}
    eng = UNetTrainEngine(params, 6, 8, 1024, 1024, device=cuda_device, loss_scale=4096.0)
    xb = synth.normalize_tiles(synth.make_tiles_u8(8, 1024, seed=2)).to(cuda_device)
    logits = eng.forward(xb)
    dl = torch.randn_like(logits) * 1e-6
    grads = eng.backward(dl)
    torch.cuda.synchronize()
    assert torch.isfinite(logits).all() and all(torch.isfinite(v).all() for v in grads.values())
    assert torch.cuda.max_memory_allocated() < 170e9


def test_train_forward_512_matches_oracle(cuda_device):
    """512^2 train-mode forward (the BASELINE config 3 extent, batch 2 of its 16) against the oracle's train-mode forward"""
    sd0, x, params, eng = _engine_pair(2, 2, 512, cuda_device)
    logits = eng.forward(x.to(cuda_device)).float().cpu()
    sd = {k: v.clone() for k, v in sd0.items()}
    with torch.no_grad():
        ref = unet_oracle.unet_forward_train(sd, x)
    r = _rel(logits, ref)
    print("train-mode forward 2x3x512x512: rel-L2 of logits %.2e" % r)
    assert r < 5e-3


def test_second_forward_before_backward_is_refused(cuda_device):
    """ADVICE r1: the training plan keeps ONE set of saved activations per input shape. A backward through a graph whose buffers a
    later forward overwrote, or a second backward through the same graph, must raise instead of returning wrong gradients."""
    from robosat_b200.losses import CrossEntropyLoss2d
    from robosat_b200.unet import UNet

    net = UNet(2, pretrained=False).to(cuda_device)
    net.load_state_dict({k[7:]: v for k, v in synth.make_state_dict(2, seed=0).items()})
    net.train()
    crit = CrossEntropyLoss2d().to(cuda_device)
    x = synth.normalize_tiles(synth.make_tiles_u8(2, 64, seed=4)).to(cuda_device)
    masks = synth.make_masks(2, 64, 2, seed=5).to(cuda_device)
    l1 = crit(net(x), masks)
    l2 = crit(net(x), masks)
    with pytest.raises(RuntimeError, match="second train-mode forward"):
        l1.backward()
    l2.backward(retain_graph=True)  # the latest graph is fine ...
    with pytest.raises(RuntimeError, match="ran twice"):
        l2.backward()               # ... once


def test_inference_plans_follow_weight_updates_through_dataparallel(cuda_device):
    """ADVICE r1: loading a checkpoint through the nn.DataParallel wrapper (the reference's usage, predict.py:63-68) or editing
    weights in place must invalidate the cached inference plans (they hold folded fp16 copies of the weights)."""
    from robosat_b200.unet import UNet

    sd_a, sd_b = synth.make_state_dict(2, seed=0), synth.make_state_dict(2, seed=5)
    x = synth.normalize_tiles(synth.make_tiles_u8(1, 64, seed=1))
    net = torch.nn.DataParallel(UNet(2, pretrained=False), device_ids=[0]).to(cuda_device)
    net.load_state_dict(sd_a)
    net.eval()
    with torch.no_grad():
        a = net(x.to(cuda_device)).cpu()
        net.load_state_dict(sd_b)          # goes through _load_from_state_dict of the wrapped module: no override is reached
        b = net(x.to(cuda_device)).cpu()
        ref_a, ref_b = unet_oracle.unet_forward(sd_a, x), unet_oracle.unet_forward(sd_b, x)
        assert _rel(a, ref_a) < 2e-4 and _rel(b, ref_b) < 2e-4 and _rel(b, ref_a) > 1e-2
        net.module.final.bias.add_(1.0)    # in-place edit in eval mode
        c = net(x.to(cuda_device)).cpu()
    assert torch.allclose(c, b + 1.0, atol=1e-3)


def test_backward_is_deterministic(cuda_device):
    """Deterministic split-K of the weight gradients (rsb_wgrad_plan_set_scratch: per-slice partials added in slice order by a
    second kernel): two backward passes over the same activations give bit-identical parameter gradients."""
    sd0, x, params, eng = _engine_pair(2, 2, 128, cuda_device)
    g = torch.Generator().manual_seed(3)
    dlogits = (torch.randn((2, 2, 128, 128), generator=g) * 1e-3).to(cuda_device)
    runs = []
    for _ in range(2):
        eng.forward(x.to(cuda_device))
        grads = eng.backward(dlogits)
        torch.cuda.synchronize()
        runs.append({k: v.clone() for k, v in grads.items()})
    assert eng._wgrad_scratch is not None, "no wgrad plan needed a scratch: the test would be vacuous"
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_graph_replay_equals_kernel_by_kernel(cuda_device):
    """The forward / backward op lists replayed from CUDA graphs (default, RSB_TRAIN_GRAPH=1: captured on the third call of a
    key) give bit-identical logits, gradients and running statistics to launching the same lists kernel by kernel, also after
    the loss scale changes (re-capture) and with a fresh input tensor at every call (static input copy)."""
    sd0, x, params_a, eng_a = _engine_pair(2, 2, 128, cuda_device)
    _, _, params_b, eng_b = _engine_pair(2, 2, 128, cuda_device)
    assert eng_a.use_graph and eng_b.use_graph
    eng_b.use_graph = False
    g = torch.Generator().manual_seed(5)
    for step in range(7):
        if step == 5:
            eng_a.loss_scale = eng_b.loss_scale = 1024.0
        xs = (x + 0.01 * step).to(cuda_device)  # a new tensor (new address) per step
        dl = (torch.randn((2, 2, 128, 128), generator=g) * 1e-3).to(cuda_device)
        la = eng_a.forward(xs).clone()
        lb = eng_b.forward(xs.clone()).clone()
        ga = {k: v.clone() for k, v in eng_a.backward(dl).items()}
        gb = {k: v.clone() for k, v in eng_b.backward(dl.clone()).items()}
        torch.cuda.synchronize()
        assert torch.equal(la, lb), step
        for k in ga:
            assert torch.equal(ga[k], gb[k]), (step, k)
    assert any(s["graph"] is not None for s in eng_a._graphs.values()), "no graph was captured: the test would be vacuous"
    assert not eng_b._graphs
    for k in params_a:
        if k.endswith("running_mean") or k.endswith("running_var") or k.endswith("num_batches_tracked"):
            assert torch.equal(params_a[k], params_b[k]), k
