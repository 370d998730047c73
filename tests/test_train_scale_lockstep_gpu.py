"""The training step op by op against float64 at the shapes the benchmark trains at: 16 x 512^2 with 2 classes and the Lovasz
loss's gradient, and 8 x 1024^2 with 6 classes and the cross-entropy gradient. The lockstep harness runs in its sampled mode
(tests/lockstep.py): convolutions and weight gradients at sampled pixels and rows, every other op element by element in
chunks. At these sizes the grid-stride loops of the helper kernels run many times and the reductions run at their capped grids
(tests/train_launch.py), which the small-shape lockstep tests never reach; at 8 x 1024^2 the stem's BatchNorm backward sums
run the longest fp32 chain of the step (155 roundings).

At 16 x 512^2 the test also replays the forward and backward op lists from CUDA graphs captured directly around the engine's
kernel-by-kernel launcher, and checks that one replay is bit-identical to the kernel-by-kernel run. That shows the op lists
replay exactly at this size; the engine's own capture path (use_graph, capture on the third call, the static input copy) is
covered at 2 x 128^2 by tests/test_train_gpu.py."""

import time

import pytest
import torch

import lockstep
import train_launch
from robosat_b200 import _lib, synth
from robosat_b200.losses import LovaszLoss2d

pytestmark = pytest.mark.gpu

SAMPLE_ABOVE = 65536  # output pixels above which a convolution is checked at sampled pixels


def _dlogits(kind, B, C, H, W, dev):
    """the logit gradient of the project's Lovasz ("lovasz") or cross-entropy ("ce") kernel on synthetic masks"""
    logits = (torch.randn((B, C, H, W), generator=torch.Generator().manual_seed(2)) * 2).to(dev)
    masks = synth.make_masks(B, max(H, W), C, seed=3)[:, :H, :W].contiguous().to(dev)
    if kind == "lovasz":
        lg = logits.requires_grad_(True)
        LovaszLoss2d().to(dev)(lg, masks).backward()
        dl = lg.grad
    else:
        lib = _lib.load()
        loss = torch.zeros(1, device=dev)
        dl = torch.empty_like(logits)
        scratch = torch.empty(2, dtype=torch.float64, device=dev)
        _lib.check(lib.rsb_cross_entropy(logits.data_ptr(), masks.data_ptr(), None, loss.data_ptr(), dl.data_ptr(), scratch.data_ptr(), B, C, H * W,
                                         _lib.current_stream_ptr()), "rsb_cross_entropy")
    torch.cuda.synchronize()
    return dl.detach().cpu().contiguous()


def _scale_lockstep(dev, C, B, H, W, loss):
    t0 = time.time()
    _, dut, twin = lockstep.make_pair(C, B, H, W, 1024.0, dev)
    x = synth.normalize_tiles(synth.make_tiles_u8(B, max(H, W), seed=1))[:, :, :H, :W].contiguous()
    dlogits = _dlogits(loss, B, C, H, W, dev)
    assert torch.isfinite(dlogits).all() and bool((dlogits != 0).any())
    # the stray-write snapshot is a second copy of the engine's buffers: on the device if it fits beside other work, else on the host
    snap_bytes = sum(t.numel() * t.element_size() for t in lockstep._bases(dut))
    free, _ = torch.cuda.mem_get_info()
    snapshot = "device" if free > snap_bytes + (8 << 30) else "host"
    print("\nstray-write snapshot: %.1f GB on the %s (%.1f GB free on the device)" % (snap_bytes / 2 ** 30, snapshot, free / 2 ** 30))
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    ls = lockstep.Lockstep(lockstep.GpuExecutor(dut), twin, sample_above=SAMPLE_ABOVE, sms=sms, snapshot=snapshot)
    t1 = time.time()
    ls.run(x, dlogits, dut_x=x.to(dev), dut_dlogits=dlogits.to(dev), log=lambda line: print(line, flush=True))
    t2 = time.time()
    print("\n%d x 3 x %d x %d, %d classes, %s dlogits (engine + twin %.0f s, lockstep %.0f s):\n%s" % (
        B, H, W, C, loss, t1 - t0, t2 - t1, ls.table()))
    print(train_launch.e_sum_note(ls.launches))
    assert len(ls.checked["fwd"]) == len(dut.fwd_ops) and len(ls.checked["bwd"]) == len(dut.bwd_ops)
    assert lockstep.n_ops(dut) == 413
    print("ops checked: %d" % (len(ls.checked["fwd"]) + len(ls.checked["bwd"])))
    # the geometry read from the engine built at this size (with the device's SM count) is the one the CPU suite restates from a
    # small plan, and every capped family has launches at its cap among the ops just checked
    _, _, small = lockstep.make_pair(C, 1, 64, 64, 1024.0, "cpu")
    key = lambda la: (la.family, la.which, la.index, la.work, la.grid, la.chain)  # noqa: E731
    assert [key(la) for la in ls.launches] == [key(la) for la in train_launch.plan_launches(small, (B, H, W), sms=sms)]
    for fam in train_launch.CAPPED_FAMILIES:
        hit = train_launch.capped(ls.launches, fam)
        assert hit, "%s: no launch reaches its cap at %d x %d^2" % (fam, B, H)
        print("%-15s %d capped launches, e.g. %r" % (fam, len(hit), hit[0]))
    for tag in ("conv", "conv.dgrad", "wgrad", "bn_stats", "bn_apply", "bn_bwd.dz", "bn_bwd.dgamma_dbeta", "final_bwd.dw_db", "maxpool_bwd"):
        assert ls.stats[tag][0] > 0, tag
    return dut, x, dlogits


def _bits_of(eng):
    return [lockstep._bits(t).clone() for t in [eng.logits, eng._grads_flat] + [v for v in eng.params.values()]]


def test_train_step_lockstep_16x512_lovasz(cuda_device):
    dut, x, dlogits = _scale_lockstep(cuda_device, 2, 16, 512, 512, "lovasz")
    # one CUDA-graph replay of the forward and backward op lists against the kernel-by-kernel run, from the same state
    xd, dd = x.to(cuda_device), dlogits.to(cuda_device)
    state = {k: v.clone() for k, v in dut.params.items()}
    dut._run(dut.fwd_ops, x=xd)
    dut._run(dut.bwd_ops, dlogits=dd)
    torch.cuda.synchronize()
    ref = _bits_of(dut)
    graphs = []
    for ops, kw in ((dut.fwd_ops, {"x": xd}), (dut.bwd_ops, {"dlogits": dd})):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            dut._run(ops, **kw)
        graphs.append(g)
    for k, v in dut.params.items():
        v.copy_(state[k])
    dut.logits.fill_(float("nan"))
    dut._grads_flat.fill_(float("nan"))
    for g in graphs:
        g.replay()
    torch.cuda.synchronize()
    got = _bits_of(dut)
    names = ["logits", "grads"] + list(dut.params)
    for n, a, b in zip(names, ref, got):
        assert torch.equal(a, b), "graph replay differs from the kernel-by-kernel run in %s" % n


def test_train_step_lockstep_8x1024_six_classes(cuda_device):
    _scale_lockstep(cuda_device, 6, 8, 1024, 1024, "ce")
