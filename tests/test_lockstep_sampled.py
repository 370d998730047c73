"""The lockstep harness's sampled mode (tests/lockstep.py) and the launch-geometry restatement (tests/train_launch.py) on the
CPU: the sampled float64 references equal the full ones where they overlap, sampled mode with the emulator passes clean and
still names each injected fault at its op and buffer, and the restatement shows which launches reach their capped grids."""

import numpy as np
import pytest
import torch

import emulate
import lockstep
import train_launch as TL
from robosat_b200 import synth
from test_lockstep import FaultyEmulator, _name


def _randomized_twin(C, B, H, W):
    _, _, twin = lockstep.make_pair(C, B, H, W, 1024.0, "cpu")
    g = torch.Generator().manual_seed(11)
    for t in twin._keep:
        if t.dtype == torch.float16:
            t.copy_((torch.randn(t.shape, generator=g) * 0.5).half())
    return twin


def _kinds(twin):
    """one conv op per (sources, phases, residual, ReLU, segments) kind of the plan, forward and backward"""
    seen, out = set(), []
    for op in twin.fwd_ops + twin.bwd_ops:
        if op[0] != "conv" or op[1].desc.mode != 0:
            continue
        d = op[1].desc
        key = (d.nsrc, d.phases, bool(d.residual), bool(d.relu), d.nseg, d.out_sx)
        if key not in seen:
            seen.add(key)
            out.append(op[1])
    return out


@pytest.mark.parametrize("C,B,H,W", [(2, 1, 64, 512), (6, 2, 64, 64)])
def test_sampled_references_equal_the_full_ones(C, B, H, W):
    twin = _randomized_twin(C, B, H, W)
    ls = lockstep.Lockstep.__new__(lockstep.Lockstep)  # only the sampler: it reads the seed and the current op
    ls.seed = 0
    convs = _kinds(twin)
    assert any(c.desc.phases == 4 for c in convs) and any(c.desc.residual for c in convs) and any(c.desc.nsrc == 4 for c in convs)
    for i, c in enumerate(convs):
        d = c.desc
        ls._cur = ("fwd", i)
        pix = ls._conv_sample(d)
        val, mag, addr = emulate.conv_f64_at(d, pix)
        full = {}
        emulate.run_desc(d, sink=lambda ptr, shape, strides, v, m, parts, plane: full.__setitem__(ptr, (v, m, strides)))
        for phase, base, shape, strides in emulate.conv_out_views(d):
            fv, fm, st = full[base]
            sel = pix[:, 3] == phase
            n, y, x = pix[sel, 0], pix[sel, 1], pix[sel, 2]
            assert np.array_equal(addr[sel], base + 2 * (n * st[0] + y * st[1] + x * st[2])), c.name
            rv, rm = fv[n, y, x], fm[n, y, x]
            assert np.all(np.abs(val[sel] - rv) <= 1e-13 * rm + 1e-300), c.name
            assert np.all(np.abs(mag[sel] - rm) <= 1e-13 * rm + 1e-300), c.name
    units = [u for u in twin.units.values()]
    for u in units[:: max(1, len(units) // 12)] + [twin.units["dec4"], twin.units["dec0"]]:
        d = u.desc
        R = d.phases * d.Cout
        rows = np.array(sorted({r for r in (0, 63, 64, 127, 128, R - 1, R // 3) if r < R}))
        ptr = u.out.data_ptr() + 2 * u.out_offset
        ref, rmag = emulate.run_wgrad(d, ptr, None, f64=True)
        got, gmag = emulate.run_wgrad_rows(d, ptr, rows, chunk_bytes=1 << 20)
        assert np.all(np.abs(got - ref[rows]) <= 1e-13 * rmag[rows] + 1e-300), u.name
        assert np.all(np.abs(gmag - rmag[rows]) <= 1e-13 * rmag[rows] + 1e-300), u.name


# ------------------------------------------------------------------------------------------------ faults in sampled mode
def _conv_last_box_unstored(ex, op, run):
    d = op[1].desc
    (_, base, shape, strides), = emulate.conv_out_views(d)
    out = emulate._view(base, shape, strides, writable=True)
    y0, x0 = (-(-d.Ht // d.TH) - 1) * d.TH, (-(-d.Wt // d.TW) - 1) * d.TW
    saved = out[:, y0:, x0:].copy()
    run()
    out[:, y0:, x0:] = saved


def _bn_apply_capped_grid_runs_once(ex, op, run):
    """the grid-stride loop stops after one pass of the capped grid. At this shape the 2112-block cap is never reached, so the
    same arithmetic runs with the cap of a one-SM part (16 blocks of 256 threads)"""
    _, b, res, y, relu = op
    flat = y.reshape(-1)
    total = b.M * b.C // 8
    done = TL.tr_blocks(total, 256, cap=16) * 256
    assert done < total
    saved = flat[8 * done:].clone()
    run()
    flat[8 * done:] = saved


def _wgrad_row_off_by_one_mma_block(ex, op, run):
    run()
    u = op[1]
    K = u.dw_packed.numel() // (u.desc.phases * u.desc.Cout)
    row = u.dw_packed.view(-1, K)[64]
    row.copy_(torch.roll(row.clone(), 16))


def _bn_bwd_drops_last_main_loop_group(ex, op, run):
    """channel_reduce without the fourth row group of its unrolled main loop (rows r + 3 step while r + 3 step < M)"""
    run()
    _, b, dy, y, dz, g_out = op
    M, C = b.M, b.C
    step = TL.reduce_blocks(M, C) * TL.reduce_rows_per_iter(C)
    keep = torch.ones(M, dtype=torch.bool)
    for r0 in range(step):
        r = r0
        while r + 3 * step < M:
            keep[r + 3 * step] = False
            r += 4 * step
    assert not keep.all()
    P = ex.eng.params
    g = dy.reshape(M, C).float()
    if y is not None:
        g = g * (y.reshape(M, C).float() > 0)
    zhat = (b.z.reshape(M, C).float() - b.mean) * b.invstd
    gk = g * keep[:, None]
    s0, s1 = gk.double().sum(0), (gk * zhat).double().sum(0)
    dz.copy_((P[b.prefix + ".weight"] * b.invstd * (g - (s0 / M).float() - zhat * (s1 / M).float())).half().reshape(dz.shape))
    ex.eng._grad(b.prefix + ".weight").copy_((s1 / ex.eng.loss_scale).float())
    ex.eng._grad(b.prefix + ".bias").copy_((s0 / ex.eng.loss_scale).float())


# (an input gradient for the conv fault: a forward conv left at zero would collapse its BatchNorm's variance and overflow the
# backward downstream, which the harness would rightly report at every later op)
SAMPLED_FAULTS = [("bwd", "conv", "resnet.layer2.1.conv1.dgrad", _conv_last_box_unstored, "resnet.layer2.1.conv1.dgrad out"),
                  ("fwd", "bn_apply", "resnet.bn1", _bn_apply_capped_grid_runs_once, "resnet.bn1 y"),
                  ("bwd", "wgrad", "resnet.layer1.0.conv3", _wgrad_row_off_by_one_mma_block, "resnet.layer1.0.conv3.dw_packed (sampled rows)"),
                  ("bwd", "bn_bwd", "resnet.bn1", _bn_bwd_drops_last_main_loop_group, "resnet.bn1")]


def _sampled_run(executor_cls, faults=()):
    _, dut, twin = lockstep.make_pair(2, 1, 64, 64, 1024.0, "cpu")
    x = synth.normalize_tiles(synth.make_tiles_u8(1, 64, seed=1))
    dlogits = torch.randn((1, 2, 64, 64), generator=torch.Generator().manual_seed(3)) * 1e-3
    ex = executor_cls(dut)
    targets = {}
    for which, kind, name, fn, buf in faults:
        ops = dut.fwd_ops if which == "fwd" else dut.bwd_ops
        hits = [i for i, op in enumerate(ops) if op[0] == kind and _name(op) == name]
        assert len(hits) == 1, (kind, name)
        ex.faults[id(ops[hits[0]])] = fn
        targets[(which, hits[0])] = (kind, name, buf)
    # 32 pixels: every convolution but layer4's is sampled; small chunks: every elementwise check runs in several pieces
    ls = lockstep.Lockstep(ex, twin, sample_above=32, chunk=1 << 12)
    failures = ls.run(x, dlogits, raise_on_fail=False)
    print(ls.table())
    return dut, twin, ls, failures, targets


def test_sampled_mode_passes_clean_and_names_each_fault():
    dut, twin, ls, failures, targets = _sampled_run(FaultyEmulator, SAMPLED_FAULTS)
    for f in failures:
        print(f)
    assert len(ls.checked["fwd"]) == len(dut.fwd_ops) and len(ls.checked["bwd"]) == len(dut.bwd_ops)
    assert lockstep.n_ops(dut) == 413
    # the faulty conv's last tile box is ragged and sampled; everything else passes
    d = [op[1].desc for op in twin.bwd_ops if op[0] == "conv" and op[1].name == "resnet.layer2.1.conv1.dgrad"][0]
    assert d.Wt % d.TW or d.Ht % d.TH
    got = {}
    for f in failures:
        got.setdefault((f.which, f.index), []).append(f)
    assert set(got) == set(targets), sorted(got)
    for key, (kind, name, buf) in targets.items():
        assert all(f.kind == kind and f.name == name for f in got[key])
        assert any(f.buffer.startswith(buf) for f in got[key]), [str(f) for f in got[key]]


# ------------------------------------------------------------------------------------------------ launch geometry
def test_launch_geometry_shows_the_capped_grids_only_the_bench_shapes_reach():
    _, _, small = lockstep.make_pair(2, 1, 64, 64, 1024.0, "cpu")
    _, _, mid = lockstep.make_pair(2, 2, 128, 128, 1024.0, "cpu")
    # the restatement scaled from a small plan equals the one read from the plan built at the size
    a, b = TL.plan_launches(small, (2, 128, 128)), TL.plan_launches(mid)
    assert [(x.family, x.which, x.index, x.work, x.grid, x.chain) for x in a] == [(x.family, x.which, x.index, x.work, x.grid, x.chain) for x in b]
    for fam in TL.CAPPED_FAMILIES:
        assert not TL.capped(b, fam), (fam, TL.capped(b, fam)[:3])
    for shape in ((16, 512, 512), (8, 1024, 1024)):
        la = TL.plan_launches(small, shape)
        for fam in TL.CAPPED_FAMILIES:
            assert TL.capped(la, fam), (shape, fam)
        print(shape, TL.e_sum_note(la))
        # every derived bound stays below the 1e-5 the harness assumed before the bounds were derived per launch
        assert max(x.e_sum() for x in la if x.chain is not None) < 1e-5
    # the stem's bn_bwd sums at 8 x 1024^2: 125 rows per thread, then 32 thread partials in shared memory
    stem = [x for x in TL.plan_launches(small, (8, 1024, 1024)) if x.family == "channel_reduce" and x.name == "resnet.bn1"][0]
    assert (stem.grid, stem.chain) == (528, 125 + 32 - 2)


def test_restated_grids_match_the_kernels_arithmetic():
    assert TL.tr_blocks(0, 256) == 1 and TL.tr_blocks(257, 256) == 2 and TL.tr_blocks(10 ** 9, 256) == 2112
    assert TL.reduce_blocks(8192, 64) == 32 and TL.reduce_blocks(1 << 24, 64) == 528
    assert TL.partials_grid(256, 64) == (8, 1, 8, 264)
    assert TL.partials_grid(1 << 20, 1024) == (132, 2, 1, 132)   # L = 2048: two column blocks of 256 threads share 2 SMs x 132
    assert TL.final_bwd_dw(16 * 512 * 512).grid == 264
