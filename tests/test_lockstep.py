"""The lockstep harness (tests/lockstep.py) run on the CPU: the emulator against a float64 replay of every op passes, and a
copy of the emulator with injected faults -- each one a bug the whole-network gradient comparisons could let through -- is
reported at exactly the faulty op, with the right kind and buffer."""

import torch

import lockstep
from robosat_b200 import synth

C, B, S = 2, 1, 64


def _run(executor_cls, faults=None):
    _, dut, twin = lockstep.make_pair(C, B, S, S, 1024.0, "cpu")
    x = synth.normalize_tiles(synth.make_tiles_u8(B, S, seed=1))
    dlogits = torch.randn((B, C, S, S), generator=torch.Generator().manual_seed(3)) * 1e-3
    ex = executor_cls(dut)
    targets = {}
    if faults:
        for which, kind, name, fn in faults:
            ops = dut.fwd_ops if which == "fwd" else dut.bwd_ops
            hits = [i for i, op in enumerate(ops) if op[0] == kind and _name(op) == name]
            assert len(hits) == 1, (kind, name)
            ex.faults[id(ops[hits[0]])] = fn
            targets[(which, hits[0])] = (kind, name)
    ls = lockstep.Lockstep(ex, twin)
    failures = ls.run(x, dlogits, raise_on_fail=False)
    print(ls.table())
    return dut, ls, failures, targets


def _name(op):
    return op[1].prefix if op[0].startswith("bn_") else op[1].name


class FaultyEmulator(lockstep.EmulatorExecutor):
    def __init__(self, eng):
        super().__init__(eng)
        self.faults = {}

    def run(self, op, x=None, dlogits=None):
        fault = self.faults.get(id(op))
        if fault is None:
            return super().run(op, x=x, dlogits=dlogits)
        fault(self, op, lambda: super(FaultyEmulator, self).run(op, x=x, dlogits=dlogits))


def _wgrad_drops_a_pixel_tile(ex, op, run):
    dy = op[2]  # the stem's dz: [N, H/2, W/2, 64]; one 8 x 8 tile = one of the kernel's 64-pixel tiles
    saved = dy.clone()
    dy[:, 8:16, 16:24] = 0
    run()
    dy.copy_(saved)


def _bn_bwd_without_mean_g_zhat(ex, op, run):
    run()
    _, b, dy, y, dz, _ = op
    c = 5
    g = dy.reshape(b.M, b.C)[:, c].double()
    if y is not None:
        g = g * (y.reshape(b.M, b.C)[:, c] > 0)
    zh = (b.z.reshape(b.M, b.C)[:, c].double() - float(b.mean[c])) * float(b.invstd[c])
    gamma = float(ex.eng.params[b.prefix + ".weight"][c])
    col = dz.reshape(b.M, b.C)[:, c]
    col.copy_((col.double() + gamma * float(b.invstd[c]) * zh * (g * zh).sum() / b.M).half())


def _dgrad_without_fan_in(ex, op, run):
    d = op[1].desc
    saved = d.residual
    assert saved
    d.residual = None
    run()
    d.residual = saved


def _dec4_writes_its_pad_column(ex, op, run):
    run()
    ex.eng.feats["dec4"][0][0, 5, 0, 7] = 1.0  # column 0 of the W-padded buffer: dec5 reads it as zero padding


def _bn_slot_left_dirty(ex, op, run):
    run()
    b = op[1]
    b.sums[2 * b.C + 3] = 0.5  # accumulator slot 1


FAULTS = [("bwd", "wgrad", "stem", _wgrad_drops_a_pixel_tile, "stem.dw_packed"),
          ("bwd", "bn_bwd", "resnet.layer2.0.bn2", _bn_bwd_without_mean_g_zhat, "dz"),
          ("bwd", "conv", "resnet.layer3.1.conv1.dgrad", _dgrad_without_fan_in, "out"),
          ("fwd", "conv", "dec4", _dec4_writes_its_pad_column, "dec4"),
          ("bwd", "bn_bwd", "resnet.layer4.0.bn1", _bn_slot_left_dirty, ".sums")]


def test_lockstep_clean_emulator_passes_every_op():
    dut, ls, failures, _ = _run(lockstep.EmulatorExecutor)
    assert not failures, "\n".join(str(f) for f in failures[:10])
    assert len(ls.checked["fwd"]) == len(dut.fwd_ops) and len(ls.checked["bwd"]) == len(dut.bwd_ops)
    assert lockstep.n_ops(dut) == 413
    for tag in ("conv", "conv.dgrad", "wgrad", "bn_stats", "bn_apply", "bn_bwd.dz", "pack_all.summed", "unpack_all", "maxpool_bwd"):
        assert ls.stats[tag][0] > 0, tag


def test_lockstep_reports_each_injected_fault_at_its_op():
    faults = [(w, k, n, fn) for w, k, n, fn, _ in FAULTS]
    _, _, failures, targets = _run(FaultyEmulator, faults)
    for f in failures:
        print(f)
    got = {(f.which, f.index): f for f in failures}
    assert len(failures) == len(FAULTS) and set(got) == set(targets), sorted(got)
    for (which, idx), (kind, name) in targets.items():
        f = got[(which, idx)]
        buf = [b for w, k, n, _, b in FAULTS if (w, k, n) == (which, kind, name)][0]
        assert f.kind == kind and f.name == name and buf in f.buffer, str(f)
    assert "stray" in str(got[[t for t, v in targets.items() if v[1] == "dec4"][0]])
    assert "not cleared" in str(got[[t for t, v in targets.items() if v[1] == "resnet.layer4.0.bn1"][0]])
