"""The convolution case matrix (tests/conv_matrix.py) reaches exactly the compiled kernel instances, and its restatement
of conv_select / rsb_rowconv_run agrees with the plan constructors' validation. No GPU needed: validation runs before
the device check (test_abi.py)."""

import pytest
import torch

import conv_matrix as CM
from robosat_b200 import _lib

RSB_E_INVALID = -1
RSB_E_NODEVICE = -3


def test_compiled_instances_are_read_from_the_dispatch():
    inst = CM.compiled_instances()
    conv = {k[1:] for k in inst if k[0] == "conv"}
    row = {k[1:] for k in inst if k[0] == "row"}
    # spot checks of the parse against the dispatch as written: the N-concatenated strict narrow tiles, the strict head,
    # the fast 256-wide paired residual (not compiled in strict precision), every statistics instance
    assert (32, 0, 1, 0, 2, 0) in conv and (32, 1, 0, 0, 2, 0) in conv and (256, 0, 1, 1, 0, 0) in conv
    assert (256, 0, 1, 1, 1, 0) not in conv and (256, 0, 1, 0, 1, 0) not in conv
    assert {k for k in conv if k[5]} == {(bn, 0, 0, 0, 0, 1) for bn in (32, 64, 128, 256)} | {(bn, 0, 0, 1, 0, 1) for bn in (128, 256)}
    assert (32, 32, 1, 3, 1, 1, 1) in row and (64, 32, 1, 3, 1, 1, 0) in row and (64, 32, 0, 2, 2, 2, 0) in row
    assert (64, 64, 0, 2, 2, 2, 0) not in row  # the fused upsample 128 -> 64 does not fit in shared memory
    assert len(conv) == 30 and len(row) == 9


def test_matrix_reaches_exactly_the_compiled_instances():
    reached = {}
    for c in CM.matrix("cpu"):
        reached.setdefault(CM.instance_of(c.desc), []).append(c.name)
    assert set(reached) == CM.compiled_instances(), (
        "not reached: %s; not compiled: %s" % (sorted(CM.compiled_instances() - set(reached)), sorted(set(reached) - CM.compiled_instances())))


def test_matrix_covers_every_box_ragged_and_multiwave():
    """per tensor-core instance: every TW x TH x TN = 128 box on a ragged tile space, and one case of more tiles than SMs
    (an odd number of spatial tiles under a CTA pair); per line-buffer instance: a ragged case and one of more units than SMs"""
    boxes, waves = {}, {}
    for c in CM.matrix("cpu"):
        d = c.desc
        inst = CM.instance_of(d)
        if c.kernel == "conv":
            box = (d.TW, d.TH, d.TN)
            sp = [-(-n // b) for n, b in zip((d.Wt, d.Ht, d.Nt), box)]
            ragged = all(n % b for n, b in zip((d.Wt, d.Ht, d.Nt), box) if b > 1)
            if c.box and ragged:
                boxes.setdefault(inst, set()).add(box)
            m = sp[0] * sp[1] * sp[2]
            if m * d.phases * (d.Cout // d.block_n) > CM.SMS and (not d.cta_pair or m % 2):
                waves.setdefault(inst, []).append(c.name)
        else:
            units = d.Nt * -(-d.Wt // 128) * d.nphase_a * -(-d.Ht // d.rows_per_unit) if d.rows_per_unit else 0
            if units > CM.SMS:
                waves.setdefault(inst, []).append(c.name)
            if d.Wt % 128 and d.rows_per_unit and d.Ht % d.rows_per_unit:
                boxes.setdefault(inst, set()).add("ragged")
    for inst in CM.compiled_instances():
        if inst[0] == "conv":
            assert boxes.get(inst) == set(CM.BOXES), inst
        else:
            assert boxes.get(inst) == {"ragged"}, inst
        assert waves.get(inst), inst


def test_matrix_covers_k_chunking_heads_and_stats():
    chunked, classes = set(), set()
    for c in CM.matrix("cpu"):
        d = c.desc
        if c.kernel != "conv":
            continue
        kb = sum(d.segs[i].cblocks for i in range(d.nseg))
        if 0 < d.kchunk < kb:
            kind = "1" if d.kchunk == 1 else "K-1" if d.kchunk == kb - 1 else "ragged" if kb % d.kchunk else "divides"
            chunked.add((d.block_n <= 64, bool(d.cta_pair), bool(d.residual), bool(d.split), kind))
        if d.mode == 1:
            classes.add((bool(d.split), d.head_classes))
    for narrow, pair in ((True, False), (False, False), (False, True)):
        for res in (False, True):
            for kind in ("1", "K-1", "ragged"):
                assert (narrow, pair, res, True, kind) in chunked, (narrow, pair, res, kind)
    assert {(s, k) for s in (False, True) for k in (1, 8)} <= classes


def _rejects(desc):
    with pytest.raises(CM.Rejected):
        CM.instance_of(desc)
    assert CM.plan_create_code(_lib.load(), desc) == RSB_E_INVALID, _lib.last_error()


def test_restatement_rejects_what_the_validator_rejects():
    def tc(**kw):
        base = dict(kind="3x3", tile=(16, 8, 2), block_n=128, cout=256, seed=1)
        base.update(kw)
        return CM.TcCase("reject", **base).desc

    d = tc(split=True, residual=True, block_n=256)                 # split + residual at 256 columns
    _rejects(d)
    d = tc(block_n=256, kchunk=4, split=True)                      # K chunking at 256 columns
    _rejects(d)
    d = tc(block_n=64, cout=128, pair=True)                        # a CTA pair below 128 columns
    _rejects(d)
    d = tc(block_n=64, cout=128)
    buf = torch.zeros(1 << 16)
    d.residual, d.stats, d.stats_bytes = buf.data_ptr(), buf.data_ptr(), buf.numel() * 4   # statistics with a residual
    _rejects(d)
    d = tc(block_n=64, cout=128, stats=True, split=True)           # statistics in strict precision
    _rejects(d)
    d = tc(kind="dec", block_n=64, cout=128, stats=True)           # statistics of a 4-phase decoder
    _rejects(d)
    d = tc(kind="head", block_n=32)                                # a paired head
    d.cta_pair = 1
    _rejects(d)
    d = tc(block_n=64, cout=96)                                    # Cout not a multiple of block_n
    _rejects(d)
    d = tc(box=(8, 8, 4))                                          # not a 128-pixel box
    _rejects(d)
    d = CM.RowCase("reject", "row3x3", (200, 13, 2), 64, 64, split=True).desc   # strict line buffer outside the head
    _rejects(d)
    d = CM.RowCase("reject", "rowup", (200, 13, 2), 128, 64).desc               # fused upsample 128 -> 64: no room for the row ring
    _rejects(d)
    assert "shared memory" in _lib.last_error()
    d = CM.RowCase("reject", "rowup", (200, 13, 2), 32, 32).desc                # no instance: fused upsample on 32 channels
    with pytest.raises(CM.Rejected):
        CM.instance_of(d)


def test_validator_accepts_every_matrix_case():
    """on a host without a GPU every descriptor of the matrix passes validation and stops at the device check"""
    if torch.cuda.is_available():
        pytest.skip("GPU present: plans would be created (test_conv_matrix_gpu.py runs them)")
    lib = _lib.load()
    for c in CM.matrix("cpu"):
        d = c.desc
        assert CM.plan_create_code(lib, d) == RSB_E_NODEVICE, (c.name, _lib.last_error())
