"""Launch geometry of the training step's helper kernels (robosat_b200/csrc/rsb_train.cu), restated in Python the way
tests/conv_matrix.py restates conv_select, and the longest fp32 summation chain of every reduction launch derived from it.

Test infrastructure only. The grids are those of the host entry points:

  tr_blocks(total, block, cap)   ceil(total / block) clamped to [1, cap]; cap 132 * 16 = 2112 unless stated
  bn_apply                       tr_blocks(M C/8, 256)                   grid-stride loop over M C/8 16-byte vectors
  bn_bwd apply pass              tr_blocks(ceil(M C/8 / 4), 256)         the same loop over M C/8 vectors
  channel_reduce (bn_bwd sums)   reduce_blocks(M, C) = tr_blocks(ceil(M / (8 rows_per_iter)), 1, 132 * 4), rows_per_iter =
                                 256 / (C/8); thread rows start at block * rows_per_iter + (thread / (C/8)), step = grid *
                                 rows_per_iter
  partial_reduce (bn_stats)      2-D grid (bx, colblocks): tpr = min(L/4, 256) threads per row of L = 2C floats, colblocks =
                                 L / (4 tpr), rows_per_iter = 256 / tpr, bx = ceil(R / (4 rows_per_iter)) clamped to
                                 [1, ceil(2 SMs / colblocks)] (the only grid that reads the device's SM count)
  relu_bwd                       tr_blocks(n/8, 256)
  maxpool_bwd (argmax, gather)   tr_blocks(N OH OW C/8, 256), tr_blocks(N H W C/8, 256)
  final_fwd, final_bwd dx        tr_blocks(P, 256)
  final_bwd dw (once per class)  tr_blocks(P, 256, 132 * 2)

fp32 chains (k = the most fp32 roundings any one term of a sum goes through before the fp64 accumulation):

  channel_reduce   each thread folds ceil(M / step) rows (its g or fma(g, z) terms: the products are exact inside the fma),
                   then one thread per channel adds the rows_per_iter thread partials of its block in shared memory:
                   k = ceil(M / step) + rows_per_iter - 2.
  partial_reduce   the terms are the conv-stats partials, each the fp32 sum of one 32-pixel quarter tile (k <= 31; z^2 of an
                   fp16 z is exact in fp32); each thread folds ceil(R / step) of them, step = bx * rows_per_iter, then thread
                   0..tpr-1 fold the rows_per_iter partials in shared memory: k = 31 + ceil(R / step) + rows_per_iter - 2.
  final_bwd dw     each thread folds ceil(P / (grid 256)) fma(g, y) terms, then a 5-level warp shuffle tree. The first fma
                   (onto 0) rounds g y, an fp32 times fp16 product, so every dW term is rounded once more than its additions:
                   k = ceil(P / (grid 256)) + 5 (db's terms g are exact and need one fewer; the dW count bounds both).

A recursively or tree-wise rounded fp32 sum errs by at most gamma_k sum |x_i|, gamma_k = k u / (1 - k u), u = 2^-24. The block
totals are then added into 8 replicated fp64 slots with atomics (at most ceil(grid / 8) per slot, then the 8 slots): that adds
(ceil(grid / 8) + 8) 2^-53 sum |x_i|. `e_sum(launch)` is the sum of both.
"""

SMS = 132          # rsb_train.cu hard-codes 132 SMs in tr_blocks / reduce_blocks / final_bwd_dw; partial_reduce asks the device
U = 2.0 ** -24
RED_SLOTS = 8
FAMILIES = ("bn_apply", "bn_bwd_apply", "channel_reduce", "partial_reduce", "relu_bwd", "maxpool_argmax", "maxpool_bwd_gather",
            "final_fwd", "final_bwd_dx", "final_bwd_dw")
CAPPED_FAMILIES = ("bn_apply", "channel_reduce", "partial_reduce")  # the families the bench shapes must run at their cap


def tr_blocks(total, block, cap=SMS * 16):
    return int(max(1, min(-(-total // block), cap)))


def reduce_rows_per_iter(C):
    return 256 // (C // 8)


def reduce_blocks(M, C):
    rpi = reduce_rows_per_iter(C)
    return tr_blocks(-(-M // (rpi * 8)), 1, SMS * 4)


def partials_grid(R, C, sms=SMS):
    """(bx, colblocks, rows_per_iter, cap) of rsb_bn_partials_finalize"""
    L = 2 * C
    tpr = min(L // 4, 256)
    colblocks = L // (tpr * 4)
    rpi = 256 // tpr
    cap = -(-2 * sms // colblocks)
    bx = max(1, min(-(-R // (rpi * 4)), cap))
    return bx, colblocks, rpi, cap


def gamma(k):
    return k * U / (1 - k * U)


class Launch:
    """one kernel launch of the plan: family, grid (x blocks), cap, the op (list, index, name) and, for reductions, the longest
    fp32 chain k and the fp64 slot count that bound its sums"""

    __slots__ = ("family", "which", "index", "name", "work", "grid", "cap", "chain", "atomics")

    def __init__(self, family, which, index, name, work, grid, cap, chain=None, atomics=0):
        self.family, self.which, self.index, self.name = family, which, index, name
        self.work, self.grid, self.cap, self.chain, self.atomics = work, grid, cap, chain, atomics

    @property
    def capped(self):
        """the grid the work asks for (`work` blocks) is larger than the cap, so the grid-stride loops run more than once"""
        return self.work > self.cap

    def e_sum(self):
        """relative error bound of the launch's sums: gamma_k in fp32, then the fp64 slot accumulation"""
        return gamma(self.chain) + (self.atomics + RED_SLOTS) * 2.0 ** -53

    def __repr__(self):
        return "%s %s[%d] %s grid %d/%d%s" % (self.family, self.which, self.index, self.name, self.grid, self.cap,
                                               "" if self.chain is None else " chain %d" % self.chain)


def bn_apply(M, C, which="fwd", index=-1, name=""):
    want = -(-(M * (C // 8)) // 256)
    return Launch("bn_apply", which, index, name, want, tr_blocks(M * (C // 8), 256), SMS * 16)


def bn_bwd_apply(M, C, which="bwd", index=-1, name=""):
    n = -(-(M * (C // 8)) // 4)
    return Launch("bn_bwd_apply", which, index, name, -(-n // 256), tr_blocks(n, 256), SMS * 16)


def channel_reduce(M, C, which="bwd", index=-1, name=""):
    rpi = reduce_rows_per_iter(C)
    grid = reduce_blocks(M, C)
    step = grid * rpi
    chain = -(-M // step) + rpi - 2
    return Launch("channel_reduce", which, index, name, -(-M // (rpi * 8)), grid, SMS * 4, max(chain, 1), -(-grid // RED_SLOTS))


def partial_reduce(R, C, sms=SMS, which="fwd", index=-1, name=""):
    bx, colblocks, rpi, cap = partials_grid(R, C, sms)
    step = bx * rpi
    chain = 31 + -(-R // step) + rpi - 2
    return Launch("partial_reduce", which, index, name, -(-R // (rpi * 4)), bx, cap, chain, -(-bx // RED_SLOTS))


def final_bwd_dw(P, which="bwd", index=-1, name="final_bwd"):
    grid = tr_blocks(P, 256, SMS * 2)
    chain = -(-P // (grid * 256)) + 5
    return Launch("final_bwd_dw", which, index, name, -(-P // 256), grid, SMS * 2, chain, grid * 8)


def conv_stats_partial():
    """the conv epilogue's per-quarter-tile partials: 32 fp32 rows (or 16 + 16 joined by one shuffle), k <= 31"""
    return gamma(31)


def _simple(family, which, i, name, total):
    return Launch(family, which, i, name, -(-total // 256), tr_blocks(total, 256), SMS * 16)


def plan_launches(eng, shape=None, sms=SMS):
    """every launch of the helper kernels in eng.fwd_ops / eng.bwd_ops (a UNetTrainEngine, plan_only or not).
    shape = (N, H, W): restate the same network at another batch and size without building it. Every activation size of the
    plan is N H W / 4^j exactly (H and W are multiples of 64), so sizes scale by N'H'W' / (N H W); the conv-stats rows come from
    the conv's tile space scaled the same way and the engine's own choose_tile."""
    from robosat_b200.engine import choose_tile

    N0, H0, W0 = eng.N, eng.H, eng.W
    N, H, W = shape if shape is not None else (N0, H0, W0)
    assert H % 64 == 0 and W % 64 == 0
    num, den = N * H * W, N0 * H0 * W0

    def sc(m):
        v = m * num
        assert v % den == 0, (m, shape)
        return v // den

    by_z = {}
    for u in eng.units.values():
        if u.stats is not None:
            by_z[id(u.out)] = u

    def numel(t):
        """elements of NHWC buffer t at the restated size (dec4 / d_dec4 are W-padded by 4 columns)"""
        n, h, w, c = t.shape
        assert n == N0
        return N * (h * H // H0) * ((W + 4) if w == W0 + 4 else w * W // W0) * c

    def stats_rows(b):
        d = by_z[id(b.z)].desc
        Wt, Ht = d.Wt * W // W0, d.Ht * H // H0
        assert Wt * W0 == d.Wt * W and Ht * H0 == d.Ht * H
        Nt = N
        tw, th, tn = choose_tile(Wt, Ht, Nt)
        return 4 * -(-Wt // tw) * -(-Ht // th) * -(-Nt // tn)

    out = []
    for which, ops in (("fwd", eng.fwd_ops), ("bwd", eng.bwd_ops)):
        for i, op in enumerate(ops):
            k = op[0]
            if k == "bn_stats":
                b = op[1]
                out.append(partial_reduce(stats_rows(b) if shape is not None else b.partial_rows, b.C, sms, which, i, b.prefix))
            elif k == "bn_apply":
                b = op[1]
                out.append(bn_apply(sc(b.M), b.C, which, i, b.prefix))
            elif k == "bn_bwd":
                b = op[1]
                out.append(channel_reduce(sc(b.M), b.C, which, i, b.prefix))
                out.append(bn_bwd_apply(sc(b.M), b.C, which, i, b.prefix))
            elif k == "relu_bwd":
                out.append(_simple("relu_bwd", which, i, "relu_bwd", numel(op[1]) // 8))
            elif k == "maxpool_bwd":
                _, xx, dy, dx, n, h, w, c, kk, s, p = op
                out.append(_simple("maxpool_argmax", which, i, "maxpool_bwd", numel(dy) // 8))
                out.append(_simple("maxpool_bwd_gather", which, i, "maxpool_bwd", numel(dx) // 8))
            elif k == "final_fwd":
                out.append(_simple("final_fwd", which, i, "final_fwd", N * H * W))
            elif k == "final_bwd":
                out.append(_simple("final_bwd_dx", which, i, "final_bwd", N * H * W))
                out.append(final_bwd_dw(N * H * W, which, i))
    return out


def by_op(launches):
    """(which, index) -> {family: Launch}"""
    d = {}
    for la in launches:
        d.setdefault((la.which, la.index), {})[la.family] = la
    return d


def capped(launches, family):
    return [la for la in launches if la.family == family and la.capped]


def longest_chain(launches):
    return max((la for la in launches if la.chain is not None), key=lambda la: la.chain)


def e_sum_note(launches):
    la = longest_chain(launches)
    return "longest fp32 chain: %d roundings (%s %s %s[%d], gamma_k = %.3g)" % (la.chain, la.family, la.name, la.which, la.index, gamma(la.chain))
