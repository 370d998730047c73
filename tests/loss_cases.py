"""Input builders for the edge cases of the loss / metric / optimiser kernels, shared by tests/test_losses_edges.py (numpy only:
shows that each input tells a right implementation from a wrong one) and tests/test_losses_edges_gpu.py (the kernels).

Everything is generated from a seed; logits are fp32 [N, C, H, W] torch tensors, targets int64 [N, H, W].

The Lovasz sort works on tiles of SORT_TILE keys and pads each image's P = C*H*W keys to a whole number of tiles, so the
shapes below are chosen by P: under one tile, several tiles with a ragged last one, an exact multiple, P = 2 and odd H*W.
"""

import numpy as np
import torch

SORT_TILE = 4096  # kSortTile of robosat_b200/csrc/rsb_loss.cu

# (N, C, H, W); P / SORT_TILE in the comment
LOVASZ_SHAPES = [
    (1, 3, 32, 32),    # 0.75 tiles
    (2, 2, 96, 96),    # 4.5
    (3, 6, 96, 160),   # 22.5, N = 3
    (5, 2, 544, 544),  # 144.5, N = 5, the largest
    (1, 2, 1, 1),      # P = 2
    (2, 1, 64, 64),    # exactly one tile, C = 1
    (7, 2, 64, 65),    # 2.03 tiles, H*W odd, N = 7
]
RAGGED_MULTI_TILE = [(2, 2, 96, 96), (3, 6, 96, 160)]  # several tiles, ragged last tile, N > 1: where the tie inputs run


def targets_random(N, C, H, W, seed):
    """Blocky label masks (8 x 8 blocks where the image is large enough), every class equally likely."""
    g = torch.Generator().manual_seed(seed)
    bh, bw = max(H // 8, 1), max(W // 8, 1)
    coarse = torch.randint(0, C, (N, 1, bh, bw), generator=g)
    return torch.nn.functional.interpolate(coarse.float(), size=(H, W), mode="nearest").long().squeeze(1).contiguous()


def _randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def signs(targets, C):
    """2 * onehot - 1 as fp32 [N, C, H, W]"""
    return (torch.nn.functional.one_hot(targets, C).permute(0, 3, 1, 2).float() * 2 - 1).contiguous()


def errors(logits, targets):
    """the margin errors the Lovasz loss sorts, fp32 like the kernel computes them"""
    return 1.0 - signs(targets, logits.shape[1]) * logits


# --------------------------------------------------------------------------------------------------
# Lovasz inputs
# --------------------------------------------------------------------------------------------------
def lovasz_gaussian(shape, seed, scale=3.0):
    N, C, H, W = shape
    return (_randn(shape, seed) * scale).contiguous(), targets_random(N, C, H, W, seed + 1)


def lovasz_fp16_rounded(shape, seed):
    """logits as a fast-precision network produces them: fp16 values, so a few thousand distinct errors among P keys"""
    logits, targets = lovasz_gaussian(shape, seed)
    return logits.half().float().contiguous(), targets


def lovasz_five_values(shape, seed):
    """logits from {-2, -1, 0, 1, 2}: five distinct errors, a fifth of them exactly 0 (logit = +1 on the target class, -1 elsewhere)"""
    N, C, H, W = shape
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-2, 3, shape, generator=g).float().contiguous(), targets_random(N, C, H, W, seed + 1)


def lovasz_all_equal(shape, seed, value=0.0):
    """every logit 0: every error is 1, the sorted order is the index order"""
    N, C, H, W = shape
    return torch.full(shape, float(value)), targets_random(N, C, H, W, seed + 1)


def lovasz_index_order_grad(targets, C):
    """Closed form of the gradient when all errors are equal and positive: no sort, element k of the flattened [C, H, W] vector of
    an image is the k-th sorted element. fp32 arithmetic of robosat/losses.py:109-115, scaled by fp32(1 / N)."""
    N = targets.shape[0]
    m = torch.nn.functional.one_hot(targets, C).permute(0, 3, 1, 2).reshape(N, -1).numpy().astype(np.float32)
    out = np.zeros_like(m)
    for n in range(N):
        G = m[n].sum(dtype=np.float32)
        inter = G - np.cumsum(m[n], dtype=np.float32)
        union = G + np.cumsum(np.float32(1) - m[n], dtype=np.float32)
        j = np.float32(1) - inter / union
        j[1:] = j[1:] - j[:-1]
        out[n] = -(m[n] * np.float32(2) - np.float32(1)) * j * (np.float32(1) / np.float32(N))
    return torch.from_numpy(out.reshape(N, C, *targets.shape[1:]))


def lovasz_one_byte(shape, seed, byte):
    """Errors whose fp32 bit patterns, hence sort keys, differ in exactly one byte: that radix pass does all the ordering and the
    other three must keep it. |error| >= 2^25, where 1 - sign * x == -sign * x exactly in fp32, so the bits of the errors are chosen
    directly. byte 0..2: 0x4D000000 + (v << 8 * byte), v in 0..255 (2^27 <= e < 2^29). byte 3: (v << 24) | 0x123456 with the
    exponent kept in [152, 254]: both signs (negative errors get gradient 0), finite, 104 distinct values."""
    N, C, H, W = shape
    rng = np.random.default_rng(seed)
    targets = targets_random(N, C, H, W, seed + 1)
    if byte < 3:
        v = rng.integers(0, 256, shape, dtype=np.int64)
        bits = 0x4D000000 + (v << (8 * byte))
    else:
        v = rng.integers(76, 128, shape, dtype=np.int64) | (rng.integers(0, 2, shape, dtype=np.int64) << 7)
        bits = (v << 24) | 0x123456
    e = torch.from_numpy(bits.astype(np.uint32).view(np.float32).reshape(shape))
    logits = (-signs(targets, C) * e).contiguous()
    got = errors(logits, targets)
    assert torch.equal(got.view(torch.int32), e.view(torch.int32)), "the errors are not the chosen bit patterns"
    return logits, targets


def lovasz_tie_block(shape, seed, count=5000, error=0.5):
    """Gaussian logits with `count` randomly placed elements per image whose error is exactly `error` (0.5 is about the median of
    the others): one run of equal keys that is longer than a sort tile and, sorted, lies across tile boundaries."""
    N, C, H, W = shape
    logits, targets = lovasz_gaussian(shape, seed)
    s = signs(targets, C)
    P = C * H * W
    assert count < P
    g = torch.Generator().manual_seed(seed + 2)
    flat, sf = logits.view(N, P), s.view(N, P)
    for n in range(N):
        where = torch.randperm(P, generator=g)[:count]
        flat[n, where] = sf[n, where] * (1.0 - error)
    return logits, targets


def tie_block_span(logits, targets, error=0.5):
    """per image (first, last) sorted position of the run of errors equal to `error`"""
    e = errors(logits, targets).reshape(logits.shape[0], -1)
    return [(int((row > error).sum()), int((row >= error).sum()) - 1) for row in e]


def lovasz_scaled(shape, seed, factor):
    logits, targets = lovasz_gaussian(shape, seed)
    return (logits * factor).contiguous(), targets


def lovasz_subnormal(shape, seed):
    """logits that are subnormal fp32 numbers of both signs: every error rounds to exactly 1 (flushing them to zero gives the same)"""
    N, C, H, W = shape
    rng = np.random.default_rng(seed)
    bits = rng.integers(1, 1 << 23, shape, dtype=np.int64) | (rng.integers(0, 2, shape, dtype=np.int64) << 31)
    return torch.from_numpy(bits.astype(np.uint32).view(np.float32).reshape(shape)).contiguous(), targets_random(N, C, H, W, seed + 1)


# name -> builder(shape, seed); the inputs on which the order of equal errors decides the gradient
LOVASZ_TIE_CASES = {
    "fp16_rounded": lovasz_fp16_rounded,
    "five_values": lovasz_five_values,
    "all_equal": lovasz_all_equal,
    "byte0": lambda shape, seed: lovasz_one_byte(shape, seed, 0),
    "byte1": lambda shape, seed: lovasz_one_byte(shape, seed, 1),
    "byte2": lambda shape, seed: lovasz_one_byte(shape, seed, 2),
    "byte3": lambda shape, seed: lovasz_one_byte(shape, seed, 3),
    "tie_block": lovasz_tie_block,
}


# --------------------------------------------------------------------------------------------------
# deliberately wrong Lovasz variants (numpy): what the inputs above must be able to tell from the right one
# --------------------------------------------------------------------------------------------------
def lovasz_variant_grad(logits, targets, order="stable", pad_first=False, scale="reciprocal"):
    """The gradient of the Lovasz loss in the fp32 arithmetic of robosat/losses.py:96-119 with the pieces that can go wrong made
    selectable. The defaults are the right ones and equal oracle.losses_oracle.lovasz_loss.

    order:     "stable"      descending, equal errors in index order (torch.sort of the reference on these sizes, and the kernel)
               "scrambled"   descending, equal errors in a fixed pseudo-random order (a ranking that is not stable)
               "reversed"    ascending stable sort, then reversed: equal errors in descending index order
    pad_first: the padding of each image to whole sort tiles counted as background elements that sort first
    scale:     "reciprocal"  g * fp32(1 / N), what autograd does for loss / N;   "divide"  g / N
    """
    x = logits.numpy().astype(np.float32)
    t = targets.numpy()
    N, C, H, W = x.shape
    P = C * H * W
    mask = np.zeros((N, C, H, W), dtype=np.float32)
    np.put_along_axis(mask, t[:, None], 1.0, axis=1)
    grad = np.zeros((N, P), dtype=np.float32)
    idx = np.arange(P)
    for n in range(N):
        m = mask[n].reshape(-1)
        sign = m * np.float32(2) - np.float32(1)
        e = np.float32(1) - sign * x[n].reshape(-1)
        if order == "stable":
            o = np.argsort(-e, kind="stable")
        elif order == "scrambled":
            o = np.lexsort(((idx * 2654435761) % 4294967296, -e))
        elif order == "reversed":
            o = np.argsort(e, kind="stable")[::-1]
        else:
            raise ValueError(order)
        ls = m[o]
        pad = (-P) % SORT_TILE if pad_first else 0
        G = ls.sum(dtype=np.float32)
        inter = G - np.cumsum(ls, dtype=np.float32)
        union = G + np.float32(pad) + np.cumsum(np.float32(1) - ls, dtype=np.float32)
        j = np.float32(1) - inter / union
        first = j[0] - ((np.float32(1) - G / (G + np.float32(pad))) if pad else np.float32(0))  # J of the last padding element
        j[1:] = j[1:] - j[:-1]
        j[0] = first
        g = np.where(e[o] > 0, -sign[o] * j, np.float32(0)).astype(np.float32)
        grad[n, o] = g
    grad = grad * (np.float32(1) / np.float32(N)) if scale == "reciprocal" else grad / np.float32(N)
    return torch.from_numpy(grad.reshape(N, C, H, W))


# --------------------------------------------------------------------------------------------------
# metrics: argmax ties
# --------------------------------------------------------------------------------------------------
def metrics_tie_cases(seed=40):
    """(name, logits, targets) where a large share of the pixels has more than one maximal class: fp16-rounded logits around 300
    (where fp16 steps by 0.25) with a spread of 0.3, a five-value set, +0.0 against -0.0 (equal: the first one wins), and targets up to C - 1 >= 2 so that
    predicted / actual is neither 0, 1, inf nor NaN for many pixels (the reference counts those nowhere)."""
    out = []
    for C, (H, W) in ((2, (96, 97)), (6, (64, 65))):
        N = 3
        shape = (N, C, H, W)
        t = targets_random(N, C, H, W, seed + C)
        out.append(("fp16 C%d" % C, (_randn(shape, seed + 1) * 0.3 + 300.0).half().float().contiguous(), t))
        g = torch.Generator().manual_seed(seed + 2)
        out.append(("five values C%d" % C, torch.randint(-2, 3, shape, generator=g).float().contiguous(), t))
        z = torch.zeros(shape)
        z[torch.rand(shape, generator=g) < 0.5] = -0.0
        out.append(("signed zeros C%d" % C, z.contiguous(), t))
    return out


def metrics_counts_variant(logits, targets, last_max=False):
    """Metrics.add summed over the batch with numpy; last_max=True is the wrong argmax (the last maximal class wins)"""
    x, t = logits.numpy(), targets.numpy()
    C = x.shape[1]
    m = (C - 1 - np.argmax(x[:, ::-1], axis=1)) if last_max else np.argmax(x, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = m.astype(np.float32) / t.astype(np.float32)
    return int(np.isnan(q).sum()), int(np.isposinf(q).sum()), int((q == 0).sum()), int((q == 1).sum())


# --------------------------------------------------------------------------------------------------
# cross entropy / focal / mIoU: the ends of the exponent range, absent and zero-weight classes, C and HW limits
# --------------------------------------------------------------------------------------------------
def softmax_edge_cases(seed=60):
    """dicts(name, logits, targets, weight or None). `undefined` names the losses for which the float64 reference itself is not
    finite on that input (see tests/test_losses_edges_gpu.py)."""
    cases = []

    def add(name, logits, targets, weight=None, undefined=()):
        cases.append(dict(name=name, logits=logits.contiguous(), targets=targets.contiguous(), weight=weight, undefined=tuple(undefined)))

    # logit gaps around the underflow of expf: exp(-87.3) is the smallest normal, exp(-103.3) the smallest subnormal, beyond that 0
    N, C, H, W = 2, 3, 16, 17
    t = targets_random(N, C, H, W, seed)
    gaps = torch.linspace(80.0, 110.0, H * W).reshape(1, 1, H, W)
    for hot, label in ((0, "on the target"), (1, "off the target")):
        x = _randn((N, C, H, W), seed + 1) * 0.5
        x = x - gaps * (1 - torch.nn.functional.one_hot((t + hot) % C, C).permute(0, 3, 1, 2).float())
        add("gaps of 80..110, maximum %s" % label, x, t, torch.tensor([0.7, 1.0, 1.6]))
    big = lambda tt: torch.where(signs(tt, C) > 0, 1e4, -1e4) * (1 + 0.01 * _randn((N, C, H, W), seed + 2))
    every = t.clone()
    every[:, 0, :C] = torch.arange(C)
    add("logits of +-1e4, every class in every image", big(every), every)
    # a class that is absent from an image and has probability exactly 0 there: its soft IoU is 0 / 0
    absent = torch.cat([t[:1] % 2, every[1:]])
    add("logits of +-1e4, class 2 absent from image 0", big(absent), absent, undefined=("miou",))
    x = _randn((N, C, H, W), seed + 3) * 2
    add("class 2 absent from image 0", x, torch.cat([t[:1] % 2, t[1:]]), torch.tensor([0.7, 1.0, 1.6]))
    add("class 1 has weight 0", x, t, torch.tensor([0.7, 0.0, 1.6]))
    add("every weight 0", x, t, torch.zeros(3), undefined=("ce", "focal"))
    add("C = 1", _randn((2, 1, 8, 9), seed + 4), torch.zeros((2, 8, 9), dtype=torch.int64))
    add("C = 64", _randn((2, 64, 8, 9), seed + 5) * 3, targets_random(2, 64, 8, 9, seed + 6), torch.rand(64, generator=torch.Generator().manual_seed(seed)) + 0.5)
    add("H*W = 1", _randn((5, 3, 1, 1), seed + 7) * 2, targets_random(5, 3, 1, 1, seed + 8))
    add("H*W odd, N = 3", _randn((3, 2, 33, 35), seed + 9) * 3, targets_random(3, 2, 33, 35, seed + 10), torch.tensor([0.4, 1.3]))
    return cases


def focal_reference(logits, targets, weight=None, gamma=2.0):
    """FocalLoss2d and its gradient in float64 in closed form (robosat_b200/csrc/rsb_loss.cu states the derivative). Equal to the
    autograd of oracle.losses_oracle.focal_loss wherever that is finite (tests/test_losses_edges.py). It is not for gamma < 1 on a
    pixel whose float64 softmax is exactly 1 at the target: autograd's pow backward gives gamma * 0^(gamma-1) = inf there, times a
    log p_t that is not exactly 0. The limit of that product is 0, which is what this takes; 1 - p_t is summed from the other
    classes instead of subtracted, so it does not cancel."""
    x = logits.detach().double()
    N, C, H, W = x.shape
    w = torch.ones(C, dtype=torch.float64) if weight is None else weight.detach().double()
    onehot = torch.zeros_like(x).scatter_(1, targets.view(N, 1, H, W), 1.0)
    p, logp = torch.softmax(x, dim=1), torch.log_softmax(x, dim=1)
    pt, logpt = (p * onehot).sum(1), (logp * onehot).sum(1)
    q = (p * (1 - onehot)).sum(1)
    wt = w[targets]
    den = wt.sum()
    pen = q ** gamma
    loss = -(wt * pen * logpt).sum() / den
    dpen = torch.zeros_like(q) if gamma == 0 else torch.where(q == 0, torch.zeros_like(q), gamma * q.clamp_min(1e-300) ** (gamma - 1) * pt * logpt)
    grad = -((wt / den) * (pen - dpen)).unsqueeze(1) * (onehot - p)
    return np.float32(loss.item()), grad.float()


# --------------------------------------------------------------------------------------------------
# Adam
# --------------------------------------------------------------------------------------------------
GRID_SWEEP = 132 * 16 * 256  # elements one sweep of the capped grid covers (blocks_for in rsb_loss.cu): 540 672
ADAM_SIZES = [1, 255, 257, GRID_SWEEP, GRID_SWEEP + 1, 3_000_001]


def adam_inputs(n, seed):
    """fp32 numpy (param, [grad step 1, 2, 3]); a tenth of the gradient elements are exactly 0 in every step, so their second
    moment stays 0 and the update's denominator is eps alone"""
    rng = np.random.default_rng(seed)
    p = rng.standard_normal(n).astype(np.float32)
    zero = rng.random(n) < 0.1
    grads = []
    for _ in range(3):
        g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 1, n)).astype(np.float32)
        g[zero] = 0.0
        grads.append(g)
    return p, grads


# --------------------------------------------------------------------------------------------------
# rsb_sort_unique_u64
# --------------------------------------------------------------------------------------------------
def sort_unique_cases(seed=80):
    """(name, uint64 keys, key_bits). The contract (include/rsb200.h): keys are below 2^key_bits; key_bits = 64 means the whole
    word, compared as unsigned. Every case here satisfies it; in_contract() is what the tests assert before calling."""
    rng = np.random.default_rng(seed)
    cases = [("n = 0", np.zeros(0, np.uint64), 36)]
    for n in (4096, 8192):
        pool = rng.integers(0, 1 << 36, n // 2, dtype=np.uint64)
        cases.append(("n = %d exactly" % n, rng.choice(pool, n), 36))
    cases.append(("all keys equal", np.full(10_000, 0x123456789, np.uint64), 36))
    cases.append(("sorted and unique already", np.arange(0, 3 * 9000, 3, dtype=np.uint64) << np.uint64(11), 36))
    cases.append(("key_bits = 0", np.zeros(5000, np.uint64), 0))
    cases.append(("key_bits = 1", rng.integers(0, 2, 5000, dtype=np.uint64), 1))
    cases.append(("key_bits = 63", rng.choice(rng.integers(0, 1 << 63, 3000, dtype=np.uint64), 9000), 63))
    top = rng.integers(0, 1 << 63, 3000, dtype=np.uint64) | (rng.integers(0, 2, 3000, dtype=np.uint64) << np.uint64(63))
    cases.append(("key_bits = 64, top bit set in half", rng.choice(top, 9000), 64))
    return cases


def in_contract(keys, key_bits):
    return keys.size == 0 or key_bits == 64 or int(keys.max()) < (1 << key_bits)
