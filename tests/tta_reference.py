"""numpy restatement of the test-time augmentation head (rsb_head_tta_accumulate / _quantize / _argmax) and of the dihedral views,
shared by tests/test_tta.py (CPU) and tests/test_tta_gpu.py (which compares the device against it)."""

import numpy as np

ONE = 2 ** 59  # fixed-point scale of one probability


def augment_forward(img, op):
    """rsb_augment_dihedral's index map restated: out[y][x] = img[src(y, x)] for an [S, S, ...] array"""
    S = img.shape[0]
    y, x = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    sy, sx = y, x
    for _ in range((op >> 1) & 3):  # undo the quarter turns: ROTATE_90 writes out[y][x] = in[x][S-1-y]
        sy, sx = sx, S - 1 - sy
    if op & 1:
        sx = S - 1 - sx
    return img[sy, sx]


def view(a, op):
    """the same transform with numpy primitives on the two leading axes: left-right flip, then k counter-clockwise quarter turns"""
    if op & 1:
        a = np.flip(a, axis=1)
    return np.rot90(a, (op >> 1) & 3, axes=(0, 1))


def unview(a, op):
    """inverse of `view`: what a view's map looks like in the tile's own orientation"""
    a = np.rot90(a, -((op >> 1) & 3), axes=(0, 1))
    if op & 1:
        a = np.flip(a, axis=1)
    return a


def forward_map(op, OH, OW, y, x):
    """where pixel (y, x) of an OH x OW crop lies in the view made by `op` (the head's map; the crop is centred)"""
    if op & 1:
        x = OW - 1 - x
    k = (op >> 1) & 3
    if k == 0:
        return y, x
    if k == 1:
        return OW - 1 - x, y
    if k == 2:
        return OH - 1 - y, OW - 1 - x
    return x, OH - 1 - y


def softmax(logits):
    """float32 softmax over axis 1 as the head computes it: max-subtracted exp, class-ordered sum, one division"""
    l = np.asarray(logits, dtype=np.float32)
    m = l.max(axis=1, keepdims=True)
    e = np.exp(l - m)
    s = np.zeros_like(m)
    for c in range(l.shape[1]):
        s = s + e[:, c:c + 1]
    return e / s


def accumulate(probs, ops, B, overlap):
    """probs float32 [V*B, C, H, W] (view-major) -> int64 [B, C, H-2o, W-2o]: per tile pixel, the sum over views of
    rint(p * 2^59) of the view's probability at the pixel the op moved it to"""
    VB, C, H, W = probs.shape
    assert VB == len(ops) * B
    OH, OW = H - 2 * overlap, W - 2 * overlap
    y, x = np.meshgrid(np.arange(OH), np.arange(OW), indexing="ij")
    acc = np.zeros((B, C, OH, OW), dtype=np.int64)
    for v, op in enumerate(ops):
        vy, vx = forward_map(op, OH, OW, y, x)
        for b in range(B):
            p = probs[v * B + b][:, vy + overlap, vx + overlap].astype(np.float64)
            acc[b] += np.rint(p * ONE).astype(np.int64)
    return acc


def mean(acc, views):
    """the mean probability as the head forms it: float32(acc * 2^-59 / views), in float64 before the rounding"""
    return (acc.astype(np.float64) * (1.0 / ONE) / views).astype(np.float32)


def quantize(acc, views):
    """2 classes: np.digitize bins of the mean foreground probability, as uint8 (256 wraps to 0 like .astype(np.uint8))"""
    return np.digitize(mean(acc[:, 1], views), np.linspace(0, 1, 256)).astype(np.uint8)


def argmax(acc):
    return acc.argmax(axis=1).astype(np.uint8)


def compose(op_a, op_b):
    """the op w with view(view(a, op_b), op_a) == view(a, w): the views of a transformed tile are a permutation of the tile's"""
    probe = np.arange(9).reshape(3, 3)
    target = view(view(probe, op_b), op_a)
    for w in range(8):
        if np.array_equal(view(probe, w), target):
            return w
    raise AssertionError("the dihedral group is closed")
