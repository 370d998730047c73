"""Test-time augmentation (TTA) for `rs predict` and `rs serve`: the network runs on flipped and rotated copies of each tile, each
copy's class probabilities are mapped back to the tile's own orientation, and their mean replaces the single view's.

Overhead imagery has no up direction and `rs train` augments with the same dihedral transforms (robosat_b200/augment.py), so the
averaged mask is smoother and less prone to orientation-dependent false positives. Everything stays on the device, one chain per
batch of B tiles:

    expand:     one `rsb_augment_dihedral` launch per view writes the view's copy of the B tiles into its slice of the engine input
    per pass:   engine.forward (E = B*V/P tiles) -> `rsb_head_tta_accumulate` (softmax, inverse map, crop, int64 fixed-point sum)
    finish:     `rsb_head_tta_quantize` (2 classes: np.digitize bins of the mean foreground) or `rsb_head_tta_argmax`

The chain is plain stream work, so a caller can capture it in a CUDA graph. The fixed-point sum makes the mean bit-identical
however the views are ordered or split into passes.
"""

import ctypes

import torch

from robosat_b200 import _lib

# op = flip | (k << 1): a left-right flip, then k counter-clockwise quarter turns (rsb_augment_dihedral's encoding)
VIEW_SETS = {"none": (0,), "flip": (0, 1), "d4": tuple(range(8))}
MODES = tuple(VIEW_SETS)

# An engine never holds more than max(B, ENGINE_CAP) tiles, so TTA needs no more activation memory than a plan of that batch.
ENGINE_CAP = 32


def views(mode):
    if mode not in VIEW_SETS:
        raise ValueError("tta must be one of %s, not %r" % (", ".join(MODES), mode))
    return VIEW_SETS[mode]


def num_passes(batch, nviews, cap=None):
    """P: the smallest divisor of V for which the engine's E = B*V/P tiles stay within max(B, cap)."""
    limit = max(batch, ENGINE_CAP if cap is None else cap)
    for p in range(1, nviews + 1):
        if nviews % p == 0 and batch * nviews // p <= limit:
            return p
    return nviews


def check_shape(mode, height, width):
    """quarter turns map a tile onto itself only when it is square"""
    if any(op >> 1 & 1 for op in views(mode)) and height != width:
        raise ValueError("tta=%r rotates tiles and needs a square image, got %dx%d; use tta='flip'" % (mode, height, width))


class TtaChain:
    """Device-resident TTA of B tiles [B, H, W, 3] uint8 through `engine` (a UNetEngine over E = B*V/P tiles of H x W)."""

    def __init__(self, engine, mode, batch, height, width, num_classes, overlap=0, device="cuda"):
        check_shape(mode, height, width)
        self.engine, self.mode = engine, mode
        self.ops = views(mode)
        self.batch, self.H, self.W, self.classes, self.overlap = batch, height, width, num_classes, overlap
        self.V = len(self.ops)
        assert engine.N % batch == 0 and self.V % (engine.N // batch) == 0, "engine batch must be B * (views per pass)"
        self.per_pass = engine.N // batch
        self.passes = self.V // self.per_pass
        self.device = torch.device(device)
        self.OH, self.OW = height - 2 * overlap, width - 2 * overlap
        self.views_in = torch.empty((engine.N, height, width, 3), dtype=torch.uint8, device=self.device)
        # per view a constant ops[B] array for the augmentation kernel, built once
        self.ops_dev = torch.tensor([[op] * batch for op in self.ops], dtype=torch.int32).to(self.device)
        self.acc = torch.empty((batch, num_classes, self.OH, self.OW), dtype=torch.int64, device=self.device)
        self._ops_host = [(ctypes.c_int32 * self.per_pass)(*self.ops[p * self.per_pass:(p + 1) * self.per_pass]) for p in range(self.passes)]

    @staticmethod
    def engine_batch(mode, batch, cap=None):
        nviews = len(views(mode))
        return batch * nviews // num_passes(batch, nviews, cap)

    def num_launches(self):
        return self.V + self.passes * (self.engine.num_launches() + 1) + 1

    def accumulate(self, x):
        """enqueue expand -> P x (forward + accumulate) for device tiles x [B, H, W, 3] uint8; returns `acc`"""
        assert x.dtype == torch.uint8 and tuple(x.shape) == (self.batch, self.H, self.W, 3) and x.is_contiguous()
        lib = _lib.load()
        stream = _lib.current_stream_ptr()
        B, S = self.batch, self.H
        for p in range(self.passes):
            for j in range(self.per_pass):
                v = p * self.per_pass + j
                dst = self.views_in[j * B:(j + 1) * B]
                if self.H == self.W:
                    _lib.check(lib.rsb_augment_dihedral(x.data_ptr(), None, self.ops_dev[v].data_ptr(), dst.data_ptr(), None, B, S, stream),
                               "rsb_augment_dihedral")
                else:
                    _lib.check(lib.rsb_augment_flip_rect(x.data_ptr(), self.ops_dev[v].data_ptr(), dst.data_ptr(), B, self.H, self.W, stream),
                               "rsb_augment_flip_rect")
            logits = self.engine.forward(self.views_in)
            _lib.check(lib.rsb_head_tta_accumulate(logits.data_ptr(), self.acc.data_ptr(), self._ops_host[p], self.per_pass, B, self.classes,
                                                   self.H, self.W, self.overlap, 1 if p else 0, stream), "rsb_head_tta_accumulate")
        return self.acc

    def quantize(self, x, out_u8):
        """2 classes: uint8 [B, H-2o, W-2o] np.digitize bins of the mean foreground probability"""
        assert self.classes == 2, "single channel requires binary model"
        self.accumulate(x)
        _lib.check(_lib.load().rsb_head_tta_quantize(self.acc.data_ptr(), out_u8.data_ptr(), self.batch, self.OH * self.OW, self.V,
                                                     _lib.current_stream_ptr()), "rsb_head_tta_quantize")
        return out_u8

    def argmax(self, x, out_u8):
        """uint8 [B, H-2o, W-2o] class of the largest mean probability"""
        self.accumulate(x)
        _lib.check(_lib.load().rsb_head_tta_argmax(self.acc.data_ptr(), out_u8.data_ptr(), self.batch, self.classes, self.OH * self.OW,
                                                   _lib.current_stream_ptr()), "rsb_head_tta_argmax")
        return out_u8
