"""numpy restatement of `rs predict` and `rs masks --dataset` for models of more than two classes (DESIGN.md §8), shared by
tests/test_multiclass.py (CPU) and tests/test_multiclass_gpu.py (which compares the device against it)."""

import numpy as np

from tta_reference import softmax

ANCHORS = np.linspace(0, 1, 256)


def crop(a, overlap):
    """unbuffer: drop `overlap` pixels on every side of the two trailing axes"""
    if overlap == 0:
        return a
    return a[..., overlap:-overlap, overlap:-overlap]


def digitize(p):
    """np.digitize bins as uint8: 256 (p >= 1) wraps to 0 like .astype(np.uint8)"""
    return np.digitize(p, ANCHORS).astype(np.uint8)


def predict_probs(logits, overlap):
    """fp32 logits [N, C, H, W] -> fp32 probabilities [N, C, H-2o, W-2o], the head's softmax"""
    return crop(softmax(logits), overlap)


def predict_bins(logits, overlap):
    """the bins `rs predict` writes for every class: uint8 [N, C, H-2o, W-2o]"""
    return digitize(predict_probs(logits, overlap))


def predict_bins_binary(logits, overlap):
    """the binary tool's bins (predict.py:87-103): softmax, foreground, unbuffer, digitize -> uint8 [N, H-2o, W-2o]"""
    return digitize(crop(softmax(logits)[:, 1], overlap))


def softvote(quant, weights=None):
    """quant uint8 [K, C, ...] -> uint8 [...]: argmax over classes of np.average(anchors[quant], axis=0, weights=w)"""
    return np.argmax(np.average(ANCHORS[np.asarray(quant)], axis=0, weights=weights), axis=0).astype(np.uint8)
