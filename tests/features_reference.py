"""numpy restatement of rsb_morph_binary (OpenCV's binary erode / dilate chain) and the CPU path of `rs features`, for the tests."""

import json
import os

import numpy as np

from robosat_b200.features import MorphOp, ellipse_spans, polygons_from_grown

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rect_spans(kh, kw):
    return [(0, kw)] * kh


def cross_spans(kh, kw, anchor=None):
    ay, ax = anchor if anchor is not None else (kh // 2, kw // 2)
    return [(0, kw) if i == ay else (ax, ax + 1) for i in range(kh)]


SHAPES = {"rect": lambda k: rect_spans(k, k), "ellipse": ellipse_spans, "cross": lambda k: cross_spans(k, k)}


def op(shape, k, dilate, anchor=None):
    return MorphOp(dilate, SHAPES[shape](k), k, anchor if anchor is not None else (k // 2, k // 2))


def element(o):
    """The op's element as a uint8 kh x kw array (what cv2.erode / cv2.dilate take)"""
    e = np.zeros((len(o.spans), o.kw), np.uint8)
    for i, (j0, j1) in enumerate(o.spans):
        e[i, j0:j1] = 1
    return e


def morph_ref(mask, ops):
    """out(y, x) = min / max over set cells (i, j) of in(y + i - ay, x + j - ax); outside pixels are 1 for erode, 0 for dilate"""
    m = mask.astype(np.uint8)
    H, W = m.shape
    for o in ops:
        P = 64
        pad = np.full((H + 2 * P, W + 2 * P), 0 if o.dilate else 1, np.uint8)
        pad[P:P + H, P:P + W] = m
        out = np.full((H, W), 0 if o.dilate else 1, np.uint8)
        ay, ax = o.anchor
        for i, (j0, j1) in enumerate(o.spans):
            for j in range(j0, j1):
                s = pad[P + i - ay:P + i - ay + H, P + j - ax:P + j - ax + W]
                out = np.maximum(out, s) if o.dilate else np.minimum(out, s)
        m = out
    return m


def cv_ref(mask, ops):
    """The same chain through OpenCV (default border value, as the reference's morphologyEx)"""
    import cv2

    m = mask.astype(np.uint8)
    for o in ops:
        fn = cv2.dilate if o.dilate else cv2.erode
        m = fn(m, element(o), anchor=(o.anchor[1], o.anchor[0]))
    return m


def cpu_grow(mask, k_denoise=20, k_grow=20):
    """robosat/features/core.py:65-92 denoise + grow with OpenCV"""
    import cv2

    e1 = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (k_denoise, k_denoise))
    e2 = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (k_grow, k_grow))
    return cv2.morphologyEx(cv2.morphologyEx(mask, cv2.MORPH_OPEN, e1), cv2.MORPH_CLOSE, e2)


def cpu_features(tile, labels, class_index):
    """Features of one tile on the CPU: OpenCV morphology, then the same host code as the device path"""
    return polygons_from_grown(tile, cpu_grow((labels == class_index).astype(np.uint8)))


def load_golden():
    with open(os.path.join(GOLDEN, "features.json")) as fp:
        meta = json.load(fp)
    z = np.load(os.path.join(GOLDEN, "features.npz"))
    for i, m in enumerate(meta):
        m["labels"], m["class"], m["grown"] = z["labels%d" % i], int(z["class%d" % i]), z["grown%d" % i]
    return meta
