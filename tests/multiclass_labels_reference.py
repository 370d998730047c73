"""numpy restatement of the two multi-class label rules: `rs rasterize --class NAME` and the per-class counts of
`rs compare --csv --dataset`.

Rasterize: for c = classes.index(NAME), a pixel gets c where GDAL's fill (tests/rasterize_reference.py) sets it and 0 elsewhere;
the tile is then merged with the label already on disk by np.maximum, as the reference merges existing files
(robosat/tools/rasterize.py:131-133). The maximum is commutative, associative and idempotent, so the result of burning several
classes does not depend on the order of the runs, the higher class index wins where classes overlap, and repeating a run
changes nothing.

Compare: per class c, tp = #(label == mask == c), fp = #(mask == c) - tp, fn = #(label == c) - tp, tn = hw - #(label == c) -
#(mask == c) + tp, iou = tp / (tp + fp + fn) (None when that is 0); values >= C are counted per plane instead.
"""

import numpy as np

import rasterize_reference as rr


def burn_class(tr, polygons, size, value):
    """uint8 [size, size]: value where the polygons fill under the transform tr, 0 elsewhere"""
    return rr.burn_transform(tr, polygons, size) * np.uint8(value)


def rasterize_class(tile, polygons, size, value, prev=None):
    """one `rs rasterize --class` run on one tile: the burn merged with the existing label `prev` (None: no file)"""
    out = burn_class(rr.transform(tile, size), polygons, size, value)
    return out if prev is None else np.maximum(out, prev)


def class_counts(label, masks, C):
    """label uint8 [hw], masks uint8 [M, hw] -> (label_hist [C], mask_hist [M, C], both_hist [M, C], out_of_range [1 + M]) int64"""
    label = np.asarray(label, np.uint8).reshape(-1)
    masks = np.asarray(masks, np.uint8).reshape(len(masks), -1)
    hist = lambda v: np.bincount(v, minlength=256).astype(np.int64)  # noqa: E731
    lh = hist(label)
    mh = np.stack([hist(m) for m in masks])
    bh = np.stack([hist(m[m == label]) for m in masks])
    oor = np.concatenate([[lh[C:].sum()], mh[:, C:].sum(axis=1)])
    return lh[:C], mh[:, :C], bh[:, :C], oor


def class_rows(label_hist, mask_hist, both_hist, hw):
    """[(m, c, tp, fp, fn, tn, iou)] per mask and class, iou None when tp + fp + fn == 0"""
    rows = []
    for m in range(len(mask_hist)):
        for c in range(len(label_hist)):
            tp = int(both_hist[m, c])
            fp, fn = int(mask_hist[m, c]) - tp, int(label_hist[c]) - tp
            tn = hw - int(label_hist[c]) - int(mask_hist[m, c]) + tp
            rows.append((m, c, tp, fp, fn, tn, tp / (tp + fp + fn) if tp + fp + fn else None))
    return rows
