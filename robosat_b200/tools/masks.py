"""`rs masks` (robosat/tools/masks.py:14-84): segmentation masks from one or more directories of quantised probabilities.

Same flags and outputs. The un-quantise / weighted soft vote / arg-max of every pixel runs on the GPU (`rsb_softvote`, float64 in
numpy's order of operations: bit-identical masks); PNG decode and encode run in a thread pool, and the probability directories
are joined by tile key instead of by directory-listing order.

`--dataset dataset.toml` with more than two classes (no reference counterpart, DESIGN.md §8): every probability root holds one
directory per class, as `rs predict` writes them for such a model, and the vote is np.argmax(np.average(P, axis=0, weights=w), axis=0)
over the C un-quantised planes of each model (`rsb_softvote_classes`); the masks use the dataset's palette. With two classes, or
without `--dataset`, the binary vote runs as before."""

import argparse
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

from robosat_b200.hostinfo import usable_cores
from robosat_b200 import _lib
from robosat_b200.colors import make_palette
from robosat_b200.config import load_config
from robosat_b200.tiles import tiles_from_slippy_map


def add_parser(subparser):
    parser = subparser.add_parser("masks", help="compute masks from prediction probabilities", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("masks", type=str, help="slippy map directory to save masks to")
    parser.add_argument("probs", type=str, nargs="+", help="slippy map directories with class probabilities")
    parser.add_argument("--weights", type=float, nargs="+", help="weights for weighted average soft-voting")
    parser.add_argument("--dataset", type=str, default=None,
                        help="dataset configuration; with more than two classes, vote over the per-class probability directories")
    parser.set_defaults(func=main)


def softvote_device(quant, weights=None):
    """quant: uint8 [K, ...] probability bins on a CUDA device -> uint8 [...] class indices (masks.py:72-84 `softvote`)."""
    assert quant.is_cuda and quant.dtype == torch.uint8 and quant.is_contiguous()
    K, n = quant.shape[0], quant[0].numel()
    mask = torch.empty(quant.shape[1:], dtype=torch.uint8, device=quant.device)
    w = torch.tensor(list(weights), dtype=torch.float64, device=quant.device) if weights is not None else None
    _lib.check(_lib.load().rsb_softvote(quant.data_ptr(), w.data_ptr() if w is not None else None, mask.data_ptr(), K, n, _lib.current_stream_ptr()),
               "rsb_softvote")
    return mask


def softvote_classes_device(quant, weights=None):
    """quant: uint8 [K, C, ...] per-class probability bins on a CUDA device -> uint8 [...] class of the largest weighted mean"""
    assert quant.is_cuda and quant.dtype == torch.uint8 and quant.is_contiguous()
    K, C, n = quant.shape[0], quant.shape[1], quant[0, 0].numel()
    mask = torch.empty(quant.shape[2:], dtype=torch.uint8, device=quant.device)
    w = torch.tensor(list(weights), dtype=torch.float64, device=quant.device) if weights is not None else None
    _lib.check(_lib.load().rsb_softvote_classes(quant.data_ptr(), w.data_ptr() if w is not None else None, mask.data_ptr(), K, C, n,
                                                _lib.current_stream_ptr()), "rsb_softvote_classes")
    return mask


def _load(path):
    return np.array(Image.open(path).convert("P"), dtype=np.uint8)  # masks.py:52


def _save(root, palette, tile, mask):
    out = Image.fromarray(mask, mode="P")
    out.putpalette(palette)
    os.makedirs(os.path.join(root, str(tile.z), str(tile.x)), exist_ok=True)
    out.save(os.path.join(root, str(tile.z), str(tile.x), str(tile.y) + ".png"), optimize=True)


def main(args, batch=64):
    if args.weights and len(args.probs) != len(args.weights):
        sys.exit("Error: number of slippy map directories and weights must be the same")
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    _lib.require_device()
    device = torch.device("cuda")
    dataset = getattr(args, "dataset", None)  # Namespaces built by callers that predate the flag have no attribute
    if dataset is not None:
        common = load_config(dataset)["common"]
        if len(common["classes"]) > 2:
            return _main_classes(args, device, common["classes"], make_palette(*common["colors"]), batch)
    indices = [dict(tiles_from_slippy_map(root)) for root in args.probs]
    keys = sorted(indices[0], key=lambda t: (int(t.z), int(t.x), int(t.y)))
    assert all(set(ix) == set(indices[0]) for ix in indices), "tilesets in sync"  # masks.py:38
    palette = make_palette("denim", "orange")
    K = len(indices)
    with ThreadPoolExecutor(max_workers=min(32, usable_cores())) as pool:
        pending = []
        for i in range(0, len(keys), batch):
            part = keys[i:i + batch]
            arrays = list(pool.map(_load, [ix[t] for ix in indices for t in part]))  # model-major, like the kernel's [K][n] layout
            shape = arrays[0].shape
            assert all(a.shape == shape for a in arrays), "probability tiles must have one size"
            host = torch.from_numpy(np.stack(arrays).reshape(K, len(part), *shape))
            masks = softvote_device(host.to(device), args.weights).cpu().numpy()
            for t, m in zip(part, masks):
                pending.append(pool.submit(_save, args.masks, palette, t, m.copy()))
        for f in pending:
            f.result()


def _main_classes(args, device, classes, palette, batch):
    """The C > 2 vote: probs/<class>/z/x/y.png of every root and class, joined by tile key"""
    for root in args.probs:
        for name in classes:
            if not os.path.isdir(os.path.join(root, name)):
                sys.exit("Error: %s has no directory for class %r" % (root, name))
    indices = [[dict(tiles_from_slippy_map(os.path.join(root, name))) for name in classes] for root in args.probs]
    keys = sorted(indices[0][0], key=lambda t: (int(t.z), int(t.x), int(t.y)))
    for root, per_class in zip(args.probs, indices):
        for name, ix in zip(classes, per_class):
            if set(ix) != set(indices[0][0]):
                sys.exit("Error: %s/%s does not hold the tile set of %s/%s" % (root, name, args.probs[0], classes[0]))
    K, C = len(indices), len(classes)
    with ThreadPoolExecutor(max_workers=min(32, usable_cores())) as pool:
        pending = []
        for i in range(0, len(keys), batch):
            part = keys[i:i + batch]
            # [K][C][tiles] order, the kernel's [K][C][n] layout
            arrays = list(pool.map(_load, [ix[t] for per_class in indices for ix in per_class for t in part]))
            shape = arrays[0].shape
            assert all(a.shape == shape for a in arrays), "probability tiles must have one size"
            host = torch.from_numpy(np.stack(arrays).reshape(K, C, len(part), *shape))
            masks = softvote_classes_device(host.to(device), args.weights).cpu().numpy()
            for t, m in zip(part, masks):
                pending.append(pool.submit(_save, args.masks, palette, t, m.copy()))
        for f in pending:
            f.result()
