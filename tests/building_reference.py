"""numpy / scipy restatement of the building rule's mask cleanup (steps 1-4 of DESIGN.md §8: opening, speck drop, hole fill) and
of rsb_label_components, plus the CPU path of `rs features --type building`, for the tests."""

import numpy as np
from scipy import ndimage

import features_reference as fr
from robosat_b200.features import BuildingHandler, building_open, polygons_from_filled

STRUCTURE = {4: ndimage.generate_binary_structure(2, 1), 8: ndimage.generate_binary_structure(2, 2)}


def components(plane, value, connectivity):
    """(roots, areas, touches): int32 [H, W] smallest pixel index y * W + x of each pixel's component of (plane == value), -1 off
    it; int32 [H, W] that component's area, 0 off it; bool [H, W] whether that component touches the image border."""
    lab, n = ndimage.label(plane == value, structure=STRUCTURE[connectivity])
    flat = lab.ravel()
    ids, first = np.unique(flat, return_index=True)  # the first occurrence of a label is its smallest pixel index
    first_of = np.full(n + 1, -1, np.int64)
    first_of[ids] = first
    first_of[0] = -1
    area = np.bincount(flat, minlength=n + 1)
    area[0] = 0
    edge = np.zeros(n + 1, bool)
    edge[np.concatenate([lab[0], lab[-1], lab[:, 0], lab[:, -1]])] = True
    edge[0] = False
    return first_of[lab].astype(np.int32), area[lab].astype(np.int32), edge[lab]


def opened(labels, class_index, k_denoise=BuildingHandler.kernel_size_denoise):
    return fr.morph_ref((labels == class_index).astype(np.uint8), building_open(k_denoise))


def clean(labels, class_index, k_denoise=BuildingHandler.kernel_size_denoise, min_area=BuildingHandler.min_area,
          min_hole_area=BuildingHandler.min_hole_area):
    """Steps 1-4 on one label image -> uint8 {0, 1} mask"""
    o = opened(labels, class_index, k_denoise)
    return fill(drop(o, min_area), min_hole_area)


def drop(mask, min_area):
    _, area, _ = components(mask, 1, 8)
    return (area >= min_area).astype(np.uint8)


def fill(mask, min_hole_area):
    roots, area, touches = components(mask, 0, 4)
    return (mask.astype(bool) | ((roots >= 0) & ~touches & (area < min_hole_area))).astype(np.uint8)


def cpu_features(tile, labels, class_index):
    """Features of one tile on the CPU: the restated cleanup, then the same host code as the device path"""
    return polygons_from_filled(tile, clean(labels, class_index), BuildingHandler.simplify_epsilon)
