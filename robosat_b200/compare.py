"""`rs compare` (robosat/tools/compare.py): side-by-side review images image | label | mask 0 | ... of slippy-map tiles, with the
coverage filter and the per-tile label agreement on the GPU.

The reference opens every tile's image, label and masks with PIL, keeps a tile when any mask's share of non-zero pixels lies in
[minimum, maximum] and pastes the kept ones side by side. Here the checks run first for every tile (missing files and size
mismatches are errors before anything is written), then tiles go in batches of one size under a byte budget:

1. the masks (and, with a CSV, the labels) are decoded to index planes plus palettes by the library's PNG reader
   (`rsb_png_read_indexed_batch`, no interpreter lock), PIL's `convert("P")` for anything else;
2. `rsb_compare_count` counts every mask's non-zero pixels and its confusion counts against the label; the coverage is that
   integer count over W * H in float64 on the host, so the filter decides exactly as numpy does in the reference; with the
   dataset's classes, `rsb_compare_class_counts` adds the per-class histograms of the CSV on the same device planes;
3. only kept tiles have their images (and labels) decoded; `rsb_compare_compose` expands the planes through their palettes and
   writes the composites into pinned host memory, which the library's RGB encoder writes out while the next batch decodes.
"""

import ctypes
import os
import struct
import time
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from PIL import Image

from robosat_b200 import _lib
from robosat_b200.cover import _alloc
from robosat_b200.hostinfo import usable_cores
from robosat_b200.tiles import tiles_from_slippy_map

DEFAULT_BUDGET = 1 << 30
NATIVE_DECODE = os.environ.get("RSB_PNG_DECODER", "native") != "pil"
NATIVE_ENCODE = os.environ.get("RSB_PNG_ENCODER", "native") != "pil"
PNG_LEVEL = min(9, max(0, int(os.environ.get("RSB_PNG_LEVEL", "6"))))
CSV_COLUMNS = ["z", "x", "y", "mask", "coverage", "tp", "fp", "fn", "tn", "fg_iou"]
CLASS_CSV_COLUMNS = ["z", "x", "y", "mask", "class", "coverage", "tp", "fp", "fn", "tn", "iou"]
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"

Job = namedtuple("Job", ["tile", "image", "label", "masks", "size"])
Job.__doc__ = "One tile: its Tile, the image path, the label path, the mask paths and the image's (width, height)."


class CompareError(ValueError):
    """An input the tool cannot compare: a missing label or mask file, or a size mismatch."""


def image_size(path):
    """(width, height) from the file's header: IHDR for a PNG, PIL's lazy open for anything else."""
    with open(path, "rb") as fp:
        head = fp.read(24)
    if head[:8] == PNG_SIGNATURE and head[12:16] == b"IHDR":
        return struct.unpack(">II", head[16:24])
    with Image.open(path) as im:
        return im.size


def plan(images, labels, masks):
    """The tiles of `images` in (z, x, y) order as Jobs. Every tile's label and masks must exist and have the image's size:
    CompareError names the first tile and file that do not, before anything is read beyond the headers."""
    tiles = sorted(tiles_from_slippy_map(images), key=lambda tp: (int(tp[0].z), int(tp[0].x), int(tp[0].y)))
    jobs = []
    for tile, path in tiles:
        z, x, y = str(tile.z), str(tile.x), str(tile.y)
        name = "%s/%s/%s" % (z, x, y)
        size = tuple(image_size(path))
        others = [os.path.join(d, z, x, "{}.png".format(y)) for d in [labels] + list(masks)]
        for other in others:
            if not os.path.isfile(other):
                raise CompareError("tile %s: %s does not exist" % (name, other))
            got = tuple(image_size(other))
            if got != size:
                raise CompareError("tile %s: %s is %dx%d, the image %s is %dx%d" % (name, other, got[0], got[1], path, size[0], size[1]))
        jobs.append(Job(tile, path, others[0], others[1:], size))
    return jobs


def pitch_of(hw):
    """bytes per index plane: H * W rounded up to 16, so that every plane starts 16-byte aligned"""
    return (hw + 15) // 16 * 16


def _native(paths):
    return [i for i, p in enumerate(paths) if NATIVE_DECODE and p.lower().endswith(".png")]


def _pil_indexed(path, plane, palette, size):
    im = Image.open(path).convert("P")
    assert im.size == size, "%s changed size" % path
    plane[:size[0] * size[1]] = np.asarray(im, dtype=np.uint8).reshape(-1)
    pal = np.asarray(im.getpalette() or [], dtype=np.uint8)[:768]
    palette.reshape(-1)[:] = 0
    palette.reshape(-1)[:len(pal)] = pal


def decode_indexed(paths, planes, palettes, size, threads, pool=None, native_only=False):
    """`Image.open(p).convert("P")` of each path: index plane i into planes[i] (uint8, at least W * H bytes) and its colour table
    into palettes[i] (uint8 [256, 3]; entries past the file's palette are black, as PIL's convert("RGB") maps them). 8-bit gray
    and palette PNGs go through ONE library call; anything it reports as unsupported, and every non-PNG file, through PIL.
    `native_only`: every file goes through the library, and one it cannot decode is an RsbError naming it (no PIL)."""
    w, h = size
    native = list(range(len(paths))) if native_only else _native(paths)
    rest = sorted(set(range(len(paths))) - set(native))
    if native:
        n = len(native)
        cpaths = (ctypes.c_char_p * n)(*[os.fsencode(paths[i]) for i in native])
        outs = (ctypes.c_void_p * n)(*[planes[i].ctypes.data for i in native])
        pals = np.empty((n, 256, 3), np.uint8)
        entries = np.empty(n, np.int32)
        rcs = (ctypes.c_int32 * n)()
        rc = _lib.load().rsb_png_read_indexed_batch(cpaths, n, outs, pals.ctypes.data, entries.ctypes.data, w, h, threads, rcs)
        if rc != 0 or (native_only and any(rcs)):
            ok = (0,) if native_only else (0, _lib.RSB_E_UNSUPPORTED)
            bad = [paths[native[k]] for k in range(n) if rcs[k] not in ok]
            raise _lib.RsbError("decoding %s failed (rc=%d): %s" % (bad[:3], rc, _lib.last_error()))
        for k, i in enumerate(native):
            if rcs[k] == 0:
                palettes[i] = pals[k]
            else:
                rest.append(i)
    run = lambda i: _pil_indexed(paths[i], planes[i], palettes[i], size)  # noqa: E731
    list(pool.map(run, rest) if pool is not None else map(run, rest))


def _pil_rgb(path, out, size):
    arr = np.asarray(Image.open(path).convert("RGB"), dtype=np.uint8)
    assert arr.shape == (size[1], size[0], 3), "%s changed size" % path
    out.reshape(-1)[:] = arr.reshape(-1)


def decode_rgb(paths, images, size, threads, pool=None):
    """`Image.open(p).convert("RGB")` of each path into images[i] (uint8, W * H * 3 bytes): 8-bit PNGs through ONE library call,
    the rest (JPEG, WebP, 16-bit PNG ...) through PIL."""
    w, h = size
    native = _native(paths)
    rest = sorted(set(range(len(paths))) - set(native))
    if native:
        n = len(native)
        cpaths = (ctypes.c_char_p * n)(*[os.fsencode(paths[i]) for i in native])
        outs = (ctypes.c_void_p * n)(*[images[i].ctypes.data for i in native])
        rcs = (ctypes.c_int32 * n)()
        rc = _lib.load().rsb_png_read_rgb_batch(cpaths, n, outs, w, h, threads, rcs)
        if rc != 0:
            bad = [paths[native[k]] for k in range(n) if rcs[k] not in (0, _lib.RSB_E_UNSUPPORTED)]
            raise _lib.RsbError("decoding %s failed (rc=%d): %s" % (bad[:3], rc, _lib.last_error()))
        rest.extend(i for k, i in enumerate(native) if rcs[k] != 0)
    run = lambda i: _pil_rgb(paths[i], images[i], size)  # noqa: E731
    list(pool.map(run, rest) if pool is not None else map(run, rest))


def pack_palettes(palettes):
    """uint8 [..., 256, 3] colour tables -> uint32 [..., 256] r | g << 8 | b << 16, the layout rsb_compare_compose stages"""
    p = palettes.astype(np.uint32)
    return p[..., 0] | (p[..., 1] << 8) | (p[..., 2] << 16)


def out_stride_of(size, planes):
    """bytes per composite in the output buffer: W * (1 + planes) * H * 3 rounded up to 16"""
    return (size[0] * (1 + planes) * size[1] * 3 + 15) // 16 * 16


def count_device(masks, labels, hw, counts=None):
    """masks: uint8 CUDA tensor [N, M, pitch]; labels: uint8 CUDA tensor [N, pitch] or None -> int64 CUDA tensor [N, M, 4] of
    (tp, fp, fn, tn), foreground meaning index != 0 (without labels the label is all background), written into `counts` when
    given. Enqueued on the current stream."""
    import torch

    N, M, pitch = masks.shape
    if counts is None:
        counts = _alloc((N, M, 4), torch.int64, masks.device, "the counts of %d tiles" % N)
    _lib.check(_lib.load().rsb_compare_count(masks.data_ptr(), labels.data_ptr() if labels is not None else None, N, M, hw, pitch,
                                             counts.data_ptr(), _lib.current_stream_ptr()), "rsb_compare_count")
    return counts


def class_counts_device(masks, labels, hw, num_classes, out=None):
    """masks: uint8 CUDA tensor [N, M, pitch]; labels: uint8 CUDA tensor [N, pitch] or None (all class 0) -> int64 CUDA tensors
    (label_hist [N, C], mask_hist [N, M, C], both_hist [N, M, C], out_of_range [N, 1 + M]) of `rsb_compare_class_counts`, written
    into `out` (a tuple of the same four) when given. Enqueued on the current stream."""
    import torch

    N, M, pitch = masks.shape
    C = num_classes
    if out is None:
        out = tuple(_alloc(shape, torch.int64, masks.device, "the class counts of %d tiles" % N) for shape in ((N, C), (N, M, C), (N, M, C), (N, 1 + M)))
    _lib.check(_lib.load().rsb_compare_class_counts(masks.data_ptr(), labels.data_ptr() if labels is not None else None, N, M, C, hw, pitch,
                                                    *(t.data_ptr() for t in out), _lib.current_stream_ptr()), "rsb_compare_class_counts")
    return out


def compose_device(images, planes, palettes, size, out):
    """images: uint8 CUDA tensor [N, H * W * 3]; planes: uint8 CUDA tensor [N, P, pitch] (label, then masks); palettes: uint32
    CUDA tensor [N, P, 256]; out: uint8 tensor [N, stride] in pinned host or device memory -> out[n, :H * (1 + P) * W * 3] is
    tile n's composite. Enqueued on the current stream."""
    N, P, pitch = planes.shape
    w, h = size
    _lib.check(_lib.load().rsb_compare_compose(images.data_ptr(), planes.data_ptr(), palettes.data_ptr(), N, P, h, w, pitch, out.data_ptr(),
                                               out.stride(0), _lib.current_stream_ptr()), "rsb_compare_compose")


def tile_bytes(size, M, with_labels, num_classes=0):
    """device plus pinned host bytes one tile of a batch needs; `num_classes` > 0 adds the per-class counts (3 * C int64 per mask)"""
    hw = size[0] * size[1]
    pitch = pitch_of(hw)
    device = M * pitch + (pitch if with_labels else 0) + M * 32 + 3 * hw + (1 + M) * (pitch + 1024) + pitch
    return device + out_stride_of(size, 1 + M) + M * 3 * num_classes * 8


def batches(jobs, M, with_labels, budget, num_classes=0):
    """runs of consecutive jobs of one size whose tile_bytes fit in `budget` (one tile at least, 65535 at most)"""
    start = 0
    while start < len(jobs):
        size = jobs[start].size
        cap = min(65535, max(1, budget // tile_bytes(size, M, with_labels, num_classes)))
        end = start + 1
        while end < len(jobs) and end - start < cap and jobs[end].size == size:
            end += 1
        yield jobs[start:end]
        start = end


def csv_rows(batch, counts, coverage):
    """`CSV_COLUMNS` rows of a batch: counts int64 [N, M, 4], coverage float64 [N, M]"""
    rows = []
    for j, c, cov in zip(batch, counts, coverage):
        for m in range(len(c)):
            tp, fp, fn, tn = (int(v) for v in c[m])
            union = tp + fp + fn
            rows.append([j.tile.z, j.tile.x, j.tile.y, m, repr(float(cov[m])), tp, fp, fn, tn, repr(tp / union) if union else ""])
    return rows


def class_csv_rows(batch, label_hist, mask_hist, both_hist, coverage, classes, hw):
    """`CLASS_CSV_COLUMNS` rows of a batch, one per (tile, mask, class) with the classes in dataset order: label_hist int64 [N, C],
    mask_hist and both_hist int64 [N, M, C], coverage float64 [N, M]; tp = both, fp = mask - both, fn = label - both,
    tn = hw - label - mask + both, iou = tp / (tp + fp + fn), empty when that is 0"""
    rows = []
    for j, lab, msk, both, cov in zip(batch, label_hist, mask_hist, both_hist, coverage):
        for m in range(len(msk)):
            for c, name in enumerate(classes):
                tp, mk, lb = int(both[m, c]), int(msk[m, c]), int(lab[c])
                fp, fn = mk - tp, lb - tp
                union = tp + fp + fn
                rows.append([j.tile.z, j.tile.x, j.tile.y, m, name, repr(float(cov[m])), tp, fp, fn, hw - lb - mk + tp,
                             repr(tp / union) if union else ""])
    return rows


def out_of_range_error(batch, out_of_range, num_classes):
    """CompareError for the first tile of the batch whose label or a mask holds a value >= C (out_of_range int64 [N, 1 + M]), or None"""
    for j, row in zip(batch, out_of_range):
        for p, count in enumerate(row):
            if count:
                path = j.label if p == 0 else j.masks[p - 1]
                return CompareError("tile %s/%s/%s: %s holds %d pixels with a value outside the dataset's %d classes 0..%d"
                                    % (j.tile.z, j.tile.x, j.tile.y, path, int(count), num_classes, num_classes - 1))
    return None


def write_csv(path, rows, columns=CSV_COLUMNS):
    import csv

    with open(path, "w", newline="") as fp:
        writer = csv.writer(fp)
        writer.writerow(columns)
        writer.writerows(rows)


def _write_pil(paths, out, size, columns):
    w, h = size
    for i, path in enumerate(paths):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        rgb = out[i, :h * w * columns * 3].reshape(h, w * columns, 3)
        Image.fromarray(rgb, mode="RGB").save(path, optimize=True)


def write_composites(paths, out, size, columns, threads):
    """out: uint8 [N, stride] composites (pinned host memory) -> the PNG files `paths`, parent directories created"""
    if not paths:
        return
    if not NATIVE_ENCODE:
        _write_pil(paths, out, size, columns)
        return
    n = len(paths)
    cpaths = (ctypes.c_char_p * n)(*[os.fsencode(p) for p in paths])
    _lib.check(_lib.load().rsb_png_write_rgb8_batch(cpaths, n, out.ctypes.data, out.strides[0], size[0] * columns, size[1], PNG_LEVEL, threads, 1),
               "rsb_png_write_rgb8_batch")


def compare_device(images, labels, masks, out, minimum=0.0, maximum=1.0, csv=None, budget=DEFAULT_BUDGET, stats=None, device=None,
                   classes=None):
    """`rs compare images labels masks... --minimum --maximum [--csv [--dataset]]`: writes out/z/x/y.png for every tile with at
    least one mask whose coverage p satisfies minimum <= p <= maximum, and the CSV of every (tile, mask) when `csv` is a path.
    With `classes` (the dataset's class names, which needs `csv`) the CSV has `CLASS_CSV_COLUMNS`, one row per (tile, mask, class),
    counted by `rsb_compare_class_counts` in the same pass as the coverage; a label or mask value >= C is a CompareError naming the
    tile and the file. The coverage filter and the composites do not change.

    `stats` (a dict) receives decode_s / device_s / encode_s (wall seconds on the calling thread; encode_s on the encode thread),
    wait_s (the calling thread waiting for the previous batch's encode), kernel_ms (CUDA events around the kernels), tiles, kept and written. CompareError before anything is written when a tile
    cannot be compared."""
    import torch

    M = len(masks)
    if not 1 <= M < _lib.RSB_COMPARE_MAX_PLANES - 1:
        raise CompareError("between 1 and %d mask directories are supported, got %d" % (_lib.RSB_COMPARE_MAX_PLANES - 2, M))
    if classes is not None and not csv:
        raise CompareError("per-class counts are written to the CSV: classes need a csv path")
    C = len(classes) if classes is not None else 0
    if classes is not None and not 2 <= C <= _lib.RSB_COMPARE_MAX_CLASSES:
        raise CompareError("between 2 and %d classes are supported, got %d" % (_lib.RSB_COMPARE_MAX_CLASSES, C))
    jobs = plan(images, labels, masks)
    dev = torch.device(device if device is not None else "cuda")
    st = stats if stats is not None else {}
    st.update(decode_s=0.0, device_s=0.0, encode_s=0.0, wait_s=0.0, kernel_ms=0.0, tiles=len(jobs), kept=0, written=0)
    threads = usable_cores()
    rows = [] if csv else None
    events = []

    def encode(paths, buf, size):
        t0 = time.perf_counter()
        write_composites(paths, buf, size, 2 + M, threads)
        st["encode_s"] += time.perf_counter() - t0
        st["written"] += len(paths)

    def pinned(shape, dtype=torch.uint8):
        return torch.empty(shape, dtype=dtype, pin_memory=True)

    with ThreadPoolExecutor(max_workers=threads) as pool, ThreadPoolExecutor(max_workers=1) as encoder:
        pending = None
        for batch in batches(jobs, M, csv is not None, budget, C):
            B, size = len(batch), batch[0].size
            hw = size[0] * size[1]
            pitch = pitch_of(hw)
            t0 = time.perf_counter()
            mask_host = pinned((B, M, pitch))
            mask_pal = np.empty((B, M, 256, 3), np.uint8)
            decode_indexed([p for j in batch for p in j.masks], mask_host.numpy().reshape(B * M, pitch), mask_pal.reshape(B * M, 256, 3), size,
                           threads, pool)
            label_host = label_pal = None
            if csv:
                label_host, label_pal = pinned((B, pitch)), np.empty((B, 256, 3), np.uint8)
                decode_indexed([j.label for j in batch], label_host.numpy(), label_pal, size, threads, pool)
            t1 = time.perf_counter()
            st["decode_s"] += t1 - t0

            d_masks = _alloc((B, M, pitch), torch.uint8, dev, "the masks of %d tiles" % B)
            d_masks.copy_(mask_host, non_blocking=True)
            d_labels = None
            if csv:
                d_labels = _alloc((B, pitch), torch.uint8, dev, "the labels of %d tiles" % B)
                d_labels.copy_(label_host, non_blocking=True)
            counts = _alloc((B, M, 4), torch.int64, dev, "the counts of %d tiles" % B)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            count_device(d_masks, d_labels, hw, counts)
            hists = class_counts_device(d_masks, d_labels, hw, C) if C else None
            e1.record()
            events.append((e0, e1))
            counts = counts.cpu().numpy()
            coverage = (counts[..., 0] + counts[..., 1]) / np.int64(hw)  # float64, as np.sum(...) / np.prod(image.size)
            keep = ((coverage >= minimum) & (coverage <= maximum)).any(axis=1)
            if hists is not None:
                label_hist, mask_hist, both_hist, out_of_range = (t.cpu().numpy() for t in hists)
                err = out_of_range_error(batch, out_of_range, C)
                if err is not None:
                    raise err
                rows.extend(class_csv_rows(batch, label_hist, mask_hist, both_hist, coverage, classes, hw))
            elif rows is not None:
                rows.extend(csv_rows(batch, counts, coverage))
            t2 = time.perf_counter()
            st["device_s"] += t2 - t1

            kept = np.flatnonzero(keep)
            K = len(kept)
            if K == 0:
                continue
            st["kept"] += K
            image_host = pinned((K, hw * 3))
            decode_rgb([batch[k].image for k in kept], image_host.numpy(), size, threads, pool)
            if d_labels is None:
                label_host, label_pal = pinned((K, pitch)), np.empty((K, 256, 3), np.uint8)
                decode_indexed([batch[k].label for k in kept], label_host.numpy(), label_pal, size, threads, pool)
            else:
                label_pal = label_pal[kept]
            t3 = time.perf_counter()
            st["decode_s"] += t3 - t2
            if pending is not None:
                pending.result()  # at most two batches of composites in host memory
                t4 = time.perf_counter()
                st["wait_s"] += t4 - t3
                t3 = t4

            kidx = torch.from_numpy(kept).to(dev)
            d_images = _alloc((K, hw * 3), torch.uint8, dev, "the images of %d tiles" % K)
            d_images.copy_(image_host, non_blocking=True)
            d_planes = _alloc((K, 1 + M, pitch), torch.uint8, dev, "the label and mask planes of %d tiles" % K)
            d_planes[:, 0].copy_(label_host if d_labels is None else d_labels.index_select(0, kidx), non_blocking=True)
            d_planes[:, 1:].copy_(d_masks.index_select(0, kidx))
            pal = np.concatenate([label_pal[:, None], mask_pal[kept]], axis=1)
            d_pal = _alloc((K, 1 + M, 256), torch.int32, dev, "the palettes of %d tiles" % K)
            d_pal.copy_(torch.from_numpy(pack_palettes(pal).view(np.int32)))
            out_host = pinned((K, out_stride_of(size, 1 + M)))
            e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e2.record()
            compose_device(d_images, d_planes, d_pal, size, out_host)
            e3.record()
            events.append((e2, e3))
            e3.synchronize()
            st["device_s"] += time.perf_counter() - t3
            paths = [os.path.join(out, str(batch[k].tile.z), str(batch[k].tile.x), "{}.png".format(batch[k].tile.y)) for k in kept]
            pending = encoder.submit(encode, paths, out_host.numpy(), size)
        if pending is not None:
            pending.result()
    torch.cuda.synchronize(dev)
    st["kernel_ms"] = sum(a.elapsed_time(b) for a, b in events)
    if csv:
        write_csv(csv, rows, CLASS_CSV_COLUMNS if C else CSV_COLUMNS)
    return st
