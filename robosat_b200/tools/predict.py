"""`rs predict`: probability masks for slippy-map tiles -- same flags, inputs and outputs as
robosat/tools/predict.py:23-113, with the batch loop replaced by the H100 path.

Per batch the reference does H2D of fp32 tensors, DataParallel forward, softmax, D2H of B x 2 x S x S fp32, then
crop / digitize / PNG on one CPU thread. The reference handles 2-class models only (predict.py:98); for C > 2 classes every class
plane c is written, in the same format, to `probs/<classes[c]>/z/x/y.png` (DESIGN.md §8). Here: the dataset yields raw uint8 tiles, `TilePredictor` normalises,
runs the U-Net plan and the softmax / crop / quantise head on the GPU and returns uint8 bins; PNG encoding runs in
a thread pool. With several GPUs the tile list is sharded by rank (one process per GPU), the checkpoint is
broadcast once over NCCL and no other collective is used.
"""

import argparse
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import torch
from PIL import Image

from robosat_b200.colors import continuous_palette_for_color
from robosat_b200.config import load_config
from robosat_b200.datasets import BufferedSlippyMapDirectory
from robosat_b200.tiles import _is_int
from robosat_b200.transforms import ImageToUint8Tensor


def add_parser(subparser):
    parser = subparser.add_parser("predict", help="predicts probability masks for slippy map tiles",
                                  formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--batch_size", type=int, default=1, help="images per batch")
    parser.add_argument("--checkpoint", type=str, required=True, help="model checkpoint to load")
    parser.add_argument("--overlap", type=int, default=32, help="tile pixel overlap to predict on")
    parser.add_argument("--tile_size", type=int, required=True, help="tile size for slippy map tiles")
    parser.add_argument("--workers", type=int, default=0, help="number of workers pre-processing images")
    parser.add_argument("tiles", type=str, help="directory to read slippy map image tiles from")
    parser.add_argument("probs", type=str, help="directory to save slippy map probability masks to")
    parser.add_argument("--model", type=str, required=True, help="path to model configuration file")
    parser.add_argument("--dataset", type=str, required=True, help="path to dataset configuration file")
    parser.add_argument("--tta", type=str, default="none", choices=["none", "flip", "d4"],
                        help="test-time augmentation: mean probability over flipped (flip) or all 8 dihedral (d4) views of each tile")
    parser.set_defaults(func=main)


NATIVE_PNG = os.environ.get("RSB_PNG_ENCODER", "native") != "pil"
PNG_LEVEL = min(9, max(0, int(os.environ.get("RSB_PNG_LEVEL", "6"))))  # zlib level of the library encoder (3: ~40 % less encode time, files 4 - 16 % larger)


def check_class_names(names):
    """The dataset's class names become directory names under `probs` for a model of more than two classes: each must be a
    non-empty, unique string without a path separator or NUL, not `.` or `..`, and not an integer (a directory `probs/<int>` would
    be read as a zoom level by `tiles_from_slippy_map`). Raises ValueError naming the first bad class."""
    seen = set()
    for i, name in enumerate(names):
        if not isinstance(name, str) or not name:
            raise ValueError("class %d (%r) must be a non-empty string" % (i, name))
        if any(ch in name for ch in ("/", "\\", "\0")):
            raise ValueError("class %r must not contain a path separator or NUL" % name)
        if name in (".", ".."):
            raise ValueError("class %r is not a usable directory name" % name)
        if _is_int(name):
            raise ValueError("class %r is an integer and would be read as a zoom level" % name)
        if name in seen:
            raise ValueError("class %r appears more than once" % name)
        seen.add(name)
    return list(names)


def _class_names(args, num_classes):
    """None for a binary model (one probability directory, as the reference writes it); else the checked class names"""
    if num_classes == 2:
        return None
    names = load_config(args.dataset)["common"]["classes"]
    assert len(names) == num_classes, "dataset lists %d classes, the model has %d" % (len(names), num_classes)
    return check_class_names(names)


def _palette_bytes(palette):
    """the PLTE payload of a flat palette list (<= 256 entries). Converted on every call: a cache keyed by id(palette) handed
    a later palette the bytes of an earlier, freed list that had occupied the same address"""
    return bytes(palette[:768])


def _save_png(root, palette, x, y, z, quantized, stats=None):
    """probs/z/x/y.png: P-mode PNG with the 256-entry palette (predict.py:105-113). Default: the library's encoder
    (`rsb_png_write_p8`, zlib level 6, no interpreter lock held -> the pool threads encode in parallel); pixel content and palette
    are identical to the reference's file, the compressed bytes are not. RSB_PNG_ENCODER=pil writes through PIL with
    optimize=True exactly like the reference."""
    t0 = time.perf_counter()
    os.makedirs(os.path.join(root, str(z), str(x)), exist_ok=True)
    path = os.path.join(root, str(z), str(x), str(y) + ".png")
    if NATIVE_PNG:
        from robosat_b200 import _lib

        pal = _palette_bytes(palette)
        q = quantized if quantized.flags["C_CONTIGUOUS"] else quantized.copy()
        _lib.check(_lib.load().rsb_png_write_p8(os.fsencode(path), q.ctypes.data, q.shape[1], q.shape[0], pal, len(pal) // 3, PNG_LEVEL), "rsb_png_write_p8")
    else:
        out = Image.fromarray(quantized, mode="P")
        out.putpalette(palette)
        out.save(path, optimize=True)
    if stats is not None:
        stats["png_cpu_s"] = stats.get("png_cpu_s", 0.0) + (time.perf_counter() - t0)  # summed over pool threads (GIL-protected add)


def _save_batch(root, palette, tiles, quantized, threads, stats=None, classes=None):
    """The PNG files of one batch through ONE library call (`rsb_png_write_p8_batch`: `threads` C++ threads, directories created
    by the library); RSB_PNG_ENCODER=pil loops over `_save_png` with PIL instead. tiles: [(x, y, z)], quantized: uint8 [n, H, W];
    with `classes` (C > 2 names) quantized is uint8 [n, C, H, W] and plane c goes to root/classes[c]/z/x/y.png."""
    if not NATIVE_PNG:
        for (x, y, z), q in zip(tiles, quantized):
            if classes is None:
                _save_png(root, palette, x, y, z, q, stats)
            else:
                for name, plane in zip(classes, q):
                    _save_png(os.path.join(root, name), palette, x, y, z, plane, stats)
        return
    import ctypes

    from robosat_b200 import _lib

    t0 = time.perf_counter()
    pal = _palette_bytes(palette)
    if classes is None:
        paths = [os.path.join(root, str(z), str(x), str(y) + ".png") for x, y, z in tiles]
    else:  # (tile, class) order: the order of the planes in quantized
        paths = [os.path.join(root, name, str(z), str(x), str(y) + ".png") for x, y, z in tiles for name in classes]
        quantized = quantized.reshape(-1, *quantized.shape[2:])
    n = len(paths)
    paths = (ctypes.c_char_p * n)(*[os.fsencode(p) for p in paths])
    q = quantized if quantized.flags["C_CONTIGUOUS"] else quantized.copy()
    _lib.check(_lib.load().rsb_png_write_p8_batch(paths, n, q.ctypes.data, q.shape[1] * q.shape[2], q.shape[2], q.shape[1], pal, len(pal) // 3, PNG_LEVEL,
                                                  threads, 1), "rsb_png_write_p8_batch")
    if stats is not None:
        stats["png_cpu_s"] = stats.get("png_cpu_s", 0.0) + (time.perf_counter() - t0)  # wall time of the batch calls


def run_shard(rank, world, args, device, sd, num_classes, stats=None):
    """This rank's share of the `rs predict` batch loop (predict.py:75-113): enumerate -> [decode -> halo stitch -> net -> bins]
    -> PNG. No collective in here: `sd` is the (already broadcast) state_dict. `stats` (optional dict) receives the stage
    times the cfg-4 benchmark reports: tiles, batches, wall_s, decode_wait_s (main thread blocked on decodes), gpu_wait_s
    (blocked on the device result), png_cpu_s (encode seconds summed over pool threads), png_drain_s (waiting for the last
    encodes after the last batch), pool_threads."""
    from torch.utils.data import DataLoader, Subset

    from robosat_b200.dist import shard_range
    from robosat_b200.predictor import TilePredictor

    t_start = time.perf_counter()
    st = stats if stats is not None else {}
    tta = getattr(args, "tta", "none")  # Namespaces built by callers that predate the flag have no attribute
    classes = _class_names(args, num_classes)
    size = args.tile_size + 2 * args.overlap
    palette = continuous_palette_for_color("pink", 256)
    # host cores of this rank -- min(affinity, cgroup CPU quota): the GPU boxes report 128 hardware threads under a quota of 16
    # cores -- split between the PNG-decode and PNG-encode pools (both run GIL-free C++ threads of the library).
    # More busy threads than the quota allows get the WHOLE process throttled for the rest of each scheduler period, the launching
    # thread included: the device then runs empty however deep the pipeline is. So: leave two cores to the
    # main / consumer threads and the driver, and split the rest by measured cost: ~2.4 ms to decode a 512x512 RGB tile with the
    # library's inflate, 1.1 - 1.4 ms to encode a probability mask (on one of those cores): two thirds decode, one third encodes.
    from robosat_b200.hostinfo import usable_cores

    cores = max(2, usable_cores() // max(world, 1))
    budget = max(2, min(72, cores - 2))
    enc_default = max(1, (budget + 1) // 3)
    pool_threads = int(os.environ.get("RSB_PNG_THREADS", "0")) or enc_default
    default_decode_threads = int(os.environ.get("RSB_DECODE_THREADS", "0")) or max(1, budget - enc_default)
    st.update(host_cores=cores)
    st.update(pool_threads=pool_threads, gpu_wait_s=0.0, png_cpu_s=0.0)

    def progress(it, total):
        if os.environ.get("RSB_QUIET"):
            return it
        try:
            from tqdm import tqdm

            return tqdm(it, total=total, desc="Eval", unit="batch", ascii=True, disable=rank != 0)
        except ImportError:  # pragma: no cover
            return it

    def collect(predictor, poll=False):
        t0 = time.perf_counter()
        q = predictor.collect(poll=poll).numpy()
        st["gpu_wait_s"] += time.perf_counter() - t0
        return q

    if os.environ.get("RSB_HOST_STITCH", "0") == "1":
        # reference-shaped input path: every buffered tile is assembled on the host (up to 9 decodes per tile) and copied over PCIe
        directory = BufferedSlippyMapDirectory(args.tiles, transform=ImageToUint8Tensor(), size=args.tile_size, overlap=args.overlap)
        assert len(directory) > 0, "at least one tile in dataset"
        lo, hi = shard_range(len(directory), rank, world)
        loader = DataLoader(Subset(directory, range(lo, hi)), batch_size=args.batch_size, num_workers=args.workers)
        predictor = TilePredictor(sd, num_classes, args.batch_size, size, overlap=args.overlap, device=device,
                                   use_graph=os.environ.get("RSB_PREDICT_GRAPH", "1") == "1", depth=int(os.environ.get("RSB_PREDICT_DEPTH", "3")),
                                   tta=tta)
        st.update(tiles=hi - lo, batches=len(loader), decode_wait_s=0.0)
        with ThreadPoolExecutor(max_workers=pool_threads) as pool:
            pending = []
            for images, tiles in progress(loader, len(loader)):
                n = images.shape[0]
                staging = predictor.pinned_input()
                staging[:n].copy_(images)
                if n < args.batch_size:
                    staging[n:].zero_()  # last, ragged batch: pad with black tiles and drop their outputs
                predictor.submit(staging)
                quantized = collect(predictor)
                for tile, q in zip(tiles, quantized[:n]):
                    x, y, z = (int(v) for v in tile)
                    if classes is None:
                        pending.append(pool.submit(_save_png, args.probs, palette, x, y, z, q.copy(), st))
                    else:
                        for name, plane in zip(classes, q):
                            pending.append(pool.submit(_save_png, os.path.join(args.probs, name), palette, x, y, z, plane.copy(), st))
            t0 = time.perf_counter()
            for f in pending:
                f.result()
            st["png_drain_s"] = time.perf_counter() - t0
    else:
        # default: decode every tile once, keep it in a device-resident cache and stitch the halo there (robosat_b200/stitch.py)
        from robosat_b200.stitch import DeviceTileCache, HaloStitcher
        from robosat_b200.tiles import tiles_from_slippy_map

        index = dict(tiles_from_slippy_map(args.tiles))
        assert len(index) > 0, "at least one tile in dataset"
        order = sorted(index, key=lambda t: (int(t.z), int(t.x), int(t.y)))  # column-major: neighbours stay resident
        lo, hi = shard_range(len(order), rank, world)
        mine = order[lo:hi]
        capacity = max(9 * args.batch_size, int(os.environ.get("RSB_TILE_CACHE", "2048")))
        decode_threads = args.workers if args.workers > 0 else default_decode_threads
        cache = DeviceTileCache(index, args.tile_size, capacity, device=device, workers=decode_threads)
        stitcher = HaloStitcher(cache, args.overlap, args.batch_size)
        predictor = TilePredictor(sd, num_classes, args.batch_size, size, overlap=args.overlap, device=device,
                                   use_graph=os.environ.get("RSB_PREDICT_GRAPH", "1") == "1", depth=int(os.environ.get("RSB_PREDICT_DEPTH", "3")),
                                   tta=tta)
        chunks = [mine[i:i + args.batch_size] for i in range(0, len(mine), args.batch_size)]
        st.update(tiles=len(mine), batches=len(chunks), decode_threads=decode_threads)
        st["setup_s"] = time.perf_counter() - t_start  # enumerate + plan (weight folding / packing) + buffers, before the first batch
        with ThreadPoolExecutor(max_workers=4) as pool:  # carries one library call per batch; the library brings its own threads
            import queue
            import threading

            pending = []
            # Results are taken off the device by a CONSUMER thread (wait for the D2H copy, copy the bins out of the pinned slot, hand
            # them to the PNG pool), so the launching thread never waits for a batch to finish: it only stitches, prefetches and
            # launches, at most `depth` batches ahead (the semaphore is released once a slot's host buffer has been copied out).
            # With the wait inside the loop, the host work of a batch and its device time would be serialised.
            submitted = queue.Queue()
            slots_free = threading.Semaphore(predictor.depth)
            failure = []

            def consumer():
                try:
                    torch.cuda.set_device(device)
                    while True:
                        tiles = submitted.get()
                        if tiles is None:
                            return
                        quantized = collect(predictor, poll=os.environ.get("RSB_COLLECT_POLL", "1") == "1")
                        coords = [(int(t.x), int(t.y), int(t.z)) for t in tiles]
                        bins = quantized[:len(tiles)].copy()
                        slots_free.release()
                        pending.append(pool.submit(_save_batch, args.probs, palette, coords, bins, pool_threads, st, classes))
                except BaseException as exc:  # surfaced by the launching thread
                    failure.append(exc)
                    slots_free.release()

            taker = threading.Thread(target=consumer, name="rsb-predict-consumer", daemon=True)
            taker.start()
            tm = {"stitch_s": 0.0, "prefetch_s": 0.0, "launch_s": 0.0, "slot_wait_s": 0.0}
            clock = time.perf_counter
            # decode runs up to two batches ahead of the GPU when the cache can keep three batches' neighbourhoods resident
            ahead = 2 if capacity >= 27 * args.batch_size else 1
            for c in chunks[:ahead]:
                stitcher.prefetch(c)
            marks = []
            for ci, tiles in enumerate(progress(chunks, len(chunks))):
                t0 = clock()
                slots_free.acquire()  # blocks only when `depth` batches are in flight, i.e. when the device is the bottleneck
                if failure:
                    break
                ta = clock()
                if stats is not None:  # device timeline of the batch: uploads + stitch + network + head, and the idle gap before it
                    marks.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
                    marks[-1][0].record()
                stitcher.stitch(tiles, predictor.device_input())  # upload what was decoded ahead, assemble the buffered batch on the device
                if stats is not None:
                    mid = torch.cuda.Event(enable_timing=True)
                    mid.record()
                    marks[-1] = marks[-1] + (mid,)
                t1 = clock()
                if ci + ahead < len(chunks):
                    stitcher.prefetch(chunks[ci + ahead])  # decode batch i+ahead on the library's threads while the GPU runs batch i
                t2 = clock()
                predictor.submit_device()
                if stats is not None:
                    marks[-1][1].record()
                submitted.put(tiles)
                t3 = clock()
                tm["slot_wait_s"] += ta - t0
                tm["stitch_s"] += t1 - ta
                tm["prefetch_s"] += t2 - t1
                tm["launch_s"] += t3 - t2
            submitted.put(None)
            taker.join()
            if failure:
                raise failure[0]
            t0 = time.perf_counter()
            for f in pending:
                f.result()
            st["png_drain_s"] = time.perf_counter() - t0
            st["main_thread_s"] = tm  # launching thread: waiting for a free slot (device-bound), stitch (incl. decode wait), prefetch, launches
            if marks:
                torch.cuda.synchronize(device)
                st["device_busy_s"] = sum(m[0].elapsed_time(m[1]) for m in marks) / 1e3        # uploads + stitch + net + head, per batch, summed
                st["device_idle_s"] = sum(marks[i][1].elapsed_time(marks[i + 1][0]) for i in range(len(marks) - 1)) / 1e3  # stream empty between batches
                st["device_stitch_s"] = sum(m[0].elapsed_time(m[2]) for m in marks) / 1e3      # of device_busy: waiting for uploads + table copy + stitch kernel
            t0 = time.perf_counter()
        st["pool_shutdown_s"] = time.perf_counter() - t0
        cache.close()
        st.update(decode_wait_s=cache.decode_wait_s, decodes=cache.decodes, cache_hits=cache.hits)
        if rank == 0 and os.environ.get("RSB_VERBOSE"):
            print("tile cache: %d decodes for %d tiles (%d cache hits)" % (cache.decodes, len(mine), cache.hits))
    st["wall_s"] = time.perf_counter() - t_start
    return st


def load_state_dict(path):
    # https://github.com/pytorch/pytorch/issues/7178 -- always deserialise to host memory first
    return torch.load(path, map_location="cpu")["state_dict"]


def _run(rank, world, args, port):
    from robosat_b200.dist import broadcast_state_dict, check_async_error, unet_state_template

    dataset = load_config(args.dataset)
    num_classes = len(dataset["common"]["classes"])
    torch.cuda.set_device(rank)
    device = torch.device("cuda", rank)

    sd = load_state_dict(args.checkpoint) if rank == 0 else None
    if world > 1:
        import torch.distributed as dist

        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", str(port))
        os.environ.setdefault("TORCH_NCCL_ASYNC_ERROR_HANDLING", "1")  # a failed collective aborts the process instead of hanging it
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
        sd = broadcast_state_dict(sd, unet_state_template(num_classes), device)  # the single collective of this tool
        check_async_error(device, "checkpoint broadcast")

    run_shard(rank, world, args, device, sd, num_classes)

    if world > 1:
        import torch.distributed as dist

        dist.barrier()
        check_async_error(device, "final barrier")
        dist.destroy_process_group()


def main(args):
    names = load_config(args.dataset)["common"]["classes"]
    if len(names) > 2:
        try:
            check_class_names(names)  # before any work: the names become directories under `probs`
        except ValueError as exc:
            sys.exit("Error: dataset %s: %s" % (args.dataset, exc))
    model = load_config(args.model)
    if not model["common"]["cuda"]:
        sys.exit("Error: robosat_b200 runs on CUDA devices only; set cuda = true in the model configuration")
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")

    world = int(os.environ.get("RSB_GPUS", torch.cuda.device_count()))
    world = max(1, min(world, torch.cuda.device_count()))
    if world == 1:
        _run(0, 1, args, 0)
    else:
        import socket

        import torch.multiprocessing as mp

        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        try:
            mp.spawn(_run, args=(world, args, port), nprocs=world, join=True)
        except Exception as exc:  # a rank died (CUDA / NCCL error, bad tile): the whole tool exits non-zero, like the reference's sys.exit
            sys.exit("Error: a predict rank failed: %s" % exc)
