"""`rs segment`: a GeoTIFF in, a 1-band mask (or probability) GeoTIFF on the same grid out, with the tiles, the network and the
mosaic kept on the GPU.

The rule is a composition and nothing else (DESIGN.md §8): the output's pixels are those of

    rs tile → rs predict → rs masks → rs mosaic --like ortho.tif

run with the same settings. So the tiles are `tile.candidate_tiles` (intersected with `--tiles`) warped by `tile.plan`'s windows
with `tile.choose_step`'s lattice (the corner lattice for `average`), a tile exists when it has a covered pixel, each existing
tile is predicted with the halo of its existing neighbours (black where a neighbour does not exist), the bins become masks with
the soft vote of one model, and the output windows are `mosaic.plan`'s over the grid of the source raster, sampled nearest with
missing tiles invalid.

Nothing is written to or read from disk between the steps. Two device stores hold what is in flight, both rings indexed by the
warped tiles in row-major order (tile i lives in slot i mod slots):
- the image store, uint8 [slots, S, S, 3]: `rsb_tile_warp` writes each window's tiles there, `rsb_stitch_halo` reads the 3 x 3
  neighbourhoods of a batch from it;
- the plane store, uint8 [slots, S, S]: the masks (or bins) of the predicted tiles, which `rsb_mosaic_warp` reads through its slot
  table.

The schedule (`plan`) is fixed before any device work, from the grid alone. Batch j holds warped tiles [jB, (j + 1) B); it runs
once every warp window holding one of its tiles' neighbours has been warped, and tiles that turn out not to exist are skipped
(their rows of the stitch table are -1). An output window runs right after the batch that predicts the last warped tile of its
reach. Images are freed once no later batch's neighbourhoods reach them, planes once no pending output window's reach does; both
lower bounds only grow, so both stores are rings and their peaks are known up front.
"""

import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from robosat_b200 import _lib
from robosat_b200 import mosaic as M
from robosat_b200 import tile as T
from robosat_b200.stitch import NEIGHBOURS

DEFAULT_BUDGET = 8 << 30  # device bytes of the image and plane stores together
DEFAULT_BATCH = 32
OUTPUTS = ("masks", "probs")
WRITES_AHEAD = 4  # output windows on their way to the writer at most (each holds a pinned copy of its pixels)


class Plan:
    """The schedule of one run.

    tiles       int64 [n, 2], the warped tiles (x, y) in row-major order; tile i is index i
    corner      whether the warps' lattice is the corner lattice of `average` (tile.plan's `corner`)
    warps       the tile.Window of `tile.plan`, in the same order; warp k writes indices [first[k], first[k + 1])
    neighbours  int64 [n, 9], the index of each tile's neighbour in `stitch.NEIGHBOURS` order, -1 when it is not warped
    batches     [(a, b)]: batch j predicts indices [a, b)
    windows     the mosaic.Window of `mosaic.plan`; reach[m] int64 [th, tw] holds the index of each tile of window m's reach, -1
                when it is not warped (None when the window reaches no tile at all)
    ops         [(kind, number, img_lo, img_hi, pl_lo, pl_hi)] in execution order, kind 'warp', 'predict' or 'mosaic'; the image
                store holds indices [img_lo, img_hi) and the plane store [pl_lo, pl_hi) while the op runs
    wait        {k: batch}: warp k overwrites slots whose last reader was that batch's stitch (absent: no earlier reader)
    image_slots, plane_slots, store_bytes: the peaks and what the two stores take (for a JPEG raster, store_bytes also holds
                decode_bytes: the staged bytes and decoder scratch of the largest warp window; for a band raster, render_bytes:
                the raw and the RGBA window buffers, each sized for the largest warp window)
    """


def _index_of(tiles):
    return {(int(x), int(y)): i for i, (x, y) in enumerate(tiles.tolist())}


def plan(raster, grid, zoom, size, batch=DEFAULT_BATCH, tiles=None, budget=DEFAULT_BUDGET, resampling="bilinear"):
    """The Plan of segmenting `raster` (a GeoTiff, or anything with width, height, spp, crs and geotransform) onto `grid` (a
    mosaic.Grid) with tiles of `size` pixels at `zoom` and batches of `batch`. `tiles` (iterable of (x, y)) restricts the candidate
    tiles as `rs tile --tiles` does; `resampling` is the image warp's, as in `rs tile`, and picks the lattice. Host only. RsbError,
    before anything is allocated, when the stores' peak exceeds `budget` or (average) a footprint exceeds the cap of `tile.plan`."""
    if batch < 1:
        raise ValueError("batch must be at least 1")
    if resampling not in T.RESAMPLINGS:
        raise ValueError("resampling must be one of %s" % ", ".join(T.RESAMPLINGS))
    cand = T.candidate_tiles(raster, zoom, size)
    if tiles is not None:
        want = {(int(x), int(y)) for x, y in tiles}
        cand = cand[np.array([(int(x), int(y)) in want for x, y in cand], bool)] if len(cand) else cand
    p = Plan()
    p.zoom, p.size, p.batch, p.budget = zoom, size, batch, budget
    p.corner = resampling == "average"
    p.candidates = len(cand)
    p.step = T.choose_step(raster, zoom, size, cand, p.corner)
    p.warps = T.plan(raster, zoom, size, cand, p.step, corner=p.corner)
    p.tiles = np.array([(x, w.y) for w in p.warps for x in w.xs], np.int64).reshape(-1, 2)
    p.first = np.cumsum([0] + [len(w.xs) for w in p.warps]).astype(np.int64)
    n = len(p.tiles)
    at = _index_of(p.tiles)
    p.neighbours = np.array([[at.get((x + dx, y + dy), -1) for dx, dy in NEIGHBOURS] for x, y in p.tiles.tolist()], np.int64).reshape(n, 9)
    p.batches = [(a, min(n, a + batch)) for a in range(0, n, batch)]
    p.mosaic_step = M.choose_step(grid, zoom, size)
    p.windows = M.plan(grid, zoom, size, p.tiles, p.mosaic_step)
    p.reach = []
    for w in p.windows:
        if w.reach is None:
            p.reach.append(None)
            continue
        tx0, ty0, tx1, ty1 = w.reach
        p.reach.append(np.array([[at.get((x, y), -1) for x in range(tx0, tx1 + 1)] for y in range(ty0, ty1 + 1)], np.int64))
    _schedule(p)
    p.store_bytes = p.image_slots * size * size * 3 + p.plane_slots * size * size
    if T.is_jpeg(raster):  # the staged bytes and decoder scratch of the largest warp window count too
        from robosat_b200 import jpeg

        p.decode_bytes = max([jpeg.extra_bytes(raster, w.row0, w.rows, w.col0, w.cols) for w in p.warps], default=0)
        p.store_bytes += p.decode_bytes
        if p.store_bytes > budget:
            raise _lib.RsbError("the image and plane stores and the JPEG decode need %d device bytes at their peak (%d tiles of %d x %d x 3, %d of "
                                "%d x %d and %d bytes of staged chunks and decoder scratch), more than the budget of %d bytes; segment fewer tiles at "
                                "once with --tiles" % (p.store_bytes, p.image_slots, size, size, p.plane_slots, size, size, p.decode_bytes, budget))
    if T.is_bands(raster):  # the raw and the RGBA window buffers count too
        p.render_bytes = max([T.raw_bytes(raster, w.rows, w.cols) for w in p.warps], default=0) + max([w.rows * w.cols * 4 for w in p.warps], default=0)
        p.store_bytes += p.render_bytes
        if p.store_bytes > budget:
            raise _lib.RsbError("the image and plane stores and the band windows need %d device bytes at their peak (%d tiles of %d x %d x 3, %d of "
                                "%d x %d and %d bytes of raw and RGBA windows), more than the budget of %d bytes; segment fewer tiles at once with "
                                "--tiles" % (p.store_bytes, p.image_slots, size, size, p.plane_slots, size, size, p.render_bytes, budget))
    if p.store_bytes > budget:
        raise _lib.RsbError("the image and plane stores need %d device bytes at their peak (%d tiles of %d x %d x 3 and %d of %d x %d), more than "
                            "the budget of %d bytes; segment fewer tiles at once with --tiles" % (
                                p.store_bytes, p.image_slots, size, size, p.plane_slots, size, size, budget))
    return p


def _schedule(p):
    n, B = len(p.tiles), p.batch
    nb = np.where(p.neighbours >= 0, p.neighbours, np.int64(n))
    nb_lo = nb.min(axis=1) if n else np.zeros(0, np.int64)  # the tile itself is its own neighbour: every row has one index
    nb_hi = np.where(p.neighbours >= 0, p.neighbours, np.int64(-1)).max(axis=1) if n else np.zeros(0, np.int64)
    need_lo = np.minimum.accumulate(nb_lo[::-1])[::-1] if n else nb_lo  # the lowest index any tile from i on reads
    # each output window: the lowest and highest warped index it reads, and the batch after which it runs
    span = {}
    for m, r in enumerate(p.reach):
        idx = r[r >= 0] if r is not None else np.zeros(0, np.int64)
        if len(idx):
            span[m] = (int(idx.min()), int(idx.max()))
    ready = {}
    for m, (lo, hi) in span.items():
        ready.setdefault(hi // B, []).append(m)
    last_read = np.full(n, -1, np.int64)  # the last batch whose stitch reads each image
    for j, (a, b) in enumerate(p.batches):
        rows = p.neighbours[a:b]
        last_read[rows[rows >= 0]] = j
    ops = [("mosaic", m, 0, 0, 0, 0) for m in range(len(p.windows)) if m not in span]  # nodata windows need nothing
    img_lo = img_hi = pl_lo = pl_hi = 0
    k = 0
    pending = set(span)
    image_slots = plane_slots = 0
    warp_at = []

    def first_pending(upto):  # planes below the lowest index a pending window reads are free (never above those produced)
        return min([span[q][0] for q in pending] + [upto])

    for j, (a, b) in enumerate(p.batches):
        img_lo = int(need_lo[a])
        need = int(nb_hi[a:b].max())
        while k < len(p.warps) and p.first[k] <= need:
            img_hi = int(p.first[k + 1])
            ops.append(("warp", k, img_lo, img_hi, pl_lo, pl_hi))
            warp_at.append((k, int(p.first[k]), img_hi))
            image_slots = max(image_slots, img_hi - img_lo)
            k += 1
        pl_lo, pl_hi = first_pending(a), b
        ops.append(("predict", j, img_lo, img_hi, pl_lo, pl_hi))
        plane_slots = max(plane_slots, pl_hi - pl_lo)
        for m in ready.get(j, []):
            ops.append(("mosaic", m, img_lo, img_hi, pl_lo, pl_hi))
            pending.discard(m)
            pl_lo = first_pending(pl_hi)
    p.ops, p.image_slots, p.plane_slots = ops, max(image_slots, 1), max(plane_slots, 1)
    # a warp reuses the slots of indices image_slots lower; the batch that read them last must be done with them first
    p.wait = {}
    for k, a, b in warp_at:
        old = last_read[max(0, a - p.image_slots):max(0, b - p.image_slots)]
        if len(old) and old.max() >= 0:
            p.wait[k] = int(old.max())


# ---- execution ----

def output_palette(flat):
    """uint8 [256, 3]: the palette `rs mosaic` builds from tiles saved with the flat putpalette list `flat` (its entries, then
    black)"""
    pal = np.zeros((256, 3), np.uint8)
    entries = np.asarray(flat[:768], np.uint8).reshape(-1, 3)
    pal[:len(entries)] = entries
    return pal


def run(raster, p, predictor, resampling="bilinear", output="masks", nodata=0, sink=None, device="cuda", stats=None, threads=None):
    """Execute Plan `p` on one device. `predictor`: a TilePredictor of p.batch tiles of p.size + 2 overlap pixels. `resampling`: the
    image warp's, as in `rs tile`, and must be the one `p` was planned for. output 'masks':
    the class of each pixel (the soft vote of one model); 'probs' (two classes only): the foreground bins. sink(window, pixels) is
    called on a writer thread for every output window, in schedule order, with pixels uint8 [rows, cols] (None: every pixel is
    nodata). Returns the number of existing tiles. `stats`, a dict, receives the counts and the seconds of decode, warp, predict
    (stitch, network, head and vote) and mosaic warp, the last three from CUDA events. For a JPEG raster, decode is the staging of the
    chunks' entropy-coded bytes on the host; their upload and device decode run on the warps' stream, outside the warp events. A band
    raster (geotiff.BandTiff) is uploaded raw and rendered to RGBA (rsb_tile_render, render_s) on the warps' stream before its warp."""
    import torch

    from robosat_b200.hostinfo import usable_cores

    if resampling not in T.RESAMPLINGS:
        raise ValueError("resampling must be one of %s" % ", ".join(T.RESAMPLINGS))
    if (resampling == "average") != p.corner:
        raise ValueError("the plan's lattice is for %s, not %s resampling" % ("average" if p.corner else "nearest or bilinear", resampling))
    if output not in OUTPUTS:
        raise ValueError("output must be one of %s" % ", ".join(OUTPUTS))
    C = predictor.classes
    if output == "probs" and C != 2:
        raise ValueError("probabilities are written for two-class models only")
    if predictor.batch != p.batch or predictor.out_size != p.size:
        raise ValueError("the predictor runs batches of %d tiles of %d pixels, the plan %d of %d" % (predictor.batch, predictor.out_size, p.batch, p.size))
    if not 0 <= nodata <= 255:
        raise ValueError("nodata must be in 0..255")
    stats = stats if stats is not None else {}
    threads = threads or usable_cores()
    S, n = p.size, len(p.tiles)
    stats.update(step=p.step, mosaic_step=p.mosaic_step, candidates=p.candidates, warped=n, existing=0, predicted=0, batches=0,
                 windows=len(p.windows), image_slots=p.image_slots, plane_slots=p.plane_slots, store_bytes=p.store_bytes, decode_s=0.0,
                 render_s=0.0, warp_s=0.0, predict_s=0.0, mosaic_s=0.0, sink_s=0.0)
    dev = torch.device(device)
    lib = _lib.load()
    plane, image = S * S, S * S * 3
    images = torch.empty((p.image_slots, S, S, 3), dtype=torch.uint8, device=dev)
    planes = torch.empty((p.plane_slots, S, S), dtype=torch.uint8, device=dev)
    exists = np.zeros(n, bool)
    main = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(device=dev)  # warps: their covered counts come back without waiting for the batches in flight
    bands = T.is_bands(raster)
    jpeg_host = T._jpeg_buffers(raster, p.warps, dev) if p.warps else None
    if p.warps:
        src_bytes = max(T.raw_bytes(raster, w.rows, w.cols) for w in p.warps)
        nmax = max(len(w.xs) for w in p.warps)
        if jpeg_host:
            src_host = jpeg_host["data"]
        else:
            src_host = [torch.empty((src_bytes,), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        src = torch.empty((src_bytes,), dtype=torch.uint8, device=dev)
        if bands:
            rgba = torch.empty((max(w.rows * w.cols * 4 for w in p.warps),), dtype=torch.uint8, device=dev)
        covered = torch.empty((nmax,), dtype=torch.int64, device=dev)
        misses = torch.zeros((2,), dtype=torch.int64, device=dev)
        counts_host = torch.empty((nmax + 2,), dtype=torch.int64, pin_memory=True)
    stitched = {}  # batch -> event recorded after its stitch (a later warp into the same image slots waits for it)
    timing = {"render_s": [], "warp_s": [], "predict_s": [], "mosaic_s": []}

    def timed(key):
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        timing[key].append(ev)
        return ev

    def decode(k):
        t0 = time.perf_counter()
        w = p.warps[k]
        if jpeg_host:
            jpeg_host["staged"][k % 2] = T._jpeg_stage(raster, w, jpeg_host, k % 2)
        else:
            raster.read_window(w.row0, w.rows, w.col0, w.cols, out=src_host[k % 2].numpy(), threads=threads)
        return time.perf_counter() - t0

    def deliver(m, pixels, done, counts):
        t0 = time.perf_counter()
        w = p.windows[m]
        if done is not None:
            done.synchronize()
            if int(counts[1]):
                raise _lib.RsbError("rsb_mosaic_warp: %d samples of output rows %d..%d, columns %d..%d fell outside their window (a planning error)" % (
                    int(counts[1]), w.row0, w.row0 + w.rows - 1, w.col0, w.col0 + w.cols - 1))
            pixels = pixels.numpy().reshape(w.rows, -1)[:, :w.cols]
        if sink is not None:
            sink(w, pixels)
        return time.perf_counter() - t0

    def warp(k, pending_decode):
        w = p.warps[k]
        a, b = int(p.first[k]), int(p.first[k + 1])
        stats["decode_s"] += pending_decode.result()
        nxt = decoder.submit(decode, k + 1) if k + 1 < len(p.warps) else None  # into the other pinned buffer, while this one warps
        with torch.cuda.stream(side):
            nbytes = T.raw_bytes(raster, w.rows, w.cols)
            if jpeg_host:
                keep = T._jpeg_decode(jpeg_host, k % 2, src[:nbytes])
            else:
                src[:nbytes].copy_(src_host[k % 2][:nbytes], non_blocking=True)
            nodes = torch.from_numpy(np.ascontiguousarray(w.nodes)).pin_memory().to(dev, non_blocking=True)
            xy = torch.from_numpy(p.tiles[a:b].copy()).pin_memory().to(dev, non_blocking=True)
            if k in p.wait:  # the stitch of that batch, or of the last batch before it that ran (stream order covers the rest)
                last = max((j for j in stitched if j <= p.wait[k]), default=None)
                if last is not None:
                    side.wait_event(stitched[last])
            pixels = src
            if bands:
                r0, r1 = timed("render_s")
                r0.record(side)
                T.render(lib, raster, src.data_ptr(), w.rows, w.cols, rgba.data_ptr())
                r1.record(side)
                pixels = rgba
            start, end = timed("warp_s")
            start.record(side)
            s0 = a % p.image_slots
            parts = [(0, min(b - a, p.image_slots - s0), s0)]
            if parts[0][1] < b - a:  # the window wraps around the end of the ring: the rest goes to slot 0 on
                parts.append((parts[0][1], b - a, 0))
            for q, (i0, i1, slot) in enumerate(parts):
                T.warp(lib, resampling, pixels.data_ptr(), w, raster, nodes.data_ptr(), p.step, xy[i0:].data_ptr(), i1 - i0, S, images[slot].data_ptr(),
                       image, covered[i0:].data_ptr(), misses[q:].data_ptr())
            end.record(side)
            counts_host[:b - a].copy_(covered[:b - a], non_blocking=True)
            counts_host[nmax:nmax + 2].copy_(misses, non_blocking=True)
        side.synchronize()  # the decode of window k + 2 reuses this window's pinned buffer; the counts decide what exists
        if jpeg_host:
            del keep
            T._jpeg_check(jpeg_host, k % 2)
        missed = int(counts_host[nmax]) + int(counts_host[nmax + 1])
        if missed:
            raise _lib.RsbError("%s: %d samples of tiles %d..%d of row %d fell outside their source window (a planning error)" % (
                T.entry_point(resampling), missed, w.xs[0], w.xs[-1], w.y))
        exists[a:b] = counts_host[:b - a].numpy() > 0
        return nxt

    def predict(j):
        a, b = p.batches[j]
        live = exists[a:b]
        if not live.any():
            return  # nothing to predict: the batch's planes stay unreferenced
        nbr = p.neighbours[a:b]
        table = np.full((p.batch, 9), -1, np.int32)
        ok = (nbr >= 0) & exists[np.maximum(nbr, 0)] & live[:, None]
        table[:b - a] = np.where(ok, nbr % p.image_slots, -1)
        start, end = timed("predict_s")
        start.record(main)
        dtable = torch.from_numpy(table).pin_memory().to(dev, non_blocking=True)
        x = predictor.device_input()
        _lib.check(lib.rsb_stitch_halo(images.data_ptr(), dtable.data_ptr(), x.data_ptr(), p.batch, S, predictor.overlap, _lib.current_stream_ptr()),
                   "rsb_stitch_halo")
        ev = torch.cuda.Event()
        ev.record(main)
        stitched[j] = ev
        q = predictor.submit_resident()
        s0 = a % p.plane_slots
        parts = [(0, min(b - a, p.plane_slots - s0), s0)]
        if parts[0][1] < b - a:
            parts.append((parts[0][1], b - a, 0))
        for i0, i1, slot in parts:
            if output == "probs":
                planes[slot:slot + i1 - i0].copy_(q[i0:i1])
            elif C == 2:
                _lib.check(lib.rsb_softvote(q[i0].data_ptr(), None, planes[slot].data_ptr(), 1, (i1 - i0) * plane, _lib.current_stream_ptr()),
                           "rsb_softvote")
            else:
                for i in range(i0, i1):  # the head's [B, C, S, S] is, per tile, the vote's [K = 1][C][n]
                    _lib.check(lib.rsb_softvote_classes(q[i].data_ptr(), None, planes[slot + i - i0].data_ptr(), 1, C, plane,
                                                        _lib.current_stream_ptr()), "rsb_softvote_classes")
        end.record(main)
        stats["batches"] += 1
        stats["predicted"] += int(live.sum())

    def mosaic(m):
        w = p.windows[m]
        r = p.reach[m]
        slots = np.where(r >= 0, r % p.plane_slots, -1) if r is not None else None
        if slots is not None:
            slots = np.where((r >= 0) & exists[np.maximum(r, 0)], slots, -1).astype(np.int32)
        if slots is None or not (slots >= 0).any():
            return writer.submit(deliver, m, None, None, None)  # no existing tile in reach: every pixel is nodata, as in rs mosaic
        pitch = (w.cols + 3) // 4 * 4
        start, end = timed("mosaic_s")
        start.record(main)
        dslots = torch.from_numpy(slots).pin_memory().to(dev, non_blocking=True)
        nodes = torch.from_numpy(np.ascontiguousarray(w.nodes)).pin_memory().to(dev, non_blocking=True)
        out = torch.empty((w.rows * pitch,), dtype=torch.uint8, device=dev)
        counts = torch.empty((2,), dtype=torch.int64, device=dev)
        _lib.check(lib.rsb_mosaic_warp(planes.data_ptr(), plane, p.plane_slots, dslots.data_ptr(), w.reach[0], w.reach[1], slots.shape[1], slots.shape[0],
                                       p.zoom, S, nodes.data_ptr(), w.kx0, w.ky0, w.nodes.shape[1], w.nodes.shape[0], p.mosaic_step, w.col0, w.row0,
                                       w.cols, w.rows, 0, nodata, out.data_ptr(), pitch, counts[0:1].data_ptr(), counts[1:2].data_ptr(),
                                       _lib.current_stream_ptr()), "rsb_mosaic_warp")
        end.record(main)
        host = torch.empty((w.rows * pitch,), dtype=torch.uint8, pin_memory=True)
        counts_out = torch.empty((2,), dtype=torch.int64, pin_memory=True)
        host.copy_(out, non_blocking=True)
        counts_out.copy_(counts, non_blocking=True)
        done = torch.cuda.Event()
        done.record(main)
        covered_counts.append(counts_out)
        return writer.submit(deliver, m, host, done, counts_out)

    covered_counts = []
    writes = []
    with ThreadPoolExecutor(1) as decoder, ThreadPoolExecutor(1) as writer:
        decoding = decoder.submit(decode, 0) if p.warps else None
        try:
            for kind, number, *_ in p.ops:
                if kind == "warp":
                    decoding = warp(number, decoding)
                elif kind == "predict":
                    predict(number)
                else:
                    if len(writes) >= WRITES_AHEAD:
                        stats["sink_s"] += writes.pop(0).result()
                    writes.append(mosaic(number))
        finally:
            if decoding is not None:
                decoding.result()
            for f in writes:
                stats["sink_s"] += f.result()
    torch.cuda.synchronize(dev)
    for key, evs in timing.items():
        stats[key] = sum(s.elapsed_time(e) for s, e in evs) / 1e3
    stats["existing"] = int(exists.sum())
    stats["covered"] = sum(int(c[0]) for c in covered_counts)
    return stats["existing"]
