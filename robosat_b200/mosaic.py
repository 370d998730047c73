"""`rs mosaic`: slippy-map mask and probability tiles back into one GeoTIFF on a raster grid, with the reprojection and the resampling
on the GPU.

The rule is this project's own (the reference never writes rasters) and is written down in DESIGN.md §8 and restated in
tests/mosaic_reference.py. It is `rs tile`'s rule with the roles swapped:

- The tiles of zoom z are a raster of 2^z S square pixels in EPSG:3857 (the world); a global pixel is valid when its tile's file
  exists.
- Output pixel (i, j) is centred at raster coordinates (i + 1/2, j + 1/2); through the grid's geotransform and
  `tile.mercator_of_model` it maps to EPSG:3857 (X, Y) and then to global pixel coordinates gx = (X + CE/2) 2^z S / CE,
  gy = (CE/2 - Y) 2^z S / CE. Global pixel g covers [g, g + 1).
- The exact (gx, gy) is computed here, in numpy, at the nodes (kG, lG) of a lattice over the output raster; `rsb_mosaic_warp`
  interpolates each pixel's cell bilinearly with the exact weights (i - kG) / G. G is the largest of 64, 32, ..., 1 for which the
  exact transform at every cell centre is within 1/8 tile pixel of the interpolation.
- A pixel is covered when (floor(gx), floor(gy)) lies in the world and is valid: nearest takes it, bilinear the four neighbours of
  (gx - 1/2, gy - 1/2) clamped to the world with invalid ones dropped and the weights renormalised. Uncovered pixels get nodata.

Work goes in windows: the output's 256-row chunk rows, split at 256-column chunk borders so that the window's reachable tiles (the
lattice's gx, gy range plus 2 pixels, intersected with the existing files), the slot table, the output and the nodes fit `budget`
device bytes. The next window's PNGs are decoded on a host thread while the current one warps, and a caller's sink (the GeoTIFF
writer of the tool) runs on another thread.
"""

import math
import os
import struct
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from robosat_b200 import _lib
from robosat_b200 import tile as T
from robosat_b200.rasterize import CE

CHUNK = 256  # output TIFF tiles are CHUNK x CHUNK
DEFAULT_BUDGET = 1 << 30
STEPS = T.STEPS
TOLERANCE = 0.125  # tile pixels between the exact transform and the lattice interpolation at every cell centre
MARGIN = 2  # tile pixels added around a window's lattice range
RESAMPLING = {"nearest": 0, "bilinear": 1}
W_COARSE = "Warning: an output pixel spans {:.1f} pixels of the zoom {} tiles; resampling aliases above 2 (mode and area resampling are not implemented)"
W_EMPTY = "Warning: no output pixel is covered by a tile"
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"


class MosaicError(ValueError):
    """An input `rs mosaic` cannot use: a tile that is not a palette or gray PNG it reads, or that disagrees with the others."""


class Grid:
    """An output raster grid: width x height pixels, crs ('3857', '4326' or ('utm', zone, south)) and geotransform (c, a, b, f, d, e)
    mapping raster coordinates (u, v) to the CRS as X = c + a u + b v, Y = f + d u + e v."""

    def __init__(self, width, height, crs, geotransform):
        self.width, self.height, self.crs, self.geotransform = int(width), int(height), crs, tuple(float(g) for g in geotransform)


# ---- inputs ----

def scan(root, zoom):
    """{(x, y): path} of every root/zoom/x/y.png"""
    base = os.path.join(root, str(zoom))
    tiles = {}
    if not os.path.isdir(base):
        return tiles
    for xd in os.listdir(base):
        if not xd.isdigit() or not os.path.isdir(os.path.join(base, xd)):
            continue
        for name in os.listdir(os.path.join(base, xd)):
            stem, ext = os.path.splitext(name)
            if ext == ".png" and stem.isdigit():
                tiles[(int(xd), int(stem))] = os.path.join(base, xd, name)
    return tiles


def png_header(path):
    """(width, height, bit depth, colour type, interlace, palette uint8 [n, 3] or None) from a PNG's IHDR and PLTE"""
    with open(path, "rb") as fp:
        head = fp.read(33)
        if len(head) < 33 or head[:8] != PNG_SIGNATURE or head[12:16] != b"IHDR":
            raise MosaicError("%s is not a PNG file" % path)
        w, h = struct.unpack(">II", head[16:24])
        depth, ctype, interlace = head[24], head[25], head[28]
        palette = None
        while ctype == 3:
            chunk = fp.read(8)
            if len(chunk) < 8:
                raise MosaicError("%s: palette PNG without PLTE" % path)
            n, kind = struct.unpack(">I", chunk[:4])[0], chunk[4:8]
            if kind in (b"IDAT", b"IEND"):
                raise MosaicError("%s: palette PNG without PLTE" % path)
            if kind == b"PLTE":
                data = fp.read(n)
                if len(data) < n or n % 3 or not 0 < n <= 768:
                    raise MosaicError("%s: PLTE of %d bytes" % (path, n))
                palette = np.frombuffer(data, np.uint8).reshape(-1, 3)
                break
            fp.seek(n + 4, 1)
    return w, h, depth, ctype, interlace, palette


def check_tiles(tiles):
    """(size, palette): the tiles' common size and the union of their palettes (uint8 [256, 3], entries no file defines black), or
    None when they are gray. MosaicError names the first file (in (x, y) order) that is not a non-interlaced palette PNG of 1, 2, 4
    or 8 bits or an 8-bit gray PNG, is another size than the first, is gray among palette files or the reverse, or has a palette
    entry that disagrees with another file's."""
    size = kind = None
    union, defined = np.zeros((256, 3), np.uint8), 0
    for key in sorted(tiles):
        path = tiles[key]
        w, h, depth, ctype, interlace, palette = png_header(path)
        if not ((ctype == 3 and depth in (1, 2, 4, 8)) or (ctype == 0 and depth == 8)) or interlace != 0:
            raise MosaicError("%s is a PNG of colour type %d, %d bits%s; rs mosaic reads palette PNGs of 1, 2, 4 or 8 bits and 8-bit gray PNGs" % (
                path, ctype, depth, ", interlaced" if interlace else ""))
        if w != h:
            raise MosaicError("%s is %dx%d; tiles must be square" % (path, w, h))
        if size is None:
            size, kind, first = w, ctype, path
        if w != size:
            raise MosaicError("%s is %dx%d, %s is %dx%d" % (path, w, h, first, size, size))
        if ctype != kind:
            raise MosaicError("%s is a %s PNG, %s is a %s PNG" % (path, "gray" if ctype == 0 else "palette", first, "gray" if kind == 0 else "palette"))
        if palette is not None:
            n = min(defined, len(palette))
            bad = np.flatnonzero((union[:n] != palette[:n]).any(axis=1))
            if len(bad):
                k = int(bad[0])
                raise MosaicError("%s: palette entry %d is %s, another tile's is %s" % (path, k, tuple(palette[k].tolist()), tuple(union[k].tolist())))
            if len(palette) > defined:
                union[defined:len(palette)] = palette[defined:]
                defined = len(palette)
    return size, (union if kind == 3 else None)


def tile_array(tiles):
    """int64 [n, 2] (x, y) of a {(x, y): path} dict, sorted"""
    return np.array(sorted(tiles), np.int64).reshape(-1, 2)


def default_grid(tiles, zoom, size):
    """the EPSG:3857 grid at the zoom's pixel size over the bounding box of the tiles: output pixel (i, j) is global pixel
    (xmin S + i, ymin S + j)"""
    t = tile_array(tiles)
    (x0, y0), (x1, y1) = t.min(axis=0), t.max(axis=0)
    px = CE / (2.0 ** zoom * size)
    return Grid((x1 - x0 + 1) * size, (y1 - y0 + 1) * size, "3857", (-CE / 2 + int(x0) * size * px, px, 0.0, CE / 2 - int(y0) * size * px, 0.0, -px))


# ---- the transform ----

def global_coords(grid, zoom, size, u, v):
    """raster coordinates (u, v) of `grid` -> continuous global pixel coordinates (gx, gy) of zoom `zoom`, tile size `size`"""
    c, a, b, f, d, e = grid.geotransform
    u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
    X, Y = T.mercator_of_model(grid.crs, c + a * u + b * v, f + d * u + e * v)
    k = 2.0 ** zoom * size / CE
    with np.errstate(invalid="ignore", over="ignore"):
        return (X + CE / 2) * k, (CE / 2 - Y) * k


def lattice(grid, zoom, size, step, kx0, kx1, ky0, ky1):
    """float64 [ky1 - ky0 + 1, kx1 - kx0 + 1, 2]: (gx, gy) at the centres of output pixels (k step, l step), kx0 <= k <= kx1,
    ky0 <= l <= ky1"""
    u = (np.arange(kx0, kx1 + 1, dtype=np.int64) * step).astype(np.float64) + 0.5
    v = (np.arange(ky0, ky1 + 1, dtype=np.int64) * step).astype(np.float64) + 0.5
    gx, gy = global_coords(grid, zoom, size, *np.meshgrid(u, v))
    return np.ascontiguousarray(np.stack([gx, gy], axis=-1))


def _lerp(a, b, t):
    return a + t * (b - a)


def step_error(grid, zoom, size, step, rows=None):
    """the largest |exact - interpolated| (gx or gy, tile pixels) at the lattice cell centres of the whole grid; NaN cells are
    skipped. Evaluated in blocks of `rows` cell rows."""
    lg = step.bit_length() - 1
    kx1, ky1 = ((grid.width - 1) >> lg) + 1, ((grid.height - 1) >> lg) + 1
    rows = rows or max(1, (1 << 20) // (kx1 + 1))
    worst = 0.0
    for l0 in range(0, ky1, rows):
        l1 = min(ky1, l0 + rows)
        n = lattice(grid, zoom, size, step, 0, kx1, l0, l1)
        mid = _lerp(_lerp(n[:-1, :-1], n[:-1, 1:], 0.5), _lerp(n[1:, :-1], n[1:, 1:], 0.5), 0.5)
        u = (np.arange(kx1, dtype=np.int64) * step).astype(np.float64) + (step / 2 + 0.5)
        v = (np.arange(l0, l1, dtype=np.int64) * step).astype(np.float64) + (step / 2 + 0.5)
        gx, gy = global_coords(grid, zoom, size, *np.meshgrid(u, v))
        with np.errstate(invalid="ignore"):
            err = np.maximum(np.abs(gx - mid[..., 0]), np.abs(gy - mid[..., 1]))
        err = err[np.isfinite(err)]
        if len(err):
            worst = max(worst, float(err.max()))
    return worst


def choose_step(grid, zoom, size):
    """the largest lattice step of STEPS that meets TOLERANCE on the whole grid"""
    for step in STEPS:
        if step_error(grid, zoom, size, step) <= TOLERANCE:
            return step
    return 1


def coarse_ratio(grid, zoom, size):
    """tile pixels per output pixel at the grid's centre (the longer of the two steps)"""
    u, v = grid.width / 2, grid.height / 2
    gx, gy = global_coords(grid, zoom, size, np.array([u, u + 1, u]), np.array([v, v, v + 1]))
    return float(max(math.hypot(gx[1] - gx[0], gy[1] - gy[0]), math.hypot(gx[2] - gx[0], gy[2] - gy[0])))


# ---- planning ----

def tile_reach(nodes, zoom, size):
    """(tx0, ty0, tx1, ty1), inclusive, of the tiles a block of lattice nodes can sample (their range plus MARGIN pixels, clipped to
    the world), or None"""
    gx, gy = nodes[..., 0], nodes[..., 1]
    ok = np.isfinite(gx) & np.isfinite(gy)
    if not ok.any():
        return None
    last = 2 ** zoom - 1
    tx0 = max(0, int(math.floor((gx[ok].min() - MARGIN) / size)))
    tx1 = min(last, int(math.floor((gx[ok].max() + MARGIN) / size)))
    ty0 = max(0, int(math.floor((gy[ok].min() - MARGIN) / size)))
    ty1 = min(last, int(math.floor((gy[ok].max() + MARGIN) / size)))
    if tx0 > tx1 or ty0 > ty1:
        return None
    return tx0, ty0, tx1, ty1


class Window:
    """output rows [row0, row0 + rows) x columns [col0, col0 + cols), the lattice nodes they read (nodes [h, w, 2] from node
    (kx0, ky0)), the tile range of their slot table (reach, inclusive; None when they reach no existing tile) and the existing tiles
    in it (int64 [n, 2])"""

    def __init__(self, row0, rows, col0, cols, kx0, ky0, nodes, reach, tiles):
        self.row0, self.rows, self.col0, self.cols = row0, rows, col0, cols
        self.kx0, self.ky0, self.nodes, self.reach, self.tiles = kx0, ky0, nodes, reach, tiles

    def device_bytes(self, size):
        return window_bytes(len(self.tiles), size, self.reach, self.rows, self.cols, self.nodes.size * 8)

    def slots(self):
        """int32 [th, tw] slot table: the position in self.tiles of each tile of the reach, -1 for no file"""
        tx0, ty0, tx1, ty1 = self.reach
        table = np.full((ty1 - ty0 + 1, tx1 - tx0 + 1), -1, np.int32)
        table[self.tiles[:, 1] - ty0, self.tiles[:, 0] - tx0] = np.arange(len(self.tiles), dtype=np.int32)
        return table


def window_bytes(n, size, reach, rows, cols, node_bytes):
    table = (reach[2] - reach[0] + 1) * (reach[3] - reach[1] + 1) * 4
    return n * size * size + table + rows * (cols + 3) // 4 * 4 + node_bytes + 64


def _in_reach(existing, reach):
    tx0, ty0, tx1, ty1 = reach
    x, y = existing[:, 0], existing[:, 1]
    return existing[(x >= tx0) & (x <= tx1) & (y >= ty0) & (y <= ty1)]


def plan(grid, zoom, size, tiles, step, budget=DEFAULT_BUDGET):
    """the windows of the output, in file order (chunk rows top to bottom, columns left to right). `tiles`: int64 [n, 2] of the
    existing tiles. RsbError when one 256 x 256 chunk alone needs more than `budget` device bytes."""
    existing = np.asarray(tiles, np.int64).reshape(-1, 2)
    lg = step.bit_length() - 1
    W, H = grid.width, grid.height
    kx1 = ((W - 1) >> lg) + 1
    windows = []
    for r0 in range(0, H, CHUNK):
        rows = min(CHUNK, H - r0)
        ky0, ky1 = r0 >> lg, ((r0 + rows - 1) >> lg) + 1
        nodes = lattice(grid, zoom, size, step, 0, kx1, ky0, ky1)
        cur = None
        for c0 in range(0, W, CHUNK):
            cols = min(CHUNK, W - c0)
            a, b = c0 >> lg, ((c0 + cols - 1) >> lg) + 1
            reach = tile_reach(nodes[:, a:b + 1], zoom, size)
            mine = _in_reach(existing, reach) if reach is not None else existing[:0]
            if not len(mine):
                if cur is not None and cur.reach is None:
                    cur.cols += cols
                else:
                    cur = Window(r0, rows, c0, cols, a, ky0, None, None, existing[:0])
                    windows.append(cur)
                continue
            alone = window_bytes(len(mine), size, reach, rows, cols, nodes[:, a:b + 1].size * 8)
            if alone > budget:
                raise _lib.RsbError("the output chunk at row %d, column %d needs %d device bytes (%d tiles of %d x %d), more than the budget of %d bytes" % (
                    r0, c0, alone, len(mine), size, size, budget))
            if cur is not None and cur.reach is not None:
                merged = (min(cur.reach[0], reach[0]), min(cur.reach[1], reach[1]), max(cur.reach[2], reach[2]), max(cur.reach[3], reach[3]))
                ca = cur.col0 >> lg
                trial = Window(r0, rows, cur.col0, cur.cols + cols, ca, ky0, nodes[:, ca:b + 1], merged, _in_reach(existing, merged))
                if trial.device_bytes(size) <= budget:
                    windows[-1] = cur = trial
                    continue
            cur = Window(r0, rows, c0, cols, a, ky0, nodes[:, a:b + 1], reach, mine)
            windows.append(cur)
    return windows


# ---- execution ----

def _pinned(n):
    import torch

    return torch.empty((max(1, n),), dtype=torch.uint8, pin_memory=True)


def run(tiles, zoom, size, grid, resampling="nearest", nodata=0, sink=None, budget=DEFAULT_BUDGET, device="cuda", stats=None, threads=None):
    """Warp the tiles {(x, y): path} of zoom `zoom` (size x size index PNGs) onto `grid`. For every window, in file order,
    sink(window, pixels) is called on a writer thread with pixels uint8 [rows, cols] (reused after the call returns), or None when
    the window reaches no tile (every pixel is nodata). Returns the number of covered output pixels. `stats`, a dict, receives the
    lattice step, the window count and seconds of decode, upload, warp (CUDA events) and sink."""
    import torch

    from robosat_b200.compare import decode_indexed
    from robosat_b200.cover import _alloc
    from robosat_b200.hostinfo import usable_cores

    if resampling not in RESAMPLING:
        raise ValueError("resampling must be one of %s" % ", ".join(RESAMPLING))
    if not 0 <= nodata <= 255:
        raise ValueError("nodata must be in 0..255")
    stats = stats if stats is not None else {}
    step = choose_step(grid, zoom, size)
    windows = plan(grid, zoom, size, tile_array(tiles), step, budget)
    stats.update(step=step, windows=len(windows), device_windows=sum(w.reach is not None for w in windows), decode_s=0.0, upload_s=0.0,
                 warp_s=0.0, sink_s=0.0)
    threads = threads or usable_cores()
    work = [k for k, w in enumerate(windows) if w.reach is not None]
    plane = size * size
    dev = torch.device(device)
    lib = _lib.load()
    if work:
        nmax = max(len(windows[k].tiles) for k in work)
        planes_host = [_pinned(nmax * plane) for _ in range(2)]
        out_host = [_pinned(max(windows[k].rows * ((windows[k].cols + 3) // 4 * 4) for k in work)) for _ in range(2)]
    counts_host = torch.empty((2,), dtype=torch.int64, pin_memory=True)
    mode = RESAMPLING[resampling]
    after = {k: work[i + 1] for i, k in enumerate(work[:-1])}
    buf = {k: i % 2 for i, k in enumerate(work)}

    def decode(k):
        t0 = time.perf_counter()
        w = windows[k]
        host = planes_host[buf[k]].numpy()
        views = [host[i * plane:(i + 1) * plane] for i in range(len(w.tiles))]
        decode_indexed([tiles[(int(x), int(y))] for x, y in w.tiles], views, np.empty((len(views), 256, 3), np.uint8), (size, size), threads,
                       native_only=True)
        return time.perf_counter() - t0

    def deliver(k, pixels):
        t0 = time.perf_counter()
        if sink is not None:
            sink(windows[k], pixels)
        return time.perf_counter() - t0

    covered_total = 0
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ThreadPoolExecutor(1) as decoder, ThreadPoolExecutor(1) as writer:
        pending = {work[0]: decoder.submit(decode, work[0])} if work else {}
        writes = []
        last_use = [None, None]  # the write of the window that last used each output buffer
        try:
            for k, w in enumerate(windows):
                if w.reach is None:
                    writes.append(writer.submit(deliver, k, None))
                    continue
                stats["decode_s"] += pending.pop(k).result()
                if k in after:
                    pending[after[k]] = decoder.submit(decode, after[k])  # into the other pinned buffer, while this window warps
                b = buf[k]
                n = len(w.tiles)
                pitch = (w.cols + 3) // 4 * 4
                t0 = time.perf_counter()
                planes = _alloc((n * plane,), torch.uint8, dev, "%d tiles of %d x %d" % (n, size, size))
                planes.copy_(planes_host[b][:n * plane], non_blocking=True)
                table = w.slots()
                slots = torch.from_numpy(table).to(dev)
                nodes = torch.from_numpy(np.ascontiguousarray(w.nodes)).to(dev)
                torch.cuda.synchronize(dev)
                stats["upload_s"] += time.perf_counter() - t0
                out = _alloc((w.rows, pitch), torch.uint8, dev, "a %d x %d output window" % (w.cols, w.rows))
                counts = torch.empty((2,), dtype=torch.int64, device=dev)
                stream = torch.cuda.current_stream(dev)
                start.record(stream)
                _lib.check(lib.rsb_mosaic_warp(planes.data_ptr(), plane, n, slots.data_ptr(), w.reach[0], w.reach[1], table.shape[1], table.shape[0],
                                               zoom, size, nodes.data_ptr(), w.kx0, w.ky0, w.nodes.shape[1], w.nodes.shape[0], step, w.col0,
                                               w.row0, w.cols, w.rows, mode, nodata, out.data_ptr(), pitch, counts[0:1].data_ptr(),
                                               counts[1:2].data_ptr(), _lib.current_stream_ptr()), "rsb_mosaic_warp")
                end.record(stream)
                if last_use[b] is not None:  # the writer is done with this output buffer before it is overwritten
                    last_use[b].result()
                out_host[b][:out.numel()].copy_(out.view(-1), non_blocking=True)
                counts_host.copy_(counts, non_blocking=True)
                torch.cuda.synchronize(dev)
                stats["warp_s"] += start.elapsed_time(end) / 1e3
                if int(counts_host[1]):
                    raise _lib.RsbError("rsb_mosaic_warp: %d samples of output rows %d..%d, columns %d..%d fell outside their window (a planning error)" % (
                        int(counts_host[1]), w.row0, w.row0 + w.rows - 1, w.col0, w.col0 + w.cols - 1))
                covered_total += int(counts_host[0])
                del planes, out
                pixels = out_host[b].numpy()[:w.rows * pitch].reshape(w.rows, pitch)[:, :w.cols]
                last_use[b] = writer.submit(deliver, k, pixels)
                writes.append(last_use[b])
        finally:
            for f in writes:
                stats["sink_s"] += f.result()
    stats["covered"] = covered_total
    return covered_total


def mosaic_device(tiles, zoom, size, grid, resampling="nearest", nodata=0, budget=DEFAULT_BUDGET, stats=None):
    """`run` collected: (uint8 [height, width] output raster, covered pixels)"""
    out = np.full((grid.height, grid.width), nodata, np.uint8)

    def sink(w, pixels):
        if pixels is not None:
            out[w.row0:w.row0 + w.rows, w.col0:w.col0 + w.cols] = pixels

    covered = run(tiles, zoom, size, grid, resampling, nodata, sink, budget, stats=stats)
    return out, covered


# ---- GeoTIFF output ----

def epsg_of(crs):
    if crs in ("3857", "4326"):
        return int(crs)
    _, zone, south = crs
    return (32700 if south else 32600) + zone


def geokeys(crs):
    """GeoKeyDirectory values: PixelIsArea, and the projected CRS in metres or EPSG:4326 in degrees"""
    if crs == "4326":
        keys = [(1024, 2), (1025, 1), (2048, 4326), (2054, 9102)]
    else:
        keys = [(1024, 1), (1025, 1), (3072, epsg_of(crs)), (3076, 9001)]
    out = [1, 1, 0, len(keys)]
    for k, v in keys:
        out += [k, 0, 1, v]
    return out


class TiffWriter:
    """A 1-band 8-bit GeoTIFF of `grid`, tiled CHUNK x CHUNK, deflate, predictor 1, little-endian; palette (ColorMap from `palette`,
    uint8 [256, 3]) or MinIsBlack (palette None); GDAL_NODATA when `nodata` is given. Windows are written in file order by `write`
    (a `run` sink); `close` writes the IFD and renames the temporary file onto `path`, `abort` removes it. BigTIFF when the worst-case
    size reaches 2^32 bytes, or when `big` says so."""

    def __init__(self, path, grid, palette=None, nodata=None, big=None, level=6, threads=None):
        from robosat_b200.hostinfo import usable_cores

        self.path, self.grid, self.palette, self.nodata = path, grid, palette, nodata
        self.fill = 0 if nodata is None else int(nodata)
        self.level, self.threads = level, threads or usable_cores()
        self.lib = _lib.load()
        self.across, self.down = -(-grid.width // CHUNK), -(-grid.height // CHUNK)
        n = self.across * self.down
        self.cap = int(self.lib.rsb_tiff_deflate_bound(CHUNK * CHUNK))
        worst = 16 + n * self.cap + n * 16 + 4096
        self.big = worst >= 2 ** 32 if big is None else bool(big)
        self.offsets = np.zeros(n, np.int64)
        self.counts = np.zeros(n, np.int64)
        self.buf = np.empty(self.across * self.cap, np.uint8)
        self.sizes = np.empty(self.across, np.int64)
        self.empty = None
        self.encode_s = self.write_s = 0.0
        d, base = os.path.split(os.path.abspath(path))
        self.tmp = os.path.join(d, ".%s.%d.tmp" % (base, os.getpid()))
        self.fp = open(self.tmp, "wb")
        self.fp.write(b"\0" * (16 if self.big else 8))

    def _encode(self, pixels, rows, cols, pitch):
        t0 = time.perf_counter()
        _lib.check(self.lib.rsb_tiff_encode_chunks(pixels.ctypes.data, pitch, rows, cols, CHUNK, self.fill, self.level, self.buf.ctypes.data, self.cap,
                                                   self.sizes.ctypes.data, self.threads), "rsb_tiff_encode_chunks")
        self.encode_s += time.perf_counter() - t0
        return [bytes(self.buf[k * self.cap:k * self.cap + int(self.sizes[k])]) for k in range(-(-cols // CHUNK))]

    def write(self, w, pixels):
        if pixels is None:
            if self.empty is None:
                self.empty = self._encode(np.full(CHUNK, self.fill, np.uint8), 1, CHUNK, CHUNK)[0]  # one fill row, padded to a fill chunk
            chunks = [self.empty] * -(-w.cols // CHUNK)
        else:
            chunks = self._encode(pixels, w.rows, w.cols, pixels.strides[0])
        t0 = time.perf_counter()
        first = (w.row0 // CHUNK) * self.across + w.col0 // CHUNK
        at = self.fp.tell()
        for k, c in enumerate(chunks):
            self.offsets[first + k], self.counts[first + k] = at, len(c)
            at += len(c)
        self.fp.write(b"".join(chunks))
        self.write_s += time.perf_counter() - t0

    def _tags(self):
        g = self.grid
        c, a, b, f, d, e = g.geotransform
        big = self.big
        t = {256: (4, [g.width]), 257: (4, [g.height]), 258: (3, [8]), 259: (3, [8]), 262: (3, [1 if self.palette is None else 3]), 277: (3, [1]),
             284: (3, [1]), 317: (3, [1]), 322: (3, [CHUNK]), 323: (3, [CHUNK]), 324: (16 if big else 4, self.offsets.tolist()),
             325: (16 if big else 4, self.counts.tolist()), 339: (3, [1]), 34735: (3, geokeys(g.crs))}
        if self.palette is not None:
            p = np.asarray(self.palette, np.uint32).reshape(256, 3) * 257
            t[320] = (3, p.T.reshape(-1).tolist())
        if b == 0 and d == 0 and a > 0 and e < 0:
            t[33550] = (12, [a, -e, 0.0])
            t[33922] = (12, [0.0, 0.0, 0.0, c, f, 0.0])
        else:
            t[34264] = (12, [a, b, 0.0, c, d, e, 0.0, f, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
        if self.nodata is not None:
            t[42113] = (2, str(int(self.nodata)))
        return t

    def close(self):
        """write the IFD, flush and rename onto the target path (an existing file is replaced)"""
        t0 = time.perf_counter()
        big = self.big
        fmt = {2: "s", 3: "H", 4: "I", 12: "d", 16: "Q"}
        tags = self._tags()
        ifd_at = self.fp.tell()
        ifd_at += ifd_at % 2
        entry, inline = (20, 8) if big else (12, 4)
        blob_at = ifd_at + (8 if big else 2) + len(tags) * entry + (8 if big else 4)
        entries, blobs = [], b""
        for tag in sorted(tags):
            typ, vals = tags[tag]
            if typ == 2:
                payload = vals.encode() + b"\0"
                count = len(payload)
            else:
                payload = struct.pack("<%d%s" % (len(vals), fmt[typ]), *vals)
                count = len(vals)
            if len(payload) <= inline:
                value = payload.ljust(inline, b"\0")
            else:
                value = struct.pack("<Q" if big else "<I", blob_at + len(blobs))
                blobs += payload + (b"\0" if len(payload) % 2 else b"")
            entries.append(struct.pack("<HHQ" if big else "<HHI", tag, typ, count) + value)
        ifd = struct.pack("<Q" if big else "<H", len(entries)) + b"".join(entries) + struct.pack("<Q" if big else "<I", 0)
        if not big and blob_at + len(blobs) >= 2 ** 32:
            raise _lib.RsbError("%s: the file outgrew a classic TIFF" % self.path)
        self.fp.seek(ifd_at)
        self.fp.write(ifd + blobs)
        self.fp.seek(0)
        self.fp.write(b"II" + (struct.pack("<HHHQ", 43, 8, 0, ifd_at) if big else struct.pack("<HI", 42, ifd_at)))
        self.fp.close()
        os.replace(self.tmp, self.path)
        self.write_s += time.perf_counter() - t0

    def abort(self):
        self.fp.close()
        if os.path.exists(self.tmp):
            os.remove(self.tmp)
