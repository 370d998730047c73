"""JPEG (Compression 7) strips and tiles of a GeoTiff (DESIGN.md §8, restated in tests/jpeg_reference.py).

`parse` runs the library's header parser (`rsb_jpeg_parse_chunks`) over every chunk when the file is opened, so a stream outside the
rule is refused before any device work; only the descriptors are kept. A window is then decoded on the device: `stage` parses the
chunks it touches again to build their table sets (GDAL gives every tile its own optimised Huffman tables, so a raster has about one
14 KB set per chunk and none is kept beyond its window), and copies their entropy-coded bytes, descriptors and sets into host buffers
(pinned ones in `rs tile` and `rs segment`); `Decoder.decode` uploads them and runs `rsb_jpeg_decode_window` into the device window
the warps read, on the current stream. Only the compressed bytes and the window's tables cross PCIe. `Decoder.check` turns a chunk's
error word into an `RsbError` that names the strip or tile.
"""

import ctypes

import numpy as np

from robosat_b200 import _lib

F = _lib.RSB_JPEG_DESC_FIELDS
SET_BYTES = _lib.RSB_JPEG_SET_WORDS * 4
OFFSET, LENGTH, SET, WIDTH, HEIGHT, H, V, RESTART, BLOCKS, FIRST_BLOCK, CHUNK = range(11)
DATA_ERRORS = {1: "invalid Huffman code", 2: "AC coefficient index past 63", 3: "unexpected marker or RST number",
               4: "extraneous bytes before a marker", 5: "data ends before the last MCU", 6: "descriptor outside the staged data (a planning error)"}


def parse(raster, buf, tables, threads, select=None, sets=None):
    """the descriptors int64 [chunks, F] of a JPEG GeoTiff whose file bytes are `buf` (uint8 numpy array) and whose JPEGTables are
    `tables` (bytes or None): of every chunk, or of the chunks `select` (int64 indices) in that order. With `sets` (an int32 array
    [room, RSB_JPEG_SET_WORDS]) the distinct table sets of those chunks are written there and (descs, count) is returned; room for one
    set per chunk always suffices. Without, the descriptors' table set is -1. RsbError names the chunk and what is outside the rule."""
    lib = _lib.load()
    n = len(raster.offsets) if select is None else len(select)
    descs = np.zeros((n, F), np.int64)
    tab = np.frombuffer(tables, np.uint8) if tables else np.zeros(1, np.uint8)
    sel = None if select is None else np.ascontiguousarray(select, np.int64)
    count = ctypes.c_int32(0)
    bad = ctypes.c_int64(-1)
    rc = lib.rsb_jpeg_parse_chunks(buf.ctypes.data, len(buf), tab.ctypes.data, len(tables) if tables else 0, raster.offsets.ctypes.data,
                                   raster.byte_counts.ctypes.data, len(raster.offsets), raster.width, raster.height, raster.chunk_w, raster.chunk_h,
                                   raster.rows_per_strip, int(raster.tiled), raster.spp, raster.photometric, None if sel is None else sel.ctypes.data,
                                   0 if sel is None else n, threads, descs.ctypes.data, None if sets is None else sets.ctypes.data,
                                   0 if sets is None else len(sets), ctypes.byref(count), ctypes.byref(bad))
    if rc != 0:
        raise _lib.RsbError("%s: %s" % (raster.path, _lib.last_error()))
    if sets is None:
        return descs
    if count.value > len(sets):
        raise _lib.RsbError("%s: %d table sets for %d chunks" % (raster.path, count.value, len(sets)))
    return descs, count.value


def touched(raster, row0, rows, col0, cols):
    """int64 indices of the chunks a window touches, row-major over their rectangle (the order rsb_jpeg_decode_window takes)"""
    across = -(-raster.width // raster.chunk_w) if raster.tiled else 1
    cr = np.arange(row0 // raster.chunk_h, (row0 + rows - 1) // raster.chunk_h + 1, dtype=np.int64)
    cc = np.arange(col0 // raster.chunk_w, (col0 + cols - 1) // raster.chunk_w + 1, dtype=np.int64)
    return (cr[:, None] * across + cc[None, :]).ravel()


def extra_bytes(raster, row0, rows, col0, cols):
    """device bytes a window's decode takes besides its pixels: the staged entropy-coded bytes, the descriptors, the error words, the
    table sets (at most one per chunk) and rsb_jpeg_scratch_bytes of its blocks"""
    d = raster.jpeg_descs[touched(raster, row0, rows, col0, cols)]
    return int(d[:, LENGTH].sum()) + len(d) * (F * 8 + 8 + SET_BYTES) + int(d[:, BLOCKS].sum()) * _lib.RSB_JPEG_SCRATCH_PER_BLOCK


class Staged:
    """what `stage` put in the host buffers: chunk indices `chunks`, `nbytes` staged bytes, `sets` table sets, `blocks` blocks"""

    def __init__(self, window, chunks, nbytes, sets, blocks):
        self.window, self.chunks, self.nbytes, self.sets, self.blocks = window, chunks, nbytes, sets, blocks


def stage_sizes(raster, windows):
    """(staged bytes, chunks) the largest of `windows` ((row0, rows, col0, cols) each) needs in the host buffers; the table sets take
    at most one RSB_JPEG_SET_WORDS row per chunk"""
    most_bytes = most_chunks = 1
    for w in windows:
        d = raster.jpeg_descs[touched(raster, *w)]
        most_bytes = max(most_bytes, int(d[:, LENGTH].sum()))
        most_chunks = max(most_chunks, len(d))
    return most_bytes, most_chunks


def stage(raster, row0, rows, col0, cols, data, descs, sets, threads=None):
    """copy the entropy-coded bytes of the chunks the window touches into `data` (uint8, at least their total), their descriptors,
    with offsets into `data` and consecutive first blocks, into `descs` (int64, at least chunks x F), and their table sets, numbered
    for this window, into `sets` (int32, at least chunks x RSB_JPEG_SET_WORDS)"""
    from robosat_b200.hostinfo import usable_cores

    idx = touched(raster, row0, rows, col0, cols)
    buf = raster.file_bytes()
    room = sets[:len(idx) * _lib.RSB_JPEG_SET_WORDS].reshape(len(idx), _lib.RSB_JPEG_SET_WORDS)
    d, nsets = parse(raster, buf, raster.jpeg_tables, threads or usable_cores(), select=idx, sets=room)
    ends = np.cumsum(d[:, LENGTH])
    starts = ends - d[:, LENGTH]
    for k in range(len(idx)):
        data[starts[k]:ends[k]] = buf[d[k, OFFSET]:d[k, OFFSET] + d[k, LENGTH]]
    d[:, OFFSET] = starts
    d[:, FIRST_BLOCK] = np.cumsum(d[:, BLOCKS]) - d[:, BLOCKS]
    descs[:d.size] = d.ravel()
    return Staged((row0, rows, col0, cols), idx, int(ends[-1]), nsets, int(d[:, BLOCKS].sum()))


class Decoder:
    """the device side of a JPEG GeoTiff's decode; each window brings its own table sets"""

    def __init__(self, raster, device):
        import torch

        self.raster = raster
        self.device = torch.device(device)

    def decode(self, st, data, descs, sets, out, errors_host):
        """enqueue on the current stream: the upload of `st`'s staged bytes, descriptors and table sets (torch uint8 / int64 / int32
        host tensors, pinned for an asynchronous copy), the decode into `out` (device uint8, rows x cols x spp of the window) and the
        copy of the error words into errors_host (int64 host tensor). Returns the device buffers, which must live until the stream has
        run them."""
        import torch

        r = self.raster
        row0, rows, col0, cols = st.window
        n = len(st.chunks)
        staged = torch.empty((max(1, st.nbytes),), dtype=torch.uint8, device=self.device)
        staged[:st.nbytes].copy_(data[:st.nbytes], non_blocking=True)
        dd = torch.empty((n * F,), dtype=torch.int64, device=self.device)
        dd.copy_(descs[:n * F], non_blocking=True)
        words = st.sets * _lib.RSB_JPEG_SET_WORDS
        ds = torch.empty((words,), dtype=torch.int32, device=self.device)
        ds.copy_(sets[:words], non_blocking=True)
        scratch = torch.empty((st.blocks * _lib.RSB_JPEG_SCRATCH_PER_BLOCK,), dtype=torch.uint8, device=self.device)
        errors = torch.empty((n,), dtype=torch.int64, device=self.device)
        _lib.check(_lib.load().rsb_jpeg_decode_window(staged.data_ptr(), st.nbytes, dd.data_ptr(), n, ds.data_ptr(), st.sets, r.width, r.height,
                                                      r.chunk_w, r.chunk_h, int(r.tiled), r.spp, r.photometric, row0, rows, col0, cols,
                                                      out.data_ptr(), scratch.data_ptr(), scratch.numel(), st.blocks, errors.data_ptr(),
                                                      _lib.current_stream_ptr()), "rsb_jpeg_decode_window")
        errors_host[:n].copy_(errors, non_blocking=True)
        return staged, dd, ds, scratch, errors

    def check(self, st, errors_host):
        """after the stream has run `decode`: RsbError naming the first chunk whose data is damaged"""
        e = errors_host[:len(st.chunks)].numpy()
        bad = np.flatnonzero(e)
        if len(bad):
            word = int(e[bad[0]])
            raise _lib.RsbError("%s: %s %d: %s at MCU %d" % (self.raster.path, "tile" if self.raster.tiled else "strip", int(st.chunks[bad[0]]),
                                                          DATA_ERRORS.get(word & 0xFF, "error %d" % (word & 0xFF)), word >> 8))


def read_window(raster, row0, rows, col0, cols, out):
    """GeoTiff.read_window of a JPEG raster: decoded on the device and copied back into `out` (uint8 numpy, rows x cols x spp)"""
    import torch

    if row0 < 0 or col0 < 0 or rows < 1 or cols < 1 or row0 + rows > raster.height or col0 + cols > raster.width:
        raise _lib.RsbError("%s: window rows [%d, %d) cols [%d, %d) outside the %d x %d raster" % (
            raster.path, row0, row0 + rows, col0, col0 + cols, raster.width, raster.height))
    _lib.require_device()
    idx = touched(raster, row0, rows, col0, cols)
    nbytes, _ = stage_sizes(raster, [(row0, rows, col0, cols)])
    data = torch.empty((nbytes,), dtype=torch.uint8)
    descs = torch.empty((len(idx) * F,), dtype=torch.int64)
    sets = torch.empty((len(idx) * _lib.RSB_JPEG_SET_WORDS,), dtype=torch.int32)
    st = stage(raster, row0, rows, col0, cols, data.numpy(), descs.numpy(), sets.numpy())
    dec = raster.jpeg_decoder("cuda")
    dev_out = torch.empty((rows * cols * raster.spp,), dtype=torch.uint8, device=dec.device)
    errors = torch.empty((len(idx),), dtype=torch.int64)
    keep = dec.decode(st, data, descs, sets, dev_out, errors)
    torch.cuda.current_stream(dec.device).synchronize()
    del keep
    dec.check(st, errors)
    out[:] = dev_out.cpu().numpy()
    return out
