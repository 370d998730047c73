"""A numpy / struct GeoTIFF writer for the band rule's tests: 8- or 16-bit samples, any number of bands, chunky (PlanarConfiguration
1) or band-interleaved (2), either byte order, classic or BigTIFF, strips or tiles (ragged edges), no compression, LZW (the encoder of
tiff_writer.py) or DEFLATE, predictor 1 or 2 on whole samples (computed on the values, then stored in the file's byte order, as
libtiff does)."""

import struct
import zlib

import numpy as np

from tiff_writer import geokeys, lzw_encode  # noqa: F401  (geokeys is re-exported for the tests)


def _predict(chunk, bits):
    """horizontal differencing of [rows, cols, spp] samples along each row, sample by sample, modulo 2^bits"""
    flat = chunk.reshape(chunk.shape[0], -1).astype(np.int64)
    spp = chunk.shape[2]
    d = flat.copy()
    d[:, spp:] = flat[:, spp:] - flat[:, :-spp]
    return (d & ((1 << bits) - 1)).reshape(chunk.shape)


def _chunks(pixels, tile, rows_per_strip):
    H, W, spp = pixels.shape
    if tile:
        tw, th = tile
        out = []
        for r in range(0, H, th):
            for c in range(0, W, tw):
                t = np.zeros((th, tw, spp), pixels.dtype)
                part = pixels[r:r + th, c:c + tw]
                t[:part.shape[0], :part.shape[1]] = part
                out.append(t)
        return out
    return [pixels[r:r + rows_per_strip] for r in range(0, H, rows_per_strip)]


def write_bands_tiff(path, pixels, *, bits=None, planar=1, big=False, order="<", tile=None, rows_per_strip=None, compression=1, predictor=1,
                     photometric=None, extra_samples=None, geo=None, scale=None, tiepoint=None, matrix=None, nodata=None, tags=None, corrupt=None):
    """pixels uint8 or uint16 [H, W, spp] (bits follows the dtype unless given). extra_samples: the ExtraSamples values (None: none
    written); corrupt: (chunk index in file order, callable bytes -> bytes); tags: {tag: (type, values)} added or replacing."""
    pixels = np.asarray(pixels)
    if pixels.ndim == 2:
        pixels = pixels[..., None]
    bits = bits or 8 * pixels.dtype.itemsize
    H, W, spp = pixels.shape
    rows_per_strip = rows_per_strip or H
    dtype = np.dtype(order + ("u1" if bits == 8 else "u2"))
    planes = [pixels] if planar == 1 else [pixels[..., b:b + 1] for b in range(spp)]
    data = []
    for plane in planes:
        for ch in _chunks(plane, tile, rows_per_strip):
            values = _predict(ch, bits) if predictor == 2 and compression != 1 else ch
            raw = np.ascontiguousarray(values).astype(dtype).tobytes()
            b = {1: lambda x: x, 5: lzw_encode, 8: zlib.compress, 32946: zlib.compress}.get(compression, lambda x: x)(raw)
            if corrupt and corrupt[0] == len(data):
                b = corrupt[1](b)
            data.append(b)
    e = order
    head = 16 if big else 8
    offsets, at = [], head
    for b in data:
        offsets.append(at)
        at += len(b)
    off_type = 16 if big else 4
    t = {256: (4, [W]), 257: (4, [H]), 258: (3, [bits] * spp), 259: (3, [compression]),
         262: (3, [photometric if photometric is not None else (1 if spp < 3 else 2)]), 277: (3, [spp]), 284: (3, [planar]), 339: (3, [1] * spp)}
    if predictor != 1:
        t[317] = (3, [predictor])
    if tile:
        t.update({322: (3, [tile[0]]), 323: (3, [tile[1]]), 324: (off_type, offsets), 325: (off_type, [len(b) for b in data])})
    else:
        t.update({273: (off_type, offsets), 278: (4, [rows_per_strip]), 279: (off_type, [len(b) for b in data])})
    if extra_samples is not None:
        t[338] = (3, list(extra_samples))
    if geo is not None:
        t[34735] = (3, geo)
    if scale is not None:
        t[33550] = (12, list(scale))
    if tiepoint is not None:
        t[33922] = (12, list(tiepoint))
    if matrix is not None:
        t[34264] = (12, list(matrix))
    if nodata is not None:
        t[42113] = (2, str(nodata))
    t.update(tags or {})
    fmt = {2: "s", 3: "H", 4: "I", 12: "d", 16: "Q"}
    entries, blobs = [], b""
    inline = 8 if big else 4
    for tag in sorted(t):
        typ, vals = t[tag]
        if typ == 2:
            payload = vals.encode() + b"\0"
            count = len(payload)
        else:
            payload = struct.pack(e + fmt[typ] * len(vals), *vals)
            count = len(vals)
        if len(payload) <= inline:
            value = payload.ljust(inline, b"\0")
        else:
            value = struct.pack(e + ("Q" if big else "I"), at + len(blobs))
            blobs += payload + (b"\0" if len(payload) % 2 else b"")
        entries.append(struct.pack(e + ("HHQ" if big else "HHI"), tag, typ, count) + value)
    ifd_at = at + len(blobs)
    ifd = struct.pack(e + ("Q" if big else "H"), len(entries)) + b"".join(entries) + struct.pack(e + ("Q" if big else "I"), 0)
    if big:
        header = (b"II" if e == "<" else b"MM") + struct.pack(e + "HHHQ", 43, 8, 0, ifd_at)
    else:
        header = (b"II" if e == "<" else b"MM") + struct.pack(e + "HI", 42, ifd_at)
    with open(path, "wb") as fp:
        fp.write(header + b"".join(data) + blobs + ifd)
    return path
