"""A small numpy / struct GeoTIFF writer for the `rs tile` tests: classic or BigTIFF, either byte order, strips or tiles (ragged
edges), no compression, LZW (its own encoder) or DEFLATE, predictor 1 or 2, and any GeoKeys or extra tags, including values the
reader must reject."""

import struct
import zlib

import numpy as np

EPSG_3857, EPSG_4326 = 3857, 4326


def lzw_encode(data):
    """TIFF 6.0 LZW: MSB-first codes, Clear first, widths grow one code early, Clear again when the table is full"""
    out, acc, nacc = bytearray(), 0, 0
    width = 9

    def emit(code):
        nonlocal acc, nacc
        acc = (acc << width) | code
        nacc += width
        while nacc >= 8:
            nacc -= 8
            out.append((acc >> nacc) & 0xff)

    table = {bytes([i]): i for i in range(256)}
    nxt = 258
    emit(256)
    w = b""
    for byte in data:
        wc = w + bytes([byte])
        if wc in table:
            w = wc
            continue
        emit(table[w])
        table[wc] = nxt
        nxt += 1
        if nxt >= 4094:
            emit(256)
            table = {bytes([i]): i for i in range(256)}
            nxt, width = 258, 9
        elif nxt >= (1 << width) and width < 12:
            width += 1
        w = bytes([byte])
    if w:
        emit(table[w])
        if nxt + 1 >= (1 << width) and width < 12:  # the decoder adds this code's entry before reading EOI
            width += 1
    emit(257)
    if nacc:
        out.append((acc << (8 - nacc)) & 0xff)
    return bytes(out)


def _predict(chunk, spp):
    """horizontal differencing of uint8 [rows, cols, spp], sample by sample along each row, modulo 256"""
    flat = chunk.reshape(chunk.shape[0], -1).astype(np.int16)
    d = flat.copy()
    d[:, spp:] = flat[:, spp:] - flat[:, :-spp]
    return (d & 0xff).astype(np.uint8)


def chunks(pixels, tile, rows_per_strip):
    """the chunks of pixels uint8 [H, W, spp] in file order: full tiles (zero-padded) or strips (the last one ragged)"""
    H, W, spp = pixels.shape
    if tile:
        tw, th = tile
        out = []
        for r in range(0, H, th):
            for c in range(0, W, tw):
                t = np.zeros((th, tw, spp), np.uint8)
                part = pixels[r:r + th, c:c + tw]
                t[:part.shape[0], :part.shape[1]] = part
                out.append(t)
        return out
    return [pixels[r:r + rows_per_strip] for r in range(0, H, rows_per_strip)]


def geokeys(model=1, epsg=EPSG_3857, raster_type=1, extra=()):
    """GeoKeyDirectory values: model type, raster type, the CRS key, plus (key, value) pairs"""
    keys = [(1024, model), (1025, raster_type), (3072 if model == 1 else 2048, epsg)] + list(extra)
    keys = sorted(keys)
    out = [1, 1, 0, len(keys)]
    for k, v in keys:
        out += [k, 0, 1, v]
    return out


def write_tiff(path, pixels, *, big=False, order="<", tile=None, rows_per_strip=None, compression=1, predictor=1, geo=None, scale=None,
               tiepoint=None, matrix=None, nodata=None, photometric=None, extra_samples=None, tags=None, corrupt=None):
    """pixels uint8 [H, W, spp]. geo: GeoKeyDirectory values (`geokeys`); scale / tiepoint / matrix: the georeferencing tags;
    tags: {tag: (type, values)} added or replacing; corrupt: (chunk index, callable bytes -> bytes) applied to one stored chunk."""
    pixels = np.asarray(pixels, np.uint8)
    if pixels.ndim == 2:
        pixels = pixels[..., None]
    H, W, spp = pixels.shape
    rows_per_strip = rows_per_strip or H
    data = []
    for k, ch in enumerate(chunks(pixels, tile, rows_per_strip)):
        raw = _predict(ch, spp).tobytes() if predictor == 2 and compression != 1 else np.ascontiguousarray(ch).tobytes()
        b = {1: lambda x: x, 5: lzw_encode, 8: zlib.compress, 32946: zlib.compress}.get(compression, lambda x: x)(raw)
        if corrupt and corrupt[0] == k:
            b = corrupt[1](b)
        data.append(b)
    e = order
    head = 16 if big else 8
    offsets, at = [], head
    for b in data:
        offsets.append(at)
        at += len(b)
    off_type = 16 if big else 4
    t = {256: (4, [W]), 257: (4, [H]), 258: (3, [8] * spp), 259: (3, [compression]), 262: (3, [photometric if photometric is not None else (1 if spp == 1 else 2)]),
         277: (3, [spp]), 284: (3, [1]), 339: (3, [1] * spp)}
    if predictor != 1:
        t[317] = (3, [predictor])
    if tile:
        t.update({322: (3, [tile[0]]), 323: (3, [tile[1]]), 324: (off_type, offsets), 325: (off_type, [len(b) for b in data])})
    else:
        t.update({273: (off_type, offsets), 278: (4, [rows_per_strip]), 279: (off_type, [len(b) for b in data])})
    if spp == 4 or extra_samples is not None:
        t[338] = (3, [extra_samples if extra_samples is not None else 2])
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
    blob_at = at
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
            value = struct.pack(e + ("Q" if big else "I"), blob_at + len(blobs))
            blobs += payload + (b"\0" if len(payload) % 2 else b"")
        entries.append(struct.pack(e + ("HHQ" if big else "HHI"), tag, typ, count) + value)
    ifd_at = blob_at + len(blobs)
    ifd = struct.pack(e + ("Q" if big else "H"), len(entries)) + b"".join(entries) + struct.pack(e + ("Q" if big else "I"), 0)
    if big:
        header = (b"II" if e == "<" else b"MM") + struct.pack(e + "HHHQ", 43, 8, 0, ifd_at)
    else:
        header = (b"II" if e == "<" else b"MM") + struct.pack(e + "HI", 42, ifd_at)
    with open(path, "wb") as fp:
        fp.write(header + b"".join(data) + blobs + ifd)
    return path
