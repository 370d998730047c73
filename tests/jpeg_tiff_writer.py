"""GeoTIFFs with JPEG (Compression 7) strips or tiles for the tests of the JPEG decoder: each chunk encoded by PIL (libjpeg-turbo),
classic or BigTIFF, either byte order, Photometric 6 (YCbCr), 2 (RGB) or 1 (MinIsBlack), full streams or abbreviated streams plus
JPEGTables, per-chunk encoder settings and a hook that corrupts a chunk."""

import io
import struct

import numpy as np
from PIL import Image, ImageFile

from tiff_writer import geokeys  # noqa: F401  (re-exported for the tests)

ImageFile.MAXBLOCK = 1 << 24  # PIL's optimize / restart encodes need the whole stream in one buffer

SUBSAMPLING_TAG = {0: (1, 1), 1: (2, 1), 2: (2, 2)}  # PIL's subsampling -> TIFF YCbCrSubSampling


def encode(pixels, photometric=6, quality=75, subsampling=2, optimize=False, restart_marker_blocks=None, restart_marker_rows=None):
    """uint8 [h, w, spp] -> one JPEG stream as PIL writes it (Photometric 2 keeps RGB, unsubsampled, with no colour transform)"""
    if pixels.shape[2] == 1:
        im = Image.fromarray(np.ascontiguousarray(pixels[..., 0]), "L")
    else:
        im = Image.fromarray(np.ascontiguousarray(pixels), "RGB")
    kw = dict(quality=quality, optimize=optimize)
    if pixels.shape[2] == 3:
        kw["subsampling"] = 0 if photometric == 2 else subsampling
        if photometric == 2:
            kw["keep_rgb"] = True
    if restart_marker_blocks:
        kw["restart_marker_blocks"] = restart_marker_blocks
    if restart_marker_rows:
        kw["restart_marker_rows"] = restart_marker_rows
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def segments(stream):
    """[(marker, whole segment bytes)] up to and including SOS, then ('data', the rest)"""
    out, at = [], 2
    while True:
        m = stream[at + 1]
        n = struct.unpack(">H", stream[at + 2:at + 4])[0]
        out.append((m, stream[at:at + 2 + n]))
        at += 2 + n
        if m == 0xDA:
            out.append(("data", stream[at:]))
            return out


def abbreviate(streams, markers=(0xDB, 0xC4)):
    """(JPEGTables, streams without the segments JPEGTables holds): JPEGTables takes the first stream's segments with `markers`
    (DQT and DHT; DQT alone is GDAL's default, which leaves each tile its own, optimised, Huffman tables)"""
    first = [seg for m, seg in segments(streams[0]) if m in markers]
    tables = b"\xff\xd8" + b"".join(first) + b"\xff\xd9"
    shared = set(first)
    out = []
    for s in streams:
        out.append(b"\xff\xd8" + b"".join(seg for m, seg in segments(s) if not (m in markers and seg in shared)))
    return tables, out


def chunk_arrays(pixels, tile, rows_per_strip, pad_last_strip=False):
    """the chunks in file order: whole tiles (edge tiles padded by repeating the last row and column), or strips (the last one
    ragged, or padded to RowsPerStrip when pad_last_strip)"""
    H, W, _ = pixels.shape
    if tile:
        tw, th = tile
        out = []
        for r in range(0, H, th):
            for c in range(0, W, tw):
                ys = np.minimum(np.arange(r, r + th), H - 1)
                xs = np.minimum(np.arange(c, c + tw), W - 1)
                out.append(pixels[ys][:, xs])
        return out
    out = [pixels[r:r + rows_per_strip] for r in range(0, H, rows_per_strip)]
    if pad_last_strip and len(out[-1]) < rows_per_strip:
        ys = np.minimum(np.arange(rows_per_strip), len(out[-1]) - 1)
        out[-1] = out[-1][ys]
    return out


def write_jpeg_tiff(path, pixels, *, big=False, order="<", tile=None, rows_per_strip=None, photometric=None, tables=False, settings=None,
                    pad_last_strip=False, geo=None, scale=None, tiepoint=None, matrix=None, nodata=None, predictor=None, tags=None, corrupt=None):
    """pixels uint8 [H, W, spp] (spp 1 or 3). settings: dict of `encode` keywords, or a callable chunk index -> such a dict. tables:
    abbreviated streams plus JPEGTables (True: DQT and DHT in JPEGTables; "dqt": DQT only, as GDAL writes it). corrupt: (chunk
    index, callable bytes -> bytes) applied to one stored chunk. Returns (path, the chunk streams as stored)."""
    pixels = np.asarray(pixels, np.uint8)
    if pixels.ndim == 2:
        pixels = pixels[..., None]
    H, W, spp = pixels.shape
    photometric = photometric if photometric is not None else (1 if spp == 1 else 6)
    rows_per_strip = rows_per_strip or H
    per = settings if callable(settings) else (lambda k: settings or {})
    streams = [encode(ch, photometric, **per(k)) for k, ch in enumerate(chunk_arrays(pixels, tile, rows_per_strip, pad_last_strip))]
    jpeg_tables = None
    if tables:
        jpeg_tables, streams = abbreviate(streams, (0xDB,) if tables == "dqt" else (0xDB, 0xC4))
    if corrupt:
        streams[corrupt[0]] = corrupt[1](streams[corrupt[0]])
    e = order
    head = 16 if big else 8
    offsets, at = [], head
    for b in streams:
        offsets.append(at)
        at += len(b)
    off_type = 16 if big else 4
    t = {256: (4, [W]), 257: (4, [H]), 258: (3, [8] * spp), 259: (3, [7]), 262: (3, [photometric]), 277: (3, [spp]), 284: (3, [1]),
         339: (3, [1] * spp)}
    if photometric == 6:
        sub = (per(0) or {}).get("subsampling", 2)
        t[530] = (3, list(SUBSAMPLING_TAG[sub]))
    if predictor is not None:
        t[317] = (3, [predictor])
    if tile:
        t.update({322: (3, [tile[0]]), 323: (3, [tile[1]]), 324: (off_type, offsets), 325: (off_type, [len(b) for b in streams])})
    else:
        t.update({273: (off_type, offsets), 278: (4, [rows_per_strip]), 279: (off_type, [len(b) for b in streams])})
    if jpeg_tables is not None:
        t[347] = (7, list(jpeg_tables))
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
    fmt = {2: "s", 3: "H", 4: "I", 7: "B", 12: "d", 16: "Q"}
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
        fp.write(header + b"".join(streams) + blobs + ifd)
    return path, streams


GEO_3857 = dict(geo=geokeys(), scale=(0.45, 0.45, 0.0), tiepoint=(0, 0, 0, 1113312.7, 6106910.3, 0))


def image(H, W, spp=3, seed=0):
    """a seeded image with smooth structure and noise, so every quality and sampling gives non-trivial blocks"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = np.sin(x / 5.0 + seed) * 60 + np.cos(y / 7.0) * 50 + 128
    a = np.stack([base, np.roll(base, 3, 1) * 0.8 + 20, 255 - base], -1) + rng.normal(0, 25, (H, W, 3))
    a = np.clip(a, 0, 255).astype(np.uint8)
    return a if spp == 3 else a[..., :1]
