"""The JPEG chunks of `rs tile` and `rs segment`, restated in numpy (DESIGN.md §8).

The rule, as the project defines it:

Accepted: IFD 0 of a classic TIFF or BigTIFF, either byte order, Compression 7 (TIFF Technical Note 2 "new-style" JPEG),
PlanarConfiguration 1, 8-bit unsigned samples in strips or tiles, and one of three layouts: 3 bands with Photometric 6 (YCbCr,
converted to RGB), 3 bands with Photometric 2 (RGB, samples taken as they are: libtiff decodes with JCS_UNKNOWN) or 1 band with
Photometric 1 (MinIsBlack). JPEGTables (tag 347) is optional; Predictor 1 or 2 is ignored, as libtiff ignores it for JPEG.

Stream: each chunk is one JPEG datastream. Its tables start as those of JPEGTables (an abbreviated stream of SOI, DQT / DHT and
EOI); the chunk's own DQT / DHT replace slots in stream order. Read are APPn / COM (skipped), DQT (8- or 16-bit entries), DHT, DRI
and SOF0 or SOF1 of precision 8; exactly one SOS, interleaving all components in frame order with Ss = 0, Se = 63, Ah = Al = 0;
entropy-coded data with RST0-7 in sequence; EOI.

Sampling: luma (1, 1), (2, 1) or (2, 2) with chroma (1, 1); one component's factors do not matter. The frame width equals the
chunk width; the frame height equals the tile height, or for a strip lies between the strip's rows and RowsPerStrip.

Everything else is refused when the file is opened, naming the value found and the strip or tile.

Pixels: exactly what libjpeg-turbo's default decompression gives: Huffman decode with the DC predictors reset at every restart,
`jpeg_idct_islow` (int64 arithmetic, the pass-1 results truncated to int, the RANGE_MASK wrap and the range limit), fancy upsampling
as `jdsample.c` (h2v1, h2v2; plain replication when the chroma is at most 2 samples wide; edges replicated at the component's true
size) and `jdcolor.c`'s integer YCbCr -> RGB tables. The chunk is then cropped to the raster.

Damaged entropy data (an invalid Huffman code, an AC index past 63, an unexpected marker or RST number, extraneous bytes before a
marker, data that ends before the last MCU) raises `DataError`; libjpeg warns and pads with zeros instead.
"""

import struct

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
                   62, 63], np.int64)  # natural index of the k-th coefficient in stream order

# data error codes (the device's error words use the same numbers)
BAD_CODE, AC_PAST_63, BAD_MARKER, EXTRANEOUS, TRUNCATED = 1, 2, 3, 4, 5
DATA_ERRORS = {BAD_CODE: "invalid Huffman code", AC_PAST_63: "AC coefficient index past 63", BAD_MARKER: "unexpected marker or RST number",
               EXTRANEOUS: "extraneous bytes before a marker", TRUNCATED: "data ends before the last MCU"}
SAMPLINGS = ((1, 1), (2, 1), (2, 2))


class Rejected(ValueError):
    """a stream outside the rule; the text names the value found"""


class DataError(ValueError):
    def __init__(self, code, mcu):
        super().__init__("%s at MCU %d" % (DATA_ERRORS[code], mcu))
        self.code, self.mcu = code, mcu


# ---- Huffman tables (libjpeg's jpeg_make_d_derived_tbl) ----

def derive(bits, vals, dc):
    """bits[1..16] counts and the symbol values -> dict(lookup int32 [256] = (length << 8) | symbol, or 9 << 8 for longer codes;
    maxcode int32 [18]; valoffset int32 [18]; huffval int32 [256]). Rejected when over-subscribed or a DC symbol exceeds 15."""
    huffsize = []
    for l in range(1, 17):
        huffsize += [l] * bits[l]
    if len(huffsize) > 256 or len(vals) < len(huffsize):
        raise Rejected("a Huffman table of %d codes" % len(huffsize))
    codes, code, si, p = [], 0, huffsize[0] if huffsize else 0, 0
    while p < len(huffsize):
        while p < len(huffsize) and huffsize[p] == si:
            codes.append(code)
            p += 1
            code += 1
        if code >= 1 << si:
            raise Rejected("an over-subscribed Huffman table")
        code <<= 1
        si += 1
    maxcode, valoffset = [-1] + [0] * 17, [0] * 18
    p = 0
    for l in range(1, 17):
        if bits[l]:
            valoffset[l] = p - codes[p]
            p += bits[l]
            maxcode[l] = codes[p - 1]
        else:
            maxcode[l] = -1
    maxcode[17] = 0xFFFFF
    lookup = [9 << 8] * 256
    p = 0
    for l in range(1, 9):
        for _ in range(bits[l]):
            look = codes[p] << (8 - l)
            for c in range(1 << (8 - l)):
                lookup[look + c] = (l << 8) | vals[p]
            p += 1
    if dc and any(v > 15 for v in vals[:len(huffsize)]):
        raise Rejected("a DC Huffman symbol above 15")
    huffval = list(vals[:len(huffsize)]) + [0] * (256 - len(huffsize))
    return dict(lookup=np.array(lookup, np.int32), maxcode=np.array(maxcode, np.int32), valoffset=np.array(valoffset, np.int32),
                huffval=np.array(huffval, np.int32))


# ---- stream parsing ----

def _segments(s, at, what):
    """(marker, payload, offset after) per marker segment from `at` until SOS (included) or EOI"""
    while True:
        if at + 2 > len(s) or s[at] != 0xFF:
            raise Rejected("%s: no marker at byte %d" % (what, at))
        while at + 1 < len(s) and s[at + 1] == 0xFF:
            at += 1  # fill bytes
        if at + 2 > len(s):
            raise Rejected("%s: no marker at byte %d" % (what, at))
        m = s[at + 1]
        if m == 0xD9:
            yield m, b"", at + 2
            return
        if at + 4 > len(s):
            raise Rejected("%s: segment 0x%02X truncated" % (what, m))
        n = struct.unpack(">H", s[at + 2:at + 4])[0]
        if n < 2 or at + 2 + n > len(s):
            raise Rejected("%s: segment 0x%02X of length %d runs past the data" % (what, m, n))
        yield m, s[at + 4:at + 2 + n], at + 2 + n
        at += 2 + n
        if m == 0xDA:
            return


def _dqt(p, q):
    i = 0
    while i < len(p):
        pq, tq = p[i] >> 4, p[i] & 15
        if pq > 1 or tq > 3:
            raise Rejected("DQT precision %d slot %d" % (pq, tq))
        n = 128 if pq else 64
        if i + 1 + n > len(p):
            raise Rejected("a truncated DQT")
        vals = struct.unpack(">64H", p[i + 1:i + 129]) if pq else tuple(p[i + 1:i + 65])
        nat = np.zeros(64, np.int32)
        nat[ZIGZAG] = vals
        q[tq] = nat
        i += 1 + n


def _dht(p, h):
    i = 0
    while i < len(p):
        tc, th = p[i] >> 4, p[i] & 15
        if tc > 1 or th > 3:
            raise Rejected("DHT class %d slot %d" % (tc, th))
        if i + 17 > len(p):
            raise Rejected("a truncated DHT")
        bits = [0] + list(p[i + 1:i + 17])
        n = sum(bits)
        if n > 256 or i + 17 + n > len(p):
            raise Rejected("a DHT of %d symbols" % n)
        h[(tc, th)] = derive(bits, list(p[i + 17:i + 17 + n]), tc == 0)
        i += 17 + n


def read_tables(tables):
    """(quant slots, huffman slots) of a JPEGTables stream"""
    q, h = {}, {}
    if tables is None:
        return q, h
    if tables[:2] != b"\xff\xd8":
        raise Rejected("JPEGTables does not start with SOI")
    for m, p, _ in _segments(tables, 2, "JPEGTables"):
        if m == 0xDB:
            _dqt(p, q)
        elif m == 0xC4:
            _dht(p, h)
        elif m == 0xDD:
            raise Rejected("DRI in JPEGTables")
        elif m == 0xD9 or 0xE0 <= m <= 0xEF or m == 0xFE:
            continue
        else:
            raise Rejected("marker 0x%02X in JPEGTables" % m)
    return q, h


def _end_of_entropy(s, at):
    """offset of the first marker after `at` that is not stuffing, fill or RSTn"""
    i = at
    while True:
        i = s.find(b"\xff", i)
        if i < 0 or i + 1 >= len(s):
            return -1
        if s[i + 1] == 0 or s[i + 1] == 0xFF or 0xD0 <= s[i + 1] <= 0xD7:
            i += 1
            continue
        return i


def parse(stream, tables, spp, photometric):
    """the header of one chunk's stream, given JPEGTables' (quant, huffman) slots -> dict(width, height, h, v, restart, start, end,
    quant [spp] int32 [64] natural order, dc / ac [spp] derived tables). Rejected names what is outside the rule."""
    q, h = dict(tables[0]), dict(tables[1])
    s = bytes(stream)
    if s[:2] != b"\xff\xd8":
        raise Rejected("does not start with SOI")
    frame, restart, scan = None, 0, None
    for m, p, after in _segments(s, 2, "stream"):
        if m == 0xDB:
            _dqt(p, q)
        elif m == 0xC4:
            _dht(p, h)
        elif m == 0xDD:
            if len(p) != 2:
                raise Rejected("a DRI of %d bytes" % len(p))
            restart = struct.unpack(">H", p)[0]
        elif m in (0xC0, 0xC1):
            if frame is not None:
                raise Rejected("two frames")
            if len(p) < 6 or p[0] != 8:
                raise Rejected("precision %d" % (p[0] if p else -1))
            hgt, wid, nf = struct.unpack(">HHB", p[1:6])
            if nf != spp:
                raise Rejected("%d components in a %d-band image" % (nf, spp))
            if len(p) != 6 + 3 * nf:
                raise Rejected("an SOF of %d bytes" % len(p))
            frame = dict(width=wid, height=hgt, comps=[(p[6 + 3 * i], p[7 + 3 * i] >> 4, p[7 + 3 * i] & 15, p[8 + 3 * i]) for i in range(nf)])
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            kind = {0xC2: "progressive", 0xC3: "lossless"}.get(m, "arithmetic or hierarchical")
            raise Rejected("%s frames (SOF%d) are not supported" % (kind, m - 0xC0))
        elif m == 0xDA:
            scan = (p, after)
        elif m == 0xD9:
            raise Rejected("no scan")
        elif 0xE0 <= m <= 0xEF or m == 0xFE:
            continue
        else:
            raise Rejected("marker 0x%02X" % m)
    if frame is None:
        raise Rejected("no SOF0 / SOF1 frame before the scan")
    comps = frame["comps"]
    if frame["width"] == 0 or frame["height"] == 0:
        raise Rejected("a %d x %d frame" % (frame["width"], frame["height"]))
    if spp == 1:
        hv = (1, 1)
    else:
        hv = (comps[0][1], comps[0][2])
        if hv not in SAMPLINGS or any((c[1], c[2]) != (1, 1) for c in comps[1:]):
            raise Rejected("sampling %s is not supported; use luma 1x1, 2x1 or 2x2 with chroma 1x1" % ",".join("%dx%d" % (c[1], c[2]) for c in comps))
        if photometric == 2 and hv != (1, 1):
            raise Rejected("subsampled RGB (sampling %dx%d)" % hv)
    p, after = scan
    ns = p[0] if p else 0
    if ns != len(comps) or len(p) != 4 + 2 * ns:
        raise Rejected("a scan of %d components in a %d-component frame" % (ns, len(comps)))
    ss, se, a = p[1 + 2 * ns], p[2 + 2 * ns], p[3 + 2 * ns]
    if ss != 0 or se != 63 or a != 0:
        raise Rejected("a scan with Ss %d, Se %d, Ah/Al 0x%02X" % (ss, se, a))
    out = dict(width=frame["width"], height=frame["height"], h=hv[0], v=hv[1], restart=restart, quant=[], dc=[], ac=[])
    for i, (cid, _, _, tq) in enumerate(comps):
        if p[1 + 2 * i] != cid:
            raise Rejected("scan component %d is not frame component %d" % (p[1 + 2 * i], cid))
        td, ta = p[2 + 2 * i] >> 4, p[2 + 2 * i] & 15
        if tq not in q:
            raise Rejected("quantisation table %d is used but not defined" % tq)
        for key, name in (((0, td), "DC"), ((1, ta), "AC")):
            if key not in h:
                raise Rejected("%s Huffman table %d is used but not defined" % (name, key[1]))
        out["quant"].append(q[tq])
        out["dc"].append(h[(0, td)])
        out["ac"].append(h[(1, ta)])
    end = _end_of_entropy(s, after)
    if end < 0:
        raise Rejected("no EOI after the scan")
    if s[end + 1] != 0xD9:
        raise Rejected("marker 0x%02X after the scan (only one scan is supported)" % s[end + 1])
    out["start"], out["end"] = after, end
    return out


def geometry(hdr, spp):
    """(mcus_x, mcus_y, blocks per MCU) of a parsed header: one component is non-interleaved, one block per MCU"""
    if spp == 1:
        return -(-hdr["width"] // 8), -(-hdr["height"] // 8), 1
    return -(-hdr["width"] // (8 * hdr["h"])), -(-hdr["height"] // (8 * hdr["v"])), hdr["h"] * hdr["v"] + 2


# ---- entropy decode ----

def _split(data):
    """the entropy-coded bytes -> [(unstuffed bytes, number of the RST that ends them or None)]"""
    segs, cur, i, n = [], bytearray(), 0, len(data)
    while i < n:
        b = data[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        nxt = data[i + 1] if i + 1 < n else None
        if nxt == 0:
            cur.append(0xFF)
            i += 2
        elif nxt is None or nxt == 0xFF:
            i += 1  # fill byte
        else:
            segs.append((bytes(cur), nxt - 0xD0))
            cur = bytearray()
            i += 2
    segs.append((bytes(cur), None))
    return segs


class _Bits:
    def __init__(self, data):
        self.d = data + b"\0\0\0\0"
        self.n = len(data) * 8
        self.pos = 0

    def peek16(self):
        i = self.pos >> 3
        return ((self.d[i] << 16 | self.d[i + 1] << 8 | self.d[i + 2]) >> (8 - (self.pos & 7))) & 0xFFFF

    def take(self, n, mcu):
        if self.pos + n > self.n:
            raise DataError(TRUNCATED, mcu)
        v = self.peek16() >> (16 - n) if n else 0
        self.pos += n
        return v

    def huff(self, t, mcu):
        look = self.peek16()
        e = int(t["lookup"][look >> 8])
        l = e >> 8
        if l <= 8:
            self.take(l, mcu)
            return e & 0xFF
        while l <= 16 and (look >> (16 - l)) > t["maxcode"][l]:
            l += 1
        if l > 16:
            raise DataError(BAD_CODE, mcu)
        code = look >> (16 - l)
        self.take(l, mcu)
        return int(t["huffval"][code + t["valoffset"][l]])


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < 1 << (s - 1) else v


def coefficients(hdr, stream, spp):
    """int16 [spp] planes of blocks [by, bx, 64] (natural order) of one chunk, each component's blocks padded to whole MCUs"""
    mx, my, _ = geometry(hdr, spp)
    hs = [hdr["h"], 1, 1][:spp] if spp == 3 else [1]
    vs = [hdr["v"], 1, 1][:spp] if spp == 3 else [1]
    planes = [np.zeros((my * vs[c], mx * hs[c], 64), np.int16) for c in range(spp)]
    segs = _split(bytes(stream)[hdr["start"]:hdr["end"]])
    R = hdr["restart"]
    total = mx * my
    seg_i = 0
    bits = _Bits(segs[0][0])
    pred = [0] * spp
    for mcu in range(total):
        if R and mcu and mcu % R == 0:
            if bits.n - ((bits.pos + 7) & ~7) >= 8:
                raise DataError(EXTRANEOUS, mcu)
            number = segs[seg_i][1]
            if number is None:
                raise DataError(TRUNCATED, mcu)
            if number != (mcu // R - 1) & 7:
                raise DataError(BAD_MARKER, mcu)
            seg_i += 1
            bits = _Bits(segs[seg_i][0])
            pred = [0] * spp
        by0, bx0 = divmod(mcu, mx)
        for c in range(spp):
            for yy in range(vs[c]):
                for xx in range(hs[c]):
                    blk = planes[c][by0 * vs[c] + yy, bx0 * hs[c] + xx]
                    s = bits.huff(hdr["dc"][c], mcu)
                    pred[c] += _extend(bits.take(s, mcu), s)
                    blk[0] = np.int32(pred[c]).astype(np.int16)
                    k = 1
                    ac = hdr["ac"][c]
                    while k < 64:
                        rs = bits.huff(ac, mcu)
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            if k > 63:
                                raise DataError(AC_PAST_63, mcu)
                            blk[ZIGZAG[k]] = _extend(bits.take(s, mcu), s)
                            k += 1
                        elif r == 15:
                            k += 16
                        else:
                            break
    if bits.n - ((bits.pos + 7) & ~7) >= 8:
        raise DataError(EXTRANEOUS, total)
    if segs[seg_i][1] is not None:
        raise DataError(BAD_MARKER, total)
    return planes


# ---- islow IDCT ----

C = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069, c2053=16819,
         c2562=20995, c3072=25172)


def _descale(x, n):
    return (x + (np.int64(1) << np.int64(n - 1))) >> np.int64(n)


def _idct_1d(i0, i1, i2, i3, i4, i5, i6, i7):
    """the even and odd parts of jidctint.c on int64 arrays; returns the 8 undescaled outputs"""
    z1 = (i2 + i6) * C["c0541"]
    tmp2 = z1 + i6 * -C["c1847"]
    tmp3 = z1 + i2 * C["c0765"]
    tmp0 = (i0 + i4) << 13
    tmp1 = (i0 - i4) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = i7, i5, i3, i1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * C["c1175"]
    o0, o1, o2, o3 = o0 * C["c0298"], o1 * C["c2053"], o2 * C["c3072"], o3 * C["c1501"]
    z1, z2, z3, z4 = z1 * -C["c0899"], z2 * -C["c2562"], z3 * -C["c1961"] + z5, z4 * -C["c0390"] + z5
    o0 = o0 + z1 + z3
    o1 = o1 + z2 + z4
    o2 = o2 + z2 + z3
    o3 = o3 + z1 + z4
    return [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]


def idct_islow(blocks, quant):
    """int16 [..., 64] natural-order coefficients, quantisation table [64] -> uint8 [..., 8, 8] samples"""
    mult = np.asarray(quant, np.int64).astype(np.int16).astype(np.int64)  # ISLOW_MULT_TYPE is a short
    x = (blocks.astype(np.int64) * mult).reshape(blocks.shape[:-1] + (8, 8))  # [..., row u, column v]
    cols = _idct_1d(*[x[..., k, :] for k in range(8)])  # pass 1 down each column: output row k of every column
    ws = np.stack([_descale(c, 11) for c in cols], axis=-2)
    ws = ws.astype(np.int32).astype(np.int64)  # (int) DESCALE(...)
    rows = _idct_1d(*[ws[..., :, k] for k in range(8)])
    out = np.stack([_descale(r, 18) for r in rows], axis=-1)
    t = (out.astype(np.int32).astype(np.int64) + 512) & 1023  # range_limit[x & RANGE_MASK] of the post-IDCT table
    return np.clip(t - 384, 0, 255).astype(np.uint8)


def component_plane(blocks, quant):
    """[by, bx, 64] coefficient blocks -> uint8 [by * 8, bx * 8] samples"""
    by, bx = blocks.shape[:2]
    px = idct_islow(blocks, quant)  # [by, bx, 8, 8]
    return px.transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)


# ---- upsampling and colour ----

def upsample(c, wc, hc, h, v, W, H):
    """chroma plane (true size wc x hc) -> int32 [H, W] as jdsample.c's fancy h2v1 / h2v2 (replication when wc <= 2)"""
    c = c[:hc, :wc].astype(np.int32)
    if h == 1 and v == 1:
        return c[:H, :W]
    X = np.arange(W)
    Y = np.arange(H)
    ci, odd = X >> 1, X & 1
    if wc <= 2:
        return c[(Y >> (v - 1))[:, None], ci[None, :]]
    if v == 1:
        rows = c[Y]
        near = rows[:, ci]
        other = rows[:, np.clip(np.where(odd == 1, ci + 1, ci - 1), 0, wc - 1)]
        even = np.where(ci == 0, near, (3 * near + other + 1) >> 2)
        oddv = np.where(ci == wc - 1, near, (3 * near + other + 2) >> 2)
        return np.where(odd == 1, oddv, even)
    ri = Y >> 1
    r2 = np.clip(np.where(Y & 1, ri + 1, ri - 1), 0, hc - 1)
    colsum = 3 * c[ri] + c[r2]  # [H, wc]
    this = colsum[:, ci]
    other = colsum[:, np.clip(np.where(odd == 1, ci + 1, ci - 1), 0, wc - 1)]
    even = np.where(ci == 0, (this * 4 + 8) >> 4, (3 * this + other + 8) >> 4)
    oddv = np.where(ci == wc - 1, (this * 4 + 7) >> 4, (3 * this + other + 7) >> 4)
    return np.where(odd == 1, oddv, even)


def ycc_to_rgb(y, cb, cr):
    """jdcolor.c's ycc_rgb_convert on int arrays -> uint8 [..., 3]"""
    x = np.arange(256, dtype=np.int64) - 128
    cr_r = (91881 * x + 32768) >> 16
    cb_b = (116130 * x + 32768) >> 16
    cr_g = -46802 * x
    cb_g = -22554 * x + 32768
    y = y.astype(np.int64)
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> 16)
    b = y + cb_b[cb]
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def decode(stream, tables=(dict(), dict()), spp=3, photometric=6):
    """one chunk's stream -> uint8 [frame height, frame width, spp]"""
    hdr = parse(stream, tables, spp, photometric)
    return decode_parsed(hdr, stream, spp, photometric)


def decode_parsed(hdr, stream, spp, photometric):
    W, H = hdr["width"], hdr["height"]
    planes = [component_plane(b, hdr["quant"][c]) for c, b in enumerate(coefficients(hdr, stream, spp))]
    if spp == 1:
        return planes[0][:H, :W, None]
    y = planes[0][:H, :W]
    h, v = hdr["h"], hdr["v"]
    wc, hc = -(-W // h), -(-H // v)
    cb = upsample(planes[1], wc, hc, h, v, W, H)
    cr = upsample(planes[2], wc, hc, h, v, W, H)
    if photometric == 2:
        return np.stack([y, cb, cr], axis=-1).astype(np.uint8)
    return ycc_to_rgb(y, cb, cr)


# ---- whole files ----

def decode_file(raster, row0=0, rows=None, col0=0, cols=None):
    """a window of a JPEG GeoTiff (robosat_b200.geotiff.GeoTiff) decoded chunk by chunk here -> uint8 [rows, cols, spp]"""
    rows = raster.height - row0 if rows is None else rows
    cols = raster.width - col0 if cols is None else cols
    data = open(raster.path, "rb").read()
    tables = read_tables(raster.jpeg_tables)
    out = np.zeros((rows, cols, raster.spp), np.uint8)
    across = -(-raster.width // raster.chunk_w) if raster.tiled else 1
    for cr in range(row0 // raster.chunk_h, (row0 + rows - 1) // raster.chunk_h + 1):
        for cc in range(col0 // raster.chunk_w, (col0 + cols - 1) // raster.chunk_w + 1):
            k = cr * across + cc
            s = data[raster.offsets[k]:raster.offsets[k] + raster.byte_counts[k]]
            px = decode(s, tables, raster.spp, raster.photometric)
            y0, x0 = cr * raster.chunk_h, cc * raster.chunk_w
            ya, yb = max(row0, y0), min(row0 + rows, y0 + raster.chunk_h, raster.height)
            xa, xb = max(col0, x0), min(col0 + cols, x0 + raster.chunk_w, raster.width)
            out[ya - row0:yb - row0, xa - col0:xb - col0] = px[ya - y0:yb - y0, xa - x0:xb - x0]
    return out
