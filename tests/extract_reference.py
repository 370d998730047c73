"""Pure-Python restatement of `rs extract` (DESIGN.md §8), independent of robosat_b200/extract.py's device path:

- a PBF writer with hand-written protobuf encoding (raw or zlib blobs, several blocks, DenseNodes and plain Nodes, any
  granularity and offsets, negative ids, packed or unpacked repeated fields, and knobs to produce every format error);
- a reader plus the handlers' rules (robosat/osm/{core,parking,building}.py), with `features.polygon_is_valid` as the validity
  test, giving the expected features and warnings.
"""

import json
import struct
import zlib

from robosat_b200.features import polygon_is_valid

W_INVALID = "Warning: invalid feature: https://www.openstreetmap.org/way/{}"
W_LOCATION = "Warning: way with a missing node or an invalid node location, skipping: https://www.openstreetmap.org/way/{}"
W_LOCATION_SUMMARY = "Warning: {} ways skipped for a missing node or an invalid node location"

# --- protobuf encoding -------------------------------------------------------------------------------------------------------


def varint(v):
    """unsigned LEB128 of v; negative v is its 64-bit two's complement (10 bytes)"""
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def zigzag(v):
    return ((v << 1) ^ (v >> 63)) & ((1 << 64) - 1)


def unzigzag(u):
    return (u >> 1) ^ -(u & 1)


def key(num, wt):
    return varint((num << 3) | wt)


def f_varint(num, v):
    return key(num, 0) + varint(v)


def f_bytes(num, b):
    return key(num, 2) + varint(len(b)) + b


def f_repeated(num, values, packed=True):
    """a repeated varint field, packed into one length-delimited field or one field per value"""
    if packed:
        return f_bytes(num, b"".join(varint(v) for v in values)) if values else b""
    return b"".join(f_varint(num, v) for v in values)


def deltas(values):
    out, prev = [], 0
    for v in values:
        out.append(v - prev)
        prev = v
    return out


# --- writer ------------------------------------------------------------------------------------------------------------------


def header_block(required=("OsmSchema-V0.6", "DenseNodes")):
    return b"".join(f_bytes(4, r.encode()) for r in required) + f_bytes(16, b"extract_reference")


def dense_group(nodes, packed=True):
    """nodes [(id, lat, lon)] in raw stored units -> a PrimitiveGroup with one DenseNodes"""
    ids, lats, lons = zip(*nodes) if nodes else ((), (), ())
    body = (f_repeated(1, [zigzag(d) for d in deltas(ids)], packed) + f_repeated(8, [zigzag(d) for d in deltas(lats)], packed)
            + f_repeated(9, [zigzag(d) for d in deltas(lons)], packed))
    return f_bytes(2, body)


def node_group(nodes, strings):
    """plain Node messages"""
    return b"".join(f_bytes(1, f_varint(1, zigzag(i)) + f_varint(8, zigzag(la)) + f_varint(9, zigzag(lo))) for i, la, lo in nodes)


def way_group(ways, strings, packed=True):
    """ways [(id, refs, {key: value})]; strings: the block's string table (a list, extended here)"""
    out = b""
    for wid, refs, tags in ways:
        ks, vs = [], []
        for k, v in tags.items():
            for s in (k, v):
                if s not in strings:
                    strings.append(s)
            ks.append(strings.index(k))
            vs.append(strings.index(v))
        body = f_varint(1, wid) + f_repeated(2, ks, packed) + f_repeated(3, vs, packed) + f_repeated(8, [zigzag(d) for d in deltas(refs)], packed)
        out += f_bytes(3, body)
    return out


def primitive_block(groups, strings, granularity=100, lat_offset=0, lon_offset=0):
    st = f_bytes(1, b"".join(f_bytes(1, s.encode()) for s in strings))
    body = st + b"".join(f_bytes(2, g) for g in groups)
    if granularity != 100:
        body += f_varint(17, granularity)
    if lat_offset:
        body += f_varint(19, lat_offset)
    if lon_offset:
        body += f_varint(20, lon_offset)
    return body


def blob(data, compression="zlib", raw_size=None):
    """a Blob message; compression 'raw', 'zlib', or a field name ('lzma', 'lz4', 'zstd', 'bzip2') holding the bytes as is"""
    if compression == "raw":
        return f_bytes(1, data)
    fields = {"zlib": 3, "lzma": 4, "bzip2": 5, "lz4": 6, "zstd": 7}
    payload = zlib.compress(data) if compression == "zlib" else data
    return f_varint(2, len(data) if raw_size is None else raw_size) + f_bytes(fields[compression], payload)


def frame(kind, blob_bytes, datasize=None):
    hdr = f_bytes(1, kind.encode()) + f_varint(3, len(blob_bytes) if datasize is None else datasize)
    return struct.pack(">I", len(hdr)) + hdr + blob_bytes


class Writer:
    """Blocks of nodes and ways in file order. Each `block(...)` call adds one OSMData blob."""

    def __init__(self, compression="zlib", required=("OsmSchema-V0.6", "DenseNodes")):
        self.compression = compression
        self.frames = [frame("OSMHeader", blob(header_block(required), compression))]

    def block(self, dense=(), nodes=(), ways=(), granularity=100, lat_offset=0, lon_offset=0, packed=True, compression=None, dense_groups=None):
        """dense / nodes: [(id, lat, lon)] raw stored units; ways: [(id, refs, tags)]. dense_groups: explicit list of dense lists."""
        strings = [""]
        groups = []
        for g in (dense_groups if dense_groups is not None else ([list(dense)] if dense else [])):
            groups.append(dense_group(g, packed))
        if nodes:
            groups.append(node_group(nodes, strings))
        if ways:
            groups.append(way_group(ways, strings, packed))
        data = primitive_block(groups, strings, granularity, lat_offset, lon_offset)
        self.frames.append(frame("OSMData", blob(data, compression or self.compression)))
        return self

    def bytes(self):
        return b"".join(self.frames)

    def write(self, path):
        with open(path, "wb") as fp:
            fp.write(self.bytes())
        return path


def raw_coord(fixed, granularity=100, offset=0):
    """the stored value that decodes to `fixed` 1e-7 degree units (granularity must divide 100 * fixed - offset)"""
    num = 100 * fixed - offset
    assert num % granularity == 0
    return num // granularity


# --- reader ------------------------------------------------------------------------------------------------------------------


class FormatError(ValueError):
    pass


def read_varint(b, i):
    v, s = 0, 0
    while True:
        if i >= len(b) or s >= 70:
            raise FormatError("bad varint")
        c = b[i]
        i += 1
        v |= (c & 0x7F) << s
        s += 7
        if not c & 0x80:
            return v & ((1 << 64) - 1), i


def fields(b):
    """[(num, wire type, value)] of a message; length-delimited values are bytes"""
    out, i = [], 0
    while i < len(b):
        k, i = read_varint(b, i)
        num, wt = k >> 3, k & 7
        if wt == 0:
            v, i = read_varint(b, i)
        elif wt == 2:
            n, i = read_varint(b, i)
            v = b[i: i + n]
            if len(v) != n:
                raise FormatError("truncated field")
            i += n
        elif wt == 1:
            v, i = b[i: i + 8], i + 8
        elif wt == 5:
            v, i = b[i: i + 4], i + 4
        else:
            raise FormatError("bad wire type")
        out.append((num, wt, v))
    return out


def repeated(fs, num):
    """values of repeated varint field `num`, packed or not"""
    out = []
    for n, wt, v in fs:
        if n != num:
            continue
        if wt == 0:
            out.append(v)
        else:
            i = 0
            while i < len(v):
                x, i = read_varint(v, i)
                out.append(x)
    return out


def to_fixed(v, granularity, offset):
    """libosmium: (offset + granularity * v) / 100 as int64 division truncating toward zero"""
    n = offset + granularity * v
    q = abs(n) // 100
    return q if n >= 0 else -q


def valid_location(x, y):
    return -1800000000 <= x <= 1800000000 and -900000000 <= y <= 900000000


def signed64(v):
    return v - (1 << 64) if v >= 1 << 63 else v


def read(data):
    """PBF bytes -> (nodes [(id, x, y)] in file order, ways [(id, refs, tags dict)] in file order)"""
    nodes, ways, i = [], [], 0
    while i < len(data):
        (hl,) = struct.unpack(">I", data[i: i + 4])
        hdr = dict((n, v) for n, _, v in fields(data[i + 4: i + 4 + hl]))
        size = hdr[3]
        b = dict((n, v) for n, _, v in fields(data[i + 4 + hl: i + 4 + hl + size]))
        i += 4 + hl + size
        raw = b[1] if 1 in b else zlib.decompress(b[3])
        if hdr[1] == b"OSMHeader":
            continue
        block = fields(raw)
        strings = [s for n, _, s in fields(next((v for n, _, v in block if n == 1), b"")) if n == 1]
        gran = next((v for n, _, v in block if n == 17), 100)
        lat_off = signed64(next((v for n, _, v in block if n == 19), 0))
        lon_off = signed64(next((v for n, _, v in block if n == 20), 0))
        for n, _, g in block:
            if n != 2:
                continue
            for gn, _, el in fields(g):
                f = fields(el)
                if gn == 1:
                    d = {n2: v for n2, _, v in f}
                    nodes.append((unzigzag(d.get(1, 0)), to_fixed(unzigzag(d.get(9, 0)), gran, lon_off), to_fixed(unzigzag(d.get(8, 0)), gran, lat_off)))
                elif gn == 2:
                    ids, lats, lons = (repeated(f, k) for k in (1, 8, 9))
                    idv = latv = lonv = 0
                    for a, la, lo in zip(ids, lats, lons):
                        idv += unzigzag(a)
                        latv += unzigzag(la)
                        lonv += unzigzag(lo)
                        nodes.append((idv, to_fixed(lonv, gran, lon_off), to_fixed(latv, gran, lat_off)))
                elif gn == 3:
                    wid = signed64(next(v for n2, _, v in f if n2 == 1))
                    ks, vs = repeated(f, 2), repeated(f, 3)
                    tags = {}
                    for k, v in zip(ks, vs):
                        tags.setdefault(strings[k].decode(), strings[v].decode())
                    ref, refs = 0, []
                    for d in repeated(f, 8):
                        ref += unzigzag(d)
                        refs.append(ref)
                    ways.append((wid, refs, tags))
    return nodes, ways


# --- the handlers --------------------------------------------------------------------------------------------------------------

PARKING_FILTER = {"underground", "sheds", "carports", "garage_boxes"}
BUILDING_FILTER = {"construction", "houseboat", "static_caravan", "stadium", "conservatory", "digester", "greenhouse", "ruins"}
LOCATION_FILTER = {"underground", "underwater"}


def is_polygon(refs):
    return len(refs) >= 4 and refs[0] == refs[-1]


def wanted(kind, tags):
    if kind == "parking":
        return tags.get("amenity") == "parking" and tags.get("parking") not in PARKING_FILTER
    return "building" in tags and tags["building"] not in BUILDING_FILTER and tags.get("location") not in LOCATION_FILTER


def expected(data, kind):
    """-> (features, warnings) of the rule on PBF bytes"""
    nodes, ways = read(data)
    loc = {}
    for nid, x, y in nodes:
        loc[nid] = (x, y)  # the later node wins
    features, warnings, skipped = [], [], 0
    for wid, refs, tags in ways:
        if not is_polygon(refs) or not wanted(kind, tags):
            continue
        pts = [loc.get(r) for r in refs]
        if any(p is None or not valid_location(*p) for p in pts):
            warnings.append(W_LOCATION.format(wid))
            skipped += 1
            continue
        if not polygon_is_valid([pts]):
            warnings.append(W_INVALID.format(wid))
            continue
        features.append({"type": "Feature", "geometry": {"type": "Polygon", "coordinates": [[[x / 1e7, y / 1e7] for x, y in pts]]}, "properties": {}})
    if skipped:
        warnings.append(W_LOCATION_SUMMARY.format(skipped))
    return features, warnings


def dumps(features):
    return json.dumps({"type": "FeatureCollection", "features": features})
