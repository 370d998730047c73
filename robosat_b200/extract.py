"""`rs extract` (robosat/tools/extract.py, robosat/osm/{core,parking,building}.py): parking-lot and building polygons from an
OpenStreetMap `.osm.pbf` file, with the DenseNodes decode, the node-location join and the ring validity check on the GPU.

The reference runs an osmium handler with node locations and keeps a way when `is_polygon` (first and last node ids equal,
>= 4 node refs), its tags pass the handler's rule and shapely finds the ring valid. This project defines the rule
(DESIGN.md §8, restated in tests/extract_reference.py):

- the file is framed, inflated and parsed on the host (`csrc/rsb_pbf.cpp`, no interpreter lock, one call per batch of blobs);
- pass 1 collects the ways that carry the handler's anchor tag (`amenity=parking` or `building`) with the values of the keys the
  rule reads, and notes the blobs that hold nodes; the tag rule and `is_polygon` run here, vectorised;
- the kept ways' refs, biased by flipping the sign bit so that negative ids sort too, are sorted and made unique on the device;
- pass 2 streams the node blobs: `rsb_pbf_dense_nodes` decodes DenseNodes, plain Nodes are decoded on the host, and
  `rsb_extract_locate` joins them to the unique refs (the later node of a repeated id wins);
- `rsb_extract_gather` builds every way's ring and flags a missing node or an invalid location; such a way is skipped with a
  warning (the reference stops with osmium's InvalidLocationError instead), and a summary count follows;
- `rsb_extract_valid` is `features.polygon_is_valid([ring])` on the integer 1e-7 degree lattice, exact; an invalid ring gets the
  reference's warning.

Coordinates are the doubles x / 1e7 and y / 1e7 of osmium's Location::lon() / lat(). osmium, shapely and geojson are not needed.
Device memory is bounded by `budget`.
"""

import os
import time

import numpy as np

from robosat_b200 import _lib
from robosat_b200.cover import _alloc

DEFAULT_BUDGET = 1 << 30
HOST_BATCH_BYTES = 256 << 20  # inflated bytes per host parse call
NODES_PER_BYTE = 1 / 3  # a DenseNodes node takes at least 3 bytes (id, lat, lon deltas), a plain Node more
NODE_RECORD_BYTES = 16  # id int64 + x, y int32
KEY_BYTES = 24  # per unique ref: the key, its best ordinal and its location
REF_BYTES = 28  # per ref of a way batch: biased id, way index, vertex, compacted vertex
WAY_BYTES = 17  # per way of a way batch: ring offset, flag, length, valid
PAIR_TILE = 64

W_INVALID = "Warning: invalid feature: https://www.openstreetmap.org/way/{}"
W_LOCATION = "Warning: way with a missing node or an invalid node location, skipping: https://www.openstreetmap.org/way/{}"
W_LOCATION_SUMMARY = "Warning: {} ways skipped for a missing node or an invalid node location"

PARKING_FILTER = {"underground", "sheds", "carports", "garage_boxes"}
BUILDING_FILTER = {"construction", "houseboat", "static_caravan", "stadium", "conservatory", "digester", "greenhouse", "ruins"}
LOCATION_FILTER = {"underground", "underwater"}

# kind -> (keys the rule reads, the first being the anchor; the anchor's required value or None)
QUERIES = {"parking": (("amenity", "parking"), "parking"), "building": (("building", "location"), None)}


def _threads():
    return max(1, min(32, os.cpu_count() or 1))


def _ptr(a):
    return a.ctypes.data_as(_lib.ctypes.c_void_p) if a is not None and a.size else None


def read_frames(data):
    """uint8 array of a whole file -> int64 [F, RSB_PBF_FRAME_FIELDS] frames (kind, compression, data offset, data length,
    raw_size, frame offset)"""
    lib = _lib.load()
    count = np.zeros(1, np.int64)
    cap = max(1, len(data) // 16)
    while True:
        frames = np.zeros((cap, _lib.RSB_PBF_FRAME_FIELDS), np.int64)
        _lib.check(lib.rsb_pbf_frames(_ptr(data), len(data), _ptr(frames), cap, _ptr(count)), "rsb_pbf_frames")
        if count[0] <= cap:
            return frames[: count[0]]
        cap = int(count[0])


def inflate(data, frames):
    """inflate the blobs of `frames` -> (buffer, offsets, sizes): blob i at buffer[offsets[i] : offsets[i] + sizes[i]]"""
    sizes = np.ascontiguousarray(frames[:, 4], dtype=np.int64)
    offsets = np.zeros(len(frames), np.int64)
    if len(frames):
        offsets[1:] = np.cumsum(sizes[:-1] + _lib.RSB_PBF_INFLATE_PAD)
    total = int(offsets[-1] + sizes[-1]) + _lib.RSB_PBF_INFLATE_PAD if len(frames) else 0
    buf = np.zeros(max(1, total), np.uint8)
    f = np.ascontiguousarray(frames, dtype=np.int64)
    _lib.check(_lib.load().rsb_pbf_inflate(_ptr(data), _ptr(f), len(frames), _ptr(buf), _ptr(offsets), _threads()), "rsb_pbf_inflate")
    return buf, offsets, sizes


def check_header(block):
    _lib.check(_lib.load().rsb_pbf_check_header(_ptr(block), len(block)), "rsb_pbf_check_header")


def parse(buf, offsets, sizes, mode, keys=(), anchor_value=None):
    """rsb_pbf_parse of the blocks buf[offsets[i] : offsets[i] + sizes[i]] -> dict of its outputs (names of RSB_PBF_OUT_*)"""
    lib = _lib.load()
    handle = _lib.ctypes.c_void_p()
    kb = b"".join(k.encode() + b"\0" for k in keys)
    av = anchor_value.encode() if anchor_value else None
    offsets = np.ascontiguousarray(offsets, np.int64)
    sizes = np.ascontiguousarray(sizes, np.int64)
    _lib.check(lib.rsb_pbf_parse(_ptr(buf), _ptr(offsets), _ptr(sizes), len(offsets), mode, kb or None, len(keys), av, _threads(),
                                 _lib.ctypes.byref(handle)), "rsb_pbf_parse")
    try:
        counts = np.zeros(_lib.RSB_PBF_OUT_COUNT, np.int64)
        _lib.check(lib.rsb_pbf_result_sizes(handle, _ptr(counts)), "rsb_pbf_result_sizes")
        out = {}
        for name, what, dtype in (("kinds", _lib.RSB_PBF_OUT_KINDS, np.int32), ("way_ids", _lib.RSB_PBF_OUT_WAY_IDS, np.int64),
                                  ("ref_offsets", _lib.RSB_PBF_OUT_REF_OFFSETS, np.int64), ("refs", _lib.RSB_PBF_OUT_REFS, np.int64),
                                  ("tags", _lib.RSB_PBF_OUT_TAGS, np.int32), ("string_offsets", _lib.RSB_PBF_OUT_STRING_OFFSETS, np.int64),
                                  ("string_bytes", _lib.RSB_PBF_OUT_STRING_BYTES, np.uint8), ("segs", _lib.RSB_PBF_OUT_SEGS, np.int64),
                                  ("host_ids", _lib.RSB_PBF_OUT_HOST_IDS, np.int64), ("host_xy", _lib.RSB_PBF_OUT_HOST_XY, np.int32)):
            a = np.zeros(int(counts[what]), dtype)
            _lib.check(lib.rsb_pbf_result_copy(handle, what, _ptr(a), a.size), "rsb_pbf_result_copy")
            out[name] = a
    finally:
        lib.rsb_pbf_result_free(handle)
    out["tags"] = out["tags"].reshape(-1, max(1, len(keys))) if keys else out["tags"].reshape(0, 0)
    out["segs"] = out["segs"].reshape(-1, _lib.RSB_PBF_SEG_FIELDS)
    out["host_xy"] = out["host_xy"].reshape(-1, 2)
    sb, so = out["string_bytes"].tobytes(), out["string_offsets"]
    out["strings"] = [sb[so[i]: so[i + 1]].decode("utf-8", "replace") for i in range(len(so) - 1)]
    return out


def _in(tags, col, strings, values):
    """per way: the value of key `col` exists and is one of `values`"""
    hit = np.array([s in values for s in strings] + [False], dtype=bool)  # index -1 (absent) -> False
    return hit[tags[:, col]]


def select(kind, parsed):
    """the handler's rule on one parse result: is_polygon and the tag filters -> boolean mask over its ways"""
    offs, refs, tags, strings = parsed["ref_offsets"], parsed["refs"], parsed["tags"], parsed["strings"]
    n = offs[1:] - offs[:-1]
    closed = np.zeros(len(n), bool)
    big = n >= 4
    closed[big] = refs[offs[:-1][big]] == refs[offs[1:][big] - 1]
    if kind == "parking":  # amenity=parking is the anchor
        return closed & ~_in(tags, 1, strings, PARKING_FILTER)
    return closed & ~_in(tags, 0, strings, BUILDING_FILTER) & ~_in(tags, 1, strings, LOCATION_FILTER)


def _batches(sizes, limit):
    """consecutive index ranges whose sizes add up to at most `limit` (a single larger item goes alone)"""
    out, start, acc = [], 0, 0
    for i, s in enumerate(sizes):
        if i > start and acc + s > limit:
            out.append((start, i))
            start, acc = i, 0
        acc += s
    if start < len(sizes):
        out.append((start, len(sizes)))
    return out


class _Clock:
    def __init__(self, stats, sync):
        self.stats, self.sync = stats, sync

    def __call__(self, name, t0):
        if self.stats is None:
            return time.perf_counter()
        if self.sync:
            import torch

            torch.cuda.synchronize()
        t1 = time.perf_counter()
        self.stats[name] = self.stats.get(name, 0.0) + (t1 - t0)
        return t1


def extract_device(path, kind, budget=DEFAULT_BUDGET, device=None, stats=None):
    """Features of `kind` ("parking" or "building") in the PBF file `path` -> (features, warnings): GeoJSON Feature dicts in way
    order and the warning lines, in order. `budget` bounds the device bytes; `stats` (a dict), when given, receives per-stage
    seconds and counts."""
    import torch

    if kind not in QUERIES:
        raise ValueError("unknown feature type %r (parking or building)" % (kind,))
    _lib.require_device()
    dev = torch.device(device if device is not None else "cuda")
    lib = _lib.load()
    stream = _lib.current_stream_ptr
    clock = _Clock(stats, True)
    keys, anchor = QUERIES[kind]

    t = time.perf_counter()
    data = np.fromfile(path, dtype=np.uint8) if os.path.getsize(path) < 16 else np.memmap(path, dtype=np.uint8, mode="r")
    frames = read_frames(data)
    headers = frames[frames[:, 0] == _lib.RSB_PBF_BLOB_HEADER]
    if len(headers):
        buf, offs, sizes = inflate(data, headers)
        for o, s in zip(offs, sizes):
            check_header(buf[o: o + s])
    blocks = frames[frames[:, 0] == _lib.RSB_PBF_BLOB_DATA]

    # pass 1: the ways, and which blocks hold nodes
    way_ids, ref_counts, refs, node_blocks = [], [], [], []
    for a, b in _batches(blocks[:, 4], HOST_BATCH_BYTES):
        buf, offs, sizes = inflate(data, blocks[a:b])
        p = parse(buf, offs, sizes, _lib.RSB_PBF_WAYS, keys, anchor)
        node_blocks.extend(a + np.flatnonzero(p["kinds"] & (_lib.RSB_PBF_HAS_NODES | _lib.RSB_PBF_HAS_DENSE)))
        keep = select(kind, p)
        ro = p["ref_offsets"]
        way_ids.append(p["way_ids"][keep])
        ref_counts.append((ro[1:] - ro[:-1])[keep])
        refs.append(np.concatenate([p["refs"][ro[i]: ro[i + 1]] for i in np.flatnonzero(keep)]) if keep.any() else np.zeros(0, np.int64))
    t = clock("read_ways_s", t)
    way_ids = np.concatenate(way_ids) if way_ids else np.zeros(0, np.int64)
    ref_counts = np.concatenate(ref_counts) if ref_counts else np.zeros(0, np.int64)
    refs = np.concatenate(refs) if refs else np.zeros(0, np.int64)
    if stats is not None:
        stats.update(ways=len(way_ids), refs=len(refs), blocks=len(blocks), node_blocks=len(node_blocks))
    if len(way_ids) == 0:
        return [], []
    ref_offsets = np.zeros(len(way_ids) + 1, np.int64)
    ref_offsets[1:] = np.cumsum(ref_counts)
    biased = (refs.view(np.uint64) ^ np.uint64(1 << 63)).view(np.int64)

    # the unique refs and their locations must fit before anything is allocated (the ref count bounds the unique count)
    nrefs = len(refs)
    fixed = nrefs * (8 + KEY_BYTES) + int(lib.rsb_sort_unique_workspace_bytes(nrefs))
    if fixed > budget:
        raise _lib.RsbError("the %d node refs of %d ways need %d bytes of device memory for their unique ids and locations, more than the "
                            "budget of %d bytes" % (nrefs, len(way_ids), fixed, budget))
    keys_dev = _alloc((nrefs,), torch.int64, dev, "the ways' node refs")
    keys_dev.copy_(torch.from_numpy(biased))
    ws = _alloc((max(1, lib.rsb_sort_unique_workspace_bytes(nrefs)),), torch.uint8, dev, "the node ref sort workspace")
    count = torch.zeros((1,), dtype=torch.int64, device=dev)
    _lib.check(lib.rsb_sort_unique_u64(keys_dev.data_ptr(), nrefs, 64, ws.data_ptr(), ws.numel(), count.data_ptr(), stream()), "rsb_sort_unique_u64")
    del ws
    nu = int(count.item())
    keys_dev = keys_dev[:nu].clone()
    best = torch.zeros((nu,), dtype=torch.int64, device=dev)
    loc = torch.zeros((nu, 2), dtype=torch.int32, device=dev)
    t = clock("sort_s", t)

    # pass 2: stream the node blocks through the decode and the locate step
    room = budget - nu * KEY_BYTES
    per_byte = 1 + NODES_PER_BYTE * NODE_RECORD_BYTES
    ordinal = 0
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    nb = blocks[np.asarray(node_blocks, dtype=np.int64)] if node_blocks else blocks[:0]
    for a, b in _batches(nb[:, 4] + _lib.RSB_PBF_INFLATE_PAD, int(room / per_byte)):
        raw = int((nb[a:b, 4] + _lib.RSB_PBF_INFLATE_PAD).sum())
        if raw * per_byte > room:
            raise _lib.RsbError("a node blob of %d bytes needs about %d bytes of device memory, more than the %d bytes the budget leaves"
                                % (raw, int(raw * per_byte), room))
        buf, offs, sizes = inflate(data, nb[a:b])
        p = parse(buf, offs, sizes, _lib.RSB_PBF_NODES)
        segs = p["segs"]
        counts = segs[:, _lib.RSB_PBF_SEG_COUNT]
        segs[:, _lib.RSB_PBF_SEG_OUT_FIRST] = np.cumsum(counts) - counts
        n = int(counts.sum())
        t = clock("read_nodes_s", t)
        if n == 0:
            continue
        ids = _alloc((n,), torch.int64, dev, "a node chunk's ids")
        xy = _alloc((n, 2), torch.int32, dev, "a node chunk's locations")
        dense = segs[:, _lib.RSB_PBF_SEG_KIND] == 0
        if dense.any():
            blk = _alloc((len(buf),), torch.uint8, dev, "a node chunk's blocks")
            blk.copy_(torch.from_numpy(buf))
            offs_dev = torch.from_numpy(offs).to(dev)
            segs_dev = torch.from_numpy(np.ascontiguousarray(segs[dense])).to(dev)
            _lib.check(lib.rsb_pbf_dense_nodes(blk.data_ptr(), offs_dev.data_ptr(), segs_dev.data_ptr(), int(dense.sum()), ids.data_ptr(), xy.data_ptr(),
                                               status.data_ptr(), stream()), "rsb_pbf_dense_nodes")
            if int(status.item()) != 0:
                raise _lib.RsbError("pbf: a DenseNodes group is malformed (a varint longer than 10 bytes or a wrong number of values)")
        for s in segs[~dense]:
            o, c, h = s[_lib.RSB_PBF_SEG_OUT_FIRST], s[_lib.RSB_PBF_SEG_COUNT], s[_lib.RSB_PBF_SEG_HOST_FIRST]
            ids[o: o + c].copy_(torch.from_numpy(p["host_ids"][h: h + c]))
            xy[o: o + c].copy_(torch.from_numpy(p["host_xy"][h: h + c]))
        t = clock("decode_s", t)
        _lib.check(lib.rsb_extract_locate(ids.data_ptr(), xy.data_ptr(), n, ordinal, keys_dev.data_ptr(), nu, best.data_ptr(), loc.data_ptr(), stream()),
                   "rsb_extract_locate")
        ordinal += n
        del ids, xy
        t = clock("locate_s", t)
    if stats is not None:
        stats.update(nodes=ordinal, unique_refs=nu)

    # rings: gather, validity, in way batches under what the budget leaves
    features, warnings, skipped = [], [], 0
    counts = ref_counts
    way_cost = counts * REF_BYTES + WAY_BYTES
    for a, b in _batches(way_cost, room):
        if int(way_cost[a:b].sum()) > room:
            raise _lib.RsbError("way %d with %d refs needs %d bytes of device memory, more than the %d bytes the budget leaves"
                                % (way_ids[a], counts[a], int(way_cost[a]), room))
        r0, r1 = ref_offsets[a], ref_offsets[b]
        R = b - a
        offs = ref_offsets[a: b + 1] - r0
        ref_way = np.repeat(np.arange(R, dtype=np.int32), counts[a:b])
        refs_dev = torch.from_numpy(biased[r0:r1]).to(dev)
        ref_way_dev = torch.from_numpy(ref_way).to(dev)
        verts = _alloc((max(1, r1 - r0), 2), torch.int32, dev, "the ways' vertices")
        flags = _alloc((R,), torch.int32, dev, "the ways' flags")
        _lib.check(lib.rsb_extract_gather(refs_dev.data_ptr(), ref_way_dev.data_ptr(), r1 - r0, R, keys_dev.data_ptr(), nu, best.data_ptr(), loc.data_ptr(),
                                          verts.data_ptr(), flags.data_ptr(), stream()), "rsb_extract_gather")
        t = clock("gather_s", t)
        valid, _ = valid_rings(verts, offs, flags)
        t = clock("valid_s", t)
        fl, ok, v = flags.cpu().numpy(), valid.cpu().numpy(), verts.cpu().numpy()
        lonlat = v.astype(np.float64) / 1e7
        for k in range(R):
            wid = int(way_ids[a + k])
            if fl[k]:
                warnings.append(W_LOCATION.format(wid))
                skipped += 1
            elif not ok[k]:
                warnings.append(W_INVALID.format(wid))
            else:
                ring = lonlat[offs[k]: offs[k + 1]].tolist()
                features.append({"type": "Feature", "geometry": {"type": "Polygon", "coordinates": [ring]}, "properties": {}})
        t = clock("features_s", t)
    if skipped:
        warnings.append(W_LOCATION_SUMMARY.format(skipped))
    if stats is not None:
        stats.update(features=len(features), invalid=len(warnings) - skipped - (1 if skipped else 0), skipped=skipped)
    return features, warnings


def valid_rings(verts, ring_offsets, flags=None):
    """rsb_extract_valid on device int32 vertices [n, 2] of closed rings (ring r at ring_offsets[r] .. ring_offsets[r + 1], numpy)
    -> (valid uint8 [R], compacted lengths int32 [R]) as device tensors. flags (device int32 [R]) != 0 skips a ring."""
    import torch

    dev = verts.device
    lib = _lib.load()
    R = len(ring_offsets) - 1
    n = ring_offsets[1:] - ring_offsets[:-1]
    if flags is None:
        flags = torch.zeros((max(1, R),), dtype=torch.int32, device=dev)
    long_rings = np.flatnonzero(n > _lib.RSB_EXTRACT_WARP_RING).astype(np.int32)
    nbl = (n[long_rings] + PAIR_TILE - 1) // PAIR_TILE
    tile_offsets = np.zeros(len(long_rings) + 1, np.int64)
    tile_offsets[1:] = np.cumsum(nbl * nbl)
    offs_dev = torch.from_numpy(np.ascontiguousarray(ring_offsets, np.int64)).to(dev)
    long_dev = torch.from_numpy(long_rings).to(dev) if len(long_rings) else None
    tiles_dev = torch.from_numpy(tile_offsets).to(dev)
    scratch = _alloc(tuple(verts.shape), torch.int32, dev, "the compacted rings")
    lens = _alloc((max(1, R),), torch.int32, dev, "the ring lengths")
    valid = _alloc((max(1, R),), torch.uint8, dev, "the validity flags")
    _lib.check(lib.rsb_extract_valid(verts.data_ptr(), offs_dev.data_ptr(), R, flags.data_ptr(), long_dev.data_ptr() if long_dev is not None else None,
                                     len(long_rings), tiles_dev.data_ptr(), scratch.data_ptr(), lens.data_ptr(), valid.data_ptr(), _lib.current_stream_ptr()),
               "rsb_extract_valid")
    return valid[:R], lens[:R]


def extract(path, kind):
    """drop-in for the reference's handler run: (features, warnings) of `kind` in `path` with the default budget on the current device"""
    return extract_device(path, kind)
