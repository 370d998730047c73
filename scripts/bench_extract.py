"""Benchmark of `rs extract` on a seeded synthetic PBF: about 2e7 nodes in DenseNodes blocks of 8000 and 2e6 closed ways, of
which about 10 % are tagged buildings or parking lots. The file is written with numpy-vectorised varint encoding into a
temporary directory; per-stage seconds go to results/h100_extract.json (or --out).

    python scripts/bench_extract.py [--nodes 20000000] [--ways 2000000] [--out results/h100_extract.json]
"""

import argparse
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def varints(v):
    """uint64 array -> (concatenated LEB128 bytes, per-value lengths)"""
    v = np.asarray(v, dtype=np.uint64)
    lens = np.ones(len(v), np.int64)
    for k in range(1, 10):
        lens += (v >> np.uint64(7 * k)) != 0
    offs = np.cumsum(lens) - lens
    out = np.zeros(int(lens.sum()), np.uint8)
    for k in range(10):
        m = lens > k
        b = ((v[m] >> np.uint64(7 * k)) & np.uint64(0x7F)).astype(np.uint8) | np.where(lens[m] > k + 1, 0x80, 0).astype(np.uint8)
        out[offs[m] + k] = b
    return out, lens


def zz(d):
    d = np.asarray(d, dtype=np.int64)
    return ((d << 1) ^ (d >> 63)).view(np.uint64)


def vb(x):
    """one non-negative varint (pure Python: numpy's per-call overhead dominates for single values)"""
    out = bytearray()
    while x > 0x7F:
        out.append((x & 0x7F) | 0x80)
        x >>= 7
    out.append(x)
    return bytes(out)


def fbytes(num, b):
    return vb((num << 3) | 2) + vb(len(b)) + b


def frame(kind, data):
    blob = vb((2 << 3) | 0) + vb(len(data)) + fbytes(3, zlib.compress(data, 6))
    hdr = fbytes(1, kind) + vb(3 << 3) + vb(len(blob))
    return struct.pack(">I", len(hdr)) + hdr + blob


def packed_deltas(num, values):
    b, _ = varints(zz(np.diff(np.asarray(values, np.int64), prepend=0)))
    return fbytes(num, b.tobytes())


def write_pbf(path, n_nodes, n_ways, seed=0, per_block=8000):
    rng = np.random.RandomState(seed)
    ids = np.cumsum(rng.randint(1, 4, n_nodes)).astype(np.int64)
    side = int(np.sqrt(n_nodes)) + 1
    gx, gy = np.arange(n_nodes) % side, np.arange(n_nodes) // side
    lon = 133000000 + gx * 200 + rng.randint(0, 50, n_nodes)   # raw units at granularity 100: 1e-7 degrees
    lat = 520000000 + gy * 200 + rng.randint(0, 50, n_nodes)
    with open(path, "wb") as fp:
        fp.write(frame(b"OSMHeader", fbytes(4, b"OsmSchema-V0.6") + fbytes(4, b"DenseNodes")))
        st = fbytes(1, b"".join(fbytes(1, s) for s in (b"", b"building", b"yes", b"amenity", b"parking", b"highway", b"residential")))
        for a in range(0, n_nodes, per_block):
            s = slice(a, a + per_block)
            dense = packed_deltas(1, ids[s]) + packed_deltas(8, lat[s]) + packed_deltas(9, lon[s])
            fp.write(frame(b"OSMData", st + fbytes(2, fbytes(2, dense))))
            if a % (250 * per_block) == 0:
                print("nodes written: %d" % a, flush=True)
        # ways: a cell of the node grid (4 corners, closed); 5 % buildings, 5 % parking, the rest highways
        c = rng.randint(0, n_nodes - side - 2, n_ways)
        corners = np.stack([c, c + 1, c + side + 1, c + side, c], axis=1)
        refs = ids[corners]
        kind = rng.rand(n_ways)
        kv = np.where(kind < 0.05, 0, np.where(kind < 0.10, 1, 2))
        keys = [(b"\x12\x01\x01\x1a\x01\x02"), (b"\x12\x01\x03\x1a\x01\x04"), (b"\x12\x01\x05\x1a\x01\x06")]
        rb, rl = varints(zz(np.diff(refs, axis=1, prepend=0).reshape(-1)))
        ro = np.concatenate([[0], np.cumsum(rl.reshape(-1, 5).sum(1))])
        rbytes = rb.tobytes()
        for a in range(0, n_ways, per_block):
            parts = []
            for w in range(a, min(n_ways, a + per_block)):
                r = rbytes[ro[w]: ro[w + 1]]
                body = vb(8) + vb(w + 1) + keys[kv[w]] + b"\x42" + vb(len(r)) + r
                parts.append(b"\x1a" + vb(len(body)) + body)
            fp.write(frame(b"OSMData", st + fbytes(2, b"".join(parts))))
    return int((kv == 0).sum()), int((kv == 1).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=20000000)
    ap.add_argument("--ways", type=int, default=2000000)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_extract.json"))
    args = ap.parse_args()

    import torch

    from robosat_b200.tools import extract as tool

    tmp = tempfile.mkdtemp(prefix="bench_extract_")
    try:
        path = os.path.join(tmp, "synthetic.osm.pbf")
        t0 = time.perf_counter()
        buildings, parking = write_pbf(path, args.nodes, args.ways)
        write_s = time.perf_counter() - t0
        print("wrote %s: %d bytes in %.1f s" % (path, os.path.getsize(path), write_s), flush=True)
        gpu = torch.cuda.get_device_name(0)
        smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
        runs = {}
        for kind in ("building", "parking", "building"):  # the first run warms up the modules and the page cache
            stats = {}
            t0 = time.perf_counter()
            tool.main(argparse.Namespace(type=kind, batch=100000, map=path, out=os.path.join(tmp, kind + ".geojson")), stats=stats)
            torch.cuda.synchronize()
            stats["total_s"] = time.perf_counter() - t0
            runs[kind] = stats
            print(kind, json.dumps(stats), flush=True)
        result = {
            "gpu": gpu, "power_limit_and_max_sm_clock": smi, "nodes": args.nodes, "ways": args.ways, "tagged_buildings": buildings,
            "tagged_parking": parking, "file_bytes": os.path.getsize(path), "write_synthetic_s": write_s, "runs": runs,
            "stages": "read_ways_s: pass-1 host read + inflate + way decode + rule; sort_s: unique refs on the device; read_nodes_s: pass-2 host "
                      "inflate + parse of node blobs; decode_s: upload + rsb_pbf_dense_nodes; locate_s; gather_s; valid_s; features_s: copies "
                      "back and feature dicts; write_s: JSON files",
        }
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fp:
            json.dump(result, fp, indent=1)
        print(json.dumps(result))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
