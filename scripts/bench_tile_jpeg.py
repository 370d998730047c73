"""The JPEG decoder of `rs tile` and `rs segment` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_tile_jpeg.py --part kernel --out results/h100_tile_jpeg_kernel.json [--launches 50]
    python scripts/bench_tile_jpeg.py --part e2e --out results/h100_tile_jpeg.json [--size 20000]

Records, with the card's name and power limit read in the same run:
1. (kernel) rsb_jpeg_decode_window on windows of 64, 256 and 1 024 chunks of 256² and 512², at 4:2:0 and 4:4:4, quality 75 and 90,
   with and without restart markers (every 8 MCUs), over 16 distinct PIL-encoded streams with the standard Huffman tables repeated
   across the window; and GDAL-style windows of 64, 256 and 1 024 distinct 256² chunks (JPEGTables holding DQT only, every chunk its
   own optimised Huffman tables, so one table set per chunk). CUDA events over `launches` launches after a warm-up, as µs per
   window, per Mpx and per compressed MB, plus each kernel's share from one torch.profiler pass of 10 launches. The upload of the
   window's bytes and table sets is not in the kernel time.
2. (kernel) the CPU comparison: the warm single-thread decode of each distinct chunk by PIL (libjpeg-turbo, `Image.load`, the best of
   5), and that time times the chunks divided by the host's cores, an ideal-scaling estimate of a decode on every core.
3. (e2e) `rs tile` (tools.tile.main) and `rs segment` (tools.segment.main) end to end on scripts/bench_tile.py's seeded UTM ortho
   written GDAL-style as 256²-tiled 4:2:0 quality-90 JPEG, against its deflate twin (the same grid, holding the JPEG's decoded
   pixels, deflate level 1, predictor 2), alternately, twice each, with each tool's stage split, and whether both inputs gave
   identical outputs.
"""

import argparse
import io
import json
import os
import struct
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image, ImageFile  # noqa: E402

from bench_tile import LAT, LON, card  # noqa: E402
from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import jpeg  # noqa: E402
from robosat_b200 import synth  # noqa: E402
from robosat_b200 import tile as T  # noqa: E402
from robosat_b200.geotiff import GeoTiff  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402
from robosat_b200.tools import segment, tile  # noqa: E402

ImageFile.MAXBLOCK = 1 << 24
SUB = {"420": 2, "444": 0}


def pixels(chunk, k, seed=0):
    """bench_tile.py's tile content: blocks of smooth colour plus noise"""
    g = np.random.default_rng(seed * 1000003 + k)
    base = g.integers(0, 256, (4, 4, 3), dtype=np.uint8)
    blk = np.repeat(np.repeat(base, chunk // 4, 0), chunk // 4, 1).astype(np.int16)
    return np.clip(blk + g.integers(-12, 13, blk.shape), 0, 255).astype(np.uint8)


def encode(px, quality, sampling, restart, optimize=False):
    b = io.BytesIO()
    kw = dict(quality=quality, subsampling=SUB[sampling], optimize=optimize)
    if restart:
        kw["restart_marker_blocks"] = restart
    Image.fromarray(px, "RGB").save(b, "JPEG", **kw)
    return b.getvalue()


def write_tiff(path, size, chunk, chunks, compression, photometric, extra=()):
    """a tiled 3-band GeoTIFF in UTM zone 32 (bench_tile.py's grid); chunks(k) -> (key, bytes) of tile k, and tiles with equal keys
    share one stored stream"""
    E, N = T.tm_forward(LON, LAT, 9.0)
    across = (size + chunk - 1) // chunk
    offsets, counts, seen = [], [], {}
    with open(path, "wb") as fp:
        fp.write(b"II" + struct.pack("<HI", 42, 0))
        for k in range(across * across):
            key, b = chunks(k)
            if key not in seen:
                seen[key] = fp.tell()
                fp.write(b)
            offsets.append(seen[key])
            counts.append(len(b))
        geo = [1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, 1, 3072, 0, 1, 32632]
        tags = sorted([(256, 4, [size]), (257, 4, [size]), (258, 3, [8, 8, 8]), (259, 3, [compression]), (262, 3, [photometric]), (277, 3, [3]),
                       (284, 3, [1]), (322, 3, [chunk]), (323, 3, [chunk]), (324, 4, offsets), (325, 4, counts), (339, 3, [1, 1, 1]),
                       (33550, 12, [0.2, 0.2, 0.0]), (33922, 12, [0, 0, 0, float(E), float(N), 0]), (34735, 3, geo)] + list(extra))
        fmt = {3: "H", 4: "I", 7: "B", 12: "d"}
        entries, blob = [], b""
        blob_at = fp.tell()
        for tag, typ, vals in tags:
            payload = struct.pack("<" + fmt[typ] * len(vals), *vals)
            if len(payload) <= 4:
                value = payload.ljust(4, b"\0")
            else:
                value = struct.pack("<I", blob_at + len(blob))
                blob += payload
            entries.append(struct.pack("<HHI", tag, typ, len(vals)) + value)
        fp.write(blob)
        ifd = fp.tell()
        fp.write(struct.pack("<H", len(entries)) + b"".join(entries) + struct.pack("<I", 0))
        fp.seek(4)
        fp.write(struct.pack("<I", ifd))


def gdal_style(streams):
    """(JPEGTables holding the first stream's DQT, the streams without that DQT): GDAL's default JPEGTABLESMODE"""
    def segs(st):
        out, at = [], 2
        while True:
            m, n = st[at + 1], struct.unpack(">H", st[at + 2:at + 4])[0]
            out.append((m, st[at:at + 2 + n]))
            at += 2 + n
            if m == 0xDA:
                return out, st[at:]
    first = [seg for m, seg in segs(streams[0])[0] if m == 0xDB]
    out = []
    for st in streams:
        head, data = segs(st)
        out.append(b"\xff\xd8" + b"".join(seg for m, seg in head if not (m == 0xDB and seg in first)) + data)
    return b"\xff\xd8" + b"".join(first) + b"\xff\xd9", out


def kernel_case(d, chunk, n, sampling, quality, restart, launches, gdal=False):
    side = int(round(n ** 0.5))
    size = side * chunk
    distinct = n if gdal else 16
    streams = [encode(pixels(chunk, k, 7), quality, sampling, 8 if restart else None, optimize=gdal) for k in range(distinct)]
    extra = [(530, 3, [2, 2] if sampling == "420" else [1, 1])]
    if gdal:
        tables, streams = gdal_style(streams)
        extra.append((347, 7, list(tables)))
    path = os.path.join(d, "k.tif")
    write_tiff(path, size, chunk, lambda k: (k % distinct, streams[k % distinct]), 7, 6, extra)
    r = GeoTiff(path)
    idx = jpeg.touched(r, 0, size, 0, size)
    nbytes, _ = jpeg.stage_sizes(r, [(0, size, 0, size)])
    data = torch.empty((nbytes,), dtype=torch.uint8, pin_memory=True)
    descs = torch.empty((len(idx) * jpeg.F,), dtype=torch.int64, pin_memory=True)
    sets = torch.empty((len(idx) * _lib.RSB_JPEG_SET_WORDS,), dtype=torch.int32, pin_memory=True)
    st = jpeg.stage(r, 0, size, 0, size, data.numpy(), descs.numpy(), sets.numpy())
    out = torch.empty((size * size * 3,), dtype=torch.uint8, device="cuda")
    staged = torch.empty((st.nbytes,), dtype=torch.uint8, device="cuda")
    staged.copy_(data[:st.nbytes])
    dd = descs[:len(idx) * jpeg.F].cuda()
    ds = sets[:st.sets * _lib.RSB_JPEG_SET_WORDS].cuda()
    scratch = torch.empty((st.blocks * 192,), dtype=torch.uint8, device="cuda")
    derr = torch.empty((len(idx),), dtype=torch.int64, device="cuda")
    lib = _lib.load()

    def launch():
        _lib.check(lib.rsb_jpeg_decode_window(staged.data_ptr(), st.nbytes, dd.data_ptr(), len(idx), ds.data_ptr(), st.sets, size, size,
                                              chunk, chunk, 1, 3, 6, 0, size, 0, size, out.data_ptr(), scratch.data_ptr(), scratch.numel(), st.blocks,
                                              derr.data_ptr(), _lib.current_stream_ptr()), "rsb_jpeg_decode_window")

    for _ in range(5):
        launch()
    torch.cuda.synchronize()
    assert int(derr.abs().sum()) == 0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        launch()
    b.record()
    b.synchronize()
    sec = a.elapsed_time(b) / 1e3 / launches
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            launch()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        for name in ("huffman_kernel", "idct_kernel", "pixel_kernel", "Memset"):
            if name in ev.key:
                split[name] = round(split.get(name, 0.0) + ev.device_time_total / 10, 1)
    # the CPU comparison: the warm single-thread libjpeg-turbo decode of each distinct chunk (the chunk's own stream, with the tables
    # of JPEGTables put back for GDAL-style chunks), the best of 5
    full = [encode(pixels(chunk, k, 7), quality, sampling, 8 if restart else None, optimize=gdal) for k in range(min(distinct, 64))]
    per = []
    for s_ in full:
        best = float("inf")
        for _ in range(5):
            t0 = time.perf_counter()
            Image.open(io.BytesIO(s_)).load()
            best = min(best, time.perf_counter() - t0)
        per.append(best)
    cpu_chunk = float(np.mean(per))
    cores = usable_cores()
    mpx = size * size / 1e6
    mb = st.nbytes / 1e6
    return {"chunk": chunk, "chunks": len(idx), "sampling": sampling, "quality": quality, "restart": bool(restart), "gdal_style": gdal,
            "table_sets": st.sets, "compressed_MB": round(mb, 2), "us": round(sec * 1e6, 1), "us_per_Mpx": round(sec * 1e6 / mpx, 1),
            "us_per_MB": round(sec * 1e6 / mb, 1), "kernel_us": split, "pil_chunk_us_one_thread": round(cpu_chunk * 1e6, 1),
            "host_cores": cores, "pil_all_cores_estimate_us": round(cpu_chunk * len(idx) / cores * 1e6, 1)}


def write_ortho(d, size):
    """the JPEG ortho and its deflate twin (decoded on the device, in bands of tile rows)"""
    chunk = 256
    across = (size + chunk - 1) // chunk
    base = np.random.default_rng(0).integers(0, 256, (across * 4 + 1, across * 4 + 1, 3), dtype=np.uint8)

    def one(k):
        r, c = divmod(k, across)
        g = np.random.default_rng(1000003 + k)
        blk = np.repeat(np.repeat(base[r * 4:r * 4 + 4, c * 4:c * 4 + 4], chunk // 4, 0), chunk // 4, 1).astype(np.int16)
        px = np.clip(blk + g.integers(-12, 13, blk.shape), 0, 255).astype(np.uint8)
        return encode(px, 90, "420", None, optimize=True)

    with ThreadPoolExecutor(usable_cores()) as pool:
        streams = list(pool.map(one, range(across * across)))
    tables, streams = gdal_style(streams)
    jpath = os.path.join(d, "ortho_jpeg.tif")
    write_tiff(jpath, size, chunk, lambda k: (k, streams[k]), 7, 6, [(530, 3, [2, 2]), (347, 7, list(tables))])
    r = GeoTiff(jpath)
    band = {}

    def deflate(k):
        tr, tc = divmod(k, across)
        if tr not in band:
            band.clear()
            rows = min(chunk, size - tr * chunk)
            px = np.zeros((chunk, across * chunk, 3), np.uint8)
            px[:rows, :size] = r.read_window(tr * chunk, rows, 0, size)
            band[tr] = px
        t = band[tr][:, tc * chunk:(tc + 1) * chunk].reshape(chunk, -1).astype(np.int16)
        dd = t.copy()
        dd[:, 3:] -= t[:, :-3]
        return zlib.compress((dd & 0xff).astype(np.uint8).tobytes(), 1)

    dpath = os.path.join(d, "ortho_deflate.tif")
    write_tiff(dpath, size, chunk, lambda k: (k, deflate(k)), 8, 2, [(317, 3, [2])])
    return jpath, dpath


def run_tile(path, out):
    stats = {}
    t0 = time.perf_counter()
    tile.main(argparse.Namespace(zoom=18, size=512, tiles=None, resampling="bilinear", raster=path, out=out), stats)
    return time.perf_counter() - t0, {k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}


def run_segment(d, path, out):
    stats = {}
    t0 = time.perf_counter()
    segment.main(argparse.Namespace(zoom=18, size=512, overlap=32, batch_size=32, tiles=None, resampling="bilinear", output="masks", tta="none",
                                    nodata=None, model=os.path.join(d, "model.toml"), dataset=os.path.join(d, "dataset.toml"),
                                    checkpoint=os.path.join(d, "ckpt.pth"), raster=path, out=out), stats)
    return time.perf_counter() - t0, {k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}


def same_tree(a, b):
    fa = sorted(os.path.relpath(os.path.join(p, f), a) for p, _, fs in os.walk(a) for f in fs)
    fb = sorted(os.path.relpath(os.path.join(p, f), b) for p, _, fs in os.walk(b) for f in fs)
    return fa == fb and all(np.array_equal(np.asarray(Image.open(os.path.join(a, f))), np.asarray(Image.open(os.path.join(b, f)))) for f in fa)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--size", type=int, default=20000)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--part", choices=("kernel", "e2e"), required=True)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_jpeg: no CUDA device")
    os.environ.update(RSB_GPUS="1", RSB_QUIET="1")
    os.environ.pop("RSB_PRECISION", None)
    rec = {"card": card(), "part": args.part}
    with tempfile.TemporaryDirectory() as d:
        if args.part == "kernel":
            rec.update(launches=args.launches, kernel=[])
            cases = [(chunk, n, sampling, quality, restart, False) for chunk in (256, 512) for n in (64, 256, 1024) for sampling in ("420", "444")
                     for quality in (75, 90) for restart in (False, True)]
            cases += [(256, n, "420", quality, False, True) for n in (64, 256, 1024) for quality in (75, 90)]
            for c in cases:
                rec["kernel"].append(kernel_case(d, *c[:5], args.launches, gdal=c[5]))
                print(json.dumps(rec["kernel"][-1]), file=sys.stderr)
            return finish(rec, args.out)
        rec["end_to_end"] = []
        torch.save({"epoch": 1, "state_dict": synth.make_state_dict(2, seed=0), "optimizer": {}}, os.path.join(d, "ckpt.pth"))
        with open(os.path.join(d, "model.toml"), "w") as fp:
            fp.write("[common]\ncuda = true\nbatch_size = 2\nimage_size = 512\ncheckpoint = '%s'\n" % d)
        with open(os.path.join(d, "dataset.toml"), "w") as fp:
            fp.write("[common]\ndataset = '%s'\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n" % d)
        t0 = time.perf_counter()
        jpath, dpath = write_ortho(d, args.size)
        rec["write_inputs_s"] = round(time.perf_counter() - t0, 1)
        rec["input_MB"] = {"jpeg": round(os.path.getsize(jpath) / 1e6, 1), "deflate": round(os.path.getsize(dpath) / 1e6, 1)}
        run_tile(jpath, os.path.join(d, "warm_j"))
        run_tile(dpath, os.path.join(d, "warm_d"))
        for i in range(2):
            for name, path in (("jpeg", jpath), ("deflate", dpath)):
                wall, stats = run_tile(path, os.path.join(d, "tiles_" + name))
                rec["end_to_end"].append({"tool": "tile", "input": name, "run": i, "wall_s": round(wall, 3), "stats": stats})
                print(rec["end_to_end"][-1], file=sys.stderr)
        rec["tile_outputs_equal"] = same_tree(os.path.join(d, "tiles_jpeg"), os.path.join(d, "tiles_deflate"))
        for i in range(2):
            for name, path in (("jpeg", jpath), ("deflate", dpath)):
                wall, stats = run_segment(d, path, os.path.join(d, "seg_%s.tif" % name))
                rec["end_to_end"].append({"tool": "segment", "input": name, "run": i, "wall_s": round(wall, 3), "stats": stats})
                print(rec["end_to_end"][-1], file=sys.stderr)
        Image.MAX_IMAGE_PIXELS = None
        rec["segment_outputs_equal"] = bool(np.array_equal(np.asarray(Image.open(os.path.join(d, "seg_jpeg.tif"))),
                                                           np.asarray(Image.open(os.path.join(d, "seg_deflate.tif")))))
    finish(rec, args.out)


def finish(rec, out):
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
