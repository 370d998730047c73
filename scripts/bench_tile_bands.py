"""The band rule of `rs tile` and `rs segment` on one GPU: prints ONE JSON line and writes the same record to --out.

    python scripts/bench_tile_bands.py --out results/h100_tile_bands.json [--launches 50] [--size 20000] [--window 8192]

Records, with the card's name and power limit read in the same run:
1. (kernel) rsb_tile_render on a --window² window at 8 and 16 bits with k = 1, 3 and 4 samples per pixel (the last with an alpha
   band), and rsb_band_histogram at 8 and 16 bits with 1 and 3 bands on smooth imagery (a few values: bin contention) and uniform
   noise. CUDA events over `launches` launches after a warm-up, as ms per launch and bytes moved per second (read plus written, from
   the shapes) against the H100 SXM data-sheet 3.35 TB/s.
2. (e2e) a seeded --size² 4-band uint16 UTM GeoTIFF (256² deflate tiles, level 1, predictor 2): `rs tile --bands 3,2,1 --stretch 2,98`,
   then `rs tile` with the printed --scale, then `rs segment` with that scale, alternately, twice, each with its stage split (the
   stretch pass, decode, upload, render, warp, sink / encode), and whether the stretch and the scale runs wrote identical tiles.
"""

import argparse
import contextlib
import io
import json
import os
import re
import shutil
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

from bench_tile import LAT, LON, card  # noqa: E402
from robosat_b200 import _lib  # noqa: E402
from robosat_b200 import synth  # noqa: E402
from robosat_b200 import tile as T  # noqa: E402
from robosat_b200.hostinfo import usable_cores  # noqa: E402
from robosat_b200.tools import segment, tile  # noqa: E402

PEAK_BW = 3.35e12  # H100 SXM HBM3, data sheet


def timed(fn, launches):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def window(side, k, bits, smooth, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    top = (1 << bits) - 1
    if smooth:  # a handful of values per band: every CTA's counts pile onto a few bins
        v = torch.randint(top // 3, top // 3 + 4, (side, side, k), device="cuda", generator=g)
    else:
        v = torch.randint(0, top + 1, (side, side, k), device="cuda", generator=g)
    if k in (2, 4):
        v[..., -1] = top
    return v


def as_bytes(v, bits):
    """the int tensor as packed uint8 or uint16 samples, viewed as bytes"""
    if bits == 8:
        return v.to(torch.uint8).reshape(-1).contiguous()
    return v.to(torch.int16).reshape(-1).contiguous().view(torch.uint8)  # int64 -> int16 keeps the low 16 bits


def kernel_cases(side, launches):
    lib = _lib.load()
    st = _lib.current_stream_ptr()
    out = torch.empty((side * side * 4,), dtype=torch.uint8, device="cuda")
    rows = []
    for bits in (8, 16):
        for k in (1, 3, 4):
            nsel, alpha = (1 if k == 1 else 3), int(k == 4)
            src = as_bytes(window(side, k, bits, False), bits)
            scale = np.array([10, (1 << bits) - 20] * nsel, np.int32)
            ms = timed(lambda: _lib.check(lib.rsb_tile_render(src.data_ptr(), side, side, bits, nsel, alpha, -1, scale.ctypes.data, out.data_ptr(),
                                                              side * 4, st), "rsb_tile_render"), launches)
            moved = src.numel() + out.numel()
            rows.append(dict(kernel="rsb_tile_render", bits=bits, k=k, pixels=side * side, ms=round(ms, 4), bytes=moved,
                             GB_per_s=round(moved / ms / 1e6, 1), share_of_3_35_TBps=round(moved / ms / 1e-3 / PEAK_BW, 3)))
            del src
    for bits in (8, 16):
        for nsel in (1, 3):
            for smooth in (True, False):
                src = as_bytes(window(side, nsel, bits, smooth), bits)
                hist = torch.zeros((nsel, 1 << bits), dtype=torch.int64, device="cuda")
                ms = timed(lambda: _lib.check(lib.rsb_band_histogram(src.data_ptr(), side, side, bits, nsel, 0, -1, hist.data_ptr(), st),
                                              "rsb_band_histogram"), launches)
                assert int(hist[0].sum()) == (launches + 1) * side * side
                moved = src.numel()
                rows.append(dict(kernel="rsb_band_histogram", bits=bits, bands=nsel, data="smooth" if smooth else "noise", pixels=side * side,
                                 ms=round(ms, 4), bytes=moved, GB_per_s=round(moved / ms / 1e6, 1),
                                 share_of_3_35_TBps=round(moved / ms / 1e-3 / PEAK_BW, 3)))
                del src, hist
    torch.cuda.empty_cache()
    return rows


def write_geotiff16(path, size, seed=0, chunk=256, bands=4):
    """a seeded 4-band uint16 GeoTIFF of size x size in UTM zone 32 (0.2 m pixels): blocks of smooth values plus noise, 256² tiles,
    deflate level 1, predictor 2"""
    rng = np.random.default_rng(seed)
    across = (size + chunk - 1) // chunk
    base = rng.integers(600, 12000, (across * 4 + 1, across * 4 + 1, bands))
    E, N = T.tm_forward(LON, LAT, 9.0)

    def one(k):
        r, c = divmod(k, across)
        g = np.random.default_rng(seed * 1000003 + k)
        blk = np.repeat(np.repeat(base[r * 4:r * 4 + 4, c * 4:c * 4 + 4], chunk // 4, 0), chunk // 4, 1)
        px = np.clip(blk + g.integers(-150, 151, blk.shape), 0, 65535)
        flat = px.reshape(chunk, -1)
        d = flat.copy()
        d[:, bands:] -= flat[:, :-bands]
        return zlib.compress((d & 0xffff).astype("<u2").tobytes(), 1)

    n = across * across
    offsets, counts = [], []
    with open(path, "wb") as fp, ThreadPoolExecutor(usable_cores()) as pool:
        fp.write(b"II" + struct.pack("<HI", 42, 0))
        for b in pool.map(one, range(n)):
            offsets.append(fp.tell())
            counts.append(len(b))
            fp.write(b)
        geo = [1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, 1, 3072, 0, 1, 32632]
        tags = [(256, 4, [size]), (257, 4, [size]), (258, 3, [16] * bands), (259, 3, [8]), (262, 3, [2]), (277, 3, [bands]), (284, 3, [1]),
                (317, 3, [2]), (322, 3, [chunk]), (323, 3, [chunk]), (324, 4, offsets), (325, 4, counts), (338, 3, [0] * (bands - 3)),
                (339, 3, [1] * bands), (33550, 12, [0.2, 0.2, 0.0]), (33922, 12, [0, 0, 0, float(E), float(N), 0]), (34735, 3, geo)]
        fmt = {3: "H", 4: "I", 12: "d"}
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


def _round(stats):
    return {k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}


def run_tile(path, out, **opts):
    stats, err = {}, io.StringIO()
    t0 = time.perf_counter()
    with contextlib.redirect_stderr(err):
        tile.main(argparse.Namespace(zoom=18, size=512, tiles=None, resampling="bilinear", raster=path, out=out, bands="3,2,1", **opts), stats)
    return time.perf_counter() - t0, _round(stats), err.getvalue()


def run_segment(d, path, out, scale):
    stats = {}
    t0 = time.perf_counter()
    segment.main(argparse.Namespace(zoom=18, size=512, overlap=32, batch_size=32, tiles=None, resampling="bilinear", output="masks", tta="none",
                                    nodata=None, model=os.path.join(d, "model.toml"), dataset=os.path.join(d, "dataset.toml"),
                                    checkpoint=os.path.join(d, "ckpt.pth"), raster=path, out=out, bands="3,2,1", scale=scale, stretch=None), stats)
    return time.perf_counter() - t0, _round(stats)


def same_tree(a, b):
    fa = sorted(os.path.relpath(os.path.join(p, f), a) for p, _, fs in os.walk(a) for f in fs)
    fb = sorted(os.path.relpath(os.path.join(p, f), b) for p, _, fs in os.walk(b) for f in fs)
    return fa == fb and all(open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read() for f in fa)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--size", type=int, default=20000)
    ap.add_argument("--window", type=int, default=8192)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_bands needs a CUDA device")
    _lib.require_device()
    rec = {"card": card(), "kernel": kernel_cases(args.window, args.launches), "end_to_end": []}
    with tempfile.TemporaryDirectory() as d:
        os.environ.setdefault("RSB_QUIET", "1")
        torch.save({"epoch": 1, "state_dict": synth.make_state_dict(2, seed=5), "optimizer": {}}, os.path.join(d, "ckpt.pth"))
        with open(os.path.join(d, "model.toml"), "w") as fp:
            fp.write("[common]\ncuda = true\nbatch_size = 2\nimage_size = 512\ncheckpoint = '%s'\n" % d)
        with open(os.path.join(d, "dataset.toml"), "w") as fp:
            fp.write("[common]\ndataset = '%s'\nclasses = ['background', 'parking']\ncolors = ['denim', 'orange']\n" % d)
        warm = os.path.join(d, "warm.tif")
        write_geotiff16(warm, 2048, seed=1)
        _, _, err = run_tile(warm, os.path.join(d, "warm"), stretch="2,98")
        run_segment(d, warm, os.path.join(d, "warm_seg.tif"), re.search(r"--scale (\S+)", err).group(1))
        path = os.path.join(d, "ortho16.tif")
        t0 = time.perf_counter()
        write_geotiff16(path, args.size)
        rec["write_input_s"] = round(time.perf_counter() - t0, 1)
        rec["input_MB"] = round(os.path.getsize(path) / 1e6, 1)
        equal = []
        for i in range(2):
            wall, stats, err = run_tile(path, os.path.join(d, "stretch%d" % i), stretch="2,98")
            scale = re.search(r"--scale (\S+)", err).group(1)
            rec["end_to_end"].append({"tool": "tile --stretch 2,98", "run": i, "wall_s": round(wall, 3), "stats": stats, "printed": err.strip()})
            wall, stats, _ = run_tile(path, os.path.join(d, "scale%d" % i), scale=scale)
            rec["end_to_end"].append({"tool": "tile --scale", "run": i, "wall_s": round(wall, 3), "stats": stats})
            equal.append(same_tree(os.path.join(d, "stretch%d" % i), os.path.join(d, "scale%d" % i)))
            wall, stats = run_segment(d, path, os.path.join(d, "seg%d.tif" % i), scale)
            rec["end_to_end"].append({"tool": "segment --scale", "run": i, "wall_s": round(wall, 3), "stats": stats})
            for sub in ("stretch%d" % i, "scale%d" % i):
                shutil.rmtree(os.path.join(d, sub))
        rec["stretch_and_scale_tiles_equal"] = all(equal)
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fp:
        fp.write(line + "\n")


if __name__ == "__main__":
    main()
