"""numpy restatement of the band rule (DESIGN.md §8) for the tests of rsb_tile_render, rsb_band_histogram, `--stretch` and
`rs tile` / `rs segment` under --bands / --scale / --stretch.

A window of raw samples [H, W, k] (the selected bands, then the alpha band) becomes 8-bit RGBA: per band v = floor((510 t + d) / (2 d))
with d = HI - LO and t = clamp(s, LO, HI) - LO (255 t / d rounded half up, in integers); one band gives R = G = B = v; A = 0 when
the alpha sample is 0 or every selected band equals nodata (tested on the raw samples), else 255. From there on the plain rule of
tests/tile_reference.py (and tile_average_reference.py) applies to that RGBA raster with alpha validity and no nodata.

The stretch: per band, N valid pixels, rank = max(1, ceil(q N / 10000)) for q in hundredths of a percent, and the value is
np.sort(valid samples)[rank - 1]; HI = LO gives HI = LO + 1 (LO = HI - 1 at the top value)."""

import numpy as np


def valid(raw, nsel, alpha, nodata):
    ok = np.ones(raw.shape[:2], bool)
    if alpha:
        ok &= raw[..., nsel] != 0
    if nodata >= 0:
        ok &= ~(raw[..., :nsel] == nodata).all(axis=-1)
    return ok


def scale_values(s, lo, hi):
    d = hi - lo
    t = np.clip(s.astype(np.int64), lo, hi) - lo
    return ((510 * t + d) // (2 * d)).astype(np.uint8)


def render(raw, nsel, alpha, nodata, scale):
    """raw [H, W, nsel + alpha] -> uint8 RGBA [H, W, 4]"""
    H, W = raw.shape[:2]
    out = np.zeros((H, W, 4), np.uint8)
    for c in range(3):
        b = 0 if nsel == 1 else c
        out[..., c] = scale_values(raw[..., b], *scale[b])
    out[..., 3] = np.where(valid(raw, nsel, alpha, nodata), 255, 0)
    return out


def histogram(raw, nsel, alpha, nodata, bits):
    ok = valid(raw, nsel, alpha, nodata)
    return np.stack([np.bincount(raw[..., b][ok].astype(np.int64), minlength=1 << bits) for b in range(nsel)])


def percentile(values, q):
    """np.sort(values)[rank - 1] with rank = max(1, ceil(q N / 10000))"""
    v = np.sort(np.asarray(values).reshape(-1))
    rank = max(1, -(-q * len(v) // 10000))
    return int(v[rank - 1])


def stretch(raw, nsel, alpha, nodata, bits, q_lo, q_hi):
    ok = valid(raw, nsel, alpha, nodata)
    top = (1 << bits) - 1
    pairs = []
    for b in range(nsel):
        lo, hi = percentile(raw[..., b][ok], q_lo), percentile(raw[..., b][ok], q_hi)
        if hi == lo:
            lo, hi = (lo, lo + 1) if lo < top else (top - 1, top)
        pairs.append((lo, hi))
    return pairs


class RgbaRaster:
    """the RGBA raster the plain rule sees: a band raster's grid with 4 samples, alpha validity and no nodata"""

    def __init__(self, raster):
        self.width, self.height, self.crs, self.geotransform = raster.width, raster.height, raster.crs, raster.geotransform
        self.spp, self.alpha, self.nodata = 4, True, -1


def rgba_of(raster, raw=None):
    """the whole band raster (geotiff.BandTiff) rendered with its scale, and its RgbaRaster"""
    raw = raster.read_window(0, raster.height, 0, raster.width) if raw is None else raw
    return render(raw, len(raster.bands), raster.alpha, raster.nodata, raster.scale), RgbaRaster(raster)
