"""GeoTIFF input of `rs tile`: the first image of a classic TIFF or BigTIFF, its georeferencing and its pixels.

`GeoTiff(path)` parses IFD 0 and the GeoKeys with `struct` and checks that the image is one `rs tile` reads (DESIGN.md §8):
8-bit unsigned chunky samples in strips or tiles, no compression, LZW or DEFLATE, predictor 1 or 2, and 1 band (MinIsBlack), 3
(RGB) or 4 (RGB plus an alpha ExtraSample); or JPEG (Compression 7) with 1 band (MinIsBlack) or 3 (RGB, or YCbCr converted to RGB),
every chunk's stream checked against the rule when the file is opened (robosat_b200/jpeg.py); georeferenced by one tiepoint plus
a pixel scale or by an affine model transformation, in EPSG:3857, EPSG:4326 or a WGS 84 UTM zone (EPSG:32601-32660, 32701-32760).
Anything else raises `RsbError` naming the value found. Overviews and sub-IFDs are ignored. `read_window` decodes a window of rows
and columns with the library's decoder (`rsb_tiff_decode_window`) over a memory map of the file, or for JPEG on the device.

`open_bands(path, bands)` reads the same container under the band rule of `rs tile --bands / --scale / --stretch` (DESIGN.md §8):
8- or 16-bit unsigned samples, chunky or planar, MinIsBlack or RGB with any number of bands, 1 or 3 of them selected plus the alpha
band, decoded by `rsb_tiff_decode_bands`. `GeoTiff(path)` keeps its own rule and messages.

`read_grid(path)` reads only the size and the georeferencing, with the same rules and messages for those, so any pixel layout
(16-bit, JPEG, palette ...) is accepted: `rs mosaic --like` takes the grid of an existing raster.
"""

import math
import mmap
import os
import struct

import numpy as np

from robosat_b200 import _lib

TYPE_SIZES = {1: 1, 2: 1, 3: 2, 4: 4, 5: 8, 6: 1, 7: 1, 8: 2, 9: 4, 10: 8, 11: 4, 12: 8, 16: 8, 17: 8, 18: 8}
TYPE_FORMATS = {1: "B", 2: "B", 3: "H", 4: "I", 5: "II", 6: "b", 7: "B", 8: "h", 9: "i", 10: "ii", 11: "f", 12: "d", 16: "Q", 17: "q", 18: "Q"}
COMPRESSIONS = {1: "none", 5: "LZW", 7: "JPEG", 8: "deflate", 32946: "deflate"}
JPEG = 7
COMPRESSION_NAMES = {2: "CCITT RLE", 3: "CCITT fax 3", 4: "CCITT fax 4", 6: "old-style JPEG", 7: "JPEG", 32773: "PackBits", 34712: "JPEG 2000",
                     34887: "LERC", 34925: "LZMA", 50000: "Zstandard", 50001: "WebP"}
PHOTOMETRIC_NAMES = {0: "MinIsWhite", 1: "MinIsBlack", 2: "RGB", 3: "palette", 4: "transparency mask", 5: "CMYK", 6: "YCbCr", 8: "CIELab"}
METRE, DEGREE = 9001, 9102
PIXEL_IS_AREA, PIXEL_IS_POINT = 1, 2
USER_DEFINED = 32767


def crs_of_epsg(code):
    """'3857', '4326' or ('utm', zone, south) for the supported EPSG codes, else None"""
    if code in (3857, 4326):
        return str(code)
    if 32601 <= code <= 32660:
        return ("utm", code - 32600, False)
    if 32701 <= code <= 32760:
        return ("utm", code - 32700, True)
    return None


def _fail(path, what):
    raise _lib.RsbError("%s: %s" % (path, what))


class _Header:
    """IFD 0's tags, its size (width, height) and its georeferencing (epsg, crs, geotransform, as `GeoTiff`); the pixel layout
    is not looked at"""

    def __init__(self, path):
        self.path = path
        with open(path, "rb") as fp:
            self._data = fp.read(16)
            size = os.fstat(fp.fileno()).st_size
        self.file_len = size
        self._map = None
        self._parse()

    def _parse(self):
        self._parse_tags()
        self._size()
        self._georeference()

    # ---- container ----

    def _read(self, offset, n):
        with open(self.path, "rb") as fp:
            fp.seek(offset)
            b = fp.read(n)
        if len(b) < n:
            _fail(self.path, "truncated file: %d bytes at offset %d are past its end (%d bytes)" % (n, offset, self.file_len))
        return b

    def _parse_tags(self):
        head = self._data
        if len(head) < 8 or head[:2] not in (b"II", b"MM"):
            _fail(self.path, "not a TIFF file (first bytes %r)" % head[:4])
        e = "<" if head[:2] == b"II" else ">"
        magic = struct.unpack(e + "H", head[2:4])[0]
        if magic == 42:
            big, ifd = False, struct.unpack(e + "I", head[4:8])[0]
        elif magic == 43:
            if len(head) < 16 or struct.unpack(e + "HH", head[4:8]) != (8, 0):
                _fail(self.path, "bad BigTIFF header")
            big, ifd = True, struct.unpack(e + "Q", head[8:16])[0]
        else:
            _fail(self.path, "not a TIFF file (version %d)" % magic)
        self.bigtiff, self.byteorder = big, e
        count_fmt, entry_size = ("Q", 20) if big else ("H", 12)
        n = struct.unpack(e + count_fmt, self._read(ifd, 8 if big else 2))[0]
        raw = self._read(ifd + (8 if big else 2), n * entry_size)
        tags = {}
        for k in range(n):
            ent = raw[k * entry_size:(k + 1) * entry_size]
            if big:
                tag, typ, count = struct.unpack(e + "HHQ", ent[:12])
                inline, value_bytes = ent[12:20], 8
            else:
                tag, typ, count = struct.unpack(e + "HHI", ent[:8])
                inline, value_bytes = ent[8:12], 4
            if typ not in TYPE_SIZES:
                continue  # unknown types are skipped, as TIFF readers must
            nbytes = TYPE_SIZES[typ] * count
            if nbytes <= value_bytes:
                blob = inline[:nbytes]
            else:
                blob = self._read(struct.unpack(e + ("Q" if big else "I"), inline)[0], nbytes)
            if typ == 2:
                tags[tag] = blob.split(b"\0")[0].decode("latin-1")
            else:
                vals = struct.unpack(e + TYPE_FORMATS[typ] * count, blob)
                if typ in (5, 10):
                    vals = tuple(vals[i] / vals[i + 1] if vals[i + 1] else float("nan") for i in range(0, len(vals), 2))
                tags[tag] = vals
        self._tags = tags

    def _tag(self, tag, default=None):
        v = self._tags.get(tag)
        return default if v is None else v

    def _size(self):
        t = self._tag
        if 256 not in self._tags or 257 not in self._tags:
            _fail(self.path, "no ImageWidth / ImageLength")
        self.width, self.height = int(t(256)[0]), int(t(257)[0])
        if self.width < 1 or self.height < 1:
            _fail(self.path, "empty image (%d x %d)" % (self.width, self.height))

    # ---- georeferencing ----

    def _geokeys(self):
        d = self._tags.get(34735)
        if d is None:
            _fail(self.path, "no GeoKeyDirectory: not a GeoTIFF")
        keys = {}
        doubles = self._tags.get(34736, ())
        for k in range(int(d[3])):
            key, loc, count, value = d[4 + 4 * k:8 + 4 * k]
            if loc == 0:
                keys[key] = value
            elif loc == 34736:
                keys[key] = doubles[value:value + count]
            else:
                keys[key] = None  # ASCII citations carry nothing the rule uses
        return keys

    def _georeference(self):
        keys = self._geokeys()
        model = keys.get(1024)
        if model == 1:
            code = keys.get(3072)
            linear = keys.get(3076)
            if linear is not None and linear != METRE:
                _fail(self.path, "ProjLinearUnitsGeoKey %s is not supported; only metres (9001) are" % (linear,))
        elif model == 2:
            code = keys.get(2048)
        else:
            _fail(self.path, "GTModelTypeGeoKey %s is not supported; use 1 (projected) or 2 (geographic)" % (model,))
        angular = keys.get(2054)
        if angular is not None and angular != DEGREE:
            _fail(self.path, "GeogAngularUnitsGeoKey %s is not supported; only degrees (9102) are" % (angular,))
        crs = crs_of_epsg(code) if isinstance(code, int) else None
        if crs is None or (model == 2) != (crs == "4326"):
            _fail(self.path, "CRS %s %s is not supported; use EPSG:3857, EPSG:4326 or a WGS 84 UTM zone (EPSG:326xx / 327xx)" % (
                "ProjectedCSTypeGeoKey" if model == 1 else "GeographicTypeGeoKey", "user-defined" if code == USER_DEFINED else code))
        self.epsg, self.crs = code, crs
        raster_type = keys.get(1025, PIXEL_IS_AREA)
        if raster_type not in (PIXEL_IS_AREA, PIXEL_IS_POINT):
            _fail(self.path, "GTRasterTypeGeoKey %s is not supported" % (raster_type,))
        shift = 0.5 if raster_type == PIXEL_IS_POINT else 0.0
        tie, scale, matrix = self._tags.get(33922), self._tags.get(33550), self._tags.get(34264)
        if matrix is not None:
            if len(matrix) != 16:
                _fail(self.path, "ModelTransformationTag has %d values, not 16" % len(matrix))
            a, b, c, d, e, f = matrix[0], matrix[1], matrix[3], matrix[4], matrix[5], matrix[7]
        elif tie is not None and scale is not None:
            if len(tie) != 6:
                _fail(self.path, "ModelTiepointTag has %d tiepoints; only one (with ModelPixelScaleTag) is supported" % (len(tie) // 6))
            if len(scale) < 2:
                _fail(self.path, "ModelPixelScaleTag has %d values" % len(scale))
            i0, j0, _, x0, y0, _ = tie
            a, b, d, e = scale[0], 0.0, 0.0, -scale[1]
            c, f = x0 - i0 * a, y0 - j0 * e
        else:
            _fail(self.path, "no georeferencing: need ModelTiepointTag with ModelPixelScaleTag, or ModelTransformationTag")
        # raster coordinates (u, v) -> model: PixelIsPoint names the centre of pixel (0, 0) at (0, 0)
        c, f = c - shift * (a + b), f - shift * (d + e)
        det = a * e - b * d
        if not np.isfinite([a, b, c, d, e, f]).all() or det == 0:
            _fail(self.path, "degenerate geotransform %r" % ((c, a, b, f, d, e),))
        self.geotransform = (float(c), float(a), float(b), float(f), float(d), float(e))


class GeoTiff(_Header):
    """IFD 0 of a GeoTIFF. Attributes: width, height, spp (1, 3 or 4), alpha (the 4th sample is alpha), nodata (-1, or the 0..255
    value of GDAL_NODATA), compression, predictor, photometric, tiled, chunk_w, chunk_h, offsets / byte_counts (int64 chunk table), epsg, crs
    (see `crs_of_epsg`) and geotransform (c, a, b, f, d, e): X = c + a u + b v, Y = f + d u + e v for raster coordinates (u, v),
    pixel (i, j) covering [i, i + 1) x [j, j + 1) (PixelIsPoint tiepoints are shifted by half a pixel, as GDAL does). JPEG rasters
    also have jpeg_tables (bytes or None) and jpeg_descs (robosat_b200.jpeg.parse); rows_per_strip is RowsPerStrip for strips."""

    def _parse(self):
        self._parse_tags()
        self._size()
        self._image()
        self._georeference()
        if self.compression == JPEG:
            from robosat_b200 import jpeg
            from robosat_b200.hostinfo import usable_cores

            tables = self._tags.get(347)
            self.jpeg_tables = bytes(bytearray(tables)) if tables else None
            self.jpeg_descs = jpeg.parse(self, self.file_bytes(), self.jpeg_tables, usable_cores())
            self._decoder = None

    def file_bytes(self):
        """the file as a uint8 array over a read-only memory map"""
        if self._map is None:
            with open(self.path, "rb") as fp:
                self._map = mmap.mmap(fp.fileno(), 0, access=mmap.ACCESS_READ)
            self._buf = np.frombuffer(self._map, np.uint8)
        return self._buf

    def jpeg_decoder(self, device):
        """the jpeg.Decoder of this raster on `device` (its table sets uploaded once)"""
        import torch

        from robosat_b200 import jpeg

        if self._decoder is None or self._decoder.device != torch.device(device):
            self._decoder = jpeg.Decoder(self, device)
        return self._decoder

    def _image(self):
        t = self._tag
        self.compression = int(t(259, (1,))[0])
        if self.compression not in COMPRESSIONS:
            _fail(self.path, "Compression %d (%s) is not supported; use none, LZW or deflate" % (
                self.compression, COMPRESSION_NAMES.get(self.compression, "unknown")))
        self.spp = int(t(277, (1,))[0])
        planar = int(t(284, (1,))[0])
        if planar != 1:
            _fail(self.path, "PlanarConfiguration %d is not supported; only 1 (chunky) is" % planar)
        bits = t(258, (1,) * self.spp)
        if any(int(b) != 8 for b in bits):
            _fail(self.path, "BitsPerSample %s is not supported; only 8 is" % (",".join(str(int(b)) for b in bits)))
        fmt = t(339, (1,) * self.spp)
        if any(int(f) != 1 for f in fmt):
            _fail(self.path, "SampleFormat %s is not supported; only 1 (unsigned integer) is" % (",".join(str(int(f)) for f in fmt)))
        photometric = int(t(262, (1 if self.spp == 1 else 2,))[0])
        extra = tuple(int(v) for v in t(338, ()))
        if self.compression == JPEG and self.spp == 3 and photometric == 6:
            photometric = 2  # YCbCr inside the JPEG streams, RGB out of the decoder
            self.photometric = 6
        else:
            self.photometric = photometric
        if self.compression == JPEG and self.spp not in (1, 3):
            _fail(self.path, "Compression 7 (JPEG) with %d bands is not supported; use 1 (gray) or 3 (RGB or YCbCr)" % self.spp)
        if self.spp == 1 and photometric != 1:
            _fail(self.path, "one band with Photometric %d (%s) is not supported; only MinIsBlack is" % (photometric, PHOTOMETRIC_NAMES.get(photometric, "unknown")))
        if self.spp in (3, 4) and photometric != 2:
            _fail(self.path, "%d bands with Photometric %d (%s) are not supported; only RGB is" % (self.spp, photometric, PHOTOMETRIC_NAMES.get(photometric, "unknown")))
        if self.spp == 4 and extra not in ((1,), (2,)):
            _fail(self.path, "4 bands with ExtraSamples %s are not supported; the 4th band must be alpha (1 or 2)" % (extra,))
        if self.spp not in (1, 3, 4):
            _fail(self.path, "%d bands are not supported; use 1 (gray), 3 (RGB) or 4 (RGB + alpha)" % self.spp)
        self.alpha = self.spp == 4
        self.predictor = int(t(317, (1,))[0])
        if self.predictor not in (1, 2):
            _fail(self.path, "Predictor %d is not supported; use 1 or 2" % self.predictor)
        if self.compression in (1, JPEG):
            self.predictor = 1  # libtiff applies the predictor only inside a codec other than JPEG; uncompressed data is stored as is
        self._chunk_table(1)
        self.nodata = self._nodata(255)

    def _chunk_table(self, planes):
        """tiled, chunk_w, chunk_h, rows_per_strip and the offsets / byte_counts of `planes` planes of chunks"""
        t = self._tag
        if 322 in self._tags:
            self.tiled = True
            self.chunk_w, self.chunk_h = int(t(322)[0]), int(t(323, (0,))[0])
            self.rows_per_strip = self.chunk_h
            offsets, counts = t(324), t(325)
            need = -(-self.width // max(1, self.chunk_w)) * -(-self.height // max(1, self.chunk_h))
        else:
            self.tiled = False
            self.rows_per_strip = int(t(278, (2 ** 32 - 1,))[0])
            self.chunk_w, self.chunk_h = self.width, min(self.height, self.rows_per_strip)
            offsets, counts = t(273), t(279)
            need = -(-self.height // max(1, self.chunk_h))
        need *= planes
        if self.chunk_w < 1 or self.chunk_h < 1:
            _fail(self.path, "chunks of %d x %d pixels" % (self.chunk_w, self.chunk_h))
        if offsets is None or counts is None or len(offsets) != need or len(counts) != need:
            _fail(self.path, "%s table has %s offsets and %s byte counts, the image needs %d" % (
                "tile" if self.tiled else "strip", None if offsets is None else len(offsets), None if counts is None else len(counts), need))
        self.offsets = np.asarray(offsets, np.int64)
        self.byte_counts = np.asarray(counts, np.int64)

    def _nodata(self, top):
        """the integer value of GDAL_NODATA in 0..top, or -1 (any other value matches no pixel)"""
        nodata = self._tags.get(42113)
        if nodata:
            try:
                value = float(nodata.strip())
            except ValueError:
                _fail(self.path, "GDAL_NODATA %r is not a number" % nodata)
            if math.isfinite(value) and value == int(value) and 0 <= value <= top:
                return int(value)
        return -1

    # ---- pixels ----

    def read_window(self, row0, rows, col0, cols, out=None, threads=None):
        """raster rows [row0, row0 + rows) x columns [col0, col0 + cols) -> uint8 [rows, cols, spp] (into `out` when given, any
        C-contiguous uint8 array of at least that many bytes, e.g. pinned host memory); RsbError names a chunk that cannot be
        decoded. A JPEG raster is decoded on the device (rsb_jpeg_decode_window) and copied back: it needs a GPU, and there is no
        CPU decoder."""
        import ctypes

        from robosat_b200.hostinfo import usable_cores

        n = rows * cols * self.spp
        if out is None:
            out = np.empty(n, np.uint8)
        view = np.frombuffer(out, np.uint8, n) if not isinstance(out, np.ndarray) else out.reshape(-1)[:n]
        if self.compression == JPEG:
            from robosat_b200 import jpeg

            jpeg.read_window(self, row0, rows, col0, cols, view)
            return view.reshape(rows, cols, self.spp)
        self.file_bytes()
        bad = ctypes.c_int64(-1)
        _lib.check(_lib.load().rsb_tiff_decode_window(self._buf.ctypes.data, self.file_len, self.offsets.ctypes.data, self.byte_counts.ctypes.data,
                                                       len(self.offsets), self.width, self.height, self.chunk_w, self.chunk_h, int(self.tiled),
                                                       self.spp, self.compression, self.predictor, row0, rows, col0, cols, view.ctypes.data,
                                                       threads or usable_cores(), ctypes.byref(bad)), "%s" % self.path)
        return view.reshape(rows, cols, self.spp)



def open_bands(path, bands=None):
    """IFD 0 of a GeoTIFF read under the band rule (DESIGN.md §8; `rs tile --bands / --scale / --stretch`): a `BandTiff` whose window
    decode gathers the 1-based `bands` (1 or 3 of them; None: 1,2,3 of an RGB raster, or the band of a single MinIsBlack band with or
    without an alpha band) and the alpha band"""
    return BandTiff(path, bands)


class BandTiff(GeoTiff):
    """A GeoTiff under the band rule. Besides GeoTiff's attributes (spp is the file's samples per pixel, nodata is in 0..2^bits - 1 or
    -1): bits (8 or 16), planar (1 chunky, 2 band-interleaved), byteorder ('<' or '>'), bands (the 0-based selected bands, 1 or 3),
    alpha_band (0-based, or None: the first band ExtraSamples declares alpha), k (the decoded samples per pixel: the selected bands,
    then the alpha band), and scale: [(LO, HI)] per selected band, the identity (0, 255) for 8-bit rasters and None for 16-bit
    ones until set (`set_scale`)."""

    def __init__(self, path, bands=None):
        self._want = None if bands is None else [int(b) for b in bands]
        super().__init__(path)

    def _parse(self):
        self._parse_tags()
        self._size()
        self._band_image()
        self._georeference()

    def _band_image(self):
        t = self._tag
        self.compression = int(t(259, (1,))[0])
        if self.compression not in COMPRESSIONS or self.compression == JPEG:
            _fail(self.path, "Compression %d (%s) is not supported with --bands, --scale or --stretch; use none, LZW or deflate" % (
                self.compression, COMPRESSION_NAMES.get(self.compression, "unknown")))
        self.spp = int(t(277, (1,))[0])
        if self.spp < 1:
            _fail(self.path, "SamplesPerPixel %d" % self.spp)
        bits = tuple(int(b) for b in t(258, (1,) * self.spp))
        if len(set(bits)) != 1 or bits[0] not in (8, 16):
            _fail(self.path, "BitsPerSample %s is not supported; use 8 or 16 for every band" % ",".join(str(b) for b in bits))
        self.bits = bits[0]
        fmt = t(339, (1,) * self.spp)
        if any(int(f) != 1 for f in fmt):
            _fail(self.path, "SampleFormat %s is not supported; only 1 (unsigned integer) is" % (",".join(str(int(f)) for f in fmt)))
        self.planar = int(t(284, (1,))[0])
        if self.planar not in (1, 2):
            _fail(self.path, "PlanarConfiguration %d is not supported; use 1 (chunky) or 2 (planar)" % self.planar)
        self.photometric = int(t(262, (1 if self.spp < 3 else 2,))[0])
        if self.photometric not in (1, 2):
            _fail(self.path, "Photometric %d (%s) is not supported; use MinIsBlack or RGB" % (
                self.photometric, PHOTOMETRIC_NAMES.get(self.photometric, "unknown")))
        if self.photometric == 2 and self.spp < 3:
            _fail(self.path, "Photometric 2 (RGB) with %d bands" % self.spp)
        extra = tuple(int(v) for v in t(338, ()))
        if len(extra) > self.spp:
            _fail(self.path, "ExtraSamples has %d values for %d bands" % (len(extra), self.spp))
        first_extra = self.spp - len(extra)
        self.alpha_band = next((first_extra + i for i, v in enumerate(extra) if v in (1, 2)), None)
        if self._want is None:
            if self.photometric == 2:
                self.bands = [0, 1, 2]
            elif self.spp == 1 or (self.spp == 2 and self.alpha_band == 1):
                self.bands = [0]
            else:
                _fail(self.path, "%d bands (Photometric %s) need --bands to say which to read" % (
                    self.spp, PHOTOMETRIC_NAMES[self.photometric]))
        else:
            if len(self._want) not in (1, 3):
                _fail(self.path, "--bands takes 1 or 3 bands, not %d" % len(self._want))
            for b in self._want:
                if not 1 <= b <= self.spp:
                    _fail(self.path, "band %d is not in this raster of %d bands" % (b, self.spp))
            self.bands = [b - 1 for b in self._want]
        self.alpha = self.alpha_band is not None
        self.k = len(self.bands) + int(self.alpha)
        self.predictor = int(t(317, (1,))[0])
        if self.predictor not in (1, 2):
            _fail(self.path, "Predictor %d is not supported; use 1 or 2" % self.predictor)
        if self.compression == 1:
            self.predictor = 1  # libtiff applies the predictor only inside a codec; uncompressed data is stored as is
        self._chunk_table(self.planar == 2 and self.spp or 1)
        self.nodata = self._nodata((1 << self.bits) - 1)
        self.scale = [(0, 255)] * len(self.bands) if self.bits == 8 else None

    def set_scale(self, pairs):
        """the (LO, HI) of every selected band (one pair: the same for all), 0 <= LO < HI <= 2^bits - 1; RsbError otherwise"""
        pairs = [tuple(int(v) for v in p) for p in pairs]
        if len(pairs) == 1:
            pairs = pairs * len(self.bands)
        if len(pairs) != len(self.bands):
            raise _lib.RsbError("--scale has %d pairs for %d bands; give one pair, or one per band" % (len(pairs), len(self.bands)))
        top = (1 << self.bits) - 1
        for lo, hi in pairs:
            if not 0 <= lo < hi <= top:
                raise _lib.RsbError("--scale %d,%d is not 0 <= LO < HI <= %d (%d-bit samples)" % (lo, hi, top, self.bits))
        self.scale = pairs

    @property
    def sample_bytes(self):
        return self.bits // 8

    def read_window(self, row0, rows, col0, cols, out=None, threads=None):
        """raster rows [row0, row0 + rows) x columns [col0, col0 + cols) -> uint8 or uint16 [rows, cols, k]: the selected bands,
        then the alpha band (into `out` when given, any C-contiguous array of at least that many bytes, e.g. pinned host memory)"""
        import ctypes

        from robosat_b200.hostinfo import usable_cores

        dtype = np.uint8 if self.bits == 8 else np.uint16
        nbytes = rows * cols * self.k * self.sample_bytes
        if out is None:
            out = np.empty(nbytes, np.uint8)
        view = np.frombuffer(out, np.uint8, nbytes) if not isinstance(out, np.ndarray) else out.reshape(-1).view(np.uint8)[:nbytes]
        select = np.asarray(self.bands + ([self.alpha_band] if self.alpha else []), np.int32)
        self.file_bytes()
        bad = ctypes.c_int64(-1)
        _lib.check(_lib.load().rsb_tiff_decode_bands(self._buf.ctypes.data, self.file_len, self.offsets.ctypes.data, self.byte_counts.ctypes.data,
                                                      len(self.offsets), self.width, self.height, self.chunk_w, self.chunk_h, int(self.tiled),
                                                      self.spp, self.bits, self.planar, int(self.byteorder == ">"), self.compression,
                                                      self.predictor, select.ctypes.data, len(select), row0, rows, col0, cols, view.ctypes.data,
                                                      threads or usable_cores(), ctypes.byref(bad)), "%s" % self.path)
        return view.view(dtype).reshape(rows, cols, self.k)


def read_grid(path):
    """(width, height, crs, geotransform) of the first image of a GeoTIFF, from its header alone: the size and the georeferencing
    must be ones `GeoTiff` accepts (RsbError names the value found otherwise), the pixel layout may be anything."""
    h = _Header(path)
    return h.width, h.height, h.crs, h.geotransform
