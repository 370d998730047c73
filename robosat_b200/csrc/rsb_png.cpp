// Host-side PNG codec for the two file formats either side of the `rs predict` hot path (SURVEY.md 8(f) rows 1-2):
//   decode: z/x/y.png RGB tiles           <- Image.open(path).convert("RGB")            robosat/tiles.py:150-159, 181
//   encode: probs/z/x/y.png P-mode masks  <- Image.fromarray(q, "P") + putpalette + save robosat/tools/predict.py:105-113
// Plain C++ over zlib (inflate / deflate / crc32); no Python, no GIL: the tools call these through ctypes from their pool
// threads, so 16-32 threads per rank really decode / encode in parallel (PIL holds the interpreter lock for part of every call,
// which starved the main thread of `rs predict`). Pixel content is identical to PIL's; the encoded bytes
// differ (zlib level), which the consumers (`rs masks`, any PNG reader) do not see.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

#include <sys/stat.h>

#include <atomic>
#include <string>
#include <thread>
#include <vector>

#include "../../include/rsb200.h"
#include "rsb_host.h"
#include "rsb_inflate.h"

using rsb::set_error;
using rsb::kInflateInPad;
using rsb::kInflateOutPad;
using rsb::rsb_inflate_zlib_padded;

namespace {

const uint8_t kSig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};

inline uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }
inline void put32(uint8_t* p, uint32_t v) {
    p[0] = uint8_t(v >> 24);
    p[1] = uint8_t(v >> 16);
    p[2] = uint8_t(v >> 8);
    p[3] = uint8_t(v);
}

// append one chunk (length, type, data, crc) to `out`
void put_chunk(std::vector<uint8_t>& out, const char type[4], const uint8_t* data, size_t n) {
    const size_t at = out.size();
    out.resize(at + 12 + n);
    put32(&out[at], uint32_t(n));
    memcpy(&out[at + 4], type, 4);
    if (n) memcpy(&out[at + 8], data, n);
    put32(&out[at + 8 + n], uint32_t(crc32(0L, &out[at + 4], uInt(4 + n))));
}

inline int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

bool read_file(const char* path, std::vector<uint8_t>& buf) {
    FILE* f = fopen(path, "rb");
    if (!f) return false;
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    if (n < 0) {
        fclose(f);
        return false;
    }
    buf.resize(size_t(n));
    const size_t got = n ? fread(buf.data(), 1, size_t(n), f) : 0;
    fclose(f);
    return got == size_t(n);
}

bool use_own_inflate() {
    static const bool own = [] {
        const char* v = getenv("RSB_INFLATE");
        return !(v && strcmp(v, "zlib") == 0);
    }();
    return own;
}

}  // namespace

namespace {

// Filtered scanlines `raw` (filter type 0) -> a complete PNG of colour type `ctype` in `out`; palette_rgb / entries only for
// colour type 3. Returns the byte count or a negative code.
// Strategy: deflate's string matcher is most of the encode time and finds nothing in noise-like rasters (soft probabilities
// of an untrained or uncertain model: 8.5 ms per 512x512 mask at level 6 for a stream as large as Huffman coding alone gives
// in 2.8 ms). A level-1 probe of a band of rows decides: if string matching does not shrink the band below 90 % of its raw
// size the image is coded with Z_RLE (run lengths + Huffman), otherwise with the default strategy at `level`.
int64_t encode_scanlines(const std::vector<uint8_t>& raw, int32_t w, int32_t h, int ctype, const uint8_t* palette_rgb, int32_t entries,
                         int32_t level, uint8_t* out, int64_t capacity) {
    const size_t line = raw.size() / size_t(h);
    const int lvl = level < 0 ? Z_DEFAULT_COMPRESSION : (level > 9 ? 9 : level);
    int strategy = Z_DEFAULT_STRATEGY;
    if (lvl != 0) {
        const int band = h < 16 ? h : 16;
        const uint8_t* mid = raw.data() + size_t((h - band) / 2) * line;
        const uLong band_bytes = uLong(band) * uLong(line);
        uLongf pn = compressBound(band_bytes);
        std::vector<uint8_t> probe(pn);
        if (compress2(probe.data(), &pn, mid, band_bytes, 1) == Z_OK && double(pn) > 0.9 * double(band_bytes)) strategy = Z_RLE;
    }
    uLongf zn = compressBound(uLong(raw.size())) + 64;
    std::vector<uint8_t> z(zn);
    {
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        if (deflateInit2(&zs, lvl, Z_DEFLATED, 15, 8, strategy) != Z_OK) return set_error(RSB_E_INVALID, "png_encode: deflateInit2 failed");
        zs.next_in = const_cast<uint8_t*>(raw.data());
        zs.avail_in = uInt(raw.size());
        zs.next_out = z.data();
        zs.avail_out = uInt(z.size());
        const int zr = deflate(&zs, Z_FINISH);
        zn = zs.total_out;
        deflateEnd(&zs);
        if (zr != Z_STREAM_END) return set_error(RSB_E_INVALID, "png_encode: deflate failed (%d)", zr);
    }
    std::vector<uint8_t> png(kSig, kSig + 8);
    png.reserve(size_t(zn) + 1024);
    uint8_t ihdr[13];
    put32(ihdr, uint32_t(w));
    put32(ihdr + 4, uint32_t(h));
    ihdr[8] = 8;   // bit depth
    ihdr[9] = uint8_t(ctype);
    ihdr[10] = ihdr[11] = ihdr[12] = 0;
    put_chunk(png, "IHDR", ihdr, 13);
    if (ctype == 3) put_chunk(png, "PLTE", palette_rgb, size_t(entries) * 3);
    put_chunk(png, "IDAT", z.data(), size_t(zn));
    put_chunk(png, "IEND", nullptr, 0);
    if (int64_t(png.size()) > capacity) return set_error(RSB_E_INVALID, "png_encode: output buffer too small (%lld > %lld)", (long long)png.size(), (long long)capacity);
    memcpy(out, png.data(), png.size());
    return int64_t(png.size());
}

// scanlines with filter type 0 (what PIL writes for palette images) of `bytes_per_row`-byte rows
std::vector<uint8_t> unfiltered_scanlines(const uint8_t* pixels, size_t bytes_per_row, int32_t h) {
    std::vector<uint8_t> raw(size_t(h) * (bytes_per_row + 1));
    for (int y = 0; y < h; ++y) {
        raw[size_t(y) * (bytes_per_row + 1)] = 0;
        memcpy(&raw[size_t(y) * (bytes_per_row + 1) + 1], pixels + size_t(y) * bytes_per_row, bytes_per_row);
    }
    return raw;
}

}  // namespace

extern "C" int64_t rsb_png_encode_p8(const uint8_t* pixels, int32_t w, int32_t h, const uint8_t* palette_rgb, int32_t entries, int32_t level,
                                     uint8_t* out, int64_t capacity) {
    if (!pixels || !out || w <= 0 || h <= 0 || !palette_rgb || entries < 1 || entries > 256) return set_error(RSB_E_INVALID, "png_encode: bad arguments");
    return encode_scanlines(unfiltered_scanlines(pixels, size_t(w), h), w, h, 3, palette_rgb, entries, level, out, capacity);
}

extern "C" int64_t rsb_png_encode_rgb8(const uint8_t* pixels, int32_t w, int32_t h, int32_t level, uint8_t* out, int64_t capacity) {
    if (!pixels || !out || w <= 0 || h <= 0) return set_error(RSB_E_INVALID, "png_encode_rgb8: bad arguments");
    return encode_scanlines(unfiltered_scanlines(pixels, size_t(w) * 3, h), w, h, 2, nullptr, 0, level, out, capacity);
}

namespace {

// encode with `encode` into a buffer of `cap` bytes, then write the file
template <typename Encode>
int write_encoded(const char* path, int64_t cap, Encode&& encode) {
    if (!path) return set_error(RSB_E_INVALID, "png_write: null path");
    std::vector<uint8_t> buf(size_t(cap > 0 ? cap : 4096));
    const int64_t n = encode(buf.data(), int64_t(buf.size()));
    if (n < 0) return int(n);
    FILE* f = fopen(path, "wb");
    if (!f) return set_error(RSB_E_INVALID, "png_write: cannot open %s", path);
    const size_t put = fwrite(buf.data(), 1, size_t(n), f);
    if (fclose(f) != 0 || put != size_t(n)) return set_error(RSB_E_INVALID, "png_write: short write to %s", path);
    return RSB_OK;
}

// an upper bound of the encoded size of `bytes` pixel bytes in h rows (deflate's stored-block worst case plus the chunks)
int64_t encoded_capacity(int64_t bytes, int32_t h) { return bytes + int64_t(h) + 4096 + bytes / 512; }

}  // namespace

extern "C" int rsb_png_write_p8(const char* path, const uint8_t* pixels, int32_t w, int32_t h, const uint8_t* palette_rgb, int32_t entries, int32_t level) {
    return write_encoded(path, encoded_capacity(int64_t(w) * h, h), [&](uint8_t* out, int64_t cap) {
        return rsb_png_encode_p8(pixels, w, h, palette_rgb, entries, level, out, cap);
    });
}

extern "C" int rsb_zlib_inflate(const uint8_t* stream, int64_t n, uint8_t* out, int64_t out_len) {
    if (!stream || !out || n < 6 || out_len < 0) return set_error(RSB_E_INVALID, "zlib_inflate: bad arguments");
    std::vector<uint8_t> in(size_t(n) + kInflateInPad, 0), buf(size_t(out_len) + kInflateOutPad);
    memcpy(in.data(), stream, size_t(n));
    const int rc = rsb_inflate_zlib_padded(in.data(), size_t(n), buf.data(), size_t(out_len));
    if (rc) return set_error(RSB_E_INVALID, "zlib_inflate: stream rejected (%d)", rc);
    memcpy(out, buf.data(), size_t(out_len));
    return RSB_OK;
}

namespace {

struct PngHeader {
    uint32_t w = 0, h = 0;
    int depth = 0, ctype = -1, interlace = 0;
    uint8_t pal[768];
    int npal = 0;
};

// walk the chunks of a PNG file: IHDR and PLTE into `hd`, the IDAT payload into `idat`; every other chunk (tRNS included) is
// skipped, as PIL's convert("RGB") and convert("P") of such files ignore it
int parse_chunks(const uint8_t* data, int64_t n, PngHeader& hd, std::vector<uint8_t>& idat) {
    if (!data || n < 8 + 25) return set_error(RSB_E_INVALID, "png_decode: bad arguments");
    if (memcmp(data, kSig, 8) != 0) return set_error(RSB_E_UNSUPPORTED, "png_decode: not a PNG");
    int64_t at = 8;
    idat.clear();
    bool end = false;
    while (!end && at + 12 <= n) {
        const uint32_t len = be32(data + at);
        const uint8_t* type = data + at + 4;
        const uint8_t* body = data + at + 8;
        if (at + 12 + int64_t(len) > n) return set_error(RSB_E_INVALID, "png_decode: truncated chunk");
        if (!memcmp(type, "IHDR", 4)) {
            if (len != 13) return set_error(RSB_E_INVALID, "png_decode: bad IHDR");
            hd.w = be32(body);
            hd.h = be32(body + 4);
            hd.depth = body[8];
            hd.ctype = body[9];
            hd.interlace = body[12];
        } else if (!memcmp(type, "PLTE", 4)) {
            hd.npal = int(len / 3) > 256 ? 256 : int(len / 3);
            memcpy(hd.pal, body, size_t(hd.npal) * 3);
        } else if (!memcmp(type, "IDAT", 4)) {
            idat.insert(idat.end(), body, body + len);
        } else if (!memcmp(type, "IEND", 4)) {
            end = true;
        }
        at += 12 + int64_t(len);
    }
    if (hd.ctype < 0 || idat.empty()) return set_error(RSB_E_INVALID, "png_decode: missing IHDR / IDAT");
    return RSB_OK;
}

// the zlib stream of the IDAT chunks -> exactly raw_size bytes of filtered scanlines in `raw` (padded for the inflater)
int inflate_scanlines(std::vector<uint8_t>& idat, std::vector<uint8_t>& raw, size_t raw_size) {
    if (raw.size() < raw_size + kInflateOutPad) raw.resize(raw_size + kInflateOutPad);
    // the library's own inflate (csrc/rsb_inflate.cpp: ~3x zlib's rate on literal-heavy PNG data); any stream it rejects -- and
    // everything when RSB_INFLATE=zlib -- goes through zlib, whose verdict is final
    const size_t idat_size = idat.size();
    idat.resize(idat_size + kInflateInPad, 0);
    if (!use_own_inflate() || rsb_inflate_zlib_padded(idat.data(), idat_size, raw.data(), raw_size) != 0) {
        uLongf rn = uLongf(raw_size);
        const int zr = uncompress(raw.data(), &rn, idat.data(), uLong(idat_size));
        if (zr != Z_OK || rn != raw_size) return set_error(RSB_E_INVALID, "png_decode: inflate failed (%d) or size mismatch", zr);
    }
    return RSB_OK;
}

// undo one scanline's filter in place: `cur` holds `stride` bytes of `bpp`-byte pixels, `up` the unfiltered line above
int unfilter_line(uint8_t* cur, const uint8_t* up, size_t stride, int bpp, int ft) {
    switch (ft) {
        case 0: break;
        case 1:
            for (size_t i = bpp; i < stride; ++i) cur[i] = uint8_t(cur[i] + cur[i - bpp]);
            break;
        case 2:
            for (size_t i = 0; i < stride; ++i) cur[i] = uint8_t(cur[i] + up[i]);
            break;
        case 3:
            for (size_t i = 0; i < size_t(bpp); ++i) cur[i] = uint8_t(cur[i] + (up[i] >> 1));
            for (size_t i = bpp; i < stride; ++i) cur[i] = uint8_t(cur[i] + ((cur[i - bpp] + up[i]) >> 1));
            break;
        case 4:
            for (size_t i = 0; i < size_t(bpp); ++i) cur[i] = uint8_t(cur[i] + up[i]);
            for (size_t i = bpp; i < stride; ++i) cur[i] = uint8_t(cur[i] + paeth(cur[i - bpp], up[i], up[i - bpp]));
            break;
        default: return set_error(RSB_E_INVALID, "png_decode: bad filter type %d", ft);
    }
    return RSB_OK;
}

}  // namespace

extern "C" int rsb_png_decode_rgb(const uint8_t* data, int64_t n, uint8_t* out_rgb, int32_t w_expected, int32_t h_expected) {
    if (!data || !out_rgb || n < 8 + 25) return set_error(RSB_E_INVALID, "png_decode: bad arguments");
    // scratch that lives as long as the calling thread: fresh 0.7 MB vectors per tile cost ~0.3 ms of page faults and zeroing
    static thread_local std::vector<uint8_t> tl_idat, tl_raw;
    std::vector<uint8_t>&idat = tl_idat, &raw = tl_raw;  // one TLS lookup each, not one per use
    PngHeader hd;
    int rc = parse_chunks(data, n, hd, idat);
    if (rc != RSB_OK) return rc;
    const uint32_t w = hd.w, h = hd.h;
    const int ctype = hd.ctype, npal = hd.npal;
    const uint8_t* pal = hd.pal;
    if (hd.depth != 8 || hd.interlace != 0 || !(ctype == 0 || ctype == 2 || ctype == 3 || ctype == 4 || ctype == 6))
        return set_error(RSB_E_UNSUPPORTED, "png_decode: only 8-bit non-interlaced gray / RGB / palette / +alpha PNGs (depth %d, colour type %d, interlace %d)", hd.depth, ctype, hd.interlace);
    if (ctype == 3 && npal == 0) return set_error(RSB_E_INVALID, "png_decode: palette image without PLTE");
    if (int32_t(w) != w_expected || int32_t(h) != h_expected)
        return set_error(RSB_E_INVALID, "png_decode: image is %ux%u, expected %dx%d", w, h, w_expected, h_expected);
    const int bpp = ctype == 0 ? 1 : (ctype == 2 ? 3 : (ctype == 3 ? 1 : (ctype == 4 ? 2 : 4)));
    const size_t stride = size_t(w) * bpp;
    const size_t raw_size = size_t(h) * (stride + 1);
    rc = inflate_scanlines(idat, raw, raw_size);
    if (rc != RSB_OK) return rc;
    if (ctype == 2) {
        // RGB (every slippy-map tile): undo the filters while moving the scanlines into the output, the row above is read from there
        static thread_local std::vector<uint8_t> tl_zero_row;
        std::vector<uint8_t>& zero_row = tl_zero_row;
        if (zero_row.size() < stride) zero_row.assign(stride, 0);
        const uint8_t* const raw_base = raw.data();
        for (uint32_t y = 0; y < h; ++y) {
            const uint8_t* __restrict src = raw_base + size_t(y) * (stride + 1);
            const int ft = *src++;
            uint8_t* __restrict o = out_rgb + size_t(y) * stride;
            const uint8_t* __restrict up = y ? o - stride : zero_row.data();
            switch (ft) {
                case 0: memcpy(o, src, stride); break;
                case 1: {
                    uint8_t a = src[0], b = src[1], c = src[2];
                    o[0] = a;
                    o[1] = b;
                    o[2] = c;
                    for (size_t i = 3; i + 2 < stride; i += 3) {  // three independent running sums
                        a = uint8_t(a + src[i]);
                        b = uint8_t(b + src[i + 1]);
                        c = uint8_t(c + src[i + 2]);
                        o[i] = a;
                        o[i + 1] = b;
                        o[i + 2] = c;
                    }
                    break;
                }
                case 2:
                    for (size_t i = 0; i < stride; ++i) o[i] = uint8_t(src[i] + up[i]);  // vectorises
                    break;
                case 3:
                    for (size_t i = 0; i < 3; ++i) o[i] = uint8_t(src[i] + (up[i] >> 1));
                    for (size_t i = 3; i < stride; ++i) o[i] = uint8_t(src[i] + ((o[i - 3] + up[i]) >> 1));
                    break;
                case 4:
                    for (size_t i = 0; i < 3; ++i) o[i] = uint8_t(src[i] + up[i]);
                    for (size_t i = 3; i < stride; ++i) o[i] = uint8_t(src[i] + paeth(o[i - 3], up[i], up[i - 3]));
                    break;
                default: return set_error(RSB_E_INVALID, "png_decode: bad filter type %d", ft);
            }
        }
        return RSB_OK;
    }
    // every other colour type: undo the per-scanline filters in place, then convert
    std::vector<uint8_t> zero(stride, 0);
    for (uint32_t y = 0; y < h; ++y) {
        uint8_t* line = &raw[size_t(y) * (stride + 1)];
        uint8_t* cur = line + 1;
        rc = unfilter_line(cur, y ? cur - (stride + 1) : zero.data(), stride, bpp, line[0]);
        if (rc != RSB_OK) return rc;
        uint8_t* o = out_rgb + size_t(y) * w * 3;
        switch (ctype) {
            case 2: memcpy(o, cur, stride); break;
            case 6:
                for (uint32_t x = 0; x < w; ++x) {
                    o[3 * x] = cur[4 * x];
                    o[3 * x + 1] = cur[4 * x + 1];
                    o[3 * x + 2] = cur[4 * x + 2];
                }
                break;
            case 0:
                for (uint32_t x = 0; x < w; ++x) o[3 * x] = o[3 * x + 1] = o[3 * x + 2] = cur[x];
                break;
            case 4:
                for (uint32_t x = 0; x < w; ++x) o[3 * x] = o[3 * x + 1] = o[3 * x + 2] = cur[2 * x];
                break;
            default:  // palette: indices past the palette map to black like PIL
                for (uint32_t x = 0; x < w; ++x) {
                    const int k = cur[x];
                    if (k < npal) {
                        o[3 * x] = pal[3 * k];
                        o[3 * x + 1] = pal[3 * k + 1];
                        o[3 * x + 2] = pal[3 * k + 2];
                    } else {
                        o[3 * x] = o[3 * x + 1] = o[3 * x + 2] = 0;
                    }
                }
        }
    }
    return RSB_OK;
}

extern "C" int rsb_png_read_rgb(const char* path, uint8_t* out_rgb, int32_t w_expected, int32_t h_expected) {
    if (!path) return set_error(RSB_E_INVALID, "png_read: null path");
    static thread_local std::vector<uint8_t> tl_buf;
    std::vector<uint8_t>& buf = tl_buf;
    if (!read_file(path, buf)) return set_error(RSB_E_INVALID, "png_read: cannot read %s", path);
    return rsb_png_decode_rgb(buf.data(), int64_t(buf.size()), out_rgb, w_expected, h_expected);
}

extern "C" int rsb_png_decode_indexed(const uint8_t* data, int64_t n, uint8_t* out_index, uint8_t* out_palette_rgb, int32_t* entries,
                                      int32_t w_expected, int32_t h_expected) {
    if (!data || !out_index || !out_palette_rgb || !entries || n < 8 + 25) return set_error(RSB_E_INVALID, "png_decode_indexed: bad arguments");
    static thread_local std::vector<uint8_t> tl_idat, tl_raw;
    std::vector<uint8_t>&idat = tl_idat, &raw = tl_raw;
    PngHeader hd;
    int rc = parse_chunks(data, n, hd, idat);
    if (rc != RSB_OK) return rc;
    const int depth = hd.depth;
    const bool palette = hd.ctype == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8);
    if (hd.interlace != 0 || !(palette || (hd.ctype == 0 && depth == 8)))
        return set_error(RSB_E_UNSUPPORTED, "png_decode_indexed: only non-interlaced palette (1/2/4/8-bit) and 8-bit gray PNGs (depth %d, colour type %d, interlace %d)",
                         depth, hd.ctype, hd.interlace);
    if (palette && hd.npal == 0) return set_error(RSB_E_INVALID, "png_decode: palette image without PLTE");
    const uint32_t w = hd.w, h = hd.h;
    if (int32_t(w) != w_expected || int32_t(h) != h_expected)
        return set_error(RSB_E_INVALID, "png_decode: image is %ux%u, expected %dx%d", w, h, w_expected, h_expected);
    const size_t stride = (size_t(w) * depth + 7) / 8;
    rc = inflate_scanlines(idat, raw, size_t(h) * (stride + 1));
    if (rc != RSB_OK) return rc;
    std::vector<uint8_t> zero(stride, 0);
    const int mask = (1 << depth) - 1;
    for (uint32_t y = 0; y < h; ++y) {
        uint8_t* line = &raw[size_t(y) * (stride + 1)];
        uint8_t* cur = line + 1;
        rc = unfilter_line(cur, y ? cur - (stride + 1) : zero.data(), stride, 1, line[0]);
        if (rc != RSB_OK) return rc;
        uint8_t* o = out_index + size_t(y) * w;
        if (depth == 8) {
            memcpy(o, cur, w);
        } else {  // packed indices, leftmost pixel in the high bits
            for (uint32_t x = 0; x < w; ++x) {
                const size_t bit = size_t(x) * depth;
                o[x] = uint8_t((cur[bit >> 3] >> (8 - depth - int(bit & 7))) & mask);
            }
        }
    }
    // PIL's convert("P"): a palette image keeps its PLTE; a gray one gets the gray ramp (index = value)
    if (palette) {
        memset(out_palette_rgb, 0, 768);
        memcpy(out_palette_rgb, hd.pal, size_t(hd.npal) * 3);
        *entries = hd.npal;
    } else {
        for (int i = 0; i < 256; ++i) out_palette_rgb[3 * i] = out_palette_rgb[3 * i + 1] = out_palette_rgb[3 * i + 2] = uint8_t(i);
        *entries = 256;
    }
    return RSB_OK;
}

extern "C" int rsb_png_read_indexed(const char* path, uint8_t* out_index, uint8_t* out_palette_rgb, int32_t* entries, int32_t w_expected, int32_t h_expected) {
    if (!path) return set_error(RSB_E_INVALID, "png_read: null path");
    static thread_local std::vector<uint8_t> tl_buf;
    std::vector<uint8_t>& buf = tl_buf;
    if (!read_file(path, buf)) return set_error(RSB_E_INVALID, "png_read: cannot read %s", path);
    return rsb_png_decode_indexed(buf.data(), int64_t(buf.size()), out_index, out_palette_rgb, entries, w_expected, h_expected);
}

// ---------------------------------------------------------------------------------------------------------------------
// Batch entry points: one call per tile batch, fanned out over `threads` std::threads inside the library. The Python tools
// submit ONE job per batch to their pool instead of one future per tile (2 x 1024 futures per 1024 tiles cost the main thread
// of `rs predict` more than the GPU needed for the network).
namespace {

template <typename F>
void parallel_for(int n, int threads, F&& fn) {
    if (threads < 1) threads = 1;
    if (threads > n) threads = n;
    if (threads <= 1) {
        for (int i = 0; i < n; ++i) fn(i);
        return;
    }
    std::atomic<int> next(0);
    std::vector<std::thread> pool;
    pool.reserve(size_t(threads));
    for (int t = 0; t < threads; ++t)
        pool.emplace_back([&]() {
            for (int i = next.fetch_add(1); i < n; i = next.fetch_add(1)) fn(i);
        });
    for (auto& th : pool) th.join();
}

// mkdir -p of the directory part of `path`
void make_parent_dirs(const char* path) {
    std::string p(path);
    for (size_t i = 1; i < p.size(); ++i) {
        if (p[i] == '/') {
            p[i] = 0;
            mkdir(p.c_str(), 0777);  // EEXIST is fine; a real failure shows up when the file is opened
            p[i] = '/';
        }
    }
}

}  // namespace

extern "C" int rsb_png_read_rgb_batch(const char* const* paths, int32_t n, uint8_t* const* outs_rgb, int32_t w_expected, int32_t h_expected,
                                      int32_t threads, int32_t* rcs) {
    if (!paths || !outs_rgb || !rcs || n < 0) return set_error(RSB_E_INVALID, "png_read_batch: bad arguments");
    parallel_for(n, threads, [&](int i) { rcs[i] = rsb_png_read_rgb(paths[i], outs_rgb[i], w_expected, h_expected); });
    int worst = RSB_OK;
    for (int i = 0; i < n; ++i)
        if (rcs[i] != RSB_OK && rcs[i] != RSB_E_UNSUPPORTED) worst = rcs[i];
    return worst;  // per-file codes in rcs (RSB_E_UNSUPPORTED entries are the caller's to decode with another library)
}

extern "C" int rsb_png_write_p8_batch(const char* const* paths, int32_t n, const uint8_t* pixels, int64_t image_stride, int32_t w, int32_t h,
                                      const uint8_t* palette_rgb, int32_t entries, int32_t level, int32_t threads, int32_t make_dirs) {
    if (!paths || !pixels || n < 0 || image_stride < int64_t(w) * h) return set_error(RSB_E_INVALID, "png_write_batch: bad arguments");
    std::vector<int> rc(size_t(n), RSB_OK);
    parallel_for(n, threads, [&](int i) {
        if (make_dirs) make_parent_dirs(paths[i]);
        rc[size_t(i)] = rsb_png_write_p8(paths[i], pixels + int64_t(i) * image_stride, w, h, palette_rgb, entries, level);
    });
    for (int i = 0; i < n; ++i)
        if (rc[size_t(i)] != RSB_OK) return set_error(rc[size_t(i)], "png_write_batch: writing %s failed", paths[i]);
    return RSB_OK;
}

extern "C" int rsb_png_read_indexed_batch(const char* const* paths, int32_t n, uint8_t* const* outs_index, uint8_t* palettes_rgb, int32_t* entries,
                                          int32_t w_expected, int32_t h_expected, int32_t threads, int32_t* rcs) {
    if (!paths || !outs_index || !palettes_rgb || !entries || !rcs || n < 0) return set_error(RSB_E_INVALID, "png_read_indexed_batch: bad arguments");
    parallel_for(n, threads, [&](int i) {
        rcs[i] = rsb_png_read_indexed(paths[i], outs_index[i], palettes_rgb + size_t(i) * 768, entries + i, w_expected, h_expected);
    });
    int worst = RSB_OK;
    for (int i = 0; i < n; ++i)
        if (rcs[i] != RSB_OK && rcs[i] != RSB_E_UNSUPPORTED) worst = rcs[i];
    return worst;
}

extern "C" int rsb_png_write_rgb8_batch(const char* const* paths, int32_t n, const uint8_t* pixels, int64_t image_stride, int32_t w, int32_t h,
                                        int32_t level, int32_t threads, int32_t make_dirs) {
    if (!paths || !pixels || n < 0 || w <= 0 || h <= 0 || image_stride < int64_t(w) * h * 3) return set_error(RSB_E_INVALID, "png_write_rgb8_batch: bad arguments");
    std::vector<int> rc(size_t(n), RSB_OK);
    parallel_for(n, threads, [&](int i) {
        if (make_dirs) make_parent_dirs(paths[i]);
        const uint8_t* image = pixels + int64_t(i) * image_stride;
        rc[size_t(i)] = write_encoded(paths[i], encoded_capacity(int64_t(w) * h * 3, h), [&](uint8_t* out, int64_t cap) {
            return rsb_png_encode_rgb8(image, w, h, level, out, cap);
        });
    });
    for (int i = 0; i < n; ++i)
        if (rc[size_t(i)] != RSB_OK) return set_error(rc[size_t(i)], "png_write_rgb8_batch: writing %s failed", paths[i]);
    return RSB_OK;
}
