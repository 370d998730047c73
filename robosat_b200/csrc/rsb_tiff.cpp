// Host side of `rs tile` and `rs mosaic` (DESIGN.md §8): decoding a window of a TIFF's strips or tiles into a caller's buffer (8-bit
// chunky, or under the band rule 8- or 16-bit, chunky or planar, with a selection of bands), and deflating the square tiles of a
// window of a 1-band 8-bit raster. Plain C++, no Python, no interpreter lock; the chunks of a window are decoded or compressed on the
// library's own threads.
//
// The IFD and GeoKey parsing stay in Python (robosat_b200/geotiff.py); this file sees the raster through its chunk table. Each chunk
// is decoded into a per-thread scratch (inflate through the library's DEFLATE decoder, or LZW), predictor 2 is undone on its rows,
// and the part of the chunk inside the window is copied out. Chunks are disjoint in the output, so the threads never share bytes.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <thread>
#include <vector>

#include "../../include/rsb200.h"
#include "rsb_host.h"
#include "rsb_inflate.h"
#include <zlib.h>

using rsb::set_error;

namespace {

// per-chunk failure codes; the first bad chunk is named in the error message
enum ChunkError {
    kOk = 0,
    kOutsideFile,      // offset + byte count beyond the end of the file
    kShortRaw,         // an uncompressed chunk holds fewer bytes than its pixels need
    kDeflateTruncated, // the DEFLATE stream ran out of input
    kDeflateInvalid,   // the zlib header or the DEFLATE stream is invalid
    kDeflateShort,     // the stream ended before the chunk's pixels
    kDeflateChecksum,  // Adler-32 mismatch
    kLzwBadCode,       // an LZW code past the table
    kLzwTruncated,     // the LZW stream ended before the chunk's pixels
    kLzwOldStyle,      // LSB-first (pre-TIFF 6) LZW
};

const char* chunk_error_text(int e) {
    switch (e) {
        case kOutsideFile: return "extends beyond the end of the file";
        case kShortRaw: return "holds fewer bytes than its pixels";
        case kDeflateTruncated: return "deflate stream truncated";
        case kDeflateInvalid: return "invalid deflate stream";
        case kDeflateShort: return "deflate stream ended before the chunk's pixels";
        case kDeflateChecksum: return "deflate stream fails its Adler-32 checksum";
        case kLzwBadCode: return "bad LZW code";
        case kLzwTruncated: return "LZW stream ended before the chunk's pixels";
        case kLzwOldStyle: return "old-style (LSB-first) LZW is not supported";
        default: return "unknown error";
    }
}

// TIFF 6.0 LZW (MSB-first codes of 9 to 12 bits, Clear = 256, EndOfInformation = 257, widths grow one code early, as libtiff
// writes them) -> exactly out_len bytes; bytes past out_len are dropped, as libtiff does
int lzw_decode(const uint8_t* in, size_t n, uint8_t* out, size_t out_len) {
    if (n >= 2 && in[0] == 0 && (in[1] & 1)) return kLzwOldStyle;
    static thread_local std::vector<uint16_t> prefix(4096);
    static thread_local std::vector<uint8_t> suffix(4096), first(4096);
    static thread_local std::vector<uint16_t> length(4096);
    for (int i = 0; i < 256; ++i) {
        prefix[i] = 0xffff;
        suffix[i] = uint8_t(i);
        first[i] = uint8_t(i);
        length[i] = 1;
    }
    size_t at = 0, bitpos = 0;
    const size_t nbits = n * 8;
    int width = 9, next = 258, prev = -1;
    while (at < out_len) {
        if (bitpos + size_t(width) > nbits) return kLzwTruncated;
        int code = 0;
        for (int b = 0; b < width; ++b, ++bitpos) code = (code << 1) | ((in[bitpos >> 3] >> (7 - (bitpos & 7))) & 1);
        if (code == 257) break;
        if (code == 256) {
            width = 9;
            next = 258;
            prev = -1;
            continue;
        }
        int emit;  // the code whose string is written; for code == next it is prev's string plus its first byte
        if (prev < 0) {
            if (code > 255) return kLzwBadCode;
            emit = code;
        } else if (code < next) {
            emit = code;
        } else if (code == next && next < 4096) {
            emit = prev;
        } else {
            return kLzwBadCode;
        }
        const int len = length[size_t(emit)];
        // the string of `emit`, written backwards from its last byte; bytes past out_len are not written
        for (int c = emit, k = len - 1; c != 0xffff; c = prefix[size_t(c)], --k)
            if (at + size_t(k) < out_len) out[at + size_t(k)] = suffix[size_t(c)];
        at += size_t(len);
        if (prev >= 0 && code == next) {
            if (at < out_len) out[at] = first[size_t(prev)];
            ++at;
        }
        if (prev >= 0 && next < 4096) {
            prefix[size_t(next)] = uint16_t(prev);
            suffix[size_t(next)] = first[size_t(code == next ? prev : code)];
            first[size_t(next)] = first[size_t(prev)];
            length[size_t(next)] = uint16_t(length[size_t(prev)] + 1);
            ++next;
            if (next >= (1 << width) - 1 && width < 12) ++width;
        }
        prev = code;
    }
    return at >= out_len ? kOk : kLzwTruncated;
}

template <class F>
void parallel_for(int64_t n, int threads, F&& fn) {
    if (threads < 1) threads = 1;
    if (threads > n) threads = int(n);
    if (threads <= 1) {
        for (int64_t i = 0; i < n; ++i) fn(i);
        return;
    }
    std::atomic<int64_t> next(0);
    std::vector<std::thread> pool;
    pool.reserve(size_t(threads));
    for (int t = 0; t < threads; ++t)
        pool.emplace_back([&]() {
            for (int64_t i = next.fetch_add(1); i < n; i = next.fetch_add(1)) fn(i);
        });
    for (auto& th : pool) th.join();
}

// The per-chunk decode both entry points share. A unit is one chunk of the window's chunk rectangle in one plane (planar 2: one per
// distinct selected band; planar 1: plane 0 holds every band). Its pixels are decoded into a per-thread scratch, byte-swapped to
// the host's order (16-bit), predictor 2 is undone on whole samples up to the window's last column, and the window's part is
// gathered into out [rows][cols][k] (copied whole rows at a time when the selection is every band in order).
struct Decode {
    const char* fn;
    const uint8_t* file;
    int64_t file_len;
    const int64_t *offsets, *counts;
    int64_t width, height;
    int32_t chunk_w, chunk_h, tiled, spp, bits, planar, swap, compression, predictor;
    const int32_t* select;
    int32_t k;
    int64_t row0, rows, col0, cols;
    uint8_t* out;
    int32_t threads;
    int64_t* bad_chunk;
};

template <class T>
int decode_units(const Decode& d) {
    const int64_t across = d.tiled ? (d.width + d.chunk_w - 1) / d.chunk_w : 1;
    const int64_t down = (d.height + d.chunk_h - 1) / d.chunk_h;
    if (d.bad_chunk) *d.bad_chunk = -1;
    const int64_t cr0 = d.row0 / d.chunk_h, cr1 = (d.row0 + d.rows - 1) / d.chunk_h;
    const int64_t cc0 = d.col0 / d.chunk_w, cc1 = (d.col0 + d.cols - 1) / d.chunk_w;
    const int64_t ncols = cc1 - cc0 + 1, rect = (cr1 - cr0 + 1) * ncols;
    std::vector<int32_t> planes;  // planar 2: the distinct selected bands, ascending
    bool identity = d.planar == 1 && d.k == d.spp;
    for (int32_t j = 0; j < d.k; ++j) {
        identity = identity && d.select[j] == j;
        if (d.planar == 2 && std::find(planes.begin(), planes.end(), d.select[j]) == planes.end()) planes.push_back(d.select[j]);
    }
    std::sort(planes.begin(), planes.end());
    if (d.planar == 1) planes.assign(1, 0);
    const int64_t n = rect * int64_t(planes.size());
    const int sppc = d.planar == 1 ? d.spp : 1;  // samples per pixel inside a chunk
    std::vector<int> rc(size_t(n), kOk);
    parallel_for(n, d.threads, [&](int64_t u) {
        const int32_t plane = planes[size_t(u / rect)];
        const int64_t k = u % rect, cr = cr0 + k / ncols, cc = cc0 + k % ncols;
        const int64_t idx = (d.planar == 2 ? plane * across * down : 0) + cr * across + cc;
        // a strip's last chunk holds only the raster's remaining rows; a tile is always chunk_w x chunk_h
        const int64_t crows = d.tiled ? d.chunk_h : std::min<int64_t>(d.chunk_h, d.height - cr * d.chunk_h);
        const size_t row_bytes = size_t(d.chunk_w) * size_t(sppc) * sizeof(T), need = size_t(crows) * row_bytes;
        const int64_t off = d.offsets[idx], len = d.counts[idx];
        if (off < 0 || len < 0 || off > d.file_len || len > d.file_len - off) {
            rc[size_t(u)] = kOutsideFile;
            return;
        }
        static thread_local std::vector<uint8_t> in, buf;
        const uint8_t* px;
        int e = kOk;
        if (d.compression == 1) {
            if (size_t(len) < need) e = kShortRaw;
            px = d.file + off;
            if ((d.predictor == 2 || sizeof(T) > 1) && e == kOk) {  // changed in place, or read as aligned 16-bit samples
                buf.assign(d.file + off, d.file + off + need);
                px = buf.data();
            }
        } else if (d.compression == 5) {
            buf.resize(need);
            e = lzw_decode(d.file + off, size_t(len), buf.data(), need);
            px = buf.data();
        } else {
            in.assign(size_t(len) + rsb::kInflateInPad, 0);
            memcpy(in.data(), d.file + off, size_t(len));
            buf.resize(need + rsb::kInflateOutPad);
            const int z = rsb::rsb_inflate_zlib_padded(in.data(), size_t(len), buf.data(), need);
            e = z == 0 ? kOk : z == -2 ? kDeflateTruncated : z == -4 ? kDeflateShort : z == -5 ? kDeflateChecksum : kDeflateInvalid;
            px = buf.data();
        }
        if (e != kOk) {
            rc[size_t(u)] = e;
            return;
        }
        // the chunk's rows and columns inside the window
        const int64_t y0 = std::max<int64_t>(d.row0, cr * d.chunk_h), y1 = std::min<int64_t>(d.row0 + d.rows, cr * d.chunk_h + crows);
        const int64_t x0 = std::max<int64_t>(d.col0, cc * d.chunk_w), x1 = std::min<int64_t>(d.col0 + d.cols, std::min<int64_t>(d.width, cc * d.chunk_w + d.chunk_w));
        T* const out = reinterpret_cast<T*>(d.out);
        for (int64_t y = y0; y < y1; ++y) {
            T* row = reinterpret_cast<T*>(const_cast<uint8_t*>(px) + size_t(y - cr * d.chunk_h) * row_bytes);
            const size_t end = size_t(x1 - cc * d.chunk_w) * size_t(sppc);
            if (sizeof(T) == 2 && d.swap)
                for (size_t i = 0; i < end; ++i) row[i] = T((row[i] >> 8) | (row[i] << 8));
            if (d.predictor == 2)  // horizontal differencing, sample by sample, modulo 2^bits (undone up to the window's last column)
                for (size_t i = size_t(sppc); i < end; ++i) row[i] = T(row[i] + row[i - size_t(sppc)]);
            T* o = out + (size_t(y - d.row0) * size_t(d.cols) + size_t(x0 - d.col0)) * size_t(d.k);
            const T* r = row + size_t(x0 - cc * d.chunk_w) * size_t(sppc);
            if (identity) {
                memcpy(o, r, size_t(x1 - x0) * size_t(d.k) * sizeof(T));
            } else if (d.planar == 1) {
                for (int64_t x = 0; x < x1 - x0; ++x, o += d.k, r += sppc)
                    for (int32_t j = 0; j < d.k; ++j) o[j] = r[d.select[j]];
            } else {
                for (int32_t j = 0; j < d.k; ++j)
                    if (d.select[j] == plane)
                        for (int64_t x = 0; x < x1 - x0; ++x) o[x * d.k + j] = r[x];
            }
        }
    });
    for (int64_t u = 0; u < n; ++u) {
        if (rc[size_t(u)] == kOk) continue;
        const int64_t k = u % rect, cr = cr0 + k / ncols, cc = cc0 + k % ncols;
        const int64_t idx = (d.planar == 2 ? planes[size_t(u / rect)] * across * down : 0) + cr * across + cc;
        if (d.bad_chunk) *d.bad_chunk = idx;
        return set_error(RSB_E_INVALID, "%s: %s %lld (offset %lld, %lld bytes): %s", d.fn, d.tiled ? "tile" : "strip", (long long)idx,
                         (long long)d.offsets[idx], (long long)d.counts[idx], chunk_error_text(rc[size_t(u)]));
    }
    return RSB_OK;
}

// the checks of the raster, the chunk table size and the window both entry points make
int check_window(const char* fn, const uint8_t* file, int64_t file_len, const int64_t* chunk_offsets, const int64_t* chunk_bytes, const void* out,
                 int64_t num_chunks, int64_t planes, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled,
                 int32_t compression, int32_t predictor, int64_t row0, int64_t rows, int64_t col0, int64_t cols) {
    if (!file || !chunk_offsets || !chunk_bytes || !out || file_len < 0) return set_error(RSB_E_INVALID, "%s: null pointer", fn);
    if (width < 1 || height < 1 || chunk_w < 1 || chunk_h < 1 || (!tiled && chunk_w != width))
        return set_error(RSB_E_INVALID, "%s: raster %lld x %lld with chunks %d x %d (tiled %d)", fn, (long long)width, (long long)height, chunk_w,
                         chunk_h, tiled);
    if (compression != 1 && compression != 5 && compression != 8 && compression != 32946)
        return set_error(RSB_E_INVALID, "%s: compression %d (need 1, 5, 8 or 32946)", fn, compression);
    if (predictor != 1 && predictor != 2) return set_error(RSB_E_INVALID, "%s: predictor %d (need 1 or 2)", fn, predictor);
    const int64_t across = tiled ? (width + chunk_w - 1) / chunk_w : 1;
    const int64_t down = (height + chunk_h - 1) / chunk_h;
    if (num_chunks != across * down * planes)
        return set_error(RSB_E_INVALID, "%s: %lld chunks, the raster needs %lld", fn, (long long)num_chunks, (long long)(across * down * planes));
    if (row0 < 0 || col0 < 0 || rows < 1 || cols < 1 || row0 + rows > height || col0 + cols > width)
        return set_error(RSB_E_INVALID, "%s: window rows [%lld, %lld) cols [%lld, %lld) outside the %lld x %lld raster", fn, (long long)row0,
                         (long long)(row0 + rows), (long long)col0, (long long)(col0 + cols), (long long)width, (long long)height);
    return RSB_OK;
}

}  // namespace

extern "C" int rsb_tiff_decode_window(const uint8_t* file, int64_t file_len, const int64_t* chunk_offsets, const int64_t* chunk_bytes,
                                      int64_t num_chunks, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled,
                                      int32_t spp, int32_t compression, int32_t predictor, int64_t row0, int64_t rows, int64_t col0,
                                      int64_t cols, uint8_t* out, int32_t threads, int64_t* bad_chunk) {
    if (spp != 1 && spp != 3 && spp != 4 && file && chunk_offsets && chunk_bytes && out && file_len >= 0)
        return set_error(RSB_E_INVALID, "tiff_decode_window: %d samples per pixel (need 1, 3 or 4)", spp);
    const int rc = check_window("tiff_decode_window", file, file_len, chunk_offsets, chunk_bytes, out, num_chunks, 1, width, height, chunk_w, chunk_h,
                                tiled, compression, predictor, row0, rows, col0, cols);
    if (rc != RSB_OK) return rc;
    const int32_t identity[4] = {0, 1, 2, 3};
    const Decode d = {"tiff_decode_window", file, file_len, chunk_offsets, chunk_bytes, width, height, chunk_w, chunk_h, tiled, spp, 8, 1, 0,
                      compression, predictor, identity, spp, row0, rows, col0, cols, out, threads, bad_chunk};
    return decode_units<uint8_t>(d);
}

extern "C" int rsb_tiff_decode_bands(const uint8_t* file, int64_t file_len, const int64_t* chunk_offsets, const int64_t* chunk_bytes,
                                     int64_t num_chunks, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled,
                                     int32_t spp, int32_t bits, int32_t planar, int32_t big_endian, int32_t compression, int32_t predictor,
                                     const int32_t* select, int32_t k, int64_t row0, int64_t rows, int64_t col0, int64_t cols, void* out,
                                     int32_t threads, int64_t* bad_chunk) {
    if (spp < 1 || spp > 65535 || (bits != 8 && bits != 16) || (planar != 1 && planar != 2))
        return set_error(RSB_E_INVALID, "tiff_decode_bands: %d samples of %d bits, planar %d (need 8 or 16 bits, planar 1 or 2)", spp, bits, planar);
    if (!select || k < 1 || k > 4) return set_error(RSB_E_INVALID, "tiff_decode_bands: %d selected bands (need 1..4)", k);
    for (int32_t j = 0; j < k; ++j)
        if (select[j] < 0 || select[j] >= spp) return set_error(RSB_E_INVALID, "tiff_decode_bands: band %d of a raster of %d", select[j], spp);
    const int rc = check_window("tiff_decode_bands", file, file_len, chunk_offsets, chunk_bytes, out, num_chunks, planar == 2 ? spp : 1, width, height,
                                chunk_w, chunk_h, tiled, compression, predictor, row0, rows, col0, cols);
    if (rc != RSB_OK) return rc;
    const uint16_t probe = 1;
    const int32_t host_big = *reinterpret_cast<const uint8_t*>(&probe) == 0;
    const Decode d = {"tiff_decode_bands", file, file_len, chunk_offsets, chunk_bytes, width, height, chunk_w, chunk_h, tiled, spp, bits, planar,
                      int32_t((big_endian != 0) != (host_big != 0)), compression, predictor, select, k, row0, rows, col0, cols,
                      static_cast<uint8_t*>(out), threads, bad_chunk};
    return bits == 8 ? decode_units<uint8_t>(d) : decode_units<uint16_t>(d);
}

extern "C" int64_t rsb_tiff_deflate_bound(int64_t n) { return n < 0 ? -1 : int64_t(compressBound(uLong(n))); }

extern "C" int rsb_tiff_encode_chunks(const uint8_t* window, int64_t pitch, int32_t rows, int32_t cols, int32_t chunk, int32_t fill, int32_t level,
                                      uint8_t* out, int64_t chunk_cap, int64_t* sizes, int32_t threads) {
    if (!window || !out || !sizes) return set_error(RSB_E_INVALID, "tiff_encode_chunks: null pointer");
    if (chunk < 16 || chunk > 4096 || chunk % 16) return set_error(RSB_E_INVALID, "tiff_encode_chunks: chunk %d (need a multiple of 16 in 16..4096)", chunk);
    if (rows < 1 || rows > chunk || cols < 1 || pitch < cols)
        return set_error(RSB_E_INVALID, "tiff_encode_chunks: window %d x %d, pitch %lld, chunk %d", cols, rows, (long long)pitch, chunk);
    if (fill < 0 || fill > 255 || level < 0 || level > 9) return set_error(RSB_E_INVALID, "tiff_encode_chunks: fill %d, level %d", fill, level);
    const size_t raw = size_t(chunk) * size_t(chunk);
    if (chunk_cap < int64_t(compressBound(uLong(raw))))
        return set_error(RSB_E_INVALID, "tiff_encode_chunks: %lld bytes per chunk, compressBound needs %lld", (long long)chunk_cap,
                         (long long)compressBound(uLong(raw)));
    const int64_t n = (int64_t(cols) + chunk - 1) / chunk;
    std::vector<int> rc(size_t(n), Z_OK);
    parallel_for(n, threads, [&](int64_t k) {
        static thread_local std::vector<uint8_t> buf;
        buf.assign(raw, uint8_t(fill));  // edge chunks are padded with the fill value
        const int64_t c0 = k * chunk, w = std::min<int64_t>(chunk, cols - c0);
        for (int32_t r = 0; r < rows; ++r) memcpy(buf.data() + size_t(r) * size_t(chunk), window + r * pitch + c0, size_t(w));
        uLongf len = uLongf(chunk_cap);
        rc[size_t(k)] = compress2(out + k * chunk_cap, &len, buf.data(), uLong(raw), level);
        sizes[k] = int64_t(len);
    });
    for (int64_t k = 0; k < n; ++k)
        if (rc[size_t(k)] != Z_OK) return set_error(RSB_E_INVALID, "tiff_encode_chunks: compress2 of chunk %lld failed (%d)", (long long)k, rc[size_t(k)]);
    return RSB_OK;
}
