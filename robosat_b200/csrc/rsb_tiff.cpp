// Host side of `rs tile` and `rs mosaic` (DESIGN.md §8): decoding a window of an 8-bit chunky TIFF's strips or tiles into a caller's
// buffer, and deflating the square tiles of a window of a 1-band 8-bit raster. Plain C++, no Python, no interpreter lock; the chunks
// of a window are decoded or compressed on the library's own threads.
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

}  // namespace

extern "C" int rsb_tiff_decode_window(const uint8_t* file, int64_t file_len, const int64_t* chunk_offsets, const int64_t* chunk_bytes,
                                      int64_t num_chunks, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled,
                                      int32_t spp, int32_t compression, int32_t predictor, int64_t row0, int64_t rows, int64_t col0,
                                      int64_t cols, uint8_t* out, int32_t threads, int64_t* bad_chunk) {
    if (!file || !chunk_offsets || !chunk_bytes || !out || file_len < 0) return set_error(RSB_E_INVALID, "tiff_decode_window: null pointer");
    if (width < 1 || height < 1 || chunk_w < 1 || chunk_h < 1 || (!tiled && chunk_w != width))
        return set_error(RSB_E_INVALID, "tiff_decode_window: raster %lld x %lld with chunks %d x %d (tiled %d)", (long long)width,
                         (long long)height, chunk_w, chunk_h, tiled);
    if (spp != 1 && spp != 3 && spp != 4) return set_error(RSB_E_INVALID, "tiff_decode_window: %d samples per pixel (need 1, 3 or 4)", spp);
    if (compression != 1 && compression != 5 && compression != 8 && compression != 32946)
        return set_error(RSB_E_INVALID, "tiff_decode_window: compression %d (need 1, 5, 8 or 32946)", compression);
    if (predictor != 1 && predictor != 2) return set_error(RSB_E_INVALID, "tiff_decode_window: predictor %d (need 1 or 2)", predictor);
    const int64_t across = tiled ? (width + chunk_w - 1) / chunk_w : 1;
    const int64_t down = (height + chunk_h - 1) / chunk_h;
    if (num_chunks != across * down)
        return set_error(RSB_E_INVALID, "tiff_decode_window: %lld chunks, the raster needs %lld", (long long)num_chunks, (long long)(across * down));
    if (row0 < 0 || col0 < 0 || rows < 1 || cols < 1 || row0 + rows > height || col0 + cols > width)
        return set_error(RSB_E_INVALID, "tiff_decode_window: window rows [%lld, %lld) cols [%lld, %lld) outside the %lld x %lld raster",
                         (long long)row0, (long long)(row0 + rows), (long long)col0, (long long)(col0 + cols), (long long)width, (long long)height);
    if (bad_chunk) *bad_chunk = -1;
    const int64_t cr0 = row0 / chunk_h, cr1 = (row0 + rows - 1) / chunk_h;
    const int64_t cc0 = col0 / chunk_w, cc1 = (col0 + cols - 1) / chunk_w;
    const int64_t ncols = cc1 - cc0 + 1, n = (cr1 - cr0 + 1) * ncols;
    std::vector<int> rc(size_t(n), kOk);
    parallel_for(n, threads, [&](int64_t k) {
        const int64_t cr = cr0 + k / ncols, cc = cc0 + k % ncols, idx = cr * across + cc;
        // a strip's last chunk holds only the raster's remaining rows; a tile is always chunk_w x chunk_h
        const int64_t crows = tiled ? chunk_h : std::min<int64_t>(chunk_h, height - cr * chunk_h);
        const size_t row_bytes = size_t(chunk_w) * size_t(spp), need = size_t(crows) * row_bytes;
        const int64_t off = chunk_offsets[idx], len = chunk_bytes[idx];
        if (off < 0 || len < 0 || off > file_len || len > file_len - off) {
            rc[size_t(k)] = kOutsideFile;
            return;
        }
        static thread_local std::vector<uint8_t> in, buf;
        const uint8_t* px;
        int e = kOk;
        if (compression == 1) {
            if (size_t(len) < need) e = kShortRaw;
            px = file + off;
            if (predictor == 2 && e == kOk) {
                buf.assign(file + off, file + off + need);
                px = buf.data();
            }
        } else if (compression == 5) {
            buf.resize(need);
            e = lzw_decode(file + off, size_t(len), buf.data(), need);
            px = buf.data();
        } else {
            in.assign(size_t(len) + rsb::kInflateInPad, 0);
            memcpy(in.data(), file + off, size_t(len));
            buf.resize(need + rsb::kInflateOutPad);
            const int z = rsb::rsb_inflate_zlib_padded(in.data(), size_t(len), buf.data(), need);
            e = z == 0 ? kOk : z == -2 ? kDeflateTruncated : z == -4 ? kDeflateShort : z == -5 ? kDeflateChecksum : kDeflateInvalid;
            px = buf.data();
        }
        if (e != kOk) {
            rc[size_t(k)] = e;
            return;
        }
        // the chunk's rows and columns inside the window
        const int64_t y0 = std::max<int64_t>(row0, cr * chunk_h), y1 = std::min<int64_t>(row0 + rows, cr * chunk_h + crows);
        const int64_t x0 = std::max<int64_t>(col0, cc * chunk_w), x1 = std::min<int64_t>(col0 + cols, std::min<int64_t>(width, cc * chunk_w + chunk_w));
        for (int64_t y = y0; y < y1; ++y) {
            uint8_t* row = const_cast<uint8_t*>(px) + size_t(y - cr * chunk_h) * row_bytes;
            if (predictor == 2) {  // horizontal differencing, sample by sample, modulo 256 (undone up to the window's last column)
                const size_t end = size_t(x1 - cc * chunk_w) * size_t(spp);
                for (size_t i = size_t(spp); i < end; ++i) row[i] = uint8_t(row[i] + row[i - size_t(spp)]);
            }
            memcpy(out + (size_t(y - row0) * size_t(cols) + size_t(x0 - col0)) * size_t(spp), row + size_t(x0 - cc * chunk_w) * size_t(spp),
                   size_t(x1 - x0) * size_t(spp));
        }
    });
    for (int64_t k = 0; k < n; ++k) {
        if (rc[size_t(k)] == kOk) continue;
        const int64_t cr = cr0 + k / ncols, cc = cc0 + k % ncols, idx = cr * across + cc;
        if (bad_chunk) *bad_chunk = idx;
        return set_error(RSB_E_INVALID, "tiff_decode_window: %s %lld (offset %lld, %lld bytes): %s", tiled ? "tile" : "strip", (long long)idx,
                         (long long)chunk_offsets[idx], (long long)chunk_bytes[idx], chunk_error_text(rc[size_t(k)]));
    }
    return RSB_OK;
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
