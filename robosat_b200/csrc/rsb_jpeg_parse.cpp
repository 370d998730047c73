// Host side of the JPEG chunks of `rs tile` and `rs segment` (DESIGN.md §8): the headers of every strip or tile of a Compression 7
// TIFF, parsed on the library's threads over the caller's bytes (a memory map of the file) when the file is opened, so every stream
// outside the rule is refused before any device work. Each chunk gets a descriptor (its entropy-coded byte range, frame, sampling,
// restart interval and block count). The table sets (quantisation tables in natural order and libjpeg's derived Huffman decode
// tables, about 14 KB each) are built only on request, for the chunks of one window: GDAL gives every tile its own optimised Huffman
// tables, so a whole raster has about one set per chunk. tests/jpeg_reference.py restates the same parse.
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <string>
#include <thread>
#include <vector>

#include "../../include/rsb200.h"
#include "rsb_host.h"
#include "rsb_jpeg.h"

using rsb::set_error;
using namespace rsb_jpeg;

namespace {

const uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                              41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// the table slots as defined so far
struct Slots {
    int32_t q[4][64];
    bool qdef[4] = {false, false, false, false};
    uint8_t bits[2][4][17];
    uint8_t vals[2][4][256];
    bool hdef[2][4] = {{false, false, false, false}, {false, false, false, false}};
};

struct Parsed {
    int64_t desc[RSB_JPEG_DESC_FIELDS];
    std::string key;  // the used tables' bytes, in component order
    std::string error;
};

// libjpeg's jpeg_make_d_derived_tbl checks: "" when the table is usable
std::string check_huffman(const uint8_t* bits, const uint8_t* vals, bool dc) {
    int n = 0;
    for (int l = 1; l <= 16; ++l) n += bits[l];
    if (n > 256) return "a Huffman table of " + std::to_string(n) + " codes";
    int code = 0;  // the next free code of each length; using the all-ones code counts as over-subscribed, as in libjpeg
    for (int l = 1; l <= 16; ++l) {
        code += bits[l];
        if (bits[l] && code >= (1 << l)) return "an over-subscribed Huffman table";
        code <<= 1;
    }
    if (dc)
        for (int i = 0; i < n; ++i)
            if (vals[i] > 15) return "a DC Huffman symbol above 15";
    return "";
}

void derive(const uint8_t* bits, const uint8_t* vals, int32_t* t) {
    int huffsize[257], huffcode[257];
    int p = 0;
    for (int l = 1; l <= 16; ++l)
        for (int i = 0; i < bits[l]; ++i) huffsize[p++] = l;
    huffsize[p] = 0;
    const int n = p;
    int code = 0, si = huffsize[0];
    p = 0;
    while (huffsize[p]) {
        while (huffsize[p] == si) huffcode[p++] = code++;
        code <<= 1;
        ++si;
    }
    p = 0;
    for (int l = 1; l <= 16; ++l) {
        if (bits[l]) {
            t[kValoffset + l] = p - huffcode[p];
            p += bits[l];
            t[kMaxcode + l] = huffcode[p - 1];
        } else {
            t[kValoffset + l] = 0;
            t[kMaxcode + l] = -1;
        }
    }
    t[kMaxcode + 0] = -1;
    t[kValoffset + 0] = 0;
    t[kMaxcode + 17] = 0xFFFFF;
    t[kValoffset + 17] = 0;
    for (int i = 0; i < 256; ++i) t[kLookup + i] = 9 << 8;
    p = 0;
    for (int l = 1; l <= 8; ++l)
        for (int i = 0; i < bits[l]; ++i, ++p) {
            const int look = huffcode[p] << (8 - l);
            for (int c = 0; c < (1 << (8 - l)); ++c) t[kLookup + look + c] = (l << 8) | vals[p];
        }
    for (int i = 0; i < 256; ++i) t[kHuffval + i] = i < n ? vals[i] : 0;
}

inline int u16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// DQT / DHT payloads into the slots; "" or what is wrong
std::string read_dqt(const uint8_t* p, int n, Slots& s) {
    for (int i = 0; i < n;) {
        const int pq = p[i] >> 4, tq = p[i] & 15;
        if (pq > 1 || tq > 3) return "DQT precision " + std::to_string(pq) + " slot " + std::to_string(tq);
        const int len = pq ? 128 : 64;
        if (i + 1 + len > n) return "a truncated DQT";
        for (int k = 0; k < 64; ++k) s.q[tq][kNatural[k]] = pq ? u16(p + i + 1 + 2 * k) : p[i + 1 + k];
        s.qdef[tq] = true;
        i += 1 + len;
    }
    return "";
}

std::string read_dht(const uint8_t* p, int n, Slots& s) {
    for (int i = 0; i < n;) {
        const int tc = p[i] >> 4, th = p[i] & 15;
        if (tc > 1 || th > 3) return "DHT class " + std::to_string(tc) + " slot " + std::to_string(th);
        if (i + 17 > n) return "a truncated DHT";
        int count = 0;
        for (int l = 1; l <= 16; ++l) count += p[i + l];
        if (count > 256 || i + 17 + count > n) return "a DHT of " + std::to_string(count) + " symbols";
        uint8_t* bits = s.bits[tc][th];
        uint8_t* vals = s.vals[tc][th];
        bits[0] = 0;
        memcpy(bits + 1, p + i + 1, 16);
        memset(vals, 0, 256);
        memcpy(vals, p + i + 17, size_t(count));
        const std::string bad = check_huffman(bits, vals, tc == 0);
        if (!bad.empty()) return bad;
        s.hdef[tc][th] = true;
        i += 17 + count;
    }
    return "";
}

// walks the marker segments from `at`; calls fn(marker, payload, length, offset after) until SOS (included) or EOI; "" or the error
template <class F>
std::string segments(const uint8_t* s, int64_t n, int64_t at, const char* what, F&& fn) {
    char buf[96];
    while (true) {
        if (at + 2 > n || s[at] != 0xFF) {
            snprintf(buf, sizeof buf, "%s: no marker at byte %lld", what, (long long)at);
            return buf;
        }
        while (at + 1 < n && s[at + 1] == 0xFF) ++at;
        if (at + 2 > n) {
            snprintf(buf, sizeof buf, "%s: no marker at byte %lld", what, (long long)at);
            return buf;
        }
        const int m = s[at + 1];
        if (m == 0xD9) return fn(m, s + at + 2, 0, at + 2);
        if (at + 4 > n) {
            snprintf(buf, sizeof buf, "%s: segment 0x%02X truncated", what, m);
            return buf;
        }
        const int len = u16(s + at + 2);
        if (len < 2 || at + 2 + len > n) {
            snprintf(buf, sizeof buf, "%s: segment 0x%02X of length %d runs past the data", what, m, len);
            return buf;
        }
        std::string r = fn(m, s + at + 4, len - 2, at + 2 + len);
        if (!r.empty() || m == 0xDA) return r;
        at += 2 + len;
    }
}

// the first marker after `at` that is not stuffing, fill or RSTn, or -1
int64_t end_of_entropy(const uint8_t* s, int64_t n, int64_t at) {
    for (int64_t i = at;;) {
        const void* f = memchr(s + i, 0xFF, size_t(n - i));
        if (!f) return -1;
        i = static_cast<const uint8_t*>(f) - s;
        if (i + 1 >= n) return -1;
        const int m = s[i + 1];
        if (m == 0 || m == 0xFF || (m >= 0xD0 && m <= 0xD7)) {
            ++i;
            continue;
        }
        return i;
    }
}

std::string fmt(const char* f, int a = 0, int b = 0, int c = 0) {
    char buf[128];
    snprintf(buf, sizeof buf, f, a, b, c);
    return buf;
}

void parse_chunk(const uint8_t* s, int64_t n, const Slots& tables, int spp, int photometric, bool want_key, Parsed& out) {
    Slots sl = tables;
    if (n < 2 || s[0] != 0xFF || s[1] != 0xD8) {
        out.error = "does not start with SOI";
        return;
    }
    bool frame = false, scan = false;
    int width = 0, height = 0, restart = 0, ncomp = 0;
    int cid[4], ch[4], cv[4], ctq[4];
    const uint8_t* sos = nullptr;
    int sos_len = 0;
    int64_t after = 0;
    std::string err = segments(s, n, 2, "stream", [&](int m, const uint8_t* p, int len, int64_t next) -> std::string {
        if (m == 0xDB) return read_dqt(p, len, sl);
        if (m == 0xC4) return read_dht(p, len, sl);
        if (m == 0xDD) {
            if (len != 2) return fmt("a DRI of %d bytes", len);
            restart = u16(p);
            return "";
        }
        if (m == 0xC0 || m == 0xC1) {
            if (frame) return "two frames";
            if (len < 6 || p[0] != 8) return fmt("precision %d", len ? p[0] : -1);
            height = u16(p + 1);
            width = u16(p + 3);
            ncomp = p[5];
            if (ncomp != spp) return fmt("%d components in a %d-band image", ncomp, spp);
            if (len != 6 + 3 * ncomp) return fmt("an SOF of %d bytes", len);
            for (int i = 0; i < ncomp; ++i) {
                cid[i] = p[6 + 3 * i];
                ch[i] = p[7 + 3 * i] >> 4;
                cv[i] = p[7 + 3 * i] & 15;
                ctq[i] = p[8 + 3 * i];
            }
            frame = true;
            return "";
        }
        if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
            const char* kind = m == 0xC2 ? "progressive" : m == 0xC3 ? "lossless" : "arithmetic or hierarchical";
            char buf[96];
            snprintf(buf, sizeof buf, "%s frames (SOF%d) are not supported", kind, m - 0xC0);
            return buf;
        }
        if (m == 0xDA) {
            scan = true;
            sos = p;
            sos_len = len;
            after = next;
            return "";
        }
        if (m == 0xD9) return "no scan";
        if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) return "";
        return fmt("marker 0x%02X", m);
    });
    if (!err.empty()) {
        out.error = err;
        return;
    }
    if (!frame) {
        out.error = "no SOF0 / SOF1 frame before the scan";
        return;
    }
    if (width == 0 || height == 0) {
        out.error = fmt("a %d x %d frame", width, height);
        return;
    }
    int h = 1, v = 1;
    if (spp == 3) {
        h = ch[0];
        v = cv[0];
        const bool ok = ((h == 1 && v == 1) || (h == 2 && v == 1) || (h == 2 && v == 2)) && ch[1] == 1 && cv[1] == 1 && ch[2] == 1 && cv[2] == 1;
        if (!ok) {
            char buf[128];
            snprintf(buf, sizeof buf, "sampling %dx%d,%dx%d,%dx%d is not supported; use luma 1x1, 2x1 or 2x2 with chroma 1x1", ch[0], cv[0], ch[1], cv[1],
                     ch[2], cv[2]);
            out.error = buf;
            return;
        }
        if (photometric == 2 && !(h == 1 && v == 1)) {
            out.error = fmt("subsampled RGB (sampling %dx%d)", h, v);
            return;
        }
    }
    const int ns = sos_len ? sos[0] : 0;
    if (ns != ncomp || sos_len != 4 + 2 * ns) {
        out.error = fmt("a scan of %d components in a %d-component frame", ns, ncomp);
        return;
    }
    const int ss = sos[1 + 2 * ns], se = sos[2 + 2 * ns], a = sos[3 + 2 * ns];
    if (ss != 0 || se != 63 || a != 0) {
        out.error = fmt("a scan with Ss %d, Se %d, Ah/Al 0x%02X", ss, se, a);
        return;
    }
    std::string key;
    for (int i = 0; i < ncomp; ++i) {
        if (sos[1 + 2 * i] != cid[i]) {
            out.error = fmt("scan component %d is not frame component %d", sos[1 + 2 * i], cid[i]);
            return;
        }
        const int td = sos[2 + 2 * i] >> 4, ta = sos[2 + 2 * i] & 15;
        if (ctq[i] > 3 || !sl.qdef[ctq[i]]) {
            out.error = fmt("quantisation table %d is used but not defined", ctq[i]);
            return;
        }
        if (td > 3 || !sl.hdef[0][td]) {
            out.error = fmt("DC Huffman table %d is used but not defined", td);
            return;
        }
        if (ta > 3 || !sl.hdef[1][ta]) {
            out.error = fmt("AC Huffman table %d is used but not defined", ta);
            return;
        }
        if (!want_key) continue;
        key.append(reinterpret_cast<const char*>(sl.q[ctq[i]]), sizeof sl.q[0]);
        key.append(reinterpret_cast<const char*>(sl.bits[0][td]), 17);
        key.append(reinterpret_cast<const char*>(sl.vals[0][td]), 256);
        key.append(reinterpret_cast<const char*>(sl.bits[1][ta]), 17);
        key.append(reinterpret_cast<const char*>(sl.vals[1][ta]), 256);
    }
    const int64_t end = end_of_entropy(s, n, after);
    if (end < 0) {
        out.error = "no EOI after the scan";
        return;
    }
    if (s[end + 1] != 0xD9) {
        out.error = fmt("marker 0x%02X after the scan (only one scan is supported)", s[end + 1]);
        return;
    }
    const int64_t mx = spp == 1 ? (width + 7) / 8 : (width + 8 * h - 1) / (8 * h);
    const int64_t my = spp == 1 ? (height + 7) / 8 : (height + 8 * v - 1) / (8 * v);
    int64_t* d = out.desc;
    d[kOffset] = after;
    d[kLength] = end - after;
    d[kSet] = 0;
    d[kWidth] = width;
    d[kHeight] = height;
    d[kH] = h;
    d[kV] = v;
    d[kRestart] = restart;
    d[kBlocks] = mx * my * (spp == 1 ? 1 : h * v + 2);
    d[kFirstBlock] = 0;
    d[kChunk] = 0;
    d[kReserved] = 0;
    out.key = std::move(key);
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
    for (int t = 0; t < threads; ++t)
        pool.emplace_back([&]() {
            for (int64_t i = next.fetch_add(1); i < n; i = next.fetch_add(1)) fn(i);
        });
    for (auto& th : pool) th.join();
}

}  // namespace

extern "C" int rsb_jpeg_parse_chunks(const uint8_t* file, int64_t file_len, const uint8_t* tables, int64_t tables_len, const int64_t* chunk_offsets,
                                     const int64_t* chunk_bytes, int64_t num_chunks, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h,
                                     int64_t rows_per_strip, int32_t tiled, int32_t spp, int32_t photometric, const int64_t* select, int64_t num_select,
                                     int32_t threads, int64_t* descs, int32_t* sets, int32_t max_sets, int32_t* num_sets, int64_t* bad_chunk) {
    if (!file || !chunk_offsets || !chunk_bytes || !descs || !num_sets || file_len < 0 || tables_len < 0 || (tables_len && !tables) || max_sets < 0 ||
        (max_sets && !sets) || num_select < 0 || (num_select && !select))
        return set_error(RSB_E_INVALID, "jpeg_parse_chunks: null pointer or negative size");
    if (width < 1 || height < 1 || chunk_w < 1 || chunk_h < 1 || (!tiled && (chunk_w != width || rows_per_strip < chunk_h)))
        return set_error(RSB_E_INVALID, "jpeg_parse_chunks: raster %lld x %lld with chunks %d x %d, RowsPerStrip %lld (tiled %d)", (long long)width,
                         (long long)height, chunk_w, chunk_h, (long long)rows_per_strip, tiled);
    if (!((spp == 1 && photometric == 1) || (spp == 3 && (photometric == 2 || photometric == 6))))
        return set_error(RSB_E_INVALID, "jpeg_parse_chunks: %d bands with Photometric %d (need 1 with 1, or 3 with 2 or 6)", spp, photometric);
    const int64_t across = tiled ? (width + chunk_w - 1) / chunk_w : 1, down = (height + chunk_h - 1) / chunk_h;
    if (num_chunks != across * down)
        return set_error(RSB_E_INVALID, "jpeg_parse_chunks: %lld chunks, the raster needs %lld", (long long)num_chunks, (long long)(across * down));
    const int64_t n = select ? num_select : num_chunks;
    for (int64_t i = 0; select && i < n; ++i)
        if (select[i] < 0 || select[i] >= num_chunks)
            return set_error(RSB_E_INVALID, "jpeg_parse_chunks: selected chunk %lld of %lld", (long long)select[i], (long long)num_chunks);
    if (bad_chunk) *bad_chunk = -1;
    const char* kind = tiled ? "tile" : "strip";
    const bool want_sets = sets != nullptr;
    Slots base;
    if (tables_len) {
        std::string err;
        if (tables_len < 2 || tables[0] != 0xFF || tables[1] != 0xD8) err = "JPEGTables does not start with SOI";
        else
            err = segments(tables, tables_len, 2, "JPEGTables", [&](int m, const uint8_t* p, int len, int64_t) -> std::string {
                if (m == 0xDB) return read_dqt(p, len, base);
                if (m == 0xC4) return read_dht(p, len, base);
                if (m == 0xDD) return "DRI in JPEGTables";
                if (m == 0xD9 || (m >= 0xE0 && m <= 0xEF) || m == 0xFE) return "";
                return fmt("marker 0x%02X in JPEGTables", m);
            });
        if (!err.empty()) return set_error(RSB_E_INVALID, "Compression 7 (JPEG) %s", err.c_str());
    }
    std::vector<Parsed> parsed(static_cast<size_t>(n));
    parallel_for(n, threads, [&](int64_t i) {
        const int64_t k = select ? select[i] : i;
        const int64_t off = chunk_offsets[k], len = chunk_bytes[k];
        Parsed& p = parsed[size_t(i)];
        if (off < 0 || len < 0 || off > file_len || len > file_len - off) {
            p.error = "extends beyond the end of the file";
            return;
        }
        parse_chunk(file + off, len, base, spp, photometric, want_sets, p);
        if (!p.error.empty()) return;
        const int64_t rows = tiled ? chunk_h : std::min<int64_t>(chunk_h, height - (k / across) * chunk_h);
        const int64_t fw = p.desc[kWidth], fh = p.desc[kHeight];
        char buf[160];
        if (fw != chunk_w) {
            snprintf(buf, sizeof buf, "a frame %lld wide in chunks %d wide", (long long)fw, chunk_w);
            p.error = buf;
        } else if (tiled ? fh != chunk_h : (fh < rows || fh > rows_per_strip)) {
            if (tiled) snprintf(buf, sizeof buf, "a frame %lld high in tiles %d high", (long long)fh, chunk_h);
            else snprintf(buf, sizeof buf, "a frame %lld high in a strip of %lld rows (RowsPerStrip %lld)", (long long)fh, (long long)rows,
                          (long long)rows_per_strip);
            p.error = buf;
        }
        p.desc[kOffset] += off;
        p.desc[kChunk] = k;
    });
    for (int64_t i = 0; i < n; ++i)
        if (!parsed[size_t(i)].error.empty()) {
            const int64_t k = select ? select[i] : i;
            if (bad_chunk) *bad_chunk = k;
            return set_error(RSB_E_INVALID, "Compression 7 (JPEG) %s %lld: %s", kind, (long long)k, parsed[size_t(i)].error.c_str());
        }
    *num_sets = 0;
    if (!want_sets) {  // the headers are checked; no table sets are built
        for (int64_t i = 0; i < n; ++i) {
            parsed[size_t(i)].desc[kSet] = -1;
            memcpy(descs + i * RSB_JPEG_DESC_FIELDS, parsed[size_t(i)].desc, sizeof parsed[0].desc);
        }
        return RSB_OK;
    }
    std::map<std::string, int32_t> ids;
    std::vector<const std::string*> order;
    for (int64_t i = 0; i < n; ++i) {
        Parsed& p = parsed[size_t(i)];
        auto it = ids.find(p.key);
        if (it == ids.end()) {
            it = ids.emplace(std::move(p.key), int32_t(order.size())).first;
            order.push_back(&it->first);
        }
        p.desc[kSet] = it->second;
        memcpy(descs + i * RSB_JPEG_DESC_FIELDS, p.desc, sizeof p.desc);
    }
    *num_sets = int32_t(order.size());
    if (int64_t(order.size()) > max_sets) return RSB_OK;  // the caller asks again with room for *num_sets
    const size_t qbytes = 64 * sizeof(int32_t), per = qbytes + 2 * (17 + 256);
    for (size_t i = 0; i < order.size(); ++i) {
        int32_t* set = sets + i * kSetWords;
        memset(set, 0, sizeof(int32_t) * kSetWords);
        const std::string& key = *order[i];
        const int comps = int(key.size() / per);
        for (int c = 0; c < comps; ++c) {
            const char* at = key.data() + c * per;
            int32_t q[64];
            memcpy(q, at, qbytes);
            for (int j = 0; j < 64; ++j) set[c * 64 + j] = int16_t(q[j]);  // ISLOW_MULT_TYPE is a short
            const uint8_t* b = reinterpret_cast<const uint8_t*>(at + qbytes);
            derive(b, b + 17, set + huff_base(c, 0));
            derive(b + 17 + 256, b + 17 + 256 + 17, set + huff_base(c, 1));
        }
    }
    return RSB_OK;
}
