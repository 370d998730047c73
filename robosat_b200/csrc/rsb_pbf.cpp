// Host side of `rs extract` (robosat/tools/extract.py, robosat/osm/*.py): framing, inflating and parsing OpenStreetMap PBF files
// (https://wiki.openstreetmap.org/wiki/PBF_Format). Plain C++ over zlib, no Python, no interpreter lock; the batch entry points fan
// out over their own threads.
//
// A file is a sequence of [uint32 big-endian length][BlobHeader][Blob] frames. rsb_pbf_frames lists them, rsb_pbf_inflate inflates
// a batch of blobs, rsb_pbf_check_header checks an OSMHeader block, and rsb_pbf_parse reads a batch of PrimitiveBlocks:
//   ways mode:  the ways that carry the anchor key (with the anchor value, when one is given), with their ids, refs and the values
//               of the requested keys; and per block which element kinds it holds;
//   nodes mode: per DenseNodes group the byte ranges of its packed id / lat / lon fields (rsb_pbf_dense_nodes decodes them on the
//               device), and the plain Nodes (and any DenseNodes group written with unpacked or split fields) decoded here.
// Packed repeated fields are accepted unpacked too, as protobuf requires.
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <zlib.h>

#include <atomic>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include "../../include/rsb200.h"
#include "rsb_host.h"
#include "rsb_inflate.h"

using rsb::set_error;

namespace {

constexpr int64_t kMaxHeader = 64 * 1024;         // BlobHeader < 64 KiB
constexpr int64_t kMaxBlob = 32 * 1024 * 1024;    // Blob and its inflated data <= 32 MiB
const char* const kCompression[] = {"raw", "zlib_data", "lzma_data", "OBSOLETE_bzip2_data", "lz4_data", "zstd_data", "no data"};

// ---- protobuf wire format ----

struct Reader {
    const uint8_t* p;
    const uint8_t* end;
    bool bad = false;

    bool more() const { return !bad && p < end; }
    uint64_t varint() {
        uint64_t v = 0;
        for (int s = 0; s < 64; s += 7) {
            if (p >= end) break;
            const uint8_t b = *p++;
            v |= uint64_t(b & 0x7f) << s;
            if (!(b & 0x80)) return v;
        }
        bad = true;
        return 0;
    }
    // one field: returns false at the end or on malformed input; wire type 2 sets (data, len), wire type 0 sets value
    bool field(uint32_t& num, int& wt, uint64_t& value, const uint8_t*& data, uint64_t& len) {
        if (!more()) return false;
        const uint64_t key = varint();
        if (bad) return false;
        num = uint32_t(key >> 3);
        wt = int(key & 7);
        switch (wt) {
            case 0: value = varint(); break;
            case 1:
                if (end - p < 8) return bad = true, false;
                p += 8;
                break;
            case 2:
                len = varint();
                if (bad || len > uint64_t(end - p)) return bad = true, false;
                data = p;
                p += len;
                break;
            case 5:
                if (end - p < 4) return bad = true, false;
                p += 4;
                break;
            default: return bad = true, false;
        }
        return !bad;
    }
};

inline int64_t zigzag(uint64_t v) { return int64_t(v >> 1) ^ -int64_t(v & 1); }

// values of a repeated scalar field occurrence, packed (wire type 2) or not (wire type 0)
template <typename F>
bool each_value(int wt, uint64_t value, const uint8_t* data, uint64_t len, F&& fn) {
    if (wt == 0) {
        fn(value);
        return true;
    }
    if (wt != 2) return false;
    Reader r{data, data + len};
    while (r.more()) {
        const uint64_t v = r.varint();
        if (r.bad) return false;
        fn(v);
    }
    return true;
}

inline uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }

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
    for (int t = 0; t < threads; ++t)
        pool.emplace_back([&]() {
            for (int i = next.fetch_add(1); i < n; i = next.fetch_add(1)) fn(i);
        });
    for (auto& th : pool) th.join();
}

// libosmium's conversion to 1e-7 degree units; INT32_MIN marks a coordinate outside +-180 / +-90 degrees
inline int32_t to_fixed(int64_t v, int64_t granularity, int64_t offset, int64_t limit) {
    const int64_t f = (offset + granularity * v) / 100;
    return (f < -limit || f > limit) ? INT32_MIN : int32_t(f);
}

// ---- parse results ----

struct Block {
    int64_t granularity = 100, lat_offset = 0, lon_offset = 0;
    std::vector<std::pair<const uint8_t*, uint64_t>> strings;
    std::vector<std::pair<const uint8_t*, uint64_t>> groups;
};

struct Segment {       // RSB_PBF_SEG_FIELDS int64 values, see rsb200.h
    int64_t v[RSB_PBF_SEG_FIELDS];
};

struct Part {           // the result of one block
    std::string error;
    int32_t kinds = 0;
    // ways mode
    std::vector<int64_t> way_ids, ref_counts, refs;
    std::vector<int32_t> tags;  // per way and key: index into `strings`, -1 when absent
    std::vector<std::string> strings;
    // nodes mode
    std::vector<Segment> segs;
    std::vector<int64_t> node_ids;
    std::vector<int32_t> node_xy;
};

bool parse_block(const uint8_t* data, uint64_t n, Block& b, std::string& err) {
    Reader r{data, data + n};
    uint32_t num;
    int wt;
    uint64_t value = 0, len = 0;
    const uint8_t* d = nullptr;
    while (r.field(num, wt, value, d, len)) {
        if (num == 1 && wt == 2) {
            Reader s{d, d + len};
            uint32_t sn;
            int swt;
            uint64_t sv = 0, sl = 0;
            const uint8_t* sd = nullptr;
            while (s.field(sn, swt, sv, sd, sl))
                if (sn == 1 && swt == 2) b.strings.emplace_back(sd, sl);
            if (s.bad) return err = "malformed string table", false;
        } else if (num == 2 && wt == 2) {
            b.groups.emplace_back(d, len);
        } else if (num == 17 && wt == 0) {
            b.granularity = int64_t(int32_t(value));
        } else if (num == 19 && wt == 0) {
            b.lat_offset = int64_t(value);
        } else if (num == 20 && wt == 0) {
            b.lon_offset = int64_t(value);
        }
    }
    if (r.bad) return err = "malformed PrimitiveBlock", false;
    return true;
}

int64_t count_terminators(const uint8_t* p, uint64_t n) {
    int64_t c = 0;
    for (uint64_t i = 0; i < n; ++i) c += !(p[i] & 0x80);
    return c;
}

struct WayQuery {
    std::vector<std::string> keys;  // keys[0] is the anchor
    std::string anchor_value;       // empty: any value
};

bool parse_ways(const Block& b, const uint8_t* gdata, uint64_t glen, const WayQuery& q, Part& part, std::string& err) {
    Reader g{gdata, gdata + glen};
    uint32_t num;
    int wt;
    uint64_t value = 0, len = 0;
    const uint8_t* d = nullptr;
    const size_t nk = q.keys.size();
    std::vector<int32_t> key_of(b.strings.size(), -1);  // string index -> requested key, or -1
    bool keys_mapped = false;
    while (g.field(num, wt, value, d, len)) {
        if (num == 1) part.kinds |= RSB_PBF_HAS_NODES;
        else if (num == 2) part.kinds |= RSB_PBF_HAS_DENSE;
        else if (num == 4) part.kinds |= RSB_PBF_HAS_RELATIONS;
        if (num != 3 || wt != 2) continue;
        part.kinds |= RSB_PBF_HAS_WAYS;
        if (!keys_mapped) {
            for (size_t s = 0; s < b.strings.size(); ++s)
                for (size_t k = 0; k < nk; ++k)
                    if (b.strings[s].second == q.keys[k].size() && !memcmp(b.strings[s].first, q.keys[k].data(), q.keys[k].size())) key_of[s] = int32_t(k);
            keys_mapped = true;
        }
        Reader w{d, d + len};
        uint32_t wn;
        int wwt;
        uint64_t wv = 0, wl = 0;
        const uint8_t* wd = nullptr;
        int64_t id = 0;
        std::vector<uint64_t> keys, vals;
        std::vector<std::tuple<int, uint64_t, const uint8_t*, uint64_t>> ref_fields;  // decoded only for kept ways
        while (w.field(wn, wwt, wv, wd, wl)) {
            if (wn == 1 && wwt == 0) id = int64_t(wv);
            else if (wn == 2 && !each_value(wwt, wv, wd, wl, [&](uint64_t v) { keys.push_back(v); })) return err = "malformed way keys", false;
            else if (wn == 3 && !each_value(wwt, wv, wd, wl, [&](uint64_t v) { vals.push_back(v); })) return err = "malformed way vals", false;
            else if (wn == 8) ref_fields.emplace_back(wwt, wv, wd, wl);
        }
        if (w.bad) return err = "malformed Way", false;
        if (keys.size() != vals.size()) return err = "way " + std::to_string(id) + ": keys and vals differ in length", false;
        std::vector<int32_t> found(nk, -1);  // string index of each requested key's value (first occurrence)
        for (size_t t = 0; t < keys.size(); ++t) {
            if (keys[t] >= b.strings.size() || vals[t] >= b.strings.size()) return err = "way " + std::to_string(id) + ": string index out of range", false;
            const int32_t k = key_of[keys[t]];
            if (k >= 0 && found[k] < 0) found[k] = int32_t(vals[t]);
        }
        if (found[0] < 0) continue;
        if (!q.anchor_value.empty()) {
            const auto& s = b.strings[size_t(found[0])];
            if (s.second != q.anchor_value.size() || memcmp(s.first, q.anchor_value.data(), s.second)) continue;
        }
        int64_t ref = 0, count = 0;
        for (const auto& f : ref_fields)
            if (!each_value(std::get<0>(f), std::get<1>(f), std::get<2>(f), std::get<3>(f), [&](uint64_t v) {
                    ref += zigzag(v);
                    part.refs.push_back(ref);
                    ++count;
                }))
                return err = "malformed way refs", false;
        part.way_ids.push_back(id);
        part.ref_counts.push_back(count);
        for (size_t k = 0; k < nk; ++k) {
            if (found[k] < 0) {
                part.tags.push_back(-1);
                continue;
            }
            const auto& s = b.strings[size_t(found[k])];
            part.tags.push_back(int32_t(part.strings.size()));
            part.strings.emplace_back(reinterpret_cast<const char*>(s.first), size_t(s.second));
        }
    }
    if (g.bad) return err = "malformed PrimitiveGroup", false;
    return true;
}

void host_node(Part& part, int64_t id, int64_t lat, int64_t lon, const Block& b) {
    part.node_ids.push_back(id);
    part.node_xy.push_back(to_fixed(lon, b.granularity, b.lon_offset, 1800000000LL));
    part.node_xy.push_back(to_fixed(lat, b.granularity, b.lat_offset, 900000000LL));
}

void add_host_segment(Part& part, int64_t first, const Block& b) {
    Segment s{};
    s.v[RSB_PBF_SEG_KIND] = 1;
    s.v[RSB_PBF_SEG_COUNT] = int64_t(part.node_ids.size()) - first;
    s.v[RSB_PBF_SEG_HOST_FIRST] = first;
    s.v[RSB_PBF_SEG_GRANULARITY] = b.granularity;
    s.v[RSB_PBF_SEG_LAT_OFFSET] = b.lat_offset;
    s.v[RSB_PBF_SEG_LON_OFFSET] = b.lon_offset;
    if (s.v[RSB_PBF_SEG_COUNT] > 0) part.segs.push_back(s);
}

bool parse_nodes(const Block& b, const uint8_t* block_base, const uint8_t* gdata, uint64_t glen, Part& part, std::string& err) {
    Reader g{gdata, gdata + glen};
    uint32_t num;
    int wt;
    uint64_t value = 0, len = 0;
    const uint8_t* d = nullptr;
    const int64_t plain_first = int64_t(part.node_ids.size());
    bool plain = false;
    while (g.field(num, wt, value, d, len)) {
        if (wt != 2) continue;
        if (num == 1) {  // Node
            Reader r{d, d + len};
            uint32_t n2;
            int w2;
            uint64_t v2 = 0, l2 = 0;
            const uint8_t* d2 = nullptr;
            int64_t id = 0, lat = 0, lon = 0;
            while (r.field(n2, w2, v2, d2, l2)) {
                if (w2 != 0) continue;
                if (n2 == 1) id = zigzag(v2);
                else if (n2 == 8) lat = zigzag(v2);
                else if (n2 == 9) lon = zigzag(v2);
            }
            if (r.bad) return err = "malformed Node", false;
            host_node(part, id, lat, lon, b);
            plain = true;
        } else if (num == 2) {  // DenseNodes
            Reader r{d, d + len};
            uint32_t n2;
            int w2;
            uint64_t v2 = 0, l2 = 0;
            const uint8_t* d2 = nullptr;
            const uint8_t* ranges[3] = {nullptr, nullptr, nullptr};
            uint64_t lens[3] = {0, 0, 0};
            int seen[3] = {0, 0, 0};
            bool packed = true;
            while (r.field(n2, w2, v2, d2, l2)) {
                const int f = n2 == 1 ? 0 : (n2 == 8 ? 1 : (n2 == 9 ? 2 : -1));
                if (f < 0) continue;
                ++seen[f];
                if (w2 == 2) {
                    ranges[f] = d2;
                    lens[f] = l2;
                } else {
                    packed = false;
                }
            }
            if (r.bad) return err = "malformed DenseNodes", false;
            if (packed && seen[0] <= 1 && seen[1] <= 1 && seen[2] <= 1) {
                const int64_t count = count_terminators(ranges[0], lens[0]);
                if (count_terminators(ranges[1], lens[1]) != count || count_terminators(ranges[2], lens[2]) != count)
                    return err = "DenseNodes: id, lat and lon hold different numbers of values", false;
                if (count == 0) continue;
                if ((lens[0] && (ranges[0][lens[0] - 1] & 0x80)) || (lens[1] && (ranges[1][lens[1] - 1] & 0x80)) || (lens[2] && (ranges[2][lens[2] - 1] & 0x80)))
                    return err = "DenseNodes: a packed field ends inside a varint", false;
                Segment s{};
                s.v[RSB_PBF_SEG_KIND] = 0;
                s.v[RSB_PBF_SEG_COUNT] = count;
                s.v[RSB_PBF_SEG_ID_OFF] = ranges[0] - block_base;
                s.v[RSB_PBF_SEG_ID_LEN] = int64_t(lens[0]);
                s.v[RSB_PBF_SEG_LAT_OFF] = ranges[1] - block_base;
                s.v[RSB_PBF_SEG_LAT_LEN] = int64_t(lens[1]);
                s.v[RSB_PBF_SEG_LON_OFF] = ranges[2] - block_base;
                s.v[RSB_PBF_SEG_LON_LEN] = int64_t(lens[2]);
                s.v[RSB_PBF_SEG_GRANULARITY] = b.granularity;
                s.v[RSB_PBF_SEG_LAT_OFFSET] = b.lat_offset;
                s.v[RSB_PBF_SEG_LON_OFFSET] = b.lon_offset;
                s.v[RSB_PBF_SEG_HOST_FIRST] = -1;
                part.segs.push_back(s);
            } else {
                // unpacked or split fields: rare enough to decode here, in order, as one host segment
                std::vector<int64_t> cols[3];
                Reader r2{d, d + len};
                while (r2.field(n2, w2, v2, d2, l2)) {
                    const int f = n2 == 1 ? 0 : (n2 == 8 ? 1 : (n2 == 9 ? 2 : -1));
                    if (f < 0) continue;
                    if (!each_value(w2, v2, d2, l2, [&](uint64_t v) { cols[f].push_back(zigzag(v)); })) return err = "malformed DenseNodes", false;
                }
                if (cols[1].size() != cols[0].size() || cols[2].size() != cols[0].size())
                    return err = "DenseNodes: id, lat and lon hold different numbers of values", false;
                const int64_t first = int64_t(part.node_ids.size());
                int64_t id = 0, lat = 0, lon = 0;
                for (size_t i = 0; i < cols[0].size(); ++i) {
                    id += cols[0][i];
                    lat += cols[1][i];
                    lon += cols[2][i];
                    host_node(part, id, lat, lon, b);
                }
                add_host_segment(part, first, b);
            }
        }
    }
    if (g.bad) return err = "malformed PrimitiveGroup", false;
    if (plain) add_host_segment(part, plain_first, b);  // the group's plain Nodes, after its DenseNodes in element order
    return true;
}

struct Result {
    int32_t mode = 0, nkeys = 0;
    std::vector<int32_t> kinds;
    std::vector<int64_t> way_ids, ref_offsets, refs, string_offsets, host_ids;
    std::vector<int32_t> tags, host_xy;
    std::vector<uint8_t> string_bytes;
    std::vector<int64_t> segs;
};

}  // namespace

extern "C" int rsb_pbf_frames(const uint8_t* file_host, int64_t n, int64_t* frames_host, int64_t capacity, int64_t* count_host) {
    if ((!file_host && n > 0) || n < 0 || !count_host || capacity < 0 || (capacity > 0 && !frames_host)) return set_error(RSB_E_INVALID, "pbf_frames: bad arguments");
    int64_t at = 0, k = 0;
    while (at < n) {
        if (n - at < 4) return set_error(RSB_E_INVALID, "pbf: truncated file: %lld bytes after the last blob at offset %lld", (long long)(n - at), (long long)at);
        const int64_t hl = be32(file_host + at);
        if (hl >= kMaxHeader) return set_error(RSB_E_INVALID, "pbf: BlobHeader of %lld bytes at offset %lld (the format allows less than 64 KiB)", (long long)hl, (long long)at);
        if (n - at - 4 < hl) return set_error(RSB_E_INVALID, "pbf: truncated file: BlobHeader at offset %lld runs past the end", (long long)at);
        Reader h{file_host + at + 4, file_host + at + 4 + hl};
        uint32_t num;
        int wt;
        uint64_t value = 0, len = 0, datasize = 0;
        const uint8_t* d = nullptr;
        int kind = RSB_PBF_BLOB_OTHER;
        bool has_size = false;
        while (h.field(num, wt, value, d, len)) {
            if (num == 1 && wt == 2) {
                if (len == 9 && !memcmp(d, "OSMHeader", 9)) kind = RSB_PBF_BLOB_HEADER;
                else if (len == 7 && !memcmp(d, "OSMData", 7)) kind = RSB_PBF_BLOB_DATA;
            } else if (num == 3 && wt == 0) {
                datasize = value;
                has_size = true;
            }
        }
        if (h.bad || !has_size) return set_error(RSB_E_INVALID, "pbf: malformed BlobHeader at offset %lld", (long long)at);
        if (int64_t(datasize) > kMaxBlob || int64_t(datasize) < 0)
            return set_error(RSB_E_INVALID, "pbf: Blob of %llu bytes at offset %lld (the format allows at most 32 MiB)", (unsigned long long)datasize, (long long)at);
        const int64_t blob = at + 4 + hl;
        if (n - blob < int64_t(datasize)) return set_error(RSB_E_INVALID, "pbf: truncated file: Blob at offset %lld runs past the end", (long long)blob);
        Reader bl{file_host + blob, file_host + blob + datasize};
        int comp = RSB_PBF_NO_DATA;
        int64_t data_off = 0, data_len = 0, raw_size = -1;
        while (bl.field(num, wt, value, d, len)) {
            if (wt == 2 && num >= 1 && num <= 7 && num != 2) {
                comp = num == 1 ? RSB_PBF_RAW : int(num) - 2;
                data_off = d - file_host;
                data_len = int64_t(len);
            } else if (num == 2 && wt == 0) {
                raw_size = int64_t(int32_t(value));
            }
        }
        if (bl.bad) return set_error(RSB_E_INVALID, "pbf: malformed Blob at offset %lld", (long long)blob);
        if (comp == RSB_PBF_RAW) raw_size = data_len;
        if (raw_size > kMaxBlob) return set_error(RSB_E_INVALID, "pbf: Blob at offset %lld inflates to %lld bytes (the format allows at most 32 MiB)", (long long)blob, (long long)raw_size);
        if (k < capacity) {
            int64_t* f = frames_host + RSB_PBF_FRAME_FIELDS * k;
            f[0] = kind;
            f[1] = comp;
            f[2] = data_off;
            f[3] = data_len;
            f[4] = raw_size;
            f[5] = at;
        }
        ++k;
        at = blob + int64_t(datasize);
    }
    *count_host = k;
    return RSB_OK;
}

extern "C" int rsb_pbf_inflate(const uint8_t* file_host, const int64_t* frames_host, int32_t n, uint8_t* out_host, const int64_t* out_offsets_host,
                               int32_t threads) {
    if (n < 0 || (n > 0 && (!file_host || !frames_host || !out_host || !out_offsets_host))) return set_error(RSB_E_INVALID, "pbf_inflate: bad arguments");
    std::vector<std::string> errs(static_cast<size_t>(n));
    parallel_for(n, threads, [&](int i) {
        const int64_t* f = frames_host + RSB_PBF_FRAME_FIELDS * int64_t(i);
        const int comp = int(f[1]);
        const int64_t off = f[2], len = f[3], raw = f[4];
        uint8_t* out = out_host + out_offsets_host[i];
        char msg[256];
        if (comp == RSB_PBF_RAW) {
            memcpy(out, file_host + off, size_t(len));
            return;
        }
        if (comp != RSB_PBF_ZLIB) {
            snprintf(msg, sizeof msg, "pbf: Blob at offset %lld uses %s, which is not supported (raw and zlib_data are)", (long long)f[5],
                     kCompression[comp >= 0 && comp <= RSB_PBF_NO_DATA ? comp : RSB_PBF_NO_DATA]);
            errs[size_t(i)] = msg;
            return;
        }
        if (raw < 0) {
            snprintf(msg, sizeof msg, "pbf: zlib Blob at offset %lld has no raw_size", (long long)f[5]);
            errs[size_t(i)] = msg;
            return;
        }
        // the library's own inflate (it succeeds only when the stream ends at exactly raw bytes and its Adler-32 matches); a
        // stream it rejects goes through zlib, whose verdict is final. The caller leaves kInflateOutPad bytes after each output.
        std::vector<uint8_t> in(size_t(len) + rsb::kInflateInPad, 0);
        memcpy(in.data(), file_host + off, size_t(len));
        if (len < 6 || rsb::rsb_inflate_zlib_padded(in.data(), size_t(len), out, size_t(raw)) != 0) {
            uLongf rn = uLongf(raw) + 1;
            std::vector<uint8_t> tmp(size_t(raw) + 1);
            const int zr = uncompress(tmp.data(), &rn, file_host + off, uLong(len));
            if (zr != Z_OK || int64_t(rn) != raw) {
                snprintf(msg, sizeof msg, "pbf: Blob at offset %lld: zlib stream %s (inflated %lld bytes, raw_size %lld)", (long long)f[5],
                         zr == Z_OK ? "does not match raw_size" : (zr == Z_BUF_ERROR ? "inflates past raw_size or is truncated" : "is corrupt"),
                         (long long)(zr == Z_OK ? int64_t(rn) : -1), (long long)raw);
                errs[size_t(i)] = msg;
                return;
            }
            memcpy(out, tmp.data(), size_t(raw));
        }
    });
    for (int i = 0; i < n; ++i)
        if (!errs[size_t(i)].empty()) return set_error(RSB_E_INVALID, "%s", errs[size_t(i)].c_str());
    return RSB_OK;
}

extern "C" int rsb_pbf_check_header(const uint8_t* block_host, int64_t n) {
    if (!block_host && n > 0) return set_error(RSB_E_INVALID, "pbf_check_header: bad arguments");
    Reader r{block_host, block_host + n};
    uint32_t num;
    int wt;
    uint64_t value = 0, len = 0;
    const uint8_t* d = nullptr;
    while (r.field(num, wt, value, d, len)) {
        if (num != 4 || wt != 2) continue;
        const std::string feature(reinterpret_cast<const char*>(d), size_t(len));
        if (feature != "OsmSchema-V0.6" && feature != "DenseNodes")
            return set_error(RSB_E_INVALID, "pbf: the file requires the feature \"%s\", which is not supported", feature.c_str());
    }
    if (r.bad) return set_error(RSB_E_INVALID, "pbf: malformed HeaderBlock");
    return RSB_OK;
}

extern "C" int rsb_pbf_parse(const uint8_t* blocks_host, const int64_t* offsets_host, const int64_t* sizes_host, int32_t n, int32_t mode,
                             const char* keys_host, int32_t nkeys, const char* anchor_value_host, int32_t threads, void** result) {
    if (!result || n < 0 || (n > 0 && (!blocks_host || !offsets_host || !sizes_host)) || (mode != RSB_PBF_WAYS && mode != RSB_PBF_NODES))
        return set_error(RSB_E_INVALID, "pbf_parse: bad arguments");
    if (mode == RSB_PBF_WAYS && (nkeys < 1 || nkeys > RSB_PBF_MAX_KEYS || !keys_host))
        return set_error(RSB_E_INVALID, "pbf_parse: ways mode needs 1..%d keys (got %d)", RSB_PBF_MAX_KEYS, nkeys);
    *result = nullptr;
    WayQuery q;
    if (mode == RSB_PBF_WAYS) {
        const char* k = keys_host;
        for (int i = 0; i < nkeys; ++i) {
            q.keys.emplace_back(k);
            k += q.keys.back().size() + 1;
        }
        q.anchor_value = anchor_value_host ? anchor_value_host : "";
    }
    std::vector<Part> parts(static_cast<size_t>(n));
    parallel_for(n, threads, [&](int i) {
        Part& part = parts[size_t(i)];
        const uint8_t* base = blocks_host + offsets_host[i];
        Block b;
        if (!parse_block(base, uint64_t(sizes_host[i]), b, part.error)) return;
        for (const auto& g : b.groups) {
            const bool ok = mode == RSB_PBF_WAYS ? parse_ways(b, g.first, g.second, q, part, part.error) : parse_nodes(b, base, g.first, g.second, part, part.error);
            if (!ok) return;
        }
    });
    for (int i = 0; i < n; ++i)
        if (!parts[size_t(i)].error.empty()) return set_error(RSB_E_INVALID, "pbf: block %d of the batch: %s", i, parts[size_t(i)].error.c_str());
    Result* res = new Result;
    res->mode = mode;
    res->nkeys = nkeys;
    res->ref_offsets.push_back(0);
    res->string_offsets.push_back(0);
    for (int i = 0; i < n; ++i) {
        Part& p = parts[size_t(i)];
        res->kinds.push_back(p.kinds);
        if (mode == RSB_PBF_WAYS) {
            const int32_t sbase = int32_t(res->string_offsets.size() - 1);
            res->way_ids.insert(res->way_ids.end(), p.way_ids.begin(), p.way_ids.end());
            for (int64_t c : p.ref_counts) res->ref_offsets.push_back(res->ref_offsets.back() + c);
            res->refs.insert(res->refs.end(), p.refs.begin(), p.refs.end());
            for (int32_t t : p.tags) res->tags.push_back(t < 0 ? -1 : t + sbase);
            for (const auto& s : p.strings) {
                res->string_bytes.insert(res->string_bytes.end(), s.begin(), s.end());
                res->string_offsets.push_back(int64_t(res->string_bytes.size()));
            }
        } else {
            const int64_t hbase = int64_t(res->host_ids.size());
            for (Segment s : p.segs) {
                s.v[RSB_PBF_SEG_BLOCK] = i;
                if (s.v[RSB_PBF_SEG_KIND] == 1) s.v[RSB_PBF_SEG_HOST_FIRST] += hbase;
                res->segs.insert(res->segs.end(), s.v, s.v + RSB_PBF_SEG_FIELDS);
            }
            res->host_ids.insert(res->host_ids.end(), p.node_ids.begin(), p.node_ids.end());
            res->host_xy.insert(res->host_xy.end(), p.node_xy.begin(), p.node_xy.end());
        }
    }
    *result = res;
    return RSB_OK;
}

extern "C" int rsb_pbf_result_sizes(const void* result, int64_t* sizes_host) {
    if (!result || !sizes_host) return set_error(RSB_E_INVALID, "pbf_result_sizes: bad arguments");
    const Result* r = static_cast<const Result*>(result);
    sizes_host[RSB_PBF_OUT_KINDS] = int64_t(r->kinds.size());
    sizes_host[RSB_PBF_OUT_WAY_IDS] = int64_t(r->way_ids.size());
    sizes_host[RSB_PBF_OUT_REF_OFFSETS] = int64_t(r->ref_offsets.size());
    sizes_host[RSB_PBF_OUT_REFS] = int64_t(r->refs.size());
    sizes_host[RSB_PBF_OUT_TAGS] = int64_t(r->tags.size());
    sizes_host[RSB_PBF_OUT_STRING_OFFSETS] = int64_t(r->string_offsets.size());
    sizes_host[RSB_PBF_OUT_STRING_BYTES] = int64_t(r->string_bytes.size());
    sizes_host[RSB_PBF_OUT_SEGS] = int64_t(r->segs.size());
    sizes_host[RSB_PBF_OUT_HOST_IDS] = int64_t(r->host_ids.size());
    sizes_host[RSB_PBF_OUT_HOST_XY] = int64_t(r->host_xy.size());
    return RSB_OK;
}

extern "C" int rsb_pbf_result_copy(const void* result, int32_t what, void* dst_host, int64_t count) {
    if (!result || (!dst_host && count > 0)) return set_error(RSB_E_INVALID, "pbf_result_copy: bad arguments");
    const Result* r = static_cast<const Result*>(result);
    const void* src = nullptr;
    int64_t have = 0, elem = 8;
    switch (what) {
        case RSB_PBF_OUT_KINDS: src = r->kinds.data(), have = int64_t(r->kinds.size()), elem = 4; break;
        case RSB_PBF_OUT_WAY_IDS: src = r->way_ids.data(), have = int64_t(r->way_ids.size()); break;
        case RSB_PBF_OUT_REF_OFFSETS: src = r->ref_offsets.data(), have = int64_t(r->ref_offsets.size()); break;
        case RSB_PBF_OUT_REFS: src = r->refs.data(), have = int64_t(r->refs.size()); break;
        case RSB_PBF_OUT_TAGS: src = r->tags.data(), have = int64_t(r->tags.size()), elem = 4; break;
        case RSB_PBF_OUT_STRING_OFFSETS: src = r->string_offsets.data(), have = int64_t(r->string_offsets.size()); break;
        case RSB_PBF_OUT_STRING_BYTES: src = r->string_bytes.data(), have = int64_t(r->string_bytes.size()), elem = 1; break;
        case RSB_PBF_OUT_SEGS: src = r->segs.data(), have = int64_t(r->segs.size()); break;
        case RSB_PBF_OUT_HOST_IDS: src = r->host_ids.data(), have = int64_t(r->host_ids.size()); break;
        case RSB_PBF_OUT_HOST_XY: src = r->host_xy.data(), have = int64_t(r->host_xy.size()), elem = 4; break;
        default: return set_error(RSB_E_INVALID, "pbf_result_copy: unknown output %d", what);
    }
    if (count != have) return set_error(RSB_E_INVALID, "pbf_result_copy: output %d holds %lld values, not %lld", what, (long long)have, (long long)count);
    if (count) memcpy(dst_host, src, size_t(count * elem));
    return RSB_OK;
}

extern "C" void rsb_pbf_result_free(void* result) { delete static_cast<Result*>(result); }
