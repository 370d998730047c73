// Device decoder of the JPEG chunks of `rs tile` and `rs segment` (DESIGN.md §8): a window of a Compression 7 TIFF decoded from the
// staged entropy-coded bytes of the chunks it touches straight into the source window the warps read, uint8 [rows][cols][spp].
//
// Three kernels on the caller's stream, over a scratch of RSB_JPEG_SCRATCH_PER_BLOCK bytes per 8 x 8 block (int16 coefficients, then
// uint8 samples, both in each chunk's MCU order):
// 1. huffman_kernel: one thread per chunk (32 chunks per warp), MCUs and restart intervals in order: the Huffman decode of
//    libjpeg (an 8-bit lookahead table, then maxcode / valoffset), DC prediction reset at every restart, the coefficients written
//    into blocks the host cleared. Every read stays inside the chunk's byte range and every write inside its block count; damaged
//    data or a descriptor inconsistent with the staged bytes, the scratch or the table sets stops the chunk with an error word
//    (code | MCU << 8) instead of libjpeg's zero padding; the next two kernels skip every chunk whose word is not 0.
// 2. idct_kernel: eight threads per block, one column each in pass 1 and one row each in pass 2 of `jpeg_idct_islow` (int64
//    arithmetic as JLONG, the pass-1 results truncated to int, the RANGE_MASK wrap and the range limit).
// 3. pixel_kernel: one thread per window pixel: jdsample.c's fancy h2v1 / h2v2 upsampling (edges replicated at the component's true
//    size, plain replication when the chroma is at most 2 samples wide), jdcolor.c's integer YCbCr -> RGB, the crop to the window.
// tests/jpeg_reference.py restates all of it in numpy.

#include <stdint.h>
#include <stdio.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"
#include "rsb_jpeg.h"

using namespace rsb;
using namespace rsb_jpeg;

namespace {

__constant__ uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Launch {
    const uint8_t* staged;
    int64_t staged_len;
    const int64_t* descs;
    int32_t n;
    const int32_t* sets;
    int32_t n_sets;
    int32_t spp, photometric, chunk_w, chunk_h;
    int64_t row0, rows, col0, cols;
    int64_t chunk_row0, chunk_col0, grid_cols;
    uint8_t* out;
    int16_t* coefs;
    uint8_t* samples;
    int64_t total_blocks;
    int64_t* errors;
};

// ---- stage 1: entropy decode ----

// MSB-first bits of one chunk's entropy-coded bytes with the 0xFF00 stuffing removed. Loading stops at a marker or the end of the
// range; past that, zero bits are shifted in and counted in `pad`, and taking them is an error.
struct Bits {
    const uint8_t* p;
    int64_t pos, end;
    uint64_t acc;  // left-aligned
    int nbits, pad;
    bool marker;

    __device__ void fill() {
        while (nbits <= 56) {
            uint32_t b = 0;
            if (!marker && pos < end) {
                b = p[pos];
                if (b == 0xFF) {
                    if (pos + 1 < end && p[pos + 1] == 0) {
                        pos += 2;
                    } else {
                        marker = true;  // an RST marker, or fill bytes before one
                        b = 0;
                        pad += 8;
                    }
                } else {
                    ++pos;
                }
            } else {
                pad += 8;
            }
            acc |= uint64_t(b) << (56 - nbits);
            nbits += 8;
        }
    }
    __device__ bool take(int n, uint32_t& v) {  // n <= 16
        if (n > nbits - pad) return false;
        v = n ? uint32_t(acc >> (64 - n)) : 0u;
        acc = n ? acc << n : acc;
        nbits -= n;
        return true;
    }
    __device__ void reset(int64_t at) {
        pos = at;
        acc = 0;
        nbits = pad = 0;
        marker = false;
    }
    // drop the bits of a partly used byte; true when no whole data byte is left before the next marker
    __device__ bool align() {
        const int drop = nbits & 7;
        acc <<= drop;
        nbits -= drop;
        if (nbits - pad > 0) return false;  // whole bytes already loaded
        if (!marker && pos < end && p[pos] != 0xFF) return false;
        if (!marker && pos + 1 < end && p[pos] == 0xFF && p[pos + 1] == 0) return false;
        return true;
    }
    // after align: skip fill bytes; the marker number (0xD0..0xFF) at pos, or -1 at the end of the range
    __device__ int next_marker() {
        while (pos + 1 < end && p[pos] == 0xFF && p[pos + 1] == 0xFF) ++pos;
        if (pos + 1 < end && p[pos] == 0xFF) return p[pos + 1];
        if (pos + 1 == end && p[pos] == 0xFF) ++pos;  // a fill byte before the marker that ends the range
        return -1;
    }
};

__device__ __forceinline__ int extend(uint32_t v, int s) { return s && v < (1u << (s - 1)) ? int(v) - (1 << s) + 1 : int(v); }

// one Huffman symbol, or -1 for an invalid code or bits past the data (*truncated set)
__device__ __forceinline__ int huff(Bits& b, const int32_t* t, bool& truncated) {
    b.fill();
    const uint32_t look = uint32_t(b.acc >> 48);
    const int e = __ldg(t + kLookup + (look >> 8));
    int l = e >> 8;
    uint32_t dummy;
    if (l <= 8) {
        if (!b.take(l, dummy)) {
            truncated = true;
            return -1;
        }
        return e & 0xFF;
    }
    while (l <= 16 && int32_t(look >> (16 - l)) > __ldg(t + kMaxcode + l)) ++l;
    if (l > 16) return -1;
    const int code = int(look >> (16 - l));
    if (!b.take(l, dummy)) {
        truncated = true;
        return -1;
    }
    return __ldg(t + kHuffval + ((code + __ldg(t + kValoffset + l)) & 0xFF));
}

__global__ void __launch_bounds__(128) huffman_kernel(const Launch L) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= L.n) return;
    const int64_t* d = L.descs + int64_t(k) * RSB_JPEG_DESC_FIELDS;
    const int64_t off = d[kOffset], len = d[kLength], set = d[kSet], blocks = d[kBlocks], first = d[kFirstBlock];
    const int64_t W = d[kWidth], H = d[kHeight], h = d[kH], v = d[kV], R = d[kRestart];
    const bool gray = L.spp == 1;
    if (off < 0 || len < 0 || off > L.staged_len || len > L.staged_len - off || set < 0 || set >= L.n_sets || first < 0 || blocks < 0 ||
        first > L.total_blocks - blocks || W < 1 || H < 1 || W > 65535 || H > 65535 || R < 0 || !((h == 1 && v == 1) || (h == 2 && (v == 1 || v == 2)))) {
        L.errors[k] = kBadDescriptor;
        return;
    }
    const int64_t mx = gray ? (W + 7) / 8 : (W + 8 * h - 1) / (8 * h), my = gray ? (H + 7) / 8 : (H + 8 * v - 1) / (8 * v);
    const int luma = gray ? 1 : int(h * v), bpm = gray ? 1 : luma + 2;
    if (mx * my * bpm != blocks) {
        L.errors[k] = kBadDescriptor;
        return;
    }
    const int32_t* tab = L.sets + set * kSetWords;
    int16_t* coef = L.coefs + first * 64;
    Bits b;
    b.p = L.staged;
    b.end = off + len;
    b.reset(off);
    int pred[3] = {0, 0, 0};
    const int64_t total = mx * my;
    int err = kOk;
    int64_t mcu = 0;
    for (; mcu < total; ++mcu) {
        if (R && mcu && mcu % R == 0) {
            if (!b.align()) {
                err = kExtraneous;
                break;
            }
            const int m = b.next_marker();
            if (m < 0) {
                err = kTruncated;
                break;
            }
            if (m != 0xD0 + int((mcu / R - 1) & 7)) {
                err = kBadMarker;
                break;
            }
            b.reset(b.pos + 2);
            pred[0] = pred[1] = pred[2] = 0;
        }
        for (int j = 0; j < bpm && err == kOk; ++j) {
            const int c = j < luma ? 0 : j - luma + 1;
            const int32_t* dc = tab + huff_base(c, 0);
            const int32_t* ac = tab + huff_base(c, 1);
            int16_t* blk = coef + (mcu * bpm + j) * 64;
            bool truncated = false;
            int s = huff(b, dc, truncated);
            if (s < 0) {
                err = truncated ? kTruncated : kBadCode;
                break;
            }
            uint32_t bits;
            b.fill();
            if (!b.take(s, bits)) {
                err = kTruncated;
                break;
            }
            pred[c] += extend(bits, s);
            blk[0] = int16_t(pred[c]);
            for (int kk = 1; kk < 64;) {
                const int rs = huff(b, ac, truncated);
                if (rs < 0) {
                    err = truncated ? kTruncated : kBadCode;
                    break;
                }
                const int r = rs >> 4;
                s = rs & 15;
                if (s) {
                    kk += r;
                    if (kk > 63) {
                        err = kAcPast63;
                        break;
                    }
                    b.fill();
                    if (!b.take(s, bits)) {
                        err = kTruncated;
                        break;
                    }
                    blk[kNatural[kk]] = int16_t(extend(bits, s));
                    ++kk;
                } else if (r == 15) {
                    kk += 16;
                } else {
                    break;
                }
            }
        }
        if (err != kOk) break;  // mcu stays the MCU that failed
    }
    if (err == kOk) {
        if (!b.align()) err = kExtraneous;
        else if (b.next_marker() >= 0) err = kBadMarker;
        else if (b.pos < b.end) err = kExtraneous;
    }
    L.errors[k] = err == kOk ? 0 : int64_t(err) | (mcu << 8);
}

// ---- stage 2: dequantisation and the islow IDCT ----

constexpr int64_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137,
                  F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

__device__ __forceinline__ void idct_1d(int64_t i0, int64_t i1, int64_t i2, int64_t i3, int64_t i4, int64_t i5, int64_t i6, int64_t i7,
                                        int64_t* o) {
    int64_t z1 = (i2 + i6) * F0541;
    const int64_t tmp2 = z1 + i6 * -F1847, tmp3 = z1 + i2 * F0765;
    const int64_t tmp0 = (i0 + i4) * 8192, tmp1 = (i0 - i4) * 8192;
    const int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    int64_t a0 = i7, a1 = i5, a2 = i3, a3 = i1;
    z1 = a0 + a3;
    int64_t z2 = a1 + a2, z3 = a0 + a2, z4 = a1 + a3;
    const int64_t z5 = (z3 + z4) * F1175;
    a0 *= F0298;
    a1 *= F2053;
    a2 *= F3072;
    a3 *= F1501;
    z1 *= -F0899;
    z2 *= -F2562;
    z3 = z3 * -F1961 + z5;
    z4 = z4 * -F0390 + z5;
    a0 += z1 + z3;
    a1 += z2 + z4;
    a2 += z2 + z3;
    a3 += z1 + z4;
    o[0] = t10 + a3;
    o[1] = t11 + a2;
    o[2] = t12 + a1;
    o[3] = t13 + a0;
    o[4] = t13 - a0;
    o[5] = t12 - a1;
    o[6] = t11 - a2;
    o[7] = t10 - a3;
}

constexpr int IDCT_THREADS = 256, IDCT_BLOCKS = IDCT_THREADS / 8;

__global__ void __launch_bounds__(IDCT_THREADS) idct_kernel(const Launch L) {
    __shared__ int32_t ws[IDCT_BLOCKS][64];
    const int lane8 = threadIdx.x & 7, slot = threadIdx.x >> 3;
    for (int64_t base = int64_t(blockIdx.x) * IDCT_BLOCKS; base < L.total_blocks; base += int64_t(gridDim.x) * IDCT_BLOCKS) {
        const int64_t blk = base + slot;
        bool live = blk < L.total_blocks;
        const int32_t* q = nullptr;
        if (live) {  // the chunk of this block: the last whose first block is <= blk
            int lo = 0, hi = L.n - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (L.descs[int64_t(mid) * RSB_JPEG_DESC_FIELDS + kFirstBlock] <= blk) lo = mid;
                else hi = mid - 1;
            }
            const int64_t* d = L.descs + int64_t(lo) * RSB_JPEG_DESC_FIELDS;
            const int64_t j = blk - d[kFirstBlock], set = d[kSet];
            live = L.errors[lo] == 0 && j >= 0 && j < d[kBlocks] && set >= 0 && set < L.n_sets;
            if (live) {
                const int bpm = L.spp == 1 ? 1 : int(d[kH] * d[kV]) + 2, luma = bpm - 2;
                const int jj = int(j % bpm);
                const int c = L.spp == 1 || jj < luma ? 0 : jj - luma + 1;
                q = L.sets + set * kSetWords + c * 64;
            }
        }
        int64_t o[8];
        if (live) {  // pass 1: column lane8
            const int16_t* in = L.coefs + blk * 64;
            int64_t x[8];
#pragma unroll
            for (int r = 0; r < 8; ++r) x[r] = int64_t(in[r * 8 + lane8]) * int64_t(__ldg(q + r * 8 + lane8));
            idct_1d(x[0], x[1], x[2], x[3], x[4], x[5], x[6], x[7], o);
#pragma unroll
            for (int r = 0; r < 8; ++r) ws[slot][r * 8 + lane8] = int32_t((o[r] + 1024) >> 11);
        }
        __syncwarp();
        if (live) {  // pass 2: row lane8
            const int32_t* w = ws[slot] + lane8 * 8;
            idct_1d(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7], o);
            uint32_t lo = 0, hi = 0;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int32_t t = (int32_t((o[c] + (int64_t(1) << 17)) >> 18) + 512) & 1023;
                const uint32_t px = uint32_t(min(max(t - 384, 0), 255));
                if (c < 4) lo |= px << (8 * c);
                else hi |= px << (8 * (c - 4));
            }
            *reinterpret_cast<uint2*>(L.samples + blk * 64 + lane8 * 8) = make_uint2(lo, hi);
        }
        __syncwarp();
    }
}

// ---- stage 3: upsampling, colour and the crop ----

struct Chunk {
    const uint8_t* s;
    int64_t mx;
    int h, v, bpm, wc, hc;
};

__device__ __forceinline__ int luma_at(const Chunk& c, int x, int y) {
    const int64_t mcu = int64_t(y / (8 * c.v)) * c.mx + x / (8 * c.h);
    const int j = ((y >> 3) % c.v) * c.h + (x >> 3) % c.h;
    return c.s[(mcu * c.bpm + j) * 64 + (y & 7) * 8 + (x & 7)];
}

__device__ __forceinline__ int chroma_at(const Chunk& c, int comp, int x, int y) {
    const int64_t mcu = int64_t(y >> 3) * c.mx + (x >> 3);
    return c.s[(mcu * c.bpm + c.bpm - 3 + comp) * 64 + (y & 7) * 8 + (x & 7)];
}

// component comp (1 or 2) at full-resolution (x, y), as jdsample.c upsamples it
__device__ int upsampled(const Chunk& c, int comp, int x, int y) {
    if (c.h == 1) return chroma_at(c, comp, x, y);
    const int ci = x >> 1, odd = x & 1;
    if (c.wc <= 2) return chroma_at(c, comp, ci, c.v == 2 ? y >> 1 : y);
    const int cj = odd ? min(ci + 1, c.wc - 1) : max(ci - 1, 0);
    if (c.v == 1) {
        const int near = chroma_at(c, comp, ci, y), other = chroma_at(c, comp, cj, y);
        if (!odd) return ci == 0 ? near : (3 * near + other + 1) >> 2;
        return ci == c.wc - 1 ? near : (3 * near + other + 2) >> 2;
    }
    const int ri = y >> 1, r2 = (y & 1) ? min(ri + 1, c.hc - 1) : max(ri - 1, 0);
    const int self = 3 * chroma_at(c, comp, ci, ri) + chroma_at(c, comp, ci, r2);
    const int other = 3 * chroma_at(c, comp, cj, ri) + chroma_at(c, comp, cj, r2);
    if (!odd) return ci == 0 ? (self * 4 + 8) >> 4 : (3 * self + other + 8) >> 4;
    return ci == c.wc - 1 ? (self * 4 + 7) >> 4 : (3 * self + other + 7) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int x) { return uint8_t(min(max(x, 0), 255)); }

__global__ void __launch_bounds__(256) pixel_kernel(const Launch L) {
    const int64_t x = int64_t(blockIdx.x) * 32 + (threadIdx.x & 31), y = int64_t(blockIdx.y) * 8 + (threadIdx.x >> 5);
    if (x >= L.cols || y >= L.rows) return;
    const int64_t gx = L.col0 + x, gy = L.row0 + y;
    const int64_t cr = gy / L.chunk_h, cc = gx / L.chunk_w;
    const int64_t k = (cr - L.chunk_row0) * L.grid_cols + (cc - L.chunk_col0);
    uint8_t* o = L.out + (y * L.cols + x) * L.spp;
    if (k < 0 || k >= L.n || L.errors[k] != 0) return;  // a failed chunk (bad data or a bad descriptor) keeps the cleared pixels
    const int64_t* d = L.descs + k * RSB_JPEG_DESC_FIELDS;
    const int X = int(gx - cc * L.chunk_w), Y = int(gy - cr * L.chunk_h);
    if (X >= d[kWidth] || Y >= d[kHeight]) return;  // not a decodable pixel: the chunk's error word says why
    Chunk c;
    c.s = L.samples + d[kFirstBlock] * 64;
    c.h = L.spp == 1 ? 1 : int(d[kH]);
    c.v = L.spp == 1 ? 1 : int(d[kV]);
    c.mx = (d[kWidth] + 8 * c.h - 1) / (8 * c.h);
    c.bpm = L.spp == 1 ? 1 : c.h * c.v + 2;
    c.wc = int((d[kWidth] + c.h - 1) / c.h);
    c.hc = int((d[kHeight] + c.v - 1) / c.v);
    const int yv = luma_at(c, X, Y);
    if (L.spp == 1) {
        o[0] = uint8_t(yv);
        return;
    }
    const int cb = upsampled(c, 1, X, Y), cr2 = upsampled(c, 2, X, Y);
    if (L.photometric == 2) {
        o[0] = uint8_t(yv);
        o[1] = uint8_t(cb);
        o[2] = uint8_t(cr2);
        return;
    }
    const int64_t xb = cb - 128, xr = cr2 - 128;
    o[0] = clamp255(yv + int((91881 * xr + 32768) >> 16));
    o[1] = clamp255(yv + int((-22554 * xb + 32768 + -46802 * xr) >> 16));
    o[2] = clamp255(yv + int((116130 * xb + 32768) >> 16));
}

}  // namespace

extern "C" int64_t rsb_jpeg_scratch_bytes(int64_t total_blocks) { return total_blocks < 0 ? -1 : total_blocks * RSB_JPEG_SCRATCH_PER_BLOCK; }

extern "C" int rsb_jpeg_decode_window(const uint8_t* staged, int64_t staged_len, const int64_t* descs, int32_t num_chunks, const int32_t* sets,
                                      int32_t num_sets, int64_t width, int64_t height, int32_t chunk_w, int32_t chunk_h, int32_t tiled, int32_t spp,
                                      int32_t photometric, int64_t row0, int64_t rows, int64_t col0, int64_t cols, uint8_t* out, void* scratch,
                                      int64_t scratch_bytes, int64_t total_blocks, int64_t* errors, void* stream) {
    if (!staged || !descs || !sets || !out || !scratch || !errors) return set_error(RSB_E_INVALID, "jpeg_decode_window: null pointer");
    if (staged_len < 0 || num_chunks < 1 || num_sets < 1 || total_blocks < 1)
        return set_error(RSB_E_INVALID, "jpeg_decode_window: %lld staged bytes, %d chunks, %d table sets, %lld blocks", (long long)staged_len,
                         num_chunks, num_sets, (long long)total_blocks);
    if (!((spp == 1 && photometric == 1) || (spp == 3 && (photometric == 2 || photometric == 6))))
        return set_error(RSB_E_INVALID, "jpeg_decode_window: %d bands with Photometric %d (need 1 with 1, or 3 with 2 or 6)", spp, photometric);
    if (width < 1 || height < 1 || chunk_w < 1 || chunk_h < 1 || chunk_w > 65535 || chunk_h > 65535 || (!tiled && chunk_w != width))
        return set_error(RSB_E_INVALID, "jpeg_decode_window: raster %lld x %lld with chunks %d x %d (tiled %d)", (long long)width, (long long)height,
                         chunk_w, chunk_h, tiled);
    if (row0 < 0 || col0 < 0 || rows < 1 || cols < 1 || row0 + rows > height || col0 + cols > width)
        return set_error(RSB_E_INVALID, "jpeg_decode_window: window rows [%lld, %lld) cols [%lld, %lld) outside the %lld x %lld raster",
                         (long long)row0, (long long)(row0 + rows), (long long)col0, (long long)(col0 + cols), (long long)width, (long long)height);
    const int64_t cr0 = row0 / chunk_h, cr1 = (row0 + rows - 1) / chunk_h, cc0 = col0 / chunk_w, cc1 = (col0 + cols - 1) / chunk_w;
    if (int64_t(num_chunks) != (cr1 - cr0 + 1) * (cc1 - cc0 + 1))
        return set_error(RSB_E_INVALID, "jpeg_decode_window: %d chunks, the window touches %lld", num_chunks, (long long)((cr1 - cr0 + 1) * (cc1 - cc0 + 1)));
    if (total_blocks > INT64_MAX / RSB_JPEG_SCRATCH_PER_BLOCK || scratch_bytes < total_blocks * RSB_JPEG_SCRATCH_PER_BLOCK)
        return set_error(RSB_E_INVALID, "jpeg_decode_window: scratch of %lld bytes, %lld blocks need %lld", (long long)scratch_bytes,
                         (long long)total_blocks, (long long)rsb_jpeg_scratch_bytes(total_blocks));
    if (reinterpret_cast<uintptr_t>(scratch) % 16) return set_error(RSB_E_INVALID, "jpeg_decode_window: scratch not 16-byte aligned");
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Launch L;
    L.staged = staged;
    L.staged_len = staged_len;
    L.descs = descs;
    L.n = num_chunks;
    L.sets = sets;
    L.n_sets = num_sets;
    L.spp = spp;
    L.photometric = photometric;
    L.chunk_w = chunk_w;
    L.chunk_h = chunk_h;
    L.row0 = row0;
    L.rows = rows;
    L.col0 = col0;
    L.cols = cols;
    L.chunk_row0 = cr0;
    L.chunk_col0 = cc0;
    L.grid_cols = cc1 - cc0 + 1;
    L.out = out;
    L.coefs = static_cast<int16_t*>(scratch);
    L.samples = static_cast<uint8_t*>(scratch) + total_blocks * 128;
    L.total_blocks = total_blocks;
    L.errors = errors;
    cudaError_t e = cudaMemsetAsync(scratch, 0, size_t(total_blocks) * 128, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(out, 0, size_t(rows * cols * spp), st);
    if (e != cudaSuccess) return set_cuda_error(e, "jpeg_decode_window: clear");
    huffman_kernel<<<(num_chunks + 127) / 128, 128, 0, st>>>(L);
    const int64_t want = (total_blocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS;
    idct_kernel<<<unsigned(want < 65535 * 8 ? want : 65535 * 8), IDCT_THREADS, 0, st>>>(L);
    pixel_kernel<<<dim3(unsigned((cols + 31) / 32), unsigned((rows + 7) / 8)), 256, 0, st>>>(L);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "jpeg_decode_window launch");
}
