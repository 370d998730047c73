// Layouts shared by the JPEG chunk parser (rsb_jpeg_parse.cpp, host) and decoder (rsb_jpeg.cu, device); the public sizes are in
// include/rsb200.h.
#pragma once
#include <stdint.h>

#include "../../include/rsb200.h"

namespace rsb_jpeg {

// a chunk's descriptor: int64 [RSB_JPEG_DESC_FIELDS]
enum DescField {
    kOffset = 0,    // the entropy-coded bytes: file offset (parse) or offset in the staged bytes (decode)
    kLength,        // their length (up to the marker after the scan)
    kSet,           // the table set
    kWidth,         // frame width and height
    kHeight,
    kH,             // luma sampling factors (1, 1 for one component)
    kV,
    kRestart,       // restart interval in MCUs, 0 for none
    kBlocks,        // 8 x 8 blocks of the chunk (whole MCUs of every component)
    kFirstBlock,    // decode: the chunk's first block in the scratch (parse: 0)
    kChunk,         // the strip or tile index in the file
    kReserved,
};

// a table set: int32 [RSB_JPEG_SET_WORDS] = quant [3][64] (natural order, as ISLOW_MULT_TYPE short), then per component the DC and
// the AC table, each HUFF_WORDS: lookup [256] ((length << 8) | symbol; 9 << 8 for codes longer than 8 bits), maxcode [18],
// valoffset [18], huffval [256] (libjpeg's d_derived_tbl)
constexpr int kLookup = 0, kMaxcode = 256, kValoffset = 274, kHuffval = 292, kHuffWords = 548;
constexpr int kQuantWords = 3 * 64;
constexpr int kSetWords = kQuantWords + 6 * kHuffWords;

static_assert(kSetWords == RSB_JPEG_SET_WORDS, "include/rsb200.h and rsb_jpeg.h disagree");

constexpr int huff_base(int comp, int ac) { return kQuantWords + (2 * comp + ac) * kHuffWords; }

// data error codes of the decoder's per-chunk error words (code | mcu << 8)
enum DataError { kOk = 0, kBadCode, kAcPast63, kBadMarker, kExtraneous, kTruncated, kBadDescriptor };

}  // namespace rsb_jpeg
