// archive_header.cuh — the gzip member header and zlib stream header grammars, shared by the host calls (api_wrappers.cu:
// swc_gzip_header_parse, swc_zlib_header_parse, the single and multi-member unarchive calls) and the device batch
// (unarchive_batch.cu).  The library is built without relocatable device code, so the one copy lives in this header.
// Reference: Sources/GZip/GzipHeader.swift:68-199, Sources/Zlib/ZlibHeader.swift:47-93.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/swcgpu.h"

namespace swc {

// bitwise CRC-32 of header / index / footer fields; payload CRCs run in checks.cu
__host__ __device__ inline uint32_t crc32_framing(const uint8_t *p, size_t n) {
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) {
        c ^= p[i];
        for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    }
    return ~c;
}

// GzipHeader.init(_: LsbBitReader), GzipHeader.swift:68-199 — one pass over the member's header that both validates it and
// records where its fields are.  Written against the Swift source (guards in source order, one `Cursor` read per
// `reader.byte()`); `left()` is `reader.bytesLeft`.  Reads the reference performs WITHOUT a guard trap there (BitByteData
// precondition): they report SWC_ERR_REFERENCE_TRAP here.
struct Cursor {
    const uint8_t *base; size_t n, at;
    __host__ __device__ size_t left() const { return n - at; }
    __host__ __device__ bool finished() const { return at >= n; }
};

__host__ __device__ inline int gzip_parse(const uint8_t *in, size_t n, size_t member_off, swc_gzip_header *h) {
    if (member_off > n) return SWC_GZIP_WRONG_MAGIC;
    Cursor c{in, n, member_off};
    swc_gzip_header out = {};
    if (c.left() < 10) return SWC_GZIP_WRONG_MAGIC;                                  // :70-71
    if (in[c.at] != 0x1f || in[c.at + 1] != 0x8b) return SWC_GZIP_WRONG_MAGIC;       // :74-76 (uint16 == 0x8b1f)
    if (in[c.at + 2] != 8) return SWC_GZIP_WRONG_COMPRESSION_METHOD;                 // :80-82
    out.compression_method = 8;
    const unsigned flg = in[c.at + 3];
    if ((flg & 0xE0) != 0) return SWC_GZIP_WRONG_FLAGS;                              // :86-88
    out.modification_time = (uint32_t)in[c.at + 4] | (uint32_t)in[c.at + 5] << 8 | (uint32_t)in[c.at + 6] << 16 | (uint32_t)in[c.at + 7] << 24;
    out.os_type = in[c.at + 9];                                                      // :103-105 (XFL at +8 is only hashed)
    out.is_text_file = (flg & 0x01) != 0;                                            // :107
    c.at += 10;
    if (flg & 0x04) {                                                                // FEXTRA :111-155
        if (c.left() < 2) return SWC_GZIP_WRONG_MAGIC;                               // :112-113
        size_t xlen = (size_t)in[c.at] | (size_t)in[c.at + 1] << 8;
        c.at += 2;
        if (!(c.left() >= xlen && xlen >= 4)) return SWC_GZIP_WRONG_MAGIC;           // :123-124
        out.extra_off = c.at; out.extra_len = xlen;
        long remaining = (long)xlen;                                                 // the reference's signed `xlen` countdown
        while (remaining > 0) {                                                      // :125
            // si1, si2, two length bytes: four unguarded reader.byte() calls (:126-140)
            if (c.left() < 2) return SWC_ERR_REFERENCE_TRAP;
            if (in[c.at + 1] == 0) return SWC_GZIP_WRONG_FLAGS;                      // :131-132 (checked before the length is read)
            if (c.left() < 4) return SWC_ERR_REFERENCE_TRAP;
            const long len = (long)in[c.at + 2] | (long)in[c.at + 3] << 8;
            c.at += 4;
            remaining -= 4;                                                          // :141
            if (remaining < len) return SWC_GZIP_WRONG_MAGIC;                        // :145-146
            if ((long)c.left() < len) return SWC_ERR_REFERENCE_TRAP;                 // :148-152 unguarded payload reads
            c.at += (size_t)len;
            remaining -= len;                                                        // :154
        }
    }
    if (flg & 0x08) {                                                                // FNAME :159-172
        out.has_file_name = 1; out.file_name_off = c.at;
        for (;;) {
            if (c.finished()) return SWC_GZIP_WRONG_MAGIC;                           // :162-163
            if (in[c.at++] == 0) break;
        }
        out.file_name_len = c.at - 1 - out.file_name_off;
    }
    if (flg & 0x10) {                                                                // FCOMMENT :177-190
        out.has_comment = 1; out.comment_off = c.at;
        for (;;) {
            if (c.finished()) return SWC_GZIP_WRONG_MAGIC;                           // :180-181
            if (in[c.at++] == 0) break;
        }
        out.comment_len = c.at - 1 - out.comment_off;
    }
    if (flg & 0x02) {                                                                // FHCRC :194-200
        if (c.left() < 2) return SWC_GZIP_WRONG_MAGIC;
        const unsigned stored = (unsigned)in[c.at] | (unsigned)in[c.at + 1] << 8;
        if ((crc32_framing(in + member_off, c.at - member_off) & 0xFFFFu) != stored) return SWC_GZIP_WRONG_HEADER_CRC;
        c.at += 2;
    }
    out.header_len = c.at - member_off;
    if (h) *h = out;
    return SWC_OK;
}

// ZlibHeader.init(_: LsbBitReader), ZlibHeader.swift:47-93
__host__ __device__ inline int zlib_parse(const uint8_t *in, size_t n, swc_zlib_header *h) {
    if (n < 2) return SWC_ZLIB_WRONG_COMPRESSION_METHOD;                             // :49-50
    const unsigned cmf = in[0], flg = in[1];
    if ((cmf & 0xF) != 8) return SWC_ZLIB_WRONG_COMPRESSION_METHOD;                  // :56-58
    const unsigned cinfo = (cmf & 0xF0) >> 4;
    if (cinfo > 7) return SWC_ZLIB_WRONG_COMPRESSION_INFO;                           // :62-64
    // CompressionLevel(rawValue: (flags & 0xC0) >> 6) covers 0...3: it cannot fail (:80-82)
    if ((((unsigned)cmf << 8) + flg) % 31 != 0) return SWC_ZLIB_WRONG_FCHECK;        // :84-85 (Swift precedence: (cmf << 8) + flags)
    size_t len = 2;
    if ((flg & 0x20) != 0) {                                                         // FDICT: four bytes are skipped (:88-92)
        if (n - 2 < 4) return SWC_ZLIB_WRONG_FCHECK;
        len = 6;
    }
    if (h) { h->compression_method = 8; h->compression_level = (int32_t)((flg & 0xC0) >> 6); h->window_size = 1 << (cinfo + 8); h->header_len = len; }
    return SWC_OK;
}

}  // namespace swc
