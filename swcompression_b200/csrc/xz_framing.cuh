// xz_framing.cuh — the XZ container grammar, shared by the host calls (api_lzma.cu: swc_xz_unarchive, swc_xz_split_unarchive
// and their backward prefetch walk) and the device batch (xz_batch.cu: swc_xz_unarchive_batch).  The library is built without
// relocatable device code, so the one copy lives in this header, next to archive_header.cuh.
// Reference: Sources/XZ/XZArchive.swift:27-218, XZBlock.swift:18-97, XZStreamHeader.swift:33-57,
// LittleEndianByteReader+XZ.swift:10-30.
//
// Every function reads through an `Rd` bounded by the archive's length: a read the reference performs without a guard traps
// there (BitByteData precondition) and reports SWC_ERR_REFERENCE_TRAP here.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/swcgpu.h"
#include "archive_header.cuh"

namespace swc {
namespace xz {

struct Rd {
    const uint8_t *p; size_t n, off;
    __host__ __device__ bool need(size_t k) const { return n - off >= k; }
};

__host__ __device__ inline uint32_t rd32(const uint8_t *q) { return (uint32_t)q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16 | (uint32_t)q[3] << 24; }

// multiByteInteger() LittleEndianByteReader+XZ.swift:10-30
__host__ __device__ inline int multibyte(Rd &r, int64_t *val) {
    if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
    int i = 1;
    int64_t result = r.p[r.off++];
    if (result <= 127) { *val = result; return SWC_OK; }
    result &= 0x7F;
    for (;;) {
        if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
        unsigned b = r.p[r.off++];
        if (i >= 9 || b == 0) return SWC_XZ_MULTI_BYTE_INTEGER_ERROR;
        result += (int64_t)(b & 0x7F) << (7 * i);
        i++;
        if ((b & 0x80) == 0) break;
    }
    *val = result;
    return SWC_OK;
}

__host__ __device__ inline int check_size(int t) { return t == 0 ? 0 : t == 1 ? 4 : t == 4 ? 8 : 32; }

__host__ __device__ inline bool is_stream_magic(const uint8_t *q) {
    return q[0] == 0xFD && q[1] == 0x37 && q[2] == 0x7A && q[3] == 0x58 && q[4] == 0x5A && q[5] == 0x00;
}

// XZStreamHeader.init XZStreamHeader.swift:33-57; *ctype is the check type
__host__ __device__ inline int stream_header(Rd &r, int *ctype) {
    if (!r.need(12)) return SWC_ERR_REFERENCE_TRAP;
    if (!is_stream_magic(r.p + r.off)) return SWC_XZ_WRONG_MAGIC;
    const uint8_t *fl = r.p + r.off + 6;
    if (crc32_framing(fl, 2) != rd32(r.p + r.off + 8)) return SWC_XZ_WRONG_INFO_CRC;
    if (!(fl[0] == 0 && (fl[1] & 0xF0) == 0)) return SWC_XZ_WRONG_FIELD;
    const int t = fl[1] & 0xF;
    if (!(t == 0 || t == 1 || t == 4 || t == 0x0A)) return SWC_XZ_WRONG_FIELD;
    r.off += 12;
    *ctype = t;
    return SWC_OK;
}

enum { FILTER_DELTA = 0x03, FILTER_LZMA2 = 0x21 };

struct BlockHeader {
    size_t hstart;                   // offset of the header-size byte
    int64_t comp_size, uncomp_size;  // -1 when the field is absent
    int nfilters;
    int kind[4], param[4];           // FILTER_LZMA2: dictionary byte; FILTER_DELTA: distance 1..256
};

// XZBlock.init XZBlock.swift:18-75, up to and including the header CRC.  `hsize_byte` (non-zero) has been read already;
// on success r.off is the block's first data byte.
__host__ __device__ inline int block_header(Rd &r, unsigned hsize_byte, BlockHeader &h) {
    h.hstart = r.off - 1;
    const size_t real = ((size_t)hsize_byte + 1) * 4;
    if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
    const unsigned flags = r.p[r.off++];
    h.nfilters = (flags & 0x03) + 1;
    if (flags & 0x3C) return SWC_XZ_WRONG_FIELD;
    h.comp_size = h.uncomp_size = -1;
    int st;
    if (flags & 0x40) { if ((st = multibyte(r, &h.comp_size))) return st; }
    if (flags & 0x80) { if ((st = multibyte(r, &h.uncomp_size))) return st; }
    for (int f = 0; f < h.nfilters; f++) {
        int64_t id, psz;
        if ((st = multibyte(r, &id))) return st;
        if ((uint64_t)id >= 0x4000000000000000ull) return SWC_XZ_WRONG_FILTER_ID;
        if (id == FILTER_LZMA2) {
            if ((st = multibyte(r, &psz))) return st;
            if (psz != 1) return SWC_LZMA2_WRONG_DICTIONARY_SIZE;
            if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
            h.kind[f] = FILTER_LZMA2; h.param[f] = r.p[r.off++];
        } else if (id == FILTER_DELTA) {
            if ((st = multibyte(r, &psz))) return st;
            if (psz != 1) return SWC_XZ_WRONG_FIELD;
            if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
            h.kind[f] = FILTER_DELTA; h.param[f] = (r.p[r.off++] + 1) & 0xFF;
            if (h.param[f] == 0) h.param[f] = 256;
        } else return SWC_XZ_WRONG_FILTER_ID;
    }
    while ((int64_t)(r.off - h.hstart) < (int64_t)real - 4) {
        if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
        if (r.p[r.off++] != 0) return SWC_XZ_WRONG_PADDING;
    }
    if (!r.need(4)) return SWC_ERR_REFERENCE_TRAP;
    const uint32_t hcrc = rd32(r.p + r.off);
    if (r.n - h.hstart < real - 4) return SWC_ERR_REFERENCE_TRAP;
    if (crc32_framing(r.p + h.hstart, real - 4) != hcrc) return SWC_XZ_WRONG_INFO_CRC;
    r.off = h.hstart + real;
    return SWC_OK;
}

// XZBlock.swift:77-97 after the filters ran: the size fields, then block padding.  r.off is behind the data, which started
// at `data_start` and decoded to `out_len` bytes; *unpadded is the index's Unpadded Size (check included).
__host__ __device__ inline int block_tail(Rd &r, const BlockHeader &h, size_t data_start, int64_t out_len, int csize, int64_t *unpadded) {
    if (!((h.comp_size < 0 || h.comp_size == (int64_t)(r.off - data_start)) && (h.uncomp_size < 0 || h.uncomp_size == out_len)))
        return SWC_XZ_WRONG_DATA_SIZE;
    const int64_t unp = (int64_t)(r.off - h.hstart);
    if (unp % 4 != 0) {
        for (int i = 0, pad = 4 - (int)(unp % 4); i < pad; i++) {
            if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
            if (r.p[r.off++] != 0) return SWC_XZ_WRONG_PADDING;
        }
    }
    *unpadded = unp + csize;
    return SWC_OK;
}

// the check field behind a block: *stored points at its check_size(ctype) bytes
__host__ __device__ inline int check_field(Rd &r, int ctype, const uint8_t **stored) {
    const size_t cs = (size_t)check_size(ctype);
    if (!r.need(cs)) return SWC_ERR_REFERENCE_TRAP;
    *stored = r.p + r.off;
    r.off += cs;
    return SWC_OK;
}

// processIndex XZArchive.swift:132-167.  The index indicator byte (0) has been read already.  `blocks(k, &unpadded,
// &uncompressed)` gives block k's record as the block walk found it; *index_size is the index's size with its CRC.  The host
// passes a host-only `blocks`, the device a device one: the pragma keeps nvcc from checking the instantiation it never uses.
#pragma nv_exec_check_disable
template <class Blocks>
__host__ __device__ inline int index(Rd &r, int64_t nblocks, Blocks &&blocks, int64_t *index_size) {
    const size_t istart = r.off - 1;
    int64_t v; int st;
    if ((st = multibyte(r, &v))) return st;
    if (v != nblocks) return SWC_XZ_WRONG_FIELD;
    for (int64_t k = 0; k < nblocks; k++) {
        int64_t unp, unc;
        blocks(k, &unp, &unc);
        if ((st = multibyte(r, &v))) return st;
        if (v != unp) return SWC_XZ_WRONG_FIELD;
        if ((st = multibyte(r, &v))) return st;
        if (v != unc) return SWC_XZ_WRONG_DATA_SIZE;
    }
    int64_t isz = (int64_t)(r.off - istart);
    if (isz % 4 != 0) {
        for (int i = 0, pad = 4 - (int)(isz % 4); i < pad; i++) {
            if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
            if (r.p[r.off++] != 0) return SWC_XZ_WRONG_PADDING;
            isz++;
        }
    }
    if (!r.need(4)) return SWC_ERR_REFERENCE_TRAP;
    if (crc32_framing(r.p + istart, (size_t)isz) != rd32(r.p + r.off)) return SWC_XZ_WRONG_INFO_CRC;
    r.off = istart + (size_t)isz + 4;
    *index_size = isz + 4;
    return SWC_OK;
}

// processFooter XZArchive.swift:169-192
__host__ __device__ inline int footer(Rd &r, int ctype, int64_t index_size) {
    if (!r.need(12)) return SWC_ERR_REFERENCE_TRAP;
    const uint32_t fcrc = rd32(r.p + r.off);
    const int64_t backward = ((int64_t)rd32(r.p + r.off + 4) + 1) * 4;
    const unsigned fflags = r.p[r.off + 8] | r.p[r.off + 9] << 8;
    if (crc32_framing(r.p + r.off + 4, 6) != fcrc) return SWC_XZ_WRONG_INFO_CRC;
    if (backward != index_size) return SWC_XZ_WRONG_FIELD;
    if (!((fflags & 0xFF) == 0 && ((fflags & 0xF00) >> 8) == (unsigned)ctype && (fflags & 0xF000) == 0)) return SWC_XZ_WRONG_FIELD;
    if (!(r.p[r.off + 10] == 0x59 && r.p[r.off + 11] == 0x5A)) return SWC_XZ_WRONG_MAGIC;
    r.off += 12;
    return SWC_OK;
}

// processPadding XZArchive.swift:194-218
__host__ __device__ inline int padding(Rd &r) {
    if (r.off >= r.n) return SWC_OK;
    int pad = 0;
    for (;;) {
        const unsigned b = r.p[r.off++];
        if (b != 0) { if (pad % 4 != 0) return SWC_XZ_WRONG_PADDING; break; }
        if (r.off >= r.n) { if (pad % 4 != 3) return SWC_XZ_WRONG_PADDING; return SWC_OK; }
        pad++;
    }
    r.off -= 1;
    return SWC_OK;
}

// ---- the backward walk: stream padding, footer and index, read from the end of the archive --------------------------
// The footer's backward size locates the index, and the index's Unpadded Sizes locate the stream header.  Nothing here is
// trusted: every size is checked against the bytes before it, and any inconsistency ends the walk (returns false).
struct BackStream {
    size_t start;          // offset of the stream header
    size_t rec_off;        // offset of the first index record
    size_t istart;         // offset of the index indicator
    size_t foot;           // offset of the stream footer (the index ends here)
    int64_t count;         // index records
    int ctype;             // check type from the footer flags
    uint64_t uncomp;       // sum of the records' Uncompressed Sizes
    bool uncomp_ok;        // false when that sum does not fit in 63 bits
};

__host__ __device__ inline bool back_stream(const uint8_t *in, size_t pos, BackStream &s) {
    while (pos >= 4 && in[pos - 1] == 0 && in[pos - 2] == 0 && in[pos - 3] == 0 && in[pos - 4] == 0) pos -= 4;   // stream padding
    if (pos < 32 || in[pos - 2] != 0x59 || in[pos - 1] != 0x5A) return false;
    const size_t foot = pos - 12;
    s.ctype = in[foot + 9] & 0xF;
    const size_t index_size = ((size_t)rd32(in + foot + 4) + 1) * 4;
    if (index_size + 12 > foot) return false;
    const size_t istart = foot - index_size;
    if (in[istart] != 0) return false;
    Rd ir{in, foot, istart + 1};
    int64_t count = 0;
    if (multibyte(ir, &count) || count < 0 || count > 1000000) return false;
    s.rec_off = ir.off;
    uint64_t blocks_total = 0, uncomp = 0;
    bool uncomp_ok = true;
    for (int64_t k = 0; k < count; k++) {             // untrusted sizes: every sum is checked against the bytes before the index
        int64_t unp, unc;
        if (multibyte(ir, &unp) || multibyte(ir, &unc) || unp <= 0 || unc < 0) return false;
        if ((uint64_t)unp > (uint64_t)istart) return false;
        const uint64_t padded = ((uint64_t)unp + 3) & ~3ull;
        if (padded > (uint64_t)istart - blocks_total) return false;
        blocks_total += padded;
        if ((uint64_t)unc > ((1ull << 63) - 1) - uncomp) uncomp_ok = false;
        else uncomp += (uint64_t)unc;
    }
    if (blocks_total + 12 > istart) return false;
    s.start = istart - (size_t)blocks_total - 12;
    if (!is_stream_magic(in + s.start)) return false;
    s.istart = istart;
    s.foot = foot;
    s.count = count;
    s.uncomp = uncomp;
    s.uncomp_ok = uncomp_ok;
    return true;
}

// the size an archive of n bytes declares: the sum of its indexes' Uncompressed Sizes, when the backward walk covers it down
// to byte 0; else 0
__host__ __device__ inline uint64_t declared_size(const uint8_t *in, size_t n) {
    size_t pos = n;
    uint64_t total = 0;
    while (pos > 0) {
        BackStream s;
        if (!back_stream(in, pos, s) || !s.uncomp_ok || s.uncomp > ((1ull << 63) - 1) - total) return 0;
        total += s.uncomp;
        pos = s.start;
    }
    return total;
}

}  // namespace xz
}  // namespace swc
