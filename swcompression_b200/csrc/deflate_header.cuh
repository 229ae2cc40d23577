// deflate_header.cuh — the Deflate block-header grammar (Deflate.swift:41-168) of the kernels that start blocks: K1L
// (inflate_lut.cu), K1w (inflate_warp.cu) and inflate_slow_kernel (inflate_slow.cu).  Each function makes the reference's
// checks in its source order and returns an swc status; tables and the copy of stored bytes stay with each kernel.
// The bit reader R provides  i64 avail() (the reference's bitsLeft),  u32 peek32() (the next 32 bits, first bit in bit 0;
// bits past the end of the input may be anything: only bits that avail() covers are used)  and  void skip(int n).
#pragma once
#include "deflate_tables.cuh"

namespace swc {
namespace inflate {
namespace hdr {

// BFINAL and BTYPE (:41-43, which read them unguarded; BTYPE 3 at :239)
template <class R>
__device__ __forceinline__ int block_start(R &r, bool &is_last, u32 &btype) {
    if (r.avail() < 3) return SWC_ERR_REFERENCE_TRAP;
    const u32 h = r.peek32() & 7;
    r.skip(3);
    is_last = (h & 1) != 0;
    btype = h >> 1;
    return btype == 3 ? SWC_DEFLATE_WRONG_BLOCK_TYPE : SWC_OK;
}

// Stored block (:45-65).  On SWC_OK the reader stands at the first of the `length` stored bytes: the caller copies and skips them.
template <class R>
__device__ __forceinline__ int stored_length(R &r, u32 &length) {
    r.skip((int)(r.avail() & 7));                        // align: the input ends on a byte boundary
    if (r.avail() < 32) return SWC_DEFLATE_WRONG_UNCOMPRESSED_BLOCK_LENGTHS;
    const u32 v = r.peek32();
    r.skip(32);
    length = v & 0xFFFFu;
    if ((length & (v >> 16)) != 0 || (r.avail() >> 3) < (i64)length) return SWC_DEFLATE_WRONG_UNCOMPRESSED_BLOCK_LENGTHS;
    return SWC_OK;
}

// HLIT, HDIST, HCLEN and the code-length code lengths of a dynamic block (:90-117); cl = the 19 lengths, 3 bits each, by symbol.
template <class R>
__device__ __forceinline__ int dynamic_counts(R &r, int &hlit, int &hdist, u64 &cl) {
    if (r.avail() < 14) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
    const u32 h = r.peek32();                            // one peek for the three fields
    hlit = (int)(h & 31) + 257;
    r.skip(5);
    if (hlit > 286) return SWC_DEFLATE_WRONG_SYMBOL;
    hdist = (int)((h >> 5) & 31) + 1;
    const int hclen = (int)((h >> 10) & 15) + 4;
    r.skip(9);
    if (r.avail() < 3 * hclen) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
    cl = 0;
    for (int i = 0; i < hclen; i++) { cl |= (u64)(r.peek32() & 7) << (3 * c_cl_order[i]); r.skip(3); }
    return SWC_OK;
}

// The HLIT + HDIST code lengths (:119-161).  decode(r, pk) returns the code-length symbol at the head of pk (= r.peek32())
// with its bits consumed, or -1 (symbolNotFound).  A code-length code has at most 7 bits, so the repeat field behind it is
// taken from the same peek.  sink(n, len, reps) receives every run of `reps` (<= 6) equal non-zero lengths from symbol n on;
// zero lengths are left to the caller's cleared table (a 17 / 18 run may overshoot the count before the final check catches it).
template <class R, class Decode, class Sink>
__device__ __forceinline__ int code_lengths(R &r, int count, Decode decode, Sink sink) {
    int n = 0, prev = 0;
    while (n < count) {
        const u32 pk = r.peek32();
        const i64 left = r.avail();
        const int sym = decode(r, pk);
        if (sym < 0) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
        const u32 x = pk >> (u32)(left - r.avail());
        int len = 0, reps = 1;
        if (sym <= 15) {
            len = sym;
        } else if (sym == 16) {
            if (n == 0) return SWC_DEFLATE_WRONG_SYMBOL;
            if (r.avail() < 2) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
            reps = (int)(x & 3) + 3;
            r.skip(2);
            if (n + reps > count) return SWC_DEFLATE_WRONG_SYMBOL;
            len = prev;
        } else if (sym == 17) {
            if (r.avail() < 3) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
            reps = (int)(x & 7) + 3;
            r.skip(3);
        } else {   // 18 (the alphabet has 19 symbols)
            if (r.avail() < 7) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
            reps = (int)(x & 127) + 11;
            r.skip(7);
        }
        if (len) sink(n, len, reps);
        n += reps;
        prev = len;
    }
    return n == count ? SWC_OK : SWC_DEFLATE_WRONG_SYMBOL;
}

// The code lengths of a fixed-Huffman block (Deflate+Constants.swift; HLIT 288, HDIST 32) through a sink of the same form
// (runs of up to 144).
template <class Sink>
__device__ __forceinline__ void fixed_lengths(Sink sink) {
    sink(0, 8, 144); sink(144, 9, 112); sink(256, 7, 24); sink(280, 8, 8); sink(288, 5, 32);
}

}  // namespace hdr
}  // namespace inflate
}  // namespace swc
