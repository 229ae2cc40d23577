// bzip2.cuh — argument block of the BZip2 kernel and its scratch rule.
#pragma once
#include "common.cuh"

namespace swc {
namespace bzip2 {

// Stream mode as BZip2.multiDecompress (BZip2.swift:40-48): after each stream's end magic the reader aligns to the byte
// and, while bytes are left, the next stream follows in the same region.  Per unit the walk starts at byte at_in[unit]
// with at_out[unit] bytes and taken[unit] streams in front of it (the ones the block stage already delivered); taken[unit]
// counts on.  Each stream that ends, and on wrongCRC the failing one, gets an entry of the stream table (its output end
// and its first byte in the unit) when it fits stream_cap[unit]; n_streams[unit] is the streams returned (0 unless OK or
// wrongCRC).
struct Multi {
    const u64 *at_in = nullptr, *at_out = nullptr;                     // at_in == nullptr: one stream per unit
    u64 *taken = nullptr;
    u64 *n_streams = nullptr;                                           // may be null on its own
    const u64 *stream_off = nullptr, *stream_cap = nullptr;             // the stream table: all four, or null
    u64 *stream_end = nullptr, *stream_in_off = nullptr;
};

struct Args : DecodeIO {
    u8 *scratch;
    const u64 *scr_off;      // per unit, bytes into scratch
    const u8 *start_bits = nullptr;   // block mode: bit offset (0..7) of the block magic inside the unit's first byte
    int32_t block_mode = 0;           // 1: every unit is one block (magic first), decode it and stop; 0: whole streams
    const u8 *run = nullptr;          // per unit: 0 = skip the unit (writes nothing, not even its results); nullptr = all run
    Multi multi = {};                 // stream mode only: the multi-stream walk (its columns null: the first stream only)
};

// Room for a block's BWT text (the RLE1 form) when the unit may write `cap` output bytes.  RLE1 turns every run of four
// equal bytes into five, so a block that fits `cap` bytes of output can carry up to 5/4 x cap + 4 bytes of text; sizing the
// text by `cap` alone reported overflow for units whose output fits exactly.
__host__ __device__ __forceinline__ u64 bwt_capacity(u64 cap) { return (cap + (cap >> 2) + 8 + 3) & ~3ull; }

// scratch of one unit of output capacity `out_cap`: bwt | succ (u32) | selectors | text, a multiple of 256 bytes
__host__ __device__ __forceinline__ size_t scratch_per_unit(u64 out_cap) {
    const u64 scr_cap = bwt_capacity(out_cap);
    return (size_t)(scr_cap + 16 + scr_cap * 4 + 16 + 32768 + 16 + scr_cap + 256 + 255) & ~(size_t)255;
}

int launch(const Args &a, cudaStream_t stream);

}  // namespace bzip2
}  // namespace swc
