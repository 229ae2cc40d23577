// bzip2_compress.cuh — batched BZip2 compression (bzip2_compress.cu), the engine behind BZip2.compress.
#pragma once
#include "common.cuh"

namespace swc {
namespace bzip2c {

constexpr u32 RAW_PER_LEVEL = 80000;     // BZip2+Compress.swift:47: a raw block is blockSize.sizeInKilobytes * 800 bytes
constexpr u32 MAX_SYMBOLS = 258;         // RUNA, RUNB, 255 MTF indices and EOB
constexpr u32 MAX_LEN = 11;              // every code length of a 50-symbol group (DESIGN §4.11, lemma 4)

struct Args : UnitIO {                  // out_len: the exact size of the .bz2 stream, also for a unit that overflows
    u32 level;                           // BlockSize.rawValue, 1...9
};

// host plan of one slice, uploaded into the front of the slice's scratch
struct BlockPlan { u64 scr, group0; u32 unit, index, raw, cap; };   // cap: RLE1 bytes the block may produce
struct UnitPlan { u64 stage, stage_bytes; u32 block0, blocks; };

inline u64 a256(u64 v) { return (v + 255) & ~255ull; }
inline u32 rle_cap(u32 raw) { return raw + raw / 4; }                  // RLE1 writes at most 5 bytes per 4
inline u64 group_slots(u32 raw) { return (rle_cap(raw) + 1 + 49) / 50; }
inline u64 block_scratch(u32 raw) { return 29 * a256(rle_cap(raw) + 8); }
// the largest stream BZip2.compress writes for a unit of n bytes (DESIGN §4.11, lemma 4)
u64 max_stream_bytes(u64 n, u32 level);
u64 unit_blocks(u64 n, u32 level);
u64 unit_scratch(u64 n, u32 level);      // per-block scratch and the unit's staging words

// every stage of one slice [first, first + count) of units; `scr` holds the plans at the offsets in `p`
struct Slice {
    const BlockPlan *blocks; const UnitPlan *units;
    u64 nblocks, ngroups;
    u8 *meta, *groups;                   // per-block results, per-group-slot results
    u8 *stage; u64 stage_bytes;          // the zero-filled staging words of every unit
    u64 max_stage, copy_chunk;           // the largest unit's staging bytes; bytes per CTA of the final copy
};
int run(const Args &a, u64 first, u64 count, const Slice &sl, cudaStream_t s);

}  // namespace bzip2c
}  // namespace swc
