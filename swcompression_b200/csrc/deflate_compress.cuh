// deflate_compress.cuh — batched Deflate compression (deflate_compress.cu), the engine behind Deflate.compress,
// GzipArchive.archive and ZlibArchive.archive.
#pragma once
#include "common.cuh"

namespace swc {
namespace deflatec {

constexpr u64 MAX_UNIT = 1ull << 32;     // units of 4 GiB or more are unsupported (positions are 32-bit)
constexpr u32 REACH = 32768;             // Deflate+Compress.swift:166 (`distance <= 32768`)
constexpr u32 TILE = 64u << 10;          // positions per link-builder tile; each tile reads REACH bytes of halo in front
constexpr u32 CHUNK = 4096;              // input bytes per emit checkpoint (> 258, so every chunk but the last starts a symbol)

struct Args : UnitIO {};                // out_len: the exact size of the Deflate stream

// one slice of units [first, first + count): per-unit scratch offsets, and prefix sums of link tiles and emit chunks
// (count + 1 entries each), all in device memory
struct Plan {
    const u64 *scr_off, *tile_start, *chunk_start;
    u64 tiles, chunks;
};

u64 unit_scratch(u64 n);                 // scratch of one unit of n input bytes (0 for an unsupported unit)
u64 unit_tiles(u64 n);
u64 unit_chunks(u64 n);
// link builder, parse, emit and seam merge of one slice
int run(const Args &a, u64 first, u64 count, u8 *scr, const Plan &p, cudaStream_t s);

}  // namespace deflatec
}  // namespace swc
