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
constexpr u64 CHECKPOINT_BYTES = 24;     // sizeof(Checkpoint) in deflate_compress.cu
constexpr u64 CHAIN_ENTRY_BYTES = 4;     // a link-builder chain entry for 3-byte keys

struct Args : UnitIO {};                // out_len: the exact size of the Deflate stream

// one slice of units [first, first + count): per-unit scratch offsets, and prefix sums of link tiles and emit chunks
// (count + 1 entries each), all in device memory.  `tiles` / `chunks` size the grids and may exceed the totals
// tile_start[count] / chunk_start[count]; the kernels stop at the totals.
struct Plan {
    const u64 *scr_off, *tile_start, *chunk_start;
    u64 tiles, chunks;
};

// ---- the sizing rule, shared by the host planner of the raw batch and the device planner of the archive batches ----
__host__ __device__ __forceinline__ u64 a256(u64 v) { return (v + 255) & ~(u64)255; }
__host__ __device__ __forceinline__ u64 keyed(u64 n) { return n >= 3 ? n - 2 : 0; }       // positions with a full key
__host__ __device__ __forceinline__ u64 unit_tiles(u64 n) { return n >= MAX_UNIT ? 0 : (keyed(n) + TILE - 1) / TILE; }
__host__ __device__ __forceinline__ u64 unit_chunks(u64 n) { return n >= MAX_UNIT ? 0 : n ? (n + CHUNK - 1) / CHUNK : 1; }
// link-builder chain entries: every keyed position, plus REACH of halo in front of every tile but the first
__host__ __device__ __forceinline__ u64 chain_entries(u64 n) {
    const u64 t = unit_tiles(n);
    return t ? keyed(n) + (t - 1) * REACH : 0;
}
// the chains, later reused for the 8-byte parse records
__host__ __device__ __forceinline__ u64 big_bytes(u64 n) {
    const u64 c = CHAIN_ENTRY_BYTES * chain_entries(n), r = 8 * (n / 3 + 2);
    return c > r ? c : r;
}
// scratch of one unit of n input bytes (0 for an unsupported unit); at most 9 n + 2048
__host__ __device__ __forceinline__ u64 unit_scratch(u64 n) {
    if (n >= MAX_UNIT) return 0;
    return 256 + a256(2 * keyed(n)) + a256(4 * ((keyed(n) + 31) / 32)) + a256(CHECKPOINT_BYTES * (unit_chunks(n) + 1)) +
           a256(8 * unit_chunks(n)) + a256(big_bytes(n));
}

// link builder, parse, emit and seam merge of one slice
int run(const Args &a, u64 first, u64 count, u8 *scr, const Plan &p, cudaStream_t s);

}  // namespace deflatec
}  // namespace swc
