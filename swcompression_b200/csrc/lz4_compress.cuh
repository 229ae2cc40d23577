// lz4_compress.cuh — batched LZ4 block compression (lz4_compress.cu), the engine behind LZ4.compress.
#pragma once
#include "common.cuh"

namespace swc {
namespace lz4c {

constexpr u64 MAX_BLOCK = 4u << 20;      // the largest block a frame holds (LZ4+Compress.swift:51); longer units are unsupported
constexpr u64 MAX_DICT = 64u << 10;      // longer dictionary windows behave exactly as their last 64 KiB (see DESIGN §4.9)

struct Args {
    const u8 *in_base;
    const u64 *in_off, *in_len;          // the block of unit i
    const u64 *dict_off, *dict_len;      // its dictionary window inside in_base (both null: no dictionary)
    u8 *out_base;
    const u64 *out_off, *out_cap;
    u64 *out_len;                        // parse: exact compressed size of the raw block
    int32_t *status;
    const u8 *stored;                    // emit only, may be null: 1 = copy the block uncompressed (frame stored blocks)
    u64 n;
};

// scratch of one unit with a window of `w` bytes (dictionary + block) and a block of `l` bytes
u64 unit_scratch(u64 w, u64 l);
// per-unit scratch offsets live in device memory (`scr_off`, one entry per unit of [first, first + count))
int parse(const Args &a, u64 first, u64 count, u8 *scr, const u64 *scr_off, cudaStream_t s);   // lz4c_chain + lz4c_parse
int emit(const Args &a, u64 first, u64 count, const u8 *scr, const u64 *scr_off, cudaStream_t s);  // lz4c_emit

}  // namespace lz4c
}  // namespace swc
