// lz4_compress.cuh — batched LZ4 block compression (lz4_compress.cu), the engine behind LZ4.compress.
#pragma once
#include "common.cuh"

namespace swc {
namespace lz4c {

constexpr u64 MAX_BLOCK = 4u << 20;      // the largest block a frame holds (LZ4+Compress.swift:51); longer units are unsupported
constexpr u64 MAX_DICT = 64u << 10;      // longer dictionary windows behave exactly as their last 64 KiB (see DESIGN §4.9)

constexpr u64 USER_DICT = 1ull << 63;   // dict_off[i] with this bit: the window is user_dict[dict_off[i] - USER_DICT ..)

struct Args : UnitIO {                  // out_len: parse: exact compressed size of the raw block
    const u64 *dict_off, *dict_len;      // unit i's dictionary window inside in_base (both null: no dictionary)
    const u8 *stored;                    // emit only, may be null: 1 = copy the block uncompressed (frame stored blocks)
    const u8 *user_dict = nullptr;       // a dictionary outside in_base, for the windows marked USER_DICT
};

// scratch of one unit with a window of `w` bytes (dictionary + block) and a block of `l` bytes
u64 unit_scratch(u64 w, u64 l);
// per-unit scratch offsets live in device memory (`scr_off`, one entry per unit of [first, first + count))
int parse(const Args &a, u64 first, u64 count, u8 *scr, const u64 *scr_off, cudaStream_t s);   // lz4c_chain + lz4c_parse
int emit(const Args &a, u64 first, u64 count, const u8 *scr, const u64 *scr_off, cudaStream_t s);  // lz4c_emit

}  // namespace lz4c
}  // namespace swc
