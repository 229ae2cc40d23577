// lz4.cuh — argument block of the LZ4 block kernel.
#pragma once
#include "common.cuh"

namespace swc {
namespace lz4 {

// in_off / in_len are indexed by block (bit 63 of in_len = stored, uncompressed block); the other columns and n by unit.
// Unit u is block u unless first_blk / n_blk are set.
struct Args : UnitIO {
    const u32 *first_blk, *n_blk;     // per unit chain, or both null: unit u = block u
    const u8 *dict;                   // prefix the first block of every unit may reference (may be null)
    u64 dict_len;
    void *scratch;                    // optional: two_phase_scratch_bytes(n, in_total) bytes enables the two-phase path
};

size_t two_phase_scratch_bytes(u64 n, u64 in_total);
int launch(const Args &a, cudaStream_t stream);

}  // namespace lz4
}  // namespace swc
