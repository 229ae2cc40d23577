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
    const u8 *no_dict;                // optional, per unit: non-zero = this unit decodes without the dictionary
};

size_t two_phase_scratch_bytes(u64 n, u64 in_total);
int launch(const Args &a, cudaStream_t stream);

// The two phases of the single-block path on their own (the frame batch sizes and places its blocks between them).
// rec_base[u] is where unit u's records start in `recs`; a block of b bytes writes at most b / 3 + 2 of them.
// launch_parse leaves out_len[u] = the decoded size and status[u] = the final status, LZ4_INTERNAL_FALLBACK standing for
// "sound, copied by the one-kernel decoder"; it stores nothing.  launch_exec copies every unit whose status is SWC_OK or
// LZ4_INTERNAL_FALLBACK to out_off[u] (out_cap[u] must hold it) and turns the latter into SWC_OK.
constexpr int LZ4_INTERNAL_FALLBACK = 9002;
int launch_parse(const Args &a, const u64 *rec_base, u64 *recs, u32 *rec_count, cudaStream_t stream);
int launch_exec(const Args &a, const u64 *rec_base, const u64 *recs, const u32 *rec_count, cudaStream_t stream);

}  // namespace lz4
}  // namespace swc
