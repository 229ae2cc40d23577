// inflate.cuh — argument block shared by the Deflate kernels and the host launcher, and the match-record format that
// carries a unit from the Huffman stage (K1L inflate_lut_kernel / K1w inflate_warp_kernel) to lz_resolve_kernel (K2).
#pragma once
#include "common.cuh"

namespace swc {
namespace inflate {

struct BatchArgs {
    const u8 *in_base;
    const u64 *in_off, *in_len;
    const u8 *start_bits;      // may be null
    u8 *out_base;
    const u64 *out_off, *out_cap;
    u64 *out_len, *consumed_bits;
    int32_t *status;
    u64 n;
    u32 *rec_base;             // match-record scratch
    u32 *rec_count;            // n entries
    unsigned long long *ticket; // unit ticket counters of the persistent-lane kernels: [0] K1w, [1] K1L (zeroed by the launcher)
};

// ---- match records ----
// The Huffman stage writes every literal (and every stored-block byte) straight to its final output position and turns
// every match, in stream order, into one 4-byte record
//     {dist - 1 : 15 | esc = 0 : 1 | len - 3 : 8 | run : 8}      run = literal bytes since the end of the previous match
// A run longer than 255 is first cut down by an escape record {skip & 0x7FFF : 15 | esc = 1 : 1 | skip >> 15 : 16} that
// only advances the output position by skip = run & ~255.  K2 places each match with a warp scan of run + len (escape:
// skip) and copies it.  Matches that end past the output capacity get no record: such a unit fails with an overflow
// status and K2 skips it.  rec_count[unit] holds the number of records written.
//
// A unit whose output region starts at byte `out_off` owns records [out_off/3, (out_off+cap)/3): every match record
// accounts for >= 3 output bytes and every escape for >= 256, so disjoint output regions give disjoint record regions
// without a prefix sum over the units.
__host__ __device__ __forceinline__ u64 rec_start(u64 out_off) { return out_off / 3; }
inline size_t scratch_bytes(u64 n, u64 out_capacity_total) {
    return (size_t)((out_capacity_total / 3 + 2) * 4 + n * 4 + 1024);
}

constexpr u32 REC_ESC = 0x8000u;   // also the padding record: an escape that skips nothing

// appends the records of a match of `len` bytes at distance `dist` that follows `run` literal bytes to rec[nrec...]
__device__ __forceinline__ void put_match(u32 *rec, u32 &nrec, u32 run, u32 len, u32 dist) {
    if (run > 255) {
        const u32 skip = run & ~255u;
        rec[nrec++] = REC_ESC | (skip & 0x7FFFu) | ((skip >> 15) << 16);
        run &= 255u;
    }
    rec[nrec++] = (dist - 1) | ((len - 3) << 16) | (run << 24);
}

struct Match {
    u32 len;    // 0 for an escape
    u32 dist;   // meaningless for an escape
    u32 adv;    // output bytes from the end of the previous match to the end of this one
};
__device__ __forceinline__ Match get_match(u32 r) {
    const bool esc = (r & REC_ESC) != 0;
    Match m;
    m.len = esc ? 0 : ((r >> 16) & 0xFF) + 3;
    m.dist = (r & 0x7FFFu) + 1;
    m.adv = esc ? ((r & 0x7FFFu) | ((r >> 16) << 15)) : (r >> 24) + m.len;
    return m;
}

int launch(const BatchArgs &a, cudaStream_t stream);
void launch_slow(const BatchArgs &a, cudaStream_t stream);
int launch_warp(const BatchArgs &a, cudaStream_t stream);    // inflate_warp.cu (K1w)
int launch_lut(const BatchArgs &a, cudaStream_t stream);     // inflate_lut.cu  (K1L: table-lookup decode, thread per unit)

}  // namespace inflate
}  // namespace swc
