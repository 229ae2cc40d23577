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
    u32 *rec_base;             // literal + match-record scratch (format below)
    u32 *rec_count;            // n entries
    unsigned long long *ticket; // unit ticket counters of the persistent-lane kernels: [0] K1w, [1] K1L (zeroed by the launcher)
};

// ---- the hand-off from the Huffman stage to K2 ----
// The Huffman stage writes nothing to the output.  It hands K2 two streams per unit:
//   literals : every literal (and every stored-block byte), packed in stream order;
//   records  : every match, in stream order, as one 4-byte record
//     {dist - 1 : 15 | esc = 0 : 1 | len - 3 : 8 | run : 8}      run = literal bytes since the end of the previous match
// A run longer than 255 is first cut down by an escape record {skip & 0x7FFF : 15 | esc = 1 : 1 | skip >> 15 : 16} that
// only advances the output position by skip = run & ~255.  K2 places each match with a warp scan of run + len (escape:
// skip), takes the literals in front of it from the literal stream and is the only writer of the output.  Literals at
// output positions >= cap are not stored and matches that end past cap get no record: such a unit fails with an overflow
// status and K2 skips it.  rec_count[unit] holds the number of records written, or REC_DIRECT for a unit that
// inflate_slow_kernel wrote straight to its output.
//
// A unit whose output region starts at byte `out_off` owns the scratch words [out_off/3, (out_off+cap)/3), so disjoint
// output regions give disjoint scratch regions without a prefix sum over the units.  The literals grow upward from the
// region's first byte (4-byte aligned), the records downward from its end: record k sits at word end - 1 - k.
// Why both fit: take L stored literals, R_m match records and R_e escapes.  They cover disjoint output bytes below cap
// and a match covers >= 3, so L + 3 R_m <= cap; an escape covers >= 256 literals, so R_e <= L / 256.  The region has
// 4 floor((out_off+cap)/3) - 4 floor(out_off/3) >= 4 floor(cap/3) bytes.  With cap = 3q + r:
//     L + 4 R_m + 4 R_e <= L + 4 floor((cap - L)/3) + L/64 <= L + 4q + 4 floor((r - L)/3) + L/64 <= 4q + (8 - L)/3 + L/64
// which is <= 4q when L >= 8.  The Huffman stage stores literals in whole 8-byte words as they fill up, so every stored
// word lies below the records; only the last, partial word of a unit with fewer than 8 literals (and records for almost
// all of its bytes) may find no room: such a unit goes to inflate_slow_kernel (SWC_INTERNAL_NEEDS_SLOW).
__host__ __device__ __forceinline__ u64 rec_start(u64 out_off) { return out_off / 3; }
inline size_t scratch_bytes(u64 n, u64 out_capacity_total) {
    return (size_t)((out_capacity_total / 3 + 2) * 4 + n * 4 + 1024);
}
// bytes of the scratch region of a unit
__device__ __forceinline__ u64 region_bytes(u64 out_off, u64 cap) { return (rec_start(out_off + cap) - rec_start(out_off)) * 4; }

constexpr u32 REC_ESC = 0x8000u;       // also the padding record: an escape that skips nothing
constexpr u32 REC_DIRECT = 0xFFFFFFFFu;  // rec_count of a unit whose output is already written

// appends the records of a match of `len` bytes at distance `dist` that follows `run` literal bytes; `rec_end` is the end
// of the unit's scratch region, record k goes to rec_end - 1 - k
__device__ __forceinline__ void put_match(u32 *rec_end, u32 &nrec, u32 run, u32 len, u32 dist) {
    if (run > 255) {
        const u32 skip = run & ~255u;
        *(rec_end - 1 - nrec) = REC_ESC | (skip & 0x7FFFu) | ((skip >> 15) << 16);
        nrec++;
        run &= 255u;
    }
    *(rec_end - 1 - nrec) = (dist - 1) | ((len - 3) << 16) | (run << 24);
    nrec++;
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
