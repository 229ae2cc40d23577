// bzip2_stream_batch.cu — batched BZip2.decompress(data:) (reference Sources/BZip2/BZip2.swift:50-95) and
// BZip2.multiDecompress(data:) (:40-48) with the blocks of every stream decoded side by side.  With a caller scratch and
// max_blocks > 0 the call is a fixed sequence of launches: no host read, no allocation (DESIGN.md §4.17, §4.21).
//
//   scan<COUNT>   warp per unit     the BZh1-9 header, then block magics at every bit offset from bit 32 up to the first
//                                   end-of-stream magic (the matcher of checks::find_bzip2_magics); multi: up to the unit
//                                   end, every stream's blocks in one run of the table
//   place         one CTA           first_blk = exclusive sum of the candidate counts; a unit whose header fails, whose first
//                                   block is not at bit 32, that has no end magic, whose candidates do not fit the table, or
//                                   that the fallback could not hold behind every unit in front of it is marked for fallback
//   scan<FILL>    warp per unit     the block table: input byte, start bit and unit of every candidate
//   per slice:
//     order       one CTA           launch order, longest compressed span first; the block kernel's inputs in that order
//     blocks      warp per entry    bzip2_kernel in block mode, launch position k into slot k of SLOT bytes
//     scatter     thread per entry  the block kernel's results back into table order
//     layout      thread per unit   where each of the slice's blocks goes in its unit's region (running offset per unit)
//     copy        CTA per slot      slot -> region, 16-byte stores, clipped to out_cap
//   resolve       warp per unit     the reference's in-order walk as a validator: block k ends at candidate k + 1 (the last
//                                   at the end magic), the stored combined CRC is the fold of the block CRCs; else fallback
//     multi:      thread per unit   the walk across streams (header, blocks that are the next table entries, end magic and
//                                   combined CRC, align); the first stream not accepted or not fitting is the resume point
//   fallback      one CTA, then     per-unit scratch offsets of the fallback units (exclusive sum inside the dead block
//                 warp per unit     area), then bzip2_kernel in stream mode over exactly those units (multi: from the
//                                   resume point, stream after stream)
#include <vector>
#include "../../include/swcgpu.h"
#include "bzip2.cuh"
#include "checks_device.cuh"
#include "host_util.h"

namespace swc {
namespace {

// The output slot of one block: the host path's rule (api_bzip2.cu) at level 9.  A block that decodes to more (RLE1 lets
// a 900 kB block expand ~50x) reports overflow in its slot and its stream takes the fallback.
constexpr u64 SLOT = 9 * 200000 + 65536;
constexpr u64 SLOT_OUT = (SLOT + 64 + 255) & ~255ull;          // the copy's aligned loads read up to 32 bytes past a block
constexpr u64 NONE = ~0ull;
enum : u8 { F_OK = 1, F_PLACED = 2 };                          // header, first block at bit 32 and an end magic / in the table

__host__ __device__ __forceinline__ u64 slot_bytes() { return SLOT_OUT + bzip2::scratch_per_unit(SLOT); }

// the per-unit columns the stages hand to each other
// multi: after the resolve, count / end_bit / run_off hold the resume point (streams taken, its input byte, its output
// byte) and first_blk the stream kernel's consumed bits
struct UnitCols {
    u64 *count;        // block candidates in front of the first end magic (multi: in the whole unit)
    u64 *end_bit;      // bit of the first end magic in the unit (NONE: none; multi: the unit's end)
    u64 *first_blk;    // the unit's first entry in the block table
    u64 *run_off;      // bytes of the unit's output placed so far (carried across slices)
    u64 *fb_off;       // fallback: scratch offset inside the area
    u8 *flags;
    u8 *run;           // 1: the fallback decodes the unit
    u64 *totals;       // [0] candidates of the units that scanned clean, [1] the fallback scratch of every unit
};

// the block table, indexed by entry
struct BlockCols {
    u64 *in_off, *in_len;           // from the candidate's byte to the end of its unit
    u8 *start_bits;
    u32 *unit;
    u64 *out_len, *consumed, *dst;  // dst = where the block goes, relative to its unit's region
    int32_t *status;
    u64 *slot_off, *slot_cap, *slot_scr;   // per slot (the first `slots` entries)
    u32 *order;                     // per slice: launch position -> entry of the slice, longest first
    // per slice, in launch order: the block kernel's input and result columns
    u64 *l_in_off, *l_in_len, *l_out_len, *l_consumed;
    u8 *l_start_bits;
    int32_t *l_status;
};

struct ScanArgs {
    const u8 *in_base;
    const u64 *in_off, *in_len;
    u64 n;
    UnitCols u;
    BlockCols b;
};

// One warp per unit.  Each trip covers 512 bytes, 16 per lane in order, so lane order is position order; a lane's masks
// of those 16 bytes stay in registers for FILL's second look.  The trip that meets the first end magic is the last; with
// MULTI the scan runs to the unit end and takes every block magic (stream headers need no scan: the resolve reads them
// where its walk puts them).
template <bool FILL, bool MULTI>
__global__ void __launch_bounds__(256) bz2s_scan_kernel(ScanArgs a) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= a.n) return;
    const u32 lane = lane_id();
    if (FILL && !(a.u.flags[unit] & F_PLACED)) return;
    const u8 *p = a.in_base + a.in_off[unit];
    const u64 L = a.in_len[unit];
    const bool header = L >= 4 && p[0] == 'B' && p[1] == 'Z' && p[2] == 'h' && p[3] >= '1' && p[3] <= '9';   // BZip2.swift:53-64
    if (!header) {
        if (!FILL && lane == 0) { a.u.count[unit] = 0; a.u.end_bit[unit] = NONE; a.u.flags[unit] = 0; }
        return;
    }
    u64 total = 0, end = NONE, slot = FILL ? a.u.first_blk[unit] : 0;
    for (u64 base = 4; base + 6 <= L && (MULTI || end == NONE); base += 512) {
        const u64 b0 = base + 16 * lane;
        u32 bm[4] = {0, 0, 0, 0}, em[4] = {0, 0, 0, 0};
        // the lane's 16 bytes and the 6 behind them: the three aligned 16-byte lines that hold them (a line that starts
        // past the unit is not read), shifted into place.  Bytes past the unit are never matched (the matcher's limit).
        const u8 *at = p + b0;
        const uint4 *line = (const uint4 *)((uintptr_t)at & ~(uintptr_t)15);
        const u8 *stop = p + L;
        u32 v[12];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const uint4 x = (const u8 *)(line + k) < stop ? __ldg(line + k) : make_uint4(0, 0, 0, 0);
            v[4 * k] = x.x; v[4 * k + 1] = x.y; v[4 * k + 2] = x.z; v[4 * k + 3] = x.w;
        }
        const u32 r = (u32)((uintptr_t)at & 15), q = r >> 2, sh = (r & 3) * 8;
        u32 win[6];                                      // window byte j = byte j & 3 of win[j >> 2]
#pragma unroll
        for (int k = 0; k < 6; k++) {
            const u32 a0 = q == 0 ? v[k] : q == 1 ? v[k + 1] : q == 2 ? v[k + 2] : v[k + 3];
            const u32 a1 = q == 0 ? v[k + 1] : q == 1 ? v[k + 2] : q == 2 ? v[k + 3] : v[k + 4];
            win[k] = __funnelshift_r(a0, a1, sh);
        }
        auto byte = [&](int j) -> u64 { return (win[j >> 2] >> (8 * (j & 3))) & 0xFF; };
        u64 w = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) w = (w << 8) | byte(k);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const u64 i = b0 + j;
            w = (w << 8) | byte(j + 6);
            if (i + 6 <= L) {
                u32 mb, me;
                checks::bzip2_magics_in_byte(w, (int)min((L - i) * 8 - 47, (u64)8), &mb, &me);
                bm[j >> 2] |= mb << (8 * (j & 3));
                em[j >> 2] |= me << (8 * (j & 3));
            }
        }
        // this lane's candidates in front of its first end magic, and that magic
        u64 cnt = 0, lane_end = NONE;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const u32 mb = (bm[j >> 2] >> (8 * (j & 3))) & 0xFF, me = (em[j >> 2] >> (8 * (j & 3))) & 0xFF;
            if (MULTI) {
                cnt += __popc(mb);
            } else if (lane_end == NONE) {
                if (me) {
                    const u32 e = __ffs(me) - 1;
                    cnt += __popc(mb & ((1u << e) - 1));
                    lane_end = (b0 + j) * 8 + e;
                } else {
                    cnt += __popc(mb);
                }
            }
        }
        const u32 ends = MULTI ? 0 : __ballot_sync(SWC_FULL, lane_end != NONE);
        const u32 fe = ends ? __ffs(ends) - 1 : 32;
        if (lane > fe) cnt = 0;
        u64 incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u64 v = __shfl_up_sync(SWC_FULL, incl, d);
            if (lane >= (u32)d) incl += v;
        }
        if (FILL && cnt) {
            u64 e = slot + incl - cnt, left = cnt;
            for (int j = 0; j < 16 && left; j++) {
                for (u32 m = (bm[j >> 2] >> (8 * (j & 3))) & 0xFF; m && left; m &= m - 1, left--, e++) {
                    const u64 bit = (b0 + j) * 8 + __ffs(m) - 1;
                    a.b.in_off[e] = a.in_off[unit] + (bit >> 3);
                    a.b.in_len[e] = L - (bit >> 3);
                    a.b.start_bits[e] = (u8)(bit & 7);
                    a.b.unit[e] = (u32)unit;
                }
            }
        }
        const u64 trip = __shfl_sync(SWC_FULL, incl, 31);
        total += trip; slot += trip;
        if (ends) end = __shfl_sync(SWC_FULL, lane_end, fe);
    }
    if (!FILL && lane == 0) {
        // the first block must sit right behind the header (bit 32 is byte aligned)
        const bool first_at_32 = L >= 10 && p[4] == 0x31 && p[5] == 0x41 && p[6] == 0x59 && p[7] == 0x26 && p[8] == 0x53 && p[9] == 0x59;
        // multi: an empty first stream has its end magic there
        const bool end_at_32 = L >= 10 && p[4] == 0x17 && p[5] == 0x72 && p[6] == 0x45 && p[7] == 0x38 && p[8] == 0x50 && p[9] == 0x90;
        a.u.count[unit] = total;
        a.u.end_bit[unit] = MULTI ? L * 8 : end;
        a.u.flags[unit] = MULTI ? (first_at_32 || end_at_32 ? F_OK : 0) : first_at_32 && end != NONE ? F_OK : 0;
    }
}

// exclusive sums, one CTA, over the units in order: the candidate counts of the units that scanned clean, and every unit's
// fallback scratch.  A unit is placed iff its candidates fit the table and the fallback could still hold it and every unit
// in front of it: its blocks are copied into its region before the resolve knows whether they validate, so a placed unit
// that fails must never find the fallback full.  Starts every unit's running offset at 0.
// totals[0] = the candidates of the units that scanned clean, totals[1] = the fallback scratch of every unit.
__global__ void __launch_bounds__(1024) bz2s_place_kernel(UnitCols c, const u64 *out_cap, u64 n, u64 max_blocks, u64 area) {
    __shared__ u64 part[2][1024];
    u64 b, e;
    cta_unit_run(n, b, e);
    u64 s = 0, sf = 0;
    for (u64 i = b; i < e; i++) {
        s += (c.flags[i] & F_OK) ? c.count[i] : 0;
        sf += bzip2::scratch_per_unit(out_cap[i]);
    }
    part[0][threadIdx.x] = s; part[1][threadIdx.x] = sf;
    cta_scan<2>(part);
    if (threadIdx.x == 1023) { c.totals[0] = part[0][1023]; c.totals[1] = part[1][1023]; }
    u64 at = part[0][threadIdx.x] - s, fat = part[1][threadIdx.x] - sf;
    for (u64 i = b; i < e; i++) {
        const bool ok = (c.flags[i] & F_OK) != 0;
        const u64 nb = ok ? c.count[i] : 0, need = bzip2::scratch_per_unit(out_cap[i]);
        const bool fits = ok && at + nb <= max_blocks && fat + need <= area;
        c.flags[i] = (ok ? F_OK : 0) | (fits ? F_PLACED : 0);
        c.first_blk[i] = at;
        c.run[i] = 1;                   // until the resolve accepts the unit's blocks
        c.run_off[i] = 0;
        at += nb; fat += need;
    }
}

__global__ void __launch_bounds__(256) bz2s_slot_init_kernel(BlockCols b, u64 slots) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= slots) return;
    b.slot_off[k] = k * slot_bytes();
    b.slot_cap[k] = SLOT;
    b.slot_scr[k] = k * slot_bytes() + SLOT_OUT;
}

// thread per unit: the offsets of the unit's blocks in entries [e0, e1) inside its region, in block order
__global__ void __launch_bounds__(256) bz2s_layout_kernel(UnitCols c, BlockCols b, u64 n, u64 e0, u64 e1) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= n || !(c.flags[unit] & F_PLACED)) return;
    const u64 f = c.first_blk[unit], l = f + c.count[unit];
    const u64 kb = f > e0 ? f : e0, ke = l < e1 ? l : e1;
    if (kb >= ke) return;
    u64 at = c.run_off[unit];
    for (u64 k = kb; k < ke; k++) { b.dst[k] = at; at += b.out_len[k]; }
    c.run_off[unit] = at;
}

// One CTA per slice: the slice's entries in launch order, the longest compressed span first (a counting sort on its leading
// zeros), and the block kernel's input columns gathered in that order.  A CTA of bzip2_kernel holds its SM resources until
// its slowest warp is done, so the long blocks go first, 4 to a CTA, and the short ones (a stream's last block, idle
// entries) fill in behind them.
__global__ void __launch_bounds__(1024) bz2s_order_kernel(const u64 *unit_len, UnitCols c, BlockCols b, u64 e0, u64 cnt) {
    auto key = [&](u64 j) -> u32 {
        const u64 e = e0 + j, len = b.in_len[e];
        if (!len) return 64;                                        // idle entry
        const u32 u = b.unit[e];
        const bool last = e + 1 == c.first_blk[u] + c.count[u];
        const u64 span = len - (last ? unit_len[u] - (c.end_bit[u] >> 3) : b.in_len[e + 1]);
        return __clzll((long long)span);
    };
    clz_order(cnt, key, [&](u64 j, u32 at) {
        const u64 e = e0 + j;
        b.order[e0 + at] = (u32)j;
        b.l_in_off[at] = b.in_off[e]; b.l_in_len[at] = b.in_len[e]; b.l_start_bits[at] = b.start_bits[e];
    });
}

// thread per launch position: the block kernel's results back into table order
__global__ void __launch_bounds__(256) bz2s_scatter_kernel(BlockCols b, u64 e0, u64 cnt) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= cnt) return;
    const u64 e = e0 + b.order[e0 + k];
    b.out_len[e] = b.l_out_len[k]; b.consumed[e] = b.l_consumed[k]; b.status[e] = b.l_status[k];
}

// bytes r .. r+15 of the 32 bytes lo | hi (little-endian), r in 0..15 and uniform across the CTA
__device__ __forceinline__ uint4 bytes_at(uint4 lo, uint4 hi, u32 r) {
    const u32 w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    const u32 q = r >> 2, sh = (r & 3) * 8;
    u32 o[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const u32 a0 = q == 0 ? w[k] : q == 1 ? w[k + 1] : q == 2 ? w[k + 2] : w[k + 3];
        const u32 a1 = q == 0 ? w[k + 1] : q == 1 ? w[k + 2] : q == 2 ? w[k + 3] : w[k + 4];
        o[k] = __funnelshift_r(a0, a1, sh);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
}

// CTA per launch position (= slot) of the slice: a block that decoded cleanly goes from its slot into its unit's region,
// never past out_cap.  The stores are 16-byte aligned; the slot (16-byte aligned) is read in aligned pairs and shifted into
// place.
__global__ void __launch_bounds__(256) bz2s_copy_kernel(UnitIO io, UnitCols c, BlockCols b, const u8 *slots, u64 e0) {
    const u64 k = blockIdx.x, e = e0 + b.order[e0 + k];
    if (b.status[e] != SWC_OK) return;
    const u32 unit = b.unit[e];
    const u64 cap = io.out_cap[unit], at = b.dst[e];
    if (at >= cap) return;
    const u64 len = b.out_len[e] < cap - at ? b.out_len[e] : cap - at;
    const u8 *s = slots + k * slot_bytes();
    u8 *d = io.out_base + io.out_off[unit] + at;
    const u32 r = (u32)((16 - ((uintptr_t)d & 15)) & 15);
    const u64 head = r < len ? r : len;
    if (threadIdx.x < head) d[threadIdx.x] = s[threadIdx.x];
    const u64 body = (len - head) & ~15ull;
    for (u64 o = threadIdx.x * 16; o < body; o += blockDim.x * 16) {
        const uint4 lo = __ldg((const uint4 *)(s + o)), hi = __ldg((const uint4 *)(s + o + 16));
        *(uint4 *)(d + head + o) = bytes_at(lo, hi, r);
    }
    const u64 t = head + body + threadIdx.x;
    if (threadIdx.x < 16 && t < len) d[t] = s[t];
}

// 32 bits from bit `bit` of the unit, MSB first (BZip2's reader order); bytes past the unit read as 0
__device__ __forceinline__ u32 bits32_at(const u8 *p, u64 L, u64 bit) {
    u64 w = 0;
    const u64 b0 = bit >> 3;
#pragma unroll
    for (int k = 0; k < 5; k++) w = (w << 8) | (b0 + k < L ? p[b0 + k] : 0);
    return (u32)(w >> (8 - (bit & 7)));
}

// One warp per placed unit, 32 blocks per trip: the reference's walk (BZip2.swift:66-95) accepts the blocks iff each decoded
// cleanly (its CRC included) and ended exactly where the next candidate starts, the last one at the end magic, and the end
// magic's CRC is the fold of the block CRCs.  Accepted units get their final results; every other unit is left to the
// fallback.
__global__ void __launch_bounds__(256) bz2s_resolve_kernel(DecodeIO io, UnitCols c, BlockCols b) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= io.n || !(c.flags[unit] & F_PLACED)) return;
    const u32 lane = lane_id();
    const u8 *p = io.in_base + io.in_off[unit];
    const u64 L = io.in_len[unit], f = c.first_blk[unit], nb = c.count[unit], end = c.end_bit[unit];
    auto pos = [&](u64 k) { return (b.in_off[f + k] - io.in_off[unit]) * 8 + b.start_bits[f + k]; };
    u32 crc = 0;
    u64 total = 0;
    bool ok = end + 80 <= L * 8;
    for (u64 g = 0; g < nb && ok; g += 32) {
        const u64 k = g + lane;
        bool fail = false;
        u64 size = 0;
        if (k < nb) {
            const u64 at = pos(k), next = k + 1 < nb ? pos(k + 1) : end;
            fail = b.status[f + k] != SWC_OK || (at & ~7ull) + b.consumed[f + k] != next;
            crc ^= __funnelshift_l(bits32_at(p, L, at + 48), bits32_at(p, L, at + 48), (u32)((nb - 1 - k) & 31));   // :83-84 unrolled
            size = b.out_len[f + k];
        }
        if (__any_sync(SWC_FULL, fail)) ok = false;
#pragma unroll
        for (int d = 16; d; d >>= 1) size += __shfl_xor_sync(SWC_FULL, size, d);
        total += size;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) crc ^= __shfl_xor_sync(SWC_FULL, crc, d);
    if (lane) return;
    if (!ok || bits32_at(p, L, end + 48) != crc) return;       // the stream kernel gives the reference's answer
    const bool over = total > io.out_cap[unit];
    io.status[unit] = over ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
    io.out_len[unit] = total;
    io.consumed[unit] = over ? 0 : end + 80;
    c.run[unit] = 0;
}

// Thread per unit: the reference's multiDecompress walk (BZip2.swift:40-95) over the unit's table entries in position order
// as a validator.  A stream at byte P needs 32 bits and the header BZh1-9; from bit (P + 4) * 8 each block must be the next
// table entry, start exactly where the walk stands, have decoded cleanly (its CRC included) and end where its consumed bits
// say; at the end magic the stored CRC must be the fold of this stream's block CRCs, and the next stream starts at
// ceil((e + 80) / 8).  A table entry the walk would step over (a look-alike in a payload, or in the CRC and padding in front
// of the next header, whose bytes the layout has counted) ends acceptance at the current stream.  Reaching the unit end
// with every stream accepted gives the final result (overflow included: its exact size); otherwise the first stream not
// accepted, or the first that does not fit out_cap, is where the stream kernel resumes: its input byte goes to end_bit,
// the output bytes in front of it to run_off and the streams taken to count.  The accepted streams' table entries are
// written here.
__global__ void __launch_bounds__(256) bz2m_resolve_kernel(UnitIO io, UnitCols c, BlockCols b, bzip2::Multi m, u32 *parallel) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= io.n) return;
    u64 at = 0, out = 0, taken = 0;                 // the resume point
    u64 P = 0, sum = 0, s = 0;                      // the walk: next stream's byte, bytes and streams accepted
    bool all = false;
    const u64 L = io.in_len[unit], cap = io.out_cap[unit];
    if (c.flags[unit] & F_PLACED) {
        const u8 *p = io.in_base + io.in_off[unit];
        const u64 f = c.first_blk[unit], nb = c.count[unit];
        auto pos = [&](u64 k) { return (b.in_off[f + k] - io.in_off[unit]) * 8 + b.start_bits[f + k]; };
        u64 k = 0;
        for (;;) {
            if (P == L) { all = true; break; }
            if (L - P < 4 || p[P] != 'B' || p[P + 1] != 'Z' || p[P + 2] != 'h' || p[P + 3] < '1' || p[P + 3] > '9') break;
            u64 bit = (P + 4) * 8, bytes = sum;
            u32 crc = 0;
            bool ok = true;
            for (;;) {
                if (bit + 80 > L * 8 || (k < nb && pos(k) < bit)) { ok = false; break; }
                if (k < nb && pos(k) == bit) {
                    if (b.status[f + k] != SWC_OK) { ok = false; break; }
                    crc = ((crc << 1) | (crc >> 31)) ^ bits32_at(p, L, bit + 48);         // :83-84
                    bytes += b.out_len[f + k];
                    bit = (bit & ~7ull) + b.consumed[f + k];
                    k++;
                    continue;
                }
                const u64 magic = ((u64)bits32_at(p, L, bit) << 16) | (bits32_at(p, L, bit + 32) >> 16);
                ok = magic == 0x177245385090ull && bits32_at(p, L, bit + 48) == crc;      // :86
                break;
            }
            if (!ok) break;
            if (m.stream_end && s < m.stream_cap[unit]) {
                m.stream_end[m.stream_off[unit] + s] = bytes;
                m.stream_in_off[m.stream_off[unit] + s] = P;
            }
            P = (bit + 80 + 7) / 8;
            sum = bytes;
            s++;
            if (sum <= cap) { at = P; out = sum; taken = s; }
        }
    }
    if (parallel) parallel[unit] = (u32)taken;
    if (all) {
        const bool over = sum > cap;
        io.status[unit] = over ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
        io.out_len[unit] = sum;
        if (m.n_streams) m.n_streams[unit] = over ? 0 : s;
        c.run[unit] = 0;
        return;
    }
    if (m.n_streams) m.n_streams[unit] = 0;        // until the stream kernel finishes the unit
    c.end_bit[unit] = at; c.run_off[unit] = out; c.count[unit] = taken;
}

// exclusive sum of scratch_per_unit(out_cap) over the fallback units inside the area, one CTA; a unit past the area reports
// SWC_ERR_UNSUPPORTED and is not run
__global__ void __launch_bounds__(1024) bz2s_fallback_place_kernel(DecodeIO io, UnitCols c, u64 area) {
    __shared__ u64 part[1][1024];
    u64 b, e;
    cta_unit_run(io.n, b, e);
    u64 s = 0;
    for (u64 i = b; i < e; i++) s += c.run[i] ? bzip2::scratch_per_unit(io.out_cap[i]) : 0;
    part[0][threadIdx.x] = s;
    cta_scan<1>(part);
    u64 at = part[0][threadIdx.x] - s;
    for (u64 i = b; i < e; i++) {
        if (!c.run[i]) continue;
        const u64 need = bzip2::scratch_per_unit(io.out_cap[i]);
        c.fb_off[i] = at;
        if (at + need > area) {
            c.run[i] = 0;
            io.status[i] = SWC_ERR_UNSUPPORTED; io.out_len[i] = 0; io.consumed[i] = 0;
        }
        at += need;
    }
}

// ---- scratch layout: the unit columns, the block columns, then the area (slots, later the fallback's scratch) ----------
struct Layout {
    UnitCols u;
    BlockCols b;
    size_t unit_bytes, fixed_bytes;
    u8 *block_part, *area;

    Layout(void *base, u64 n, u64 nblk) {
        Carver c(base);
        c.cols(n, u.count, u.end_bit, u.first_blk, u.run_off, u.fb_off, u.flags, u.run);
        c.cols(2, u.totals);
        unit_bytes = c.at;
        block_part = c.end();
        c.cols(nblk, b.in_off, b.in_len, b.start_bits, b.unit, b.out_len, b.consumed, b.dst, b.status, b.slot_off, b.slot_cap,
               b.slot_scr, b.order, b.l_in_off, b.l_in_len, b.l_out_len, b.l_consumed, b.l_start_bits, b.l_status);
        fixed_bytes = c.at;
        area = c.end();
    }
};

size_t fixed_bytes_for(u64 n, u64 nblk) { return Layout(nullptr, n, nblk).fixed_bytes; }
// an upper bound of the fallback's scratch when every unit falls back: scratch_per_unit(c) <= 6 (c + c / 4 + 11) + 33 600
u64 fallback_bound(u64 n, u64 out_total) { return 6 * (out_total + out_total / 4 + 11 * n) + 33600 * n; }

// multi: the stream table and parallel_streams of swc_bzip2_multi_decompress_batch (the resume columns are filled in by
// decode())
struct Mode {
    bool multi = false;
    bzip2::Multi table = {};
    u32 *parallel = nullptr;
};

struct Call {
    DecodeIO io;                // multi: consumed is null (the stream kernel's goes to a dead unit column)
    cudaStream_t s;
    Mode mode;
};

// the scan, unless the unit columns of `l` already hold it (`counted`), and the placement in a table of max_blocks entries
// beside an area of `area` bytes
int count_and_place(const Call &q, const Layout &l, u64 max_blocks, u64 area, bool counted) {
    const unsigned warps = (unsigned)((q.io.n * 32 + 255) / 256);
    const ScanArgs sa{q.io.in_base, q.io.in_off, q.io.in_len, q.io.n, l.u, l.b};
    if (!counted && q.mode.multi) bz2s_scan_kernel<false, true><<<warps, 256, 0, q.s>>>(sa);
    if (!counted && !q.mode.multi) bz2s_scan_kernel<false, false><<<warps, 256, 0, q.s>>>(sa);
    bz2s_place_kernel<<<1, 1024, 0, q.s>>>(l.u, q.io.out_cap, q.io.n, max_blocks, area);
    count_launch(counted ? 1 : 2);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// `counted`: the unit columns of `l` already hold this batch's scan; `slots` block slots and an area of `area` bytes follow
// the columns
int decode(const Call &q, const Layout &l, u64 nblk, u64 slots, u64 area, bool counted) {
    const u64 n = q.io.n;
    const unsigned unit_warps = (unsigned)((n * 32 + 255) / 256), unit_threads = (unsigned)((n + 255) / 256);
    int st;
    timing_mark(q.s);
    if ((st = count_and_place(q, l, nblk, area, counted))) return st;
    // idle table entries have no input and fail at once
    SWC_CUDA_TRY(cudaMemsetAsync(l.block_part, 0, l.fixed_bytes - l.unit_bytes, q.s));
    bz2s_slot_init_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, q.s>>>(l.b, slots);
    const ScanArgs sa{q.io.in_base, q.io.in_off, q.io.in_len, n, l.u, l.b};
    if (q.mode.multi) bz2s_scan_kernel<true, true><<<unit_warps, 256, 0, q.s>>>(sa);
    else bz2s_scan_kernel<true, false><<<unit_warps, 256, 0, q.s>>>(sa);
    count_launch(2);
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(q.s);
    for (u64 e0 = 0; e0 < nblk; e0 += slots) {
        const u64 cnt = nblk - e0 < slots ? nblk - e0 : slots;
        bz2s_order_kernel<<<1, 1024, 0, q.s>>>(q.io.in_len, l.u, l.b, e0, cnt);
        count_launch();
        bzip2::Args blocks{{{q.io.in_base, l.b.l_in_off, l.b.l_in_len, l.area, l.b.slot_off, l.b.slot_cap, l.b.l_out_len, l.b.l_status,
                             cnt}, l.b.l_consumed},
                           l.area, l.b.slot_scr, l.b.l_start_bits, 1};
        if ((st = bzip2::launch(blocks, q.s))) return st;
        bz2s_scatter_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, q.s>>>(l.b, e0, cnt);
        bz2s_layout_kernel<<<unit_threads, 256, 0, q.s>>>(l.u, l.b, n, e0, e0 + cnt);
        bz2s_copy_kernel<<<(unsigned)cnt, 256, 0, q.s>>>(q.io, l.u, l.b, l.area, e0);
        count_launch(3);
        SWC_CUDA_TRY(cudaGetLastError());
    }
    timing_mark(q.s);
    DecodeIO io = q.io;
    if (q.mode.multi) {
        bz2m_resolve_kernel<<<unit_threads, 256, 0, q.s>>>(io, l.u, l.b, q.mode.table, q.mode.parallel);
        io.consumed = l.u.first_blk;
    } else {
        bz2s_resolve_kernel<<<unit_warps, 256, 0, q.s>>>(io, l.u, l.b);
    }
    count_launch();
    timing_mark(q.s);
    // the block stage is over: its whole area is the fallback's scratch
    bz2s_fallback_place_kernel<<<1, 1024, 0, q.s>>>(io, l.u, area);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    bzip2::Args fb{io, l.area, l.u.fb_off};
    fb.run = l.u.run;
    if (q.mode.multi) {
        fb.multi = q.mode.table;
        fb.multi.at_in = l.u.end_bit; fb.multi.at_out = l.u.run_off; fb.multi.taken = l.u.count;
    }
    if ((st = bzip2::launch(fb, q.s))) return st;
    timing_mark(q.s);
    return SWC_OK;
}

// both entry points after their argument checks: size and seat the scratch, then decode
int run_batch(const Call &q, u64 max_blocks, void *scratch, size_t scratch_bytes) {
    const u64 n = q.io.n;
    int st;
    u64 nblk = max_blocks;
    u64 fb_need = 0;
    SplitScratch sc(scratch, q.s);
    if (max_blocks == 0) {
        // the library counts first: the scan on the unit columns alone, then the totals back
        auto launch = [&](void *base, const u64 **t) {
            const Layout l(base, n, 0);
            *t = l.u.totals;
            return count_and_place(q, l, ~0ull, ~0ull, false);
        };
        u64 totals[2];
        if ((st = sc.count_first(scratch_bytes, Layout(nullptr, n, 0).unit_bytes, 2, totals, launch))) return st;
        if (totals[0] > 0xFFFFFFFFull) return SWC_ERR_UNSUPPORTED;
        nblk = totals[0] ? totals[0] : 1;
        fb_need = totals[1];
        if (scratch) {
            // the largest table that leaves the area one slot and the fallback of every unit: the units past it fall back,
            // so a scratch of swc_bzip2_stream_batch_scratch_bytes(n, 0, ...) gives every unit its exact status
            const u64 want = fb_need > slot_bytes() ? fb_need : slot_bytes();
            nblk = largest_table(nblk, scratch_bytes, [&](u64 m) { return fixed_bytes_for(n, m) + want; });
        }
    }
    const size_t fixed = fixed_bytes_for(n, nblk);
    u64 area = 0;
    if (scratch) {
        if (scratch_bytes < fixed + slot_bytes()) return SWC_ERR_INVALID_ARG;
        area = scratch_bytes - fixed;
    } else {
        // the pool: every unit's fallback scratch (counted above, or out_cap read back: one synchronisation) and as many
        // slots as the table needs, within half the free memory
        u64 fb = fb_need;
        if (max_blocks) {
            std::vector<u64> caps;
            if ((st = read_lens(q.io.out_cap, n, q.s, caps))) return st;
            for (u64 c : caps) fb += bzip2::scratch_per_unit(c);
        }
        size_t free_b = 0, total_b = 0;
        SWC_CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        u64 slots = free_b / 2 / slot_bytes();
        slots = slots < 1 ? 1 : slots > nblk ? nblk : slots;
        area = slots * slot_bytes() > fb ? slots * slot_bytes() : fb;
        if ((st = sc.seat(fixed + area))) return st;
    }
    const u64 slots_fit = area / slot_bytes();
    const u64 slots = slots_fit < nblk ? slots_fit : nblk;
    return decode(q, Layout(sc.p, n, nblk), nblk, slots, area, sc.counted);
}

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

size_t swc_bzip2_stream_batch_scratch_bytes(uint64_t n, uint64_t max_blocks, uint64_t out_capacity_total) {
    const u64 nblk = max_blocks ? max_blocks : 1;
    const u64 blocks = nblk * slot_bytes(), fb = fallback_bound(n, out_capacity_total);
    return fixed_bytes_for(n, nblk) + (blocks > fb ? blocks : fb);
}

int32_t swc_bzip2_stream_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                          uint64_t *out_len, uint64_t *consumed_bits, int32_t *status,
                                          uint64_t n, uint64_t max_blocks,
                                          void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    const Call q{{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bits}, (cudaStream_t)cuda_stream, {}};
    if (missing(q.io) || max_blocks > 0xFFFFFFFFull || n > 0xFFFFFFFFull) return SWC_ERR_INVALID_ARG;
    return run_batch(q, max_blocks, scratch, scratch_bytes);
}

int32_t swc_bzip2_multi_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                         uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                         uint64_t *out_len, int32_t *status,
                                         uint64_t *n_streams, const uint64_t *stream_off, const uint64_t *stream_cap,
                                         uint64_t *stream_end, uint64_t *stream_in_off, uint32_t *parallel_streams,
                                         uint64_t n, uint64_t max_blocks,
                                         void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    Call q{{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, nullptr}, (cudaStream_t)cuda_stream, {}};
    const int tables = !!stream_off + !!stream_cap + !!stream_end + !!stream_in_off;
    if (missing((const UnitIO &)q.io) || (tables != 0 && tables != 4) || max_blocks > 0xFFFFFFFFull || n > 0xFFFFFFFFull)
        return SWC_ERR_INVALID_ARG;
    q.mode.multi = true;
    q.mode.table.n_streams = n_streams;
    q.mode.table.stream_off = stream_off; q.mode.table.stream_cap = stream_cap;
    q.mode.table.stream_end = stream_end; q.mode.table.stream_in_off = stream_in_off;
    q.mode.parallel = parallel_streams;
    return run_batch(q, max_blocks, scratch, scratch_bytes);
}

}  // extern "C"
