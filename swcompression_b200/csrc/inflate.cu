// inflate.cu — batched Deflate decode for sm_90a: the LZ77 stage and the launcher.  Replaces Deflate.decompress(_: LsbBitReader)
// (reference Sources/Deflate/Deflate.swift:30-249) + Code.huffmanCodes / DecodingTree (Sources/Common/CodingTree).
//
// Two kernels per batch (DESIGN.md §4.1):
//   K1 the Huffman stage — K1L inflate_lut_kernel (inflate_lut.cu, one thread per unit) for large batches, K1w
//        inflate_warp_kernel (inflate_warp.cu, one warp per unit) for small ones.  Literals go to a packed stream,
//        every match becomes a record (format in inflate.cuh).
//   K2 lz_resolve_kernel (here) — ONE WARP PER UNIT, the only writer of the output.  Builds the unit in order in a
//        shared-memory ring from the literal stream and the records, and writes it out in whole 16-byte chunks.
//
// Semantics are those of the reference, including its error cases and the inputs on which it traps
// (SWC_ERR_REFERENCE_TRAP).  Code sets whose Kraft sum exceeds 1 (which the reference accepts through heap-slot
// overwrites) are routed to the generic serial decoder in inflate_slow.cu via SWC_INTERNAL_NEEDS_SLOW.
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "inflate.cuh"
#include "host_util.h"

namespace swc {
namespace inflate {

// ------------------------------------------------------------------------------------------------ K2
// One warp per unit, the only writer of the unit's output, which it builds in order in a per-warp ring of RING bytes of
// shared memory (output byte p lives at ring[(p + phase) % RING], phase = the output's address mod 16, so that aligned
// 16-byte chunks of the output are aligned 16-byte chunks of the ring).  A batch is a run of consecutive records whose
// output ends at most SPAN bytes past the batch start; lane j holds record j.  Per batch:
//   scan     : inclusive warp scans of (literal run + length) and of the literal run give every record its position and
//              the offset of its literals in the batch's part of the literal stream;
//   literals : the batch's literals are copied from the packed stream into shared memory with 16-byte loads, then every
//              lane places literals: a binary search over the records' literal offsets (shuffles) finds each one's position;
//   matches  : replayed 8 at a time by 4-lane sub-groups.  A record is READY when everything it reads is final: its source
//              ends at or before the start of the oldest still-pending record of the 8 (bytes before that point are literals,
//              older matches or earlier batches) — or it IS that oldest record.  Far matches therefore run 8-wide in one
//              pass, chains of near matches (RLE-like data) degrade to in-order execution.  Overlapping copies (dist < len)
//              replicate the period: every source byte lies in [start-dist, start), never in what the match itself writes.
//              A source byte less than RING bytes behind the batch end is still in the ring; an older one has been written
//              to the output by this warp and is read back from there;
//   flush    : every whole 16-byte chunk of the output below the batch end goes out with one 16-byte store; the output's
//              first and last partial chunks are written byte by byte, so no byte outside [0, out_len) is touched.
// A batch stays within SPAN + 15 bytes of the first unflushed byte, so nothing is overwritten in the ring before it is
// flushed.  A literal run too long for one batch (an escape of more than SPAN bytes, or the literals after the last match)
// is placed in pieces of SPAN bytes.
namespace k2 {
constexpr int WARPS = 8;
constexpr int CTAS_PER_SM = 4;
constexpr u32 RING = 2048;
constexpr u32 SPAN = RING / 2;       // >= 255 + 258: one record of any kind but an escape fits a batch
constexpr u32 LITBUF = SPAN + 32;    // a batch's literals plus the 16-byte alignment slack at both ends
struct __align__(16) WarpSmem {
    uint4 stage[32];                 // {start, length, distance} of the batch's records
    u8 ring[RING];
    u8 lit[LITBUF];
};
}  // namespace k2

__global__ void __launch_bounds__(k2::WARPS * 32, k2::CTAS_PER_SM)
lz_resolve_kernel(BatchArgs a) {
    using namespace k2;
    __shared__ WarpSmem smem[WARPS];
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= a.n) return;
    if (a.status[unit] != SWC_OK) return;
    const u32 nrec = a.rec_count[unit];
    if (nrec == REC_DIRECT) return;
    WarpSmem &S = smem[(threadIdx.x >> 5) & (WARPS - 1)];
    const u32 lane = threadIdx.x & 31;
    const u32 sub = lane >> 2, t = lane & 3;
    const u64 off = a.out_off[unit];
    const u32 len = (u32)a.out_len[unit];
    u8 *out = a.out_base + off;
    const u32 *rec = a.rec_base + rec_start(off + a.out_cap[unit]);      // record k at rec - 1 - k
    const u8 *lits = (const u8 *)(a.rec_base + rec_start(off));
    const u32 ph = (u32)((uintptr_t)out & 15);
    const u32 M = RING - 1;
    u32 done = 0;          // output bytes placed by earlier batches
    u32 flushed = 0;       // output bytes written to global memory
    u32 lit = 0;           // literals consumed
    u32 g = 0;             // next record
    u32 part = 0;          // bytes of record g already placed (an escape longer than SPAN)
    // writes output bytes [flushed, to) from the ring: whole aligned chunks as 16-byte stores, the rest byte by byte
    auto flush = [&](u32 to) {
        const u32 c0 = (flushed + ph) >> 4, c1 = (to + ph + 15) >> 4;
        for (u32 c = c0 + lane; c < c1; c += 32) {
            const int cs = (int)(c * 16) - (int)ph;                     // chunk start as an output position
            const u32 lo = cs < (int)flushed ? flushed : (u32)cs, hi = (u32)(cs + 16) < to ? (u32)(cs + 16) : to;
            if ((int)lo == cs && hi == (u32)(cs + 16)) {
                *(uint4 *)(out + cs) = *(const uint4 *)(S.ring + ((c * 16) & M));
            } else {
                for (u32 p = lo; p < hi; p++) out[p] = S.ring[(p + ph) & M];
            }
        }
        flushed = to;
    };
    for (;;) {
        // ---- the batch: records g.. whose output ends within SPAN bytes of `done`
        const bool real = g + lane < nrec;
        u32 rv = REC_ESC;
        if (real) rv = *(rec - 1 - (g + lane));
        const Match m = get_match(rv);
        const u32 adv = m.adv - (lane == 0 ? part : 0u);
        const u32 run = adv - m.len;
        u32 end = adv, lend = run;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 v = __shfl_up_sync(SWC_FULL, end, d), w = __shfl_up_sync(SWC_FULL, lend, d);
            if (lane >= (u32)d) { end += v; lend += w; }
        }
        const u32 k = __popc(__ballot_sync(SWC_FULL, real && end <= SPAN));   // a prefix: `end` does not decrease
        u32 span, nl;
        u32 delta;         // output position of a literal minus its index in the batch's literals (the lane's record)
        if (k > 0) {
            span = __shfl_sync(SWC_FULL, end, k - 1);
            nl = __shfl_sync(SWC_FULL, lend, k - 1);
            delta = done + end - adv - (lend - run);
            if (lane >= k) lend = 0xFFFFFFFFu;
            g += k;
            part = 0;
        } else {
            // a literal run longer than SPAN: an escape (g < nrec) or the literals after the last match
            const u32 adv0 = __shfl_sync(SWC_FULL, adv, 0);      // what is left of escape g
            const u32 rem = g < nrec ? adv0 : len - done;
            if (rem == 0) break;
            span = nl = rem < SPAN ? rem : SPAN;
            if (g < nrec) part += span;
            delta = done;
            lend = lane == 0 ? nl : 0xFFFFFFFFu;
        }
        S.stage[lane] = make_uint4(done + end - m.len, lane < k ? m.len : 0u, m.dist, 0u);
        // ---- literals: packed stream -> shared memory (16-byte loads) -> their positions in the ring
        const uintptr_t lsrc = (uintptr_t)(lits + lit);
        const uint4 *lchunk = (const uint4 *)(lsrc & ~(uintptr_t)15);
        const u32 lofs = (u32)(lsrc & 15), nch = (lofs + nl + 15) >> 4;
        for (u32 c = lane; c < nch; c += 32) ((uint4 *)S.lit)[c] = __ldg(lchunk + c);
        __syncwarp();
        for (u32 j0 = 0; j0 < nl; j0 += 32) {
            const u32 j = j0 + lane;
            u32 r = 0;                                           // records whose literals all precede literal j
#pragma unroll
            for (u32 step = 16; step > 0; step >>= 1)
                if (__shfl_sync(SWC_FULL, lend, r + step - 1) <= j) r += step;
            const u32 p = j + __shfl_sync(SWC_FULL, delta, r);
            if (j < nl) S.ring[(p + ph) & M] = S.lit[lofs + j];
        }
        lit += nl;
        const u32 bend = done + span;                            // batch end
        __syncwarp();
        // ---- matches
        auto src_byte = [&](u32 q) -> u8 { return q + RING >= bend ? S.ring[(q + ph) & M] : out[q]; };
#pragma unroll 1
        for (u32 b0 = 0; b0 < k; b0 += 8) {
            const uint4 rc = S.stage[b0 + sub];                  // this sub-group's record
            const u32 s = rc.x, l = rc.y, d = rc.z;
            const u32 src_end = s - d + (l < d ? l : d);
            bool pend = l != 0;
            u32 pmask = __ballot_sync(SWC_FULL, pend && t == 0); // bit 4*sub per pending record
            while (pmask) {
                const u32 oldest = (__ffs(pmask) - 1) >> 2;       // sub-group index of the oldest pending record
                const u32 frontier = S.stage[b0 + oldest].x;
                const bool ready = pend && (sub == oldest || src_end <= frontier);
                if (ready) {
                    const u32 q0 = s - d;
                    if (d >= l) {
                        // four bytes per lane and trip, all four loads issued before the first store
                        for (u32 i = t; i < l; i += 16) {
                            const bool p1 = i + 4 < l, p2 = i + 8 < l, p3 = i + 12 < l;
                            const u8 v0 = src_byte(q0 + i);
                            u8 v1 = 0, v2 = 0, v3 = 0;
                            if (p1) v1 = src_byte(q0 + i + 4);
                            if (p2) v2 = src_byte(q0 + i + 8);
                            if (p3) v3 = src_byte(q0 + i + 12);
                            S.ring[(s + i + ph) & M] = v0;
                            if (p1) S.ring[(s + i + 4 + ph) & M] = v1;
                            if (p2) S.ring[(s + i + 8 + ph) & M] = v2;
                            if (p3) S.ring[(s + i + 12 + ph) & M] = v3;
                        }
                    } else {
                        for (u32 i = t; i < l; i += 4) S.ring[(s + i + ph) & M] = src_byte(q0 + i % d);
                    }
                    pend = false;
                }
                __syncwarp();
                pmask = __ballot_sync(SWC_FULL, pend && t == 0);
            }
        }
        done = bend;
        __syncwarp();
        // ---- flush the whole chunks below the batch end
        const u32 to = ((done + ph) & ~15u) - ph;
        if (done + ph >= 16 && to > flushed) flush(to);
        __syncwarp();
    }
    flush(len);
}

// ------------------------------------------------------------------------------------------------ host
int launch(const BatchArgs &a, cudaStream_t stream) {
    if (a.n == 0) return SWC_OK;
    // Huffman stage.
    //   large batches : K1L (inflate_lut.cu) — one lane per stream, table-lookup decode.
    //   small batches (and the single-stream API calls) cannot fill the chip with one lane per stream, so they take the
    //                   warp-per-unit decoder K1w (32 lanes on every stream, ~10 x lower latency per stream).
    //   SWC_DEFLATE_K1 = lut | warp forces K1L / K1w; any other value keeps the choice by batch size.
    static const int forced = [] {
        const char *e = getenv("SWC_DEFLATE_K1");
        return !e ? -1 : !strcmp(e, "lut") ? 0 : !strcmp(e, "warp") ? 1 : -1;
    }();
    const bool use_lut = forced >= 0 ? forced == 0 : a.n >= 20000;
    SWC_CUDA_TRY(cudaMemsetAsync(a.ticket, 0, 16, stream));
    timing_mark(stream);
    const int st = use_lut ? launch_lut(a, stream) : launch_warp(a, stream);
    if (st) return st;
    timing_mark(stream);
    launch_slow(a, stream);          // no-op unless a Huffman stage flagged a unit (over-subscribed code set)
    timing_mark(stream);
    const u64 per_cta = k2::WARPS;
    lz_resolve_kernel<<<(unsigned)((a.n + per_cta - 1) / per_cta), k2::WARPS * 32, 0, stream>>>(a);
    count_launch();
    timing_mark(stream);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace inflate
}  // namespace swc
