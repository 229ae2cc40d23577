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
// output ends at most SPAN bytes past the batch start; lane j holds record j, loaded one batch ahead.  Per batch:
//   scan     : inclusive warp scans of (literal run + length) and of the literal run give every record its position and
//              the offset of its literals in the batch's part of the literal stream;
//   gather   : one round of 16-byte cp.async copies brings in the batch's literals from the packed stream and the sources
//              of its FAR matches from the output.  A match is far when its first source byte is more than RING bytes behind
//              the batch end (bend): with len <= 258 and bend - RING <= done - SPAN, its whole source then lies in output this
//              warp has already flushed, and dist > RING - SPAN >= len.  Every other match reads only bytes that are still
//              in the ring.  A far source takes at most len/16 + 2 aligned chunks, so a batch (<= 32 records, their lengths
//              summing to <= SPAN) needs at most 128 of them, which a warp-wide scan packs into a 2 KiB staging buffer;
//              the part of the output's first chunk that lies before out[0] is never read (that chunk is copied byte by
//              byte);
//   literals : every lane places literals: a binary search over the records' literal offsets (shuffles) finds each
//              one's position;
//   matches  : replayed 8 at a time by 4-lane sub-groups, reading shared memory only (far ones from the staging buffer,
//              the others from the ring).  A record is READY when everything it reads is final: its source ends at or
//              before the start of the oldest still-pending record of the 8 (bytes before that point are literals, older
//              matches or earlier batches) — or it IS that oldest record.  Far matches therefore run 8-wide in one pass,
//              chains of near matches (RLE-like data) degrade to in-order execution.  Overlapping copies (dist < len)
//              replicate the period: every source byte lies in [start-dist, start), never in what the match itself writes;
//   flush    : every whole 16-byte chunk of the output below the batch end goes out with one 16-byte store; the output's
//              first and last partial chunks are written byte by byte, so no byte outside [0, out_len) is touched.
// A batch stays within SPAN + 15 bytes of the first unflushed byte, so nothing is overwritten in the ring before it is
// flushed.  A literal run too long for one batch (an escape of more than SPAN bytes, or the literals after the last match)
// is placed in pieces of SPAN bytes.  So a batch waits on global memory once: its records were loaded during the batch
// before, its literals and far sources arrive together.
namespace k2 {
constexpr int WARPS = 8;
constexpr int CTAS_PER_SM = 4;
constexpr u32 RING = 2048;
constexpr u32 SPAN = RING / 2;       // >= 255 + 258: one record of any kind but an escape fits a batch
constexpr u32 LITBUF = SPAN + 32;    // a batch's literals plus the 16-byte alignment slack at both ends
constexpr u32 FARBUF = 128 * 16;     // the far sources of a batch: at most 32 * 2 + SPAN / 16 chunks
constexpr u32 NEAR = 0xFFFFFFFFu;    // staging offset of a match that reads the ring
struct __align__(16) WarpSmem {
    uint4 stage[32];                 // {start, length, distance, staging offset of the first source byte | NEAR}
    u8 ring[RING];
    u8 lit[LITBUF];
    u8 far[FARBUF];
};
__device__ __forceinline__ void cp_async16(void *dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((u32)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }
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
    u32 rv = lane < nrec ? __ldg(rec - 1 - lane) : REC_ESC;              // record g + lane
    for (;;) {
        // ---- the batch: records g.. whose output ends within SPAN bytes of `done`
        const bool real = g + lane < nrec;
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
        if (k > 0) rv = g + lane < nrec ? __ldg(rec - 1 - (g + lane)) : REC_ESC;   // the next batch's records
        const u32 bend = done + span;                            // batch end
        // ---- gather: the literals (packed stream) and the far match sources (flushed output) -> shared memory
        const uintptr_t lsrc = (uintptr_t)(lits + lit);
        const u8 *lchunk = (const u8 *)(lsrc & ~(uintptr_t)15);
        const u32 lofs = (u32)(lsrc & 15), nch = (lofs + nl + 15) >> 4;
        for (u32 c = lane; c < nch; c += 32) cp_async16(S.lit + c * 16, lchunk + c * 16);
        const u32 ms = done + end - m.len, mq = ms - m.dist;      // the lane's match: start, first source byte
        const bool far = lane < k && m.len != 0 && mq + RING < bend;
        const u32 c0 = (mq + ph) >> 4;                           // first source chunk (output chunk index)
        const u32 fch = far ? ((mq + m.len - 1 + ph) >> 4) - c0 + 1 : 0u;
        u32 fend = fch;                                          // inclusive scan: staging chunks up to this record
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 v = __shfl_up_sync(SWC_FULL, fend, d);
            if (lane >= (u32)d) fend += v;
        }
        const u32 fbeg = fend - fch;
        const u8 *outa = out - ph;                               // 16-byte aligned: output chunk c starts at outa + 16 c
        for (u32 c = 0; c < fch; c++) {
            u8 *dst = S.far + (fbeg + c) * 16;
            if (c0 + c > 0 || ph == 0) {
                cp_async16(dst, outa + (c0 + c) * 16);
            } else {
                for (u32 b = ph; b < 16; b++) dst[b] = outa[b];  // the output's first chunk starts before out[0]
            }
        }
        S.stage[lane] = make_uint4(ms, lane < k ? m.len : 0u, m.dist, far ? fbeg * 16 + ((mq + ph) & 15) : NEAR);
        cp_async_wait_all();
        __syncwarp();
        // ---- literals -> their positions in the ring
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
        __syncwarp();
        // ---- matches
#pragma unroll 1
        for (u32 b0 = 0; b0 < k; b0 += 8) {
            const uint4 rc = S.stage[b0 + sub];                  // this sub-group's record
            const u32 s = rc.x, l = rc.y, d = rc.z;
            const u32 src_end = s - d + (l < d ? l : d);
            // source byte i of the match: a far one from the staging buffer, a near one from the ring
            const bool fr = rc.w != NEAR;
            const u8 *sb = fr ? S.far : S.ring;
            const u32 s0 = fr ? rc.w : s - d + ph, sm = fr ? 0xFFFFFFFFu : M;
            const u32 alim = fr ? FARBUF : M - 3;               // source index of 4 bytes that do not wrap around
            auto src_byte = [&](u32 i) -> u8 { return sb[(s0 + i) & sm]; };
            bool pend = l != 0;
            u32 pmask = __ballot_sync(SWC_FULL, pend && t == 0); // bit 4*sub per pending record
            while (pmask) {
                const u32 oldest = (__ffs(pmask) - 1) >> 2;       // sub-group index of the oldest pending record
                const u32 frontier = S.stage[b0 + oldest].x;
                const bool ready = pend && (sub == oldest || src_end <= frontier);
                if (ready) {
                    if (d >= l) {
                        // four consecutive bytes per lane and trip, all four loads issued before the first store; one
                        // source and one ring address per trip unless the four bytes wrap around the ring
                        for (u32 i = 4 * t; i < l; i += 16) {
                            const bool p1 = i + 1 < l, p2 = i + 2 < l, p3 = i + 3 < l;
                            const u32 a = (s0 + i) & sm, b = (s + i + ph) & M;
                            u32 v0, v1 = 0, v2 = 0, v3 = 0;
                            if (a <= alim && b <= M - 3) {
                                const u8 *src = sb + a;
                                u8 *dst = S.ring + b;
                                v0 = src[0];
                                if (p1) v1 = src[1];
                                if (p2) v2 = src[2];
                                if (p3) v3 = src[3];
                                dst[0] = v0;
                                if (p1) dst[1] = v1;
                                if (p2) dst[2] = v2;
                                if (p3) dst[3] = v3;
                            } else {
                                v0 = src_byte(i);
                                if (p1) v1 = src_byte(i + 1);
                                if (p2) v2 = src_byte(i + 2);
                                if (p3) v3 = src_byte(i + 3);
                                S.ring[b] = v0;
                                if (p1) S.ring[(b + 1) & M] = v1;
                                if (p2) S.ring[(b + 2) & M] = v2;
                                if (p3) S.ring[(b + 3) & M] = v3;
                            }
                        }
                    } else {
                        for (u32 i = t; i < l; i += 4) S.ring[(s + i + ph) & M] = src_byte(i % d);
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
