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
// output ends at most SPAN bytes past the batch start, at most BATCH = 64 of them; lane j holds records 2j and 2j + 1,
// loaded one batch ahead.  Per batch:
//   scan     : inclusive scans of (literal run + length) and of the literal run — each lane adds its pair, a warp scan
//              adds the pair sums — give every record its position and the offset of its literals in the batch's part of
//              the literal stream;
//   gather   : one round of 16-byte cp.async copies brings in the batch's literals from the packed stream and the sources
//              of its FAR matches from the output, both into one staging buffer (literals first, far sources behind
//              them).  A match is far when its first source byte is more than RING bytes behind the batch end (bend):
//              with len <= 258 and bend - RING <= done - SPAN, its whole source then lies in output this warp has already
//              flushed, and dist > RING - SPAN >= len.  Every other match reads only bytes that are still in the ring.
//              The nl literals take at most (nl + 30)/16 aligned chunks, a far source of len bytes at most
//              (len + 30)/16; the batch's literal runs and lengths sum to <= SPAN, so with <= 64 records the buffer needs
//              at most (SPAN + 30 + 30 * 64)/16, i.e. 185 chunks.  A warp-wide scan packs the far sources; the part
//              of the output's first chunk that lies before out[0] is never read (that chunk is copied byte by byte);
//   literals : each lane copies the literal runs of its two records into the ring, eight bytes per trip (a binary
//              search over the records for every literal, one per lane and round, was slower);
//   matches  : replayed PASS = 16 at a time by 2-lane sub-groups, reading shared memory only (far ones from the staging
//              buffer, the others from the ring).  A record is READY when everything it reads is final: its source ends
//              at or before the start of the oldest still-pending record of the pass (bytes before that point are
//              literals, older matches or earlier batches) — or it IS that oldest record.  Far matches therefore run
//              16-wide in one pass, chains of near matches (RLE-like data) degrade to in-order execution.  Overlapping
//              copies (dist < len) replicate the period: every source byte lies in [start-dist, start), never in what
//              the match itself writes;
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
constexpr u32 BATCH = 64;            // records per batch at most: two per lane
constexpr u32 SUBW = 2;              // lanes per replay sub-group (4-lane sub-groups, 8 records per pass: slower)
constexpr u32 PASS = 32 / SUBW;      // records replayed per pass
constexpr u32 BPL = 16 / SUBW;       // bytes per lane and trip of a copy
constexpr u32 STAGEBUF = (SPAN + 30 + 30 * BATCH) / 16 * 16;   // a batch's literals, then its far sources
constexpr u32 NEAR = 0xFFFFFFFFu;    // staging offset of a match that reads the ring
struct __align__(16) WarpSmem {
    uint4 stage[BATCH];              // {start, length, distance, staging offset of the first source byte | NEAR}
    u8 ring[RING];
    u8 buf[STAGEBUF];
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
    const u32 sub = lane / SUBW, t = lane % SUBW;
    const u64 off = a.out_off[unit];
    const u32 len = (u32)a.out_len[unit];
    u8 *out = a.out_base + off;
    const u32 *rec = a.rec_base + rec_start(off + a.out_cap[unit]);      // record k at rec - 1 - k
    const u8 *lits = (const u8 *)(a.rec_base + rec_start(off));
    const u32 ph = (u32)((uintptr_t)out & 15);
    u8 *const outa = out - ph;       // 16-byte aligned: output chunk c starts at outa + 16 c
    const u32 M = RING - 1;
    u32 done = 0;          // output bytes placed by earlier batches
    u32 flushed = 0;       // output bytes written to global memory
    u32 lit = 0;           // literals consumed
    u32 g = 0;             // next record
    u32 part = 0;          // bytes of record g already placed (an escape longer than SPAN)
    // writes output bytes [flushed, to) from the ring: whole aligned chunks as 16-byte stores, the rest byte by byte.
    // Positions are taken relative to the aligned base out - ph (output byte p is byte p + ph of it), where every value up
    // to len + ph <= OUT_MAX + 15 fits a u32; only the first chunk starts before out[0], and its flushed + ph - cb >= ph
    // keeps those bytes out of the copy.  The chunk end cb + 16 is never formed: it wraps for the output's last chunk.
    auto flush = [&](u32 to) {
        const u32 q0 = flushed + ph, q1 = to + ph;
        const u32 c0 = q0 >> 4, c1 = (q1 >> 4) + ((q1 & 15) != 0);
        for (u32 c = c0 + lane; c < c1; c += 32) {
            const u32 cb = c * 16;                                      // chunk start relative to outa
            const u32 lo = q0 > cb ? q0 - cb : 0u, hi = q1 - cb < 16 ? q1 - cb : 16u;   // bytes [lo, hi) of the chunk
            if (lo == 0 && hi == 16) {
                *(uint4 *)(outa + cb) = *(const uint4 *)(S.ring + (cb & M));
            } else {
                for (u32 i = lo; i < hi; i++) outa[cb + i] = S.ring[(cb + i) & M];
            }
        }
        flushed = to;
    };
    // records g + 2 lane (x) and g + 2 lane + 1 (y)
    auto load = [&](u32 i) -> u32 { return i < nrec ? __ldg(rec - 1 - i) : REC_ESC; };
    u32 rx = load(2 * lane), ry = load(2 * lane + 1);
    for (;;) {
        // ---- the batch: records g.. whose output ends within SPAN bytes of `done`, at most BATCH of them
        const u32 ix = 2 * lane, iy = ix + 1;                    // record indices within the batch
        const Match mx = get_match(rx), my = get_match(ry);
        const u32 advx = mx.adv - (lane == 0 ? part : 0u), advy = my.adv;
        const u32 runx = advx - mx.len, runy = advy - my.len;
        u32 end = advx + advy, lend = runx + runy;               // inclusive scans over the pairs: record y's values
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 v = __shfl_up_sync(SWC_FULL, end, d), w = __shfl_up_sync(SWC_FULL, lend, d);
            if (lane >= (u32)d) { end += v; lend += w; }
        }
        const u32 endx = end - advy, lendx = lend - runy;        // record x's
        // a prefix: `end` does not decrease along the records
        const u32 k = __popc(__ballot_sync(SWC_FULL, g + ix < nrec && endx <= SPAN)) +
                      __popc(__ballot_sync(SWC_FULL, g + iy < nrec && end <= SPAN));
        u32 span, nl;
        u32 deltax, deltay;  // output position of a literal minus its index in the batch's literals (records x, y)
        u32 litx, lity, nx, ny;   // first literal (index in the batch's literals) and literal count of records x, y
        if (k > 0) {
            const bool ly = ((k - 1) & 1) != 0;                  // the batch's last record is a y
            span = __shfl_sync(SWC_FULL, ly ? end : endx, (k - 1) >> 1);
            nl = __shfl_sync(SWC_FULL, ly ? lend : lendx, (k - 1) >> 1);
            deltax = done + endx - advx - (lendx - runx);
            deltay = done + end - advy - (lend - runy);
            litx = lendx - runx;
            lity = lendx;
            nx = ix < k ? runx : 0u;
            ny = iy < k ? runy : 0u;
            g += k;
            part = 0;
        } else {
            // a literal run longer than SPAN: an escape (g < nrec) or the literals after the last match
            const u32 adv0 = __shfl_sync(SWC_FULL, advx, 0);     // what is left of escape g
            const u32 rem = g < nrec ? adv0 : len - done;
            if (rem == 0) break;
            span = nl = rem < SPAN ? rem : SPAN;
            if (g < nrec) part += span;
            deltax = deltay = done;
            litx = lity = 0;
            nx = lane == 0 ? nl : 0u;
            ny = 0;
        }
        if (k > 0) {                                             // the next batch's records
            rx = load(g + ix);
            ry = load(g + iy);
        }
        const u32 bend = done + span;                            // batch end
        // ---- gather: the literals (packed stream) and the far match sources (flushed output) -> shared memory
        const uintptr_t lsrc = (uintptr_t)(lits + lit);
        const u8 *lchunk = (const u8 *)(lsrc & ~(uintptr_t)15);
        const u32 lofs = (u32)(lsrc & 15), nch = (lofs + nl + 15) >> 4;
        for (u32 c = lane; c < nch; c += 32) cp_async16(S.buf + c * 16, lchunk + c * 16);
        const u32 msx = done + endx - mx.len, mqx = msx - mx.dist;      // the lane's matches: start, first source byte
        const u32 msy = done + end - my.len, mqy = msy - my.dist;
        const bool farx = ix < k && mx.len != 0 && bend - mqx > RING;  // mqx + RING would wrap near the 2^32 ceiling
        const bool fary = iy < k && my.len != 0 && bend - mqy > RING;
        const u32 c0x = (mqx + ph) >> 4, c0y = (mqy + ph) >> 4;          // first source chunks (output chunk index)
        const u32 fchx = farx ? ((mqx + mx.len - 1 + ph) >> 4) - c0x + 1 : 0u;
        const u32 fchy = fary ? ((mqy + my.len - 1 + ph) >> 4) - c0y + 1 : 0u;
        u32 fend = fchx + fchy;                                  // inclusive scan: staging chunks up to this pair
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 v = __shfl_up_sync(SWC_FULL, fend, d);
            if (lane >= (u32)d) fend += v;
        }
        const u32 fbx = nch + fend - fchx - fchy, fby = fbx + fchx;      // first staging chunks of x and y
        for (u32 c = 0; c < fchx + fchy; c++) {
            const u32 oc = c < fchx ? c0x + c : c0y + c - fchx;  // output chunk
            u8 *dst = S.buf + (fbx + c) * 16;
            if (oc > 0 || ph == 0) {
                cp_async16(dst, outa + oc * 16);
            } else {
                for (u32 b = ph; b < 16; b++) dst[b] = outa[b];  // the output's first chunk starts before out[0]
            }
        }
        S.stage[ix] = make_uint4(msx, ix < k ? mx.len : 0u, mx.dist, farx ? fbx * 16 + ((mqx + ph) & 15) : NEAR);
        S.stage[iy] = make_uint4(msy, iy < k ? my.len : 0u, my.dist, fary ? fby * 16 + ((mqy + ph) & 15) : NEAR);
        cp_async_wait_all();
        __syncwarp();
        // ---- literals -> their positions in the ring: each lane copies the literal runs of its two records, eight
        // bytes per trip, all loads before the first store
        auto place = [&](u32 li, u32 delta, u32 n, u32 i) {
            if (i >= n) return;
            const u8 *src = S.buf + lofs + li + i;
            const u32 b = (li + delta + i + ph) & M;
            u32 v[8];
#pragma unroll
            for (u32 q = 0; q < 8; q++) v[q] = i + q < n ? src[q] : 0u;
            if (b <= M - 7) {
#pragma unroll
                for (u32 q = 0; q < 8; q++)
                    if (i + q < n) S.ring[b + q] = (u8)v[q];
            } else {
#pragma unroll
                for (u32 q = 0; q < 8; q++)
                    if (i + q < n) S.ring[(b + q) & M] = (u8)v[q];
            }
        };
        for (u32 i = 0; i < (nx > ny ? nx : ny); i += 8) {
            place(litx, deltax, nx, i);
            place(lity, deltay, ny, i);
        }
        lit += nl;
        __syncwarp();
        // ---- matches
#pragma unroll 1
        for (u32 b0 = 0; b0 < k; b0 += PASS) {
            const uint4 rc = S.stage[b0 + sub];                  // this sub-group's record
            const u32 s = rc.x, l = rc.y, d = rc.z;
            const u32 src_end = s - d + (l < d ? l : d);
            // source byte i of the match: a far one from the staging buffer, a near one from the ring
            const bool fr = rc.w != NEAR;
            const u8 *sb = fr ? S.buf : S.ring;
            const u32 s0 = fr ? rc.w : s - d + ph, sm = fr ? 0xFFFFFFFFu : M;
            const u32 alim = fr ? STAGEBUF : M - (BPL - 1);     // source index of BPL bytes that do not wrap around
            auto src_byte = [&](u32 i) -> u8 { return sb[(s0 + i) & sm]; };
            bool pend = l != 0;
            u32 pmask = __ballot_sync(SWC_FULL, pend && t == 0); // bit SUBW*sub per pending record
            while (pmask) {
                const u32 oldest = (__ffs(pmask) - 1) / SUBW;     // sub-group index of the oldest pending record
                const u32 frontier = S.stage[b0 + oldest].x;
                const bool ready = pend && (sub == oldest || src_end <= frontier);
                if (ready) {
                    if (d >= l) {
                        // BPL consecutive bytes per lane and trip, all loads issued before the first store; one source
                        // and one ring address per trip unless the bytes wrap around the ring
                        for (u32 i = BPL * t; i < l; i += 16) {
                            const u32 a = (s0 + i) & sm, b = (s + i + ph) & M;
                            u32 v[BPL];
                            if (a <= alim && b <= M - (BPL - 1)) {
                                const u8 *src = sb + a;
                                u8 *dst = S.ring + b;
#pragma unroll
                                for (u32 q = 0; q < BPL; q++) v[q] = i + q < l ? src[q] : 0u;
#pragma unroll
                                for (u32 q = 0; q < BPL; q++)
                                    if (i + q < l) dst[q] = (u8)v[q];
                            } else {
#pragma unroll
                                for (u32 q = 0; q < BPL; q++) v[q] = i + q < l ? src_byte(i + q) : 0u;
#pragma unroll
                                for (u32 q = 0; q < BPL; q++)
                                    if (i + q < l) S.ring[(b + q) & M] = (u8)v[q];
                            }
                        }
                    } else {
                        for (u32 i = t; i < l; i += SUBW) S.ring[(s + i + ph) & M] = src_byte(i % d);
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
void seat_scratch(BatchArgs &a, void *scratch, u64 n, u64 first, int tickets, int ticket) {
    u8 *s = (u8 *)scratch;
    a.ticket = (unsigned long long *)(s + (size_t)256 * ticket);
    a.rec_count = (u32 *)(s + (size_t)256 * tickets) + first;
    a.rec_base = (u32 *)(s + scratch_header(n, tickets));
}

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
