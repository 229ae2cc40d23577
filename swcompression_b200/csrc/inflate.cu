// inflate.cu — batched Deflate decode for sm_90a: the LZ77 stage and the launcher.  Replaces Deflate.decompress(_: LsbBitReader)
// (reference Sources/Deflate/Deflate.swift:30-249) + Code.huffmanCodes / DecodingTree (Sources/Common/CodingTree).
//
// Two kernels per batch (DESIGN.md §4.1):
//   K1 the Huffman stage — K1L inflate_lut_kernel (inflate_lut.cu, one thread per unit) for large batches, K1w
//        inflate_warp_kernel (inflate_warp.cu, one warp per unit) for small ones.  Literals go straight to their final
//        output position, every match becomes a record (format in inflate.cuh).
//   K2 lz_resolve_kernel (here) — ONE WARP PER UNIT.  Replays the records 8 at a time on 4-lane sub-groups
//        (period-replicating when distance < length).  Positions come from a warp inclusive scan of the records.
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
// One warp per unit: replay the match records in order.  Lane j holds record j of a 32-record group; an inclusive warp
// scan of (literal-run + length) gives every match its absolute position; {start, length, distance} are staged in shared
// memory.  The group is then executed 8 records at a time by 4-lane sub-groups (one 16-byte load fetches the record).  A record is READY when everything it reads is final: its source ends at or before the
// start of the oldest still-pending record of the batch (bytes before that point were placed by K1 literals or by
// completed matches) — or it IS that oldest record.  Far matches therefore run 8-wide in one pass; chains of
// near matches (RLE-like data) degrade gracefully to in-order execution.  Overlapping copies (dist < len) replicate the
// period: every source byte lies in [start-dist, start), never in what the match itself writes.
__global__ void __launch_bounds__(256)
lz_resolve_kernel(BatchArgs a) {
    __shared__ uint4 stage[8][32];                       // {start, length, distance} of the warp's current 32 records
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= a.n) return;
    if (a.status[unit] != SWC_OK) return;
    const u32 lane = threadIdx.x & 31;
    const u32 sub = lane >> 2, t = lane & 3;
    uint4 *st = stage[(threadIdx.x >> 5) & 7];
    const u32 nrec = a.rec_count[unit];
    const u32 *rec = a.rec_base + rec_start(a.out_off[unit]);
    u8 *out = a.out_base + a.out_off[unit];
    u32 base = 0;
    for (u32 g = 0; g < nrec; g += 32) {
        const Match m = get_match((g + lane < nrec) ? rec[g + lane] : REC_ESC);
        u32 end = m.adv;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 v = __shfl_up_sync(SWC_FULL, end, d);
            if (lane >= (u32)d) end += v;
        }
        // a sub-group fetches its record with one 16-byte shared-memory load instead of three shuffles
        st[lane] = make_uint4(base + end - m.len, m.len, m.dist, 0u);
        base += __shfl_sync(SWC_FULL, end, 31);
        __syncwarp();
#pragma unroll 1
        for (u32 b0 = 0; b0 < 32; b0 += 8) {
            const uint4 rc = st[b0 + sub];                               // this sub-group's record
            const u32 s = rc.x, l = rc.y, d = rc.z;
            const u32 src_end = s - d + (l < d ? l : d);
            bool pend = l != 0;
            u32 pmask = __ballot_sync(SWC_FULL, pend && t == 0);         // bit 4*sub per pending record
            while (pmask) {
                const u32 oldest = (__ffs(pmask) - 1) >> 2;                // sub-group index of the oldest pending record
                const u32 frontier = st[b0 + oldest].x;
                const bool ready = pend && (sub == oldest || src_end <= frontier);
                if (ready) {
                    const u8 *src = out + s - d;
                    u8 *dst = out + s;
                    if (d >= l) {
                        // four bytes per lane and trip, all four loads issued before the first store (a match is 15 bytes on
                        // average: one trip covers 16)
                        for (u32 k = t; k < l; k += 16) {
                            const bool p1 = k + 4 < l, p2 = k + 8 < l, p3 = k + 12 < l;
                            const u8 b0v = src[k];
                            u8 b1 = 0, b2 = 0, b3 = 0;
                            if (p1) b1 = src[k + 4];
                            if (p2) b2 = src[k + 8];
                            if (p3) b3 = src[k + 12];
                            dst[k] = b0v;
                            if (p1) dst[k + 4] = b1;
                            if (p2) dst[k + 8] = b2;
                            if (p3) dst[k + 12] = b3;
                        }
                    } else {
                        for (u32 i = t; i < l; i += 4) dst[i] = src[i % d];
                    }
                    pend = false;
                }
                __syncwarp();
                pmask = __ballot_sync(SWC_FULL, pend && t == 0);
            }
        }
        __syncwarp();                                                    // the stage is rewritten for the next group
    }
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
    const u64 g2 = (a.n * 32 + 255) / 256;
    lz_resolve_kernel<<<(unsigned)g2, 256, 0, stream>>>(a);
    count_launch();
    timing_mark(stream);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace inflate
}  // namespace swc
