// lz4.cu — batched LZ4 block decode for sm_90a.  Replaces LZ4.process(block:_:) (reference
// Sources/LZ4/LZ4.swift:332-413) and the per-block part of LZ4.process(frame:) (:278-318).
//
// ONE WARP PER UNIT.  A unit is a chain of one or more blocks that are decoded in order into one contiguous output
// region (chains model frames with dependent blocks, LZ4.swift:307-313; independent blocks are one-block units).
// All 32 lanes parse the sequence stream in lock-step from a 32-byte register window (one coalesced load per
// sequence in the common case, bytes exchanged with warp shuffles), then copy literals and matches cooperatively.
#include <cstdlib>
#include "common.cuh"
#include "lz4.cuh"

namespace swc {
namespace lz4 {

struct Window {
    const u8 *in;
    u64 n;        // block length
    u64 base;     // offset of window byte 0
    u32 w;        // this lane's byte
    __device__ __forceinline__ void load(u64 at) {
        base = at;
        w = (at + lane_id() < n) ? in[at + lane_id()] : 0;
    }
    // make [at, at+need) visible (need <= 32)
    __device__ __forceinline__ void ensure(u64 at, u32 need) {
        if (at < base || at + need > base + 32) load(at);
    }
    __device__ __forceinline__ u32 get(u64 at) const { return __shfl_sync(SWC_FULL, w, (int)(at - base)); }
};

// warp-cooperative forward copy of n bytes, regions do not overlap (or dst > src + 32*16)
__device__ __forceinline__ void warp_copy(u8 *dst, const u8 *src, u64 n) {
    const u32 lane = lane_id();
    if (n >= 256 && (((uintptr_t)dst ^ (uintptr_t)src) & 15) == 0) {
        u64 head = (16 - ((uintptr_t)dst & 15)) & 15;
        if (lane < head) dst[lane] = src[lane];
        u64 body = (n - head) >> 4;
        const uint4 *s4 = (const uint4 *)(src + head);
        uint4 *d4 = (uint4 *)(dst + head);
        for (u64 i = lane; i < body; i += 32) d4[i] = s4[i];
        u64 done = head + (body << 4);
        if (done + lane < n) dst[done + lane] = src[done + lane];
        return;
    }
    for (u64 i = lane; i < n; i += 32) dst[i] = src[i];
}

// length-extension bytes (LZ4.swift:347-363 / :386-401). Returns false on truncation. `ip` ends after the last byte.
__device__ __forceinline__ bool read_extension(Window &win, u64 &ip, u64 &value) {
    const u32 lane = lane_id();
    for (;;) {
        if (ip >= win.n) return false;
        win.ensure(ip, 1);
        u32 pos = (u32)(ip - win.base);
        u32 m = __ballot_sync(SWC_FULL, win.w != 255) & (0xFFFFFFFFu << pos);
        if (m) {
            u32 j = __ffs(m) - 1;
            if (win.base + j >= win.n) return false;        // ran off the block inside the 255-run
            value += 255ull * (j - pos) + __shfl_sync(SWC_FULL, win.w, j);
            ip = win.base + j + 1;
            return true;
        }
        value += 255ull * (32 - pos);
        ip = win.base + 32;
        (void)lane;
    }
}

template <bool ONLY_FLAGGED>
__device__ __forceinline__ void lz4_block_body(const Args &a) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= a.n) return;
    if (ONLY_FLAGGED && a.status[unit] != 9002) return;
    const u32 lane = lane_id();
    u8 *out = a.out_base + a.out_off[unit];
    const u64 cap = a.out_cap[unit];
    const u64 b0 = a.first_blk ? a.first_blk[unit] : unit;
    const u64 nb = a.n_blk ? a.n_blk[unit] : 1;
    const i64 dict_len = (a.no_dict && a.no_dict[unit]) ? 0 : (i64)a.dict_len;
    const u8 *dict_end = a.dict + a.dict_len;       // dict bytes sit at virtual positions [-dict_len, 0)
    u64 op = 0, fail_blk = 0;
    int status = SWC_OK;

    for (u64 b = 0; b < nb && status == SWC_OK; b++) {
        fail_blk = b;
        const u64 blen_raw = a.in_len[b0 + b];
        const bool stored = (blen_raw >> 63) != 0;
        const u64 n = blen_raw & ~(1ull << 63);
        const u8 *in = a.in_base + a.in_off[b0 + b];
        if (stored) {                                                   // LZ4.swift:314-316
            if (op + n <= cap) warp_copy(out + op, in, n);
            op += n;
            __syncwarp();
            continue;
        }
        // lowest addressable virtual position for this block (LZ4.swift:305-313)
        const i64 lo = (op == 0) ? -dict_len : (i64)(op > 65536 ? op - 65536 : 0);   // `out.isEmpty` rule, :307
        Window win; win.in = in; win.n = n; win.base = 0; win.w = 0;
        u64 ip = 0;
        u64 seq = 0;
        i64 last_match_start = -1;
        bool have_match = false;
        if (n > 0) win.load(0);
        for (;;) {
            seq++;
            if (ip >= n) { status = SWC_DATA_TRUNCATED; break; }                         // :343
            win.ensure(ip, 1);
            const u32 token = win.get(ip);
            ip++;
            u64 lit = token >> 4;
            if (lit == 15 && !read_extension(win, ip, lit)) { status = SWC_DATA_TRUNCATED; break; }
            if (n - ip < lit) { status = SWC_DATA_TRUNCATED; break; }                    // :364
            if (op + lit <= cap) warp_copy(out + op, in + ip, lit);
            op += lit;
            ip += lit;
            if (ip == n) {                                                               // :369-377
                if (!(lit >= 5 || seq == 1)) status = SWC_DATA_CORRUPTED;
                else if (have_match && (i64)op - last_match_start < 12) status = SWC_DATA_CORRUPTED;
                break;
            }
            if (n - ip < 2) { status = SWC_DATA_TRUNCATED; break; }                      // :379
            win.ensure(ip, 2);
            const u64 offset = win.get(ip) | (win.get(ip + 1) << 8);
            ip += 2;
            if (offset == 0 || (i64)offset > (i64)op - lo) { status = SWC_DATA_CORRUPTED; break; }   // :383
            u64 mlen = 4 + (token & 15);
            if (mlen == 19 && !read_extension(win, ip, mlen)) { status = SWC_DATA_TRUNCATED; break; }
            last_match_start = (i64)op; have_match = true;                               // :405
            if (op + mlen <= cap) {
                __syncwarp();     // literals just written by other lanes may be match sources
                const i64 src = (i64)op - (i64)offset;
                if (src >= 0 && offset >= mlen && offset >= 16 * 32) {
                    warp_copy(out + op, out + src, mlen);
                } else {
                    for (u64 i = lane; i < mlen; i += 32) {
                        const i64 s = src + (i64)(offset >= mlen ? i : i % offset);
                        out[op + i] = s >= 0 ? out[s] : dict_end[s];
                    }
                }
                __syncwarp();
            }
            op += mlen;
        }
    }
    if (lane == 0) {
        if (status == SWC_OK && op > cap) status = SWC_ERR_OUTPUT_OVERFLOW;
        // chains report WHICH block failed so the host can order errors like the reference's sequential loop
        a.out_len[unit] = (a.n_blk && status != SWC_OK && status != SWC_ERR_OUTPUT_OVERFLOW) ? fail_blk : op;
        a.status[unit] = status;
    }
}

// =====================================================================================================================
// Two-phase path for single-block units (the batched raw-block API and independent-block frames):
//   P1 lz4_parse_kernel — ONE THREAD PER BLOCK walks the token / length / offset bytes only (no payload is touched),
//      applies every check of LZ4.process(block:_:) in the reference's order (so the status is final here) and writes one
//      8-byte record per sequence {literal length:24 | match length:24 | offset:16}.
//   P2 lz4_exec_kernel  — ONE WARP PER BLOCK: warp scans over 32 records give each sequence its input and output
//      positions; literals (sources in the compressed block: no hazards) are copied first, then matches run 8 at a time on
//      4-lane sub-groups under the same "oldest pending record" readiness rule as the Deflate resolve kernel; long copies
//      (>= 64 bytes: incompressible or zero-filled blocks) are done by the whole warp.
// Units whose lengths do not fit 24 bits, and units that read or write 4 GiB or more, are flagged for the one-kernel
// decoder above.

__device__ __forceinline__ u32 ext_bytes(u32 len_field_value /* length minus its base */) {
    return len_field_value < 15 ? 0u : 1u + (len_field_value - 15u) / 255u;
}

__global__ void __launch_bounds__(128) lz4_parse_kernel(Args a, const u64 *rec_base_idx, u64 *recs, u32 *rec_count) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= a.n) return;
    const u8 *in = a.in_base + a.in_off[unit];
    const u64 n = a.in_len[unit] & ~(1ull << 63);
    const bool stored = (a.in_len[unit] >> 63) != 0;
    const u64 cap = a.out_cap[unit];
    u64 *rec = recs + rec_base_idx[unit];
    u32 nrec = 0;
    int status = SWC_OK;
    u64 ip = 0, op = 0, seq = 0;
    const u64 prefix = a.dict && !(a.no_dict && a.no_dict[unit]) ? a.dict_len : 0;
    i64 last_match_start = -1;
    // a stored block, or a field that does not fit a record: the walk goes on without records, so that the size and the
    // status are final here, and the one-kernel decoder does the copying
    bool no_records = stored;
    if (stored) { op = n; }
    else for (;;) {
        seq++;
        if (ip >= n) { status = SWC_DATA_TRUNCATED; break; }                                     // LZ4.swift:343
        const u32 token = in[ip++];
        u64 lit = token >> 4;
        if (lit == 15) {
            bool ok = false;
            while (ip < n) { const u32 b = in[ip++]; lit += b; if (b != 255) { ok = true; break; } }
            if (!ok) { status = SWC_DATA_TRUNCATED; break; }
        }
        if (n - ip < lit) { status = SWC_DATA_TRUNCATED; break; }                                // :364
        op += lit; ip += lit;
        if (ip == n) {                                                                           // :369-377
            if (!(lit >= 5 || seq == 1)) status = SWC_DATA_CORRUPTED;
            else if (last_match_start >= 0 && (i64)op - last_match_start < 12) status = SWC_DATA_CORRUPTED;
            else if (lit >= (1u << 24)) no_records = true;
            else if (!no_records) rec[nrec++] = lit;
            break;
        }
        if (n - ip < 2) { status = SWC_DATA_TRUNCATED; break; }                                  // :379
        const u32 offset = (u32)in[ip] | ((u32)in[ip + 1] << 8);
        ip += 2;
        if (offset == 0 || (u64)offset > op + prefix) { status = SWC_DATA_CORRUPTED; break; }    // :383
        u64 mlen = 4 + (token & 15);
        if (mlen == 19) {
            bool ok = false;
            while (ip < n) { const u32 b = in[ip++]; mlen += b; if (b != 255) { ok = true; break; } }
            if (!ok) { status = SWC_DATA_TRUNCATED; break; }
        }
        last_match_start = (i64)op;
        if (lit >= (1u << 24) || mlen >= (1u << 24)) no_records = true;
        if (!no_records) rec[nrec++] = lit | (mlen << 24) | ((u64)offset << 48);
        op += mlen;
    }
    if (status == SWC_OK && op > cap) status = SWC_ERR_OUTPUT_OVERFLOW;
    // the exec kernel keeps input and output positions in 32 bits: a block that reads or writes 4 GiB or more goes to the
    // fallback (after the capacity check, so that an overflowing unit still reports its exact size)
    if (status == SWC_OK && (no_records || (op >> 32) != 0 || (n >> 32) != 0)) status = LZ4_INTERNAL_FALLBACK;
    a.out_len[unit] = op;
    a.status[unit] = status;
    rec_count[unit] = nrec;
}

// n (< 64) bytes by a 4-lane sub-group, non-overlapping: four bytes per lane and trip, the loads issued before the first store
__device__ __forceinline__ void group_copy(u8 *dst, const u8 *src, u32 n, u32 t) {
    for (u32 k = t; k < n; k += 16) {
        const bool p1 = k + 4 < n, p2 = k + 8 < n, p3 = k + 12 < n;
        const u8 b0 = src[k];
        u8 b1 = 0, b2 = 0, b3 = 0;
        if (p1) b1 = src[k + 4];
        if (p2) b2 = src[k + 8];
        if (p3) b3 = src[k + 12];
        dst[k] = b0;
        if (p1) dst[k + 4] = b1;
        if (p2) dst[k + 8] = b2;
        if (p3) dst[k + 12] = b3;
    }
}

// 4 CTAs per SM (64 registers): at 8 CTAs (32 registers) or 6 (40) sm_90a spills hundreds of bytes per thread on the copy
// path, and on an H100 the 262 144-block LZ4 batch of tools/bench_codecs.py took 113 / 93 ms there against 83 ms here
__global__ void __launch_bounds__(256, 4) lz4_exec_kernel(Args a, const u64 *rec_base_idx, const u64 *recs, const u32 *rec_count) {
    // the warp's current 32 sequences: [0] = {literal source, literal destination, literal length}, [1] = {match start, match
    // length, offset}; a sub-group fetches its sequence with one 16-byte load instead of three shuffles
    __shared__ uint4 stage[8][2][32];
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= a.n) return;
    if (a.status[unit] != SWC_OK) return;
    const u32 lane = lane_id(), sub = lane >> 2, t = lane & 3;
    uint4 (*st)[32] = stage[(threadIdx.x >> 5) & 7];
    const u8 *in = a.in_base + a.in_off[unit];
    u8 *out = a.out_base + a.out_off[unit];
    const u64 *rec = recs + rec_base_idx[unit];
    const u32 nrec = rec_count[unit];
    const u8 *dict_end = a.dict ? a.dict + a.dict_len : nullptr;
    u32 in_base = 0, out_base = 0;
    for (u32 g = 0; g < nrec; g += 32) {
        const u64 r = (g + lane < nrec) ? rec[g + lane] : 0ull;
        const bool have = g + lane < nrec;
        const u32 lit = (u32)r & 0xFFFFFFu, mlen = (u32)(r >> 24) & 0xFFFFFFu, offset = (u32)(r >> 48);
        const u32 in_adv = have ? 1u + ext_bytes(lit) + lit + (mlen ? 2u + ext_bytes(mlen - 4u) : 0u) : 0u;
        const u32 out_adv = lit + mlen;
        u32 ie = in_adv, oe = out_adv;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 vi = __shfl_up_sync(SWC_FULL, ie, d), vo = __shfl_up_sync(SWC_FULL, oe, d);
            if (lane >= (u32)d) { ie += vi; oe += vo; }
        }
        const u32 lit_src = in_base + ie - in_adv + 1u + ext_bytes(lit);
        const u32 lit_dst = out_base + oe - out_adv;
        in_base += __shfl_sync(SWC_FULL, ie, 31);
        out_base += __shfl_sync(SWC_FULL, oe, 31);
        st[0][lane] = make_uint4(lit_src, lit_dst, lit, 0u);
        st[1][lane] = make_uint4(lit_dst + lit, mlen, offset, 0u);
        __syncwarp();
        // ---- literals: long runs by the whole warp, short ones by sub-groups
        u32 big = __ballot_sync(SWC_FULL, lit >= 64);
        while (big) {
            const int k = __ffs(big) - 1; big &= big - 1;
            const uint4 q = st[0][k];
            warp_copy(out + q.y, in + q.x, q.z);
        }
#pragma unroll 1
        for (u32 b0 = 0; b0 < 32; b0 += 8) {
            const uint4 q = st[0][b0 + sub];
            if (q.z < 64) group_copy(out + q.y, in + q.x, q.z, t);
        }
        __syncwarp();
        // ---- matches
#pragma unroll 1
        for (u32 b0 = 0; b0 < 32; b0 += 8) {
            const uint4 q = st[1][b0 + sub];
            const u32 s = q.x, l = q.y, d = q.z;
            const i64 src0 = (i64)s - (i64)d;
            const i64 src_end = src0 + (i64)(l < d ? l : d);
            bool pend = l != 0;
            u32 pmask = __ballot_sync(SWC_FULL, pend && t == 0);
            while (pmask) {
                const u32 oldest = (__ffs(pmask) - 1) >> 2;
                const uint4 f = st[1][b0 + oldest];
                const u32 fs = f.x, fl = f.y, fd = f.z;
                if (fl >= 64) {                                       // long match: the whole warp copies the oldest record
                    const i64 fsrc = (i64)fs - (i64)fd;
                    if (fsrc >= 0 && fd >= fl && fd >= 512) warp_copy(out + fs, out + fsrc, fl);
                    else for (u32 i = lane; i < fl; i += 32) {
                        const i64 qq = fsrc + (i64)(fd >= fl ? i : i % fd);
                        out[fs + i] = qq >= 0 ? out[qq] : dict_end[qq];
                    }
                    if (sub == oldest) pend = false;
                } else {
                    const bool ready = pend && l < 64 && (sub == oldest || src_end <= (i64)fs);
                    if (ready) {
                        if (src0 >= 0 && d >= l) {
                            group_copy(out + s, out + src0, l, t);
                        } else {
                            for (u32 i = t; i < l; i += 4) {
                                const i64 qq = src0 + (i64)(d >= l ? i : i % d);
                                out[s + i] = qq >= 0 ? out[qq] : dict_end[qq];
                            }
                        }
                        pend = false;
                    }
                }
                __syncwarp();
                pmask = __ballot_sync(SWC_FULL, pend && t == 0);
            }
        }
        __syncwarp();                                                 // the stage is rewritten for the next group
    }
}

// exclusive prefix sum of per-unit record capacities (in_len / 3 + 2), one block
__global__ void __launch_bounds__(1024) lz4_rec_scan_kernel(const u64 *blk_len, u64 n, u64 *base) {
    __shared__ u64 part[1][1024];
    u64 b, e;
    cta_unit_run(n, b, e);
    u64 sum = 0;
    for (u64 i = b; i < e; i++) sum += (blk_len[i] & ~(1ull << 63)) / 3 + 2;
    part[0][threadIdx.x] = sum;
    cta_scan<1>(part);
    u64 run = part[0][threadIdx.x] - sum;
    for (u64 i = b; i < e; i++) { base[i] = run; run += (blk_len[i] & ~(1ull << 63)) / 3 + 2; }
}


size_t two_phase_scratch_bytes(u64 n, u64 in_total) {
    return (size_t)(n * 8 + n * 4 + (in_total / 3 + 2 * n + 16) * 8 + 1024);
}

__global__ void __launch_bounds__(256) lz4_block_kernel(Args a) { lz4_block_body<false>(a); }
__global__ void __launch_bounds__(256) lz4_fallback_kernel(Args a) { lz4_block_body<true>(a); }

int launch_parse(const Args &a, const u64 *rec_base, u64 *recs, u32 *rec_count, cudaStream_t stream) {
    lz4_parse_kernel<<<(unsigned)((a.n + 127) / 128), 128, 0, stream>>>(a, rec_base, recs, rec_count);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

int launch_exec(const Args &a, const u64 *rec_base, const u64 *recs, const u32 *rec_count, cudaStream_t stream) {
    lz4_exec_kernel<<<(unsigned)((a.n * 32 + 255) / 256), 256, 0, stream>>>(a, rec_base, recs, rec_count);
    timing_mark(stream);
    lz4_fallback_kernel<<<(unsigned)((a.n * 32 + 255) / 256), 256, 0, stream>>>(a);
    count_launch(2);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

int launch(const Args &a, cudaStream_t stream) {
    if (a.n == 0) return SWC_OK;
    if (a.first_blk == nullptr && a.scratch != nullptr) {
        u64 *base = (u64 *)a.scratch;
        u32 *cnt = (u32 *)(base + a.n);
        u64 *recs = (u64 *)(((uintptr_t)(cnt + a.n) + 255) & ~(uintptr_t)255);
        timing_mark(stream);
        lz4_rec_scan_kernel<<<1, 1024, 0, stream>>>(a.in_len, a.n, base);
        count_launch();
        if (int st = launch_parse(a, base, recs, cnt, stream)) return st;
        timing_mark(stream);
        return launch_exec(a, base, recs, cnt, stream);
    }
    const u64 g = (a.n * 32 + 255) / 256;
    lz4_block_kernel<<<(unsigned)g, 256, 0, stream>>>(a);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace lz4
}  // namespace swc
