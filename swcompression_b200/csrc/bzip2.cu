// bzip2.cu — batched BZip2 stream decode for sm_90a.  Replaces BZip2.decompress(_: MsbBitReader)
// (reference Sources/BZip2/BZip2.swift:50-270), BurrowsWheeler.reverse (BurrowsWheeler.swift:29-64) and
// CheckSums.bzip2crc32 (Sources/Common/CheckSums.swift:30-37).
//
// ONE WARP PER UNIT (one .bz2 stream).  The warp executes the bit-serial parts in lock-step (every lane holds the same
// bit buffer, so control flow is uniform) and uses its 32 lanes where the format allows it:
//   - the compressed stream is fetched 128 B at a time (one coalesced load, double-buffered), words handed out by shuffle;
//   - Huffman code length = 1 + popc(ballot(code >= limit[lane])): 20 comparisons in one instruction;
//   - the 256-entry move-to-front list lives in registers, 8 bytes per lane, and is rotated with one shuffle;
//   - RUNA/RUNB runs are filled by all lanes; MTF output goes through a 128-byte shared staging line;
//   - inverse BWT: per-byte histogram -> stable scatter builds the successor array, then the n-step pointer chase is split
//     over the 32 lanes with the splitter (sparse-ruler) list-ranking trick; RLE1 undo + block CRC run on lane 0.
#include <cstdio>
#include "common.cuh"
#include "bzip2.cuh"
#include "host_util.h"

namespace swc {
namespace bzip2 {

constexpr int WARPS = 4;
constexpr int MAX_SYMS = 258;
constexpr int MAX_LEN = 20;
constexpr int NCH = 4;           // chains a lane keeps in flight in the chase (8 measured slower: one warp is issue-latency-bound on the bookkeeping)
constexpr int NSEG = 512;        // chain pieces of the inverse BWT (see the chase)

// Room for a block's BWT text (the RLE1 form) when the unit may write `cap` output bytes.  RLE1 turns every run of four
// equal bytes into five, so a block that fits `cap` bytes of output can carry up to 5/4 x cap + 4 bytes of text; sizing the
// text by `cap` alone reported overflow for units whose output fits exactly.
__host__ __device__ __forceinline__ u64 bwt_capacity(u64 cap) { return (cap + (cap >> 2) + 8 + 3) & ~3ull; }

struct WarpSmem {
    u16 syms[6][MAX_SYMS + 2];      // symbols sorted by (length, symbol) per table
    u32 limit[6][32];               // limit[t][L-1] = left-justified (20-bit) end of the length-L code range; [20..31] = 1<<20
    u32 base[6][MAX_LEN + 2];       // first left-justified code of length L
    u16 first[6][MAX_LEN + 2];      // index of the first symbol of length L
    u8 lens[MAX_SYMS + 2];
    u8 used[256];
    u32 counts[256];
    u32 stage[32];                  // 128-byte output staging line
    u32 split_next[32], split_len[32];
};

__constant__ u32 c_bzcrc[256];      // filled by the host at first launch

// ---------------------------------------------------------------- MSB-first bit reader, warp-uniform
struct Bits {
    const u8 *base;      // 128-byte aligned chunk base pointer arithmetic is done on (in_base + in_off) & ~127
    u64 first_chunk;     // absolute chunk index of cur
    u64 end_byte;        // absolute address one past the unit's last byte
    u32 cur, nxt;        // this lane's word of the current / next 128-byte chunk (raw little-endian load)
    int k;               // next word index in cur (0..31)
    u64 bb;              // left-justified bit buffer
    int bc;
    i64 avail;
    const u32 *chunkp;   // address of the NEXT chunk to prefetch

    __device__ __forceinline__ u32 load_chunk() {
        const u32 *p = chunkp + lane_id();
        chunkp += 32;
        return ((u64)(uintptr_t)p < end_byte) ? __ldg(p) : 0u;
    }
    __device__ void init(const u8 *p, u64 len) {
        uintptr_t a = (uintptr_t)p;
        end_byte = (u64)a + len;
        chunkp = (const u32 *)(a & ~(uintptr_t)127);
        cur = load_chunk();
        nxt = load_chunk();
        k = (int)((a & 127) >> 2);
        bb = 0; bc = 0;
        avail = (i64)len * 8;
        refill();
        const int drop = (int)(a & 3) * 8;
        bb <<= drop; bc -= drop;
        need32();
    }
    __device__ __forceinline__ void refill() {           // requires bc <= 32
        u32 w = __shfl_sync(SWC_FULL, cur, k);
        w = __byte_perm(w, 0, 0x0123);                   // big-endian: first byte in memory = most significant
        bb |= (u64)w << (32 - bc);
        bc += 32;
        if (++k == 32) { cur = nxt; nxt = load_chunk(); k = 0; }
    }
    __device__ __forceinline__ void need32() { if (bc <= 32) refill(); }
    __device__ __forceinline__ u32 peek(int n) const { return n ? (u32)(bb >> (64 - n)) : 0; }
    __device__ __forceinline__ void skip(int n) { bb <<= n; bc -= n; avail -= n; }
    __device__ __forceinline__ u32 get(int n) { need32(); u32 v = peek(n); skip(n); return v; }   // n <= 32
};

// ---------------------------------------------------------------- register-resident MTF list (8 bytes per lane)
__device__ __forceinline__ u32 mtf_front(u64 v) { return (u32)__shfl_sync(SWC_FULL, (u32)v, 0) & 0xFF; }
// move element at index i (0..255) to the front; returns it
// (the result is only meaningful on lane 0 when i < 8 — BwtOut::put() stores from lane 0; the general path returns it everywhere)
__device__ __forceinline__ u32 mtf_move(u64 &v, u32 i) {
    const u32 lane = lane_id();
    if (i < 8) {                                      // warp-uniform; ~2/3 of all symbols: the whole move stays inside lane 0's word
        const u32 sh = i * 8;
        const u64 e = (v >> sh) & 0xFF;
        if (lane == 0) {
            const u64 below = v & ((1ull << sh) - 1);                     // bytes 0..i-1
            const u64 above = sh == 56 ? 0ull : (v >> (sh + 8)) << (sh + 8);
            v = above | (below << 8) | e;
        }
        return (u32)e;
    }
    const u32 q = i >> 3, r = i & 7;
    const u32 lo = (u32)v, hi = (u32)(v >> 32);
    const u32 src = r < 4 ? __shfl_sync(SWC_FULL, lo, q) : __shfl_sync(SWC_FULL, hi, q);
    const u32 e = (src >> ((r & 3) * 8)) & 0xFF;
    const u32 prev_top = __shfl_up_sync(SWC_FULL, hi, 1) >> 24;          // byte 7 of the previous lane
    const u64 carry = lane == 0 ? (u64)e : (u64)prev_top;
    if (lane < q) {
        v = (v << 8) | carry;
    } else if (lane == q) {
        const u64 keep_mask = r == 7 ? 0ull : (~0ull << ((r + 1) * 8));  // bytes above r stay
        const u64 low = (v << 8) | carry;                                 // bytes 0..r shifted up by one
        v = (v & keep_mask) | (low & ~keep_mask);
    }
    return e;
}

// ---------------------------------------------------------------- output of the MTF stage (BWT bytes) via staging line
struct BwtOut {
    u8 *bwt; u64 cap; u64 n; u32 fill;   // fill = bytes in the staging line
    WarpSmem *S;
    __device__ __forceinline__ void flush() {
        if (fill) {
            __syncwarp();
            const u32 lane = lane_id();
            u64 pos = n - fill;                       // staging line always starts 4-byte aligned in bwt (n-fill % 4 == 0)
            if (lane * 4 < fill && pos + lane * 4 + 4 <= cap + 3) *(u32 *)(bwt + pos + lane * 4) = S->stage[lane];
            __syncwarp();
            fill = 0;
        }
    }
    __device__ __forceinline__ void put(u32 byte) {
        if (lane_id() == 0) ((u8 *)S->stage)[fill] = (u8)byte;
        fill++; n++;
        if (fill == 128) flush();
    }
    __device__ void run(u32 byte, u64 count) {
        // top the staging line up to a 4-byte boundary, flush, then fill wide
        while (count && (fill & 3)) { put(byte); count--; }
        if (count >= 4) {                     // fill is a multiple of 4 here, so the flush keeps n word-aligned
            flush();
            const u32 lane = lane_id();
            const u32 w = byte * 0x01010101u;
            u64 words = count >> 2;
            if (n + count <= cap) for (u64 i = lane; i < words; i += 32) *(u32 *)(bwt + n + i * 4) = w;
            n += words * 4;
            count -= words * 4;
            __syncwarp();
        }
        while (count) { put(byte); count--; }
    }
};

// ---- GF(2) helpers for the MSB-first CRC-32 (poly 0x04C11DB7): crc(A||B) = crc(A) * x^(8|B|) + crc(B) for conditioned values
__device__ __forceinline__ u32 mulmod_bz(u32 a, u32 b) {
    u32 p = 0;
    while (a) {
        if (a & 1) p ^= b;
        a >>= 1;
        b = (b & 0x80000000u) ? (b << 1) ^ 0x04C11DB7u : b << 1;
    }
    return p;
}
__device__ __forceinline__ u32 xpow_bz(u64 nbytes) {
    u32 p = 1, sq = 1u << 8;
    while (nbytes) { if (nbytes & 1) p = mulmod_bz(sq, p); sq = mulmod_bz(sq, sq); nbytes >>= 1; }
    return p;
}

// ---------------------------------------------------------------- the kernel
__global__ void __launch_bounds__(WARPS * 32) bzip2_kernel(Args a) {
    __shared__ WarpSmem smem[WARPS];
    const u32 lane = lane_id(), warp = threadIdx.x >> 5;
    const u64 unit = (u64)blockIdx.x * WARPS + warp;
    if (unit >= a.n) return;
    WarpSmem &S = smem[warp];
    const u64 cap = a.out_cap[unit];
    u8 *out = a.out_base + a.out_off[unit];
    // per-unit scratch: bwt bytes [scr_cap] | successor array u32 [scr_cap] | selectors u8 [32768]
    const u64 scr_cap = bwt_capacity(cap);
    u8 *scr = a.scratch + a.scr_off[unit];
    u8 *bwt = scr;
    u32 *succ = (u32 *)(scr + scr_cap + 16);
    u8 *selectors = (u8 *)(succ + scr_cap) + 16;

    Bits br;
    br.init(a.in_base + a.in_off[unit], a.in_len[unit]);
    const i64 total_bits = br.avail;
    int status = SWC_OK;
    u64 op = 0;
    u32 total_crc = 0;
#define FAIL(c) do { status = (c); goto done; } while (0)

    // block mode (host-side block discovery, api_bzip2.cu): the unit is ONE block that starts `start_bits` bits into its
    // first byte, at its 48-bit magic; the stream header is not here and decoding stops after this block
    const bool block_mode = a.block_mode != 0;
    if (block_mode) {
        const u32 sb = a.start_bits ? a.start_bits[unit] : 0;
        if (br.avail < (i64)sb) FAIL(SWC_BZIP2_WRONG_MAGIC);
        if (sb) (void)br.get((int)sb);
    } else {
        if (br.avail < 32) FAIL(SWC_BZIP2_WRONG_MAGIC);                                  // BZip2.swift:53
        if (br.get(16) != 0x425A) FAIL(SWC_BZIP2_WRONG_MAGIC);                           // 'B','Z' (uint16() == 0x5a42 LE)
        if (br.get(8) != 104) FAIL(SWC_BZIP2_WRONG_VERSION);
        { u32 bs = br.get(8); if (bs < 0x31 || bs > 0x39) FAIL(SWC_BZIP2_WRONG_BLOCK_SIZE); }
    }

    for (bool first = true;; first = false) {
        if (block_mode && !first) break;                                             // exactly one block
        if (br.avail < 80) FAIL(SWC_BZIP2_WRONG_MAGIC);                              // :71
        const u64 magic = ((u64)br.get(24) << 24) | br.get(24);
        const u32 block_crc = br.get(32);
        if (magic == 0x177245385090ull) {
            if (total_crc != block_crc) FAIL(SWC_BZIP2_WRONG_CRC);                   // :86
            break;
        }
        if (magic != 0x314159265359ull) FAIL(SWC_BZIP2_WRONG_BLOCK_TYPE);

        // ------------------------------------------------ decode(_:_:) BZip2.swift:97-270
        if (br.avail < 41) FAIL(SWC_BZIP2_WRONG_MAGIC);
        if (br.get(1) != 0) FAIL(SWC_BZIP2_RANDOMIZED_BLOCK);
        const u32 orig_ptr = br.get(24);
        const u32 used_map = br.get(16);
        if (br.avail < (i64)(16 * __popc(used_map) + 18)) FAIL(SWC_BZIP2_WRONG_MAGIC);
        int nused = 0;
        for (int blk = 0; blk < 16; blk++) {
            if (used_map & (0x8000u >> blk)) {
                const u32 m = br.get(16);
                if (lane == 0) for (int s = 0; s < 16; s++) if (m & (0x8000u >> s)) S.used[nused + __popc(m >> (16 - s))] = (u8)(blk * 16 + s);
                nused += __popc(m);
            }
        }
        __syncwarp();
        const int used_count = nused + 2;
        u64 mtf = 0;                                  // lane l holds list entries 8l..8l+7
        for (int k = 0; k < 8; k++) { int idx = lane * 8 + k; if (idx < nused) mtf |= (u64)S.used[idx] << (8 * k); }
        const int ntab = (int)br.get(3);
        if (ntab < 2 || ntab > 6) FAIL(SWC_BZIP2_WRONG_HUFFMAN_GROUPS);
        const int nsel = (int)br.get(15);
        {                                             // selectors :155-173 (MTF over table indices, in a register)
            u32 tm = 0x543210;                        // nibble k = table index at MTF position k
            for (int i = 0; i < nsel; i++) {
                int c = 0;
                while (br.avail > 0) { u32 b = br.get(1); if (b == 0) break; c++; }
                if (c >= ntab) FAIL(SWC_BZIP2_WRONG_SELECTOR);
                const u32 el = (tm >> (4 * c)) & 0xF;
                const u32 below = tm & ((1u << (4 * c)) - 1);
                tm = (tm & ~((1u << (4 * (c + 1))) - 1)) | (below << 4) | el;
                if (lane == 0) selectors[i] = (u8)el;
            }
        }
        bool any_over = false;
        for (int t = 0; t < ntab; t++) {              // code lengths :177-203
            if (br.avail < 5) FAIL(SWC_BZIP2_WRONG_HUFFMAN_CODE_LENGTH);
            int length = (int)br.get(5);
            for (int i = 0; i < used_count; i++) {
                if (length < 0 || length > 20) FAIL(SWC_BZIP2_WRONG_HUFFMAN_CODE_LENGTH);
                while (br.avail > 0) {
                    if (br.get(1) == 0) break;
                    if (br.avail <= 0) FAIL(SWC_BZIP2_WRONG_HUFFMAN_CODE_LENGTH);
                    length -= (int)br.get(1) * 2 - 1;
                }
                if (i == used_count - 1 && length > 20) FAIL(SWC_ERR_REFERENCE_TRAP);   // unbounded tree in the reference
                if (lane == 0) S.lens[i] = (u8)(length < 0 ? 0 : length);
            }
            __syncwarp();
            // canonical tables (Code.huffmanCodes + DecodingTree semantics for Kraft <= 1)
            u32 code = 0, idx = 0;
            bool over = false;
            for (int L = 1; L <= MAX_LEN; L++) {
                if (lane == 0) { S.base[t][L] = code; S.first[t][L] = (u16)idx; }
                for (int s = 0; s < used_count; s++) {
                    if (S.lens[s] == L) {
                        if (code >= (1u << 20)) over = true;
                        if (lane == 0) S.syms[t][idx] = (u16)s;
                        idx++;
                        code += 1u << (20 - L);
                    }
                }
                if (lane == 0) S.limit[t][L - 1] = code > (1u << 20) ? (1u << 20) : code;
            }
            if (lane == 0) for (int L = MAX_LEN; L < 32; L++) S.limit[t][L] = 1u << 20;
            any_over = any_over || over;              // reported after ALL tables are read: a bad length further on comes first in the reference
            __syncwarp();
        }
        if (any_over) FAIL(SWC_ERR_UNSUPPORTED);      // over-subscribed set (heap-overwrite semantics): not taken by this kernel
        __syncwarp();
        if (nsel == 0) FAIL(SWC_ERR_REFERENCE_TRAP);                                 // selectors[0]

#ifdef SWC_BZ_PROFILE
        long long t_hdr = clock64();
#endif
        // ------------------------------------------------ symbol loop :212-246
        BwtOut bo; bo.bwt = bwt; bo.cap = scr_cap; bo.n = 0; bo.fill = 0; bo.S = &S;
        {
            int decoded = 0, sel_idx = 1;
            int table = selectors[0];
            u32 my_limit = S.limit[table][lane];
            const u32 *t_base = S.base[table];
            const u16 *t_first = S.first[table], *t_syms = S.syms[table];
            u64 run_length = 0, repeat_power = 1;
            for (;;) {
                if (decoded >= 50) {
                    if (sel_idx >= nsel) FAIL(SWC_BZIP2_WRONG_SELECTOR);
                    table = selectors[sel_idx++];
                    my_limit = S.limit[table][lane];
                    t_base = S.base[table]; t_first = S.first[table]; t_syms = S.syms[table];
                    decoded = 0;
                }
                br.need32();
                const u32 r20 = br.peek(20);
                const int L = 1 + __popc(__ballot_sync(SWC_FULL, r20 >= my_limit));
                if (L > MAX_LEN || br.avail < L) FAIL(SWC_BZIP2_SYMBOL_NOT_FOUND);
                const u32 sidx = t_first[L] + ((r20 - t_base[L]) >> (20 - L));
                const int symbol = t_syms[sidx];
                br.skip(L);
                decoded++;
                if (symbol < 2) {                                                    // RUNA / RUNB :226-230
                    run_length += repeat_power << symbol;
                    repeat_power <<= 1;
                    continue;
                }
                if (run_length > 0) {
                    if (nused == 0) FAIL(SWC_ERR_REFERENCE_TRAP);
                    if (bo.n + run_length > scr_cap) { bo.n += run_length; FAIL(SWC_ERR_OUTPUT_OVERFLOW); }
                    bo.run(mtf_front(mtf), run_length);
                    run_length = 0; repeat_power = 1;
                }
                if (symbol == used_count - 1) break;                                 // EOB :239
                // capacity: put() only writes the shared staging line and flush() fences global stores, so the test is
                // made once per 128-byte line (and once after the loop) instead of per symbol
                if (bo.fill == 127 && bo.n + 1 > scr_cap) FAIL(SWC_ERR_OUTPUT_OVERFLOW);
                bo.put(mtf_move(mtf, (u32)symbol - 1));                              // :243-245
            }
            if (bo.n > scr_cap) FAIL(SWC_ERR_OUTPUT_OVERFLOW);
            // pad the staging line so the final flush writes whole words
            bo.flush();
        }
        {
#ifdef SWC_BZ_PROFILE
            long long t_dec = clock64();
#endif
            // ------------------------------------------------ BurrowsWheeler.reverse
            const u64 n = bo.n;
            __syncwarp();
            if (n > 0) {
                if (orig_ptr >= n) FAIL(SWC_ERR_REFERENCE_TRAP);
                // histogram (per-lane partial counts folded through shared atomics)
                for (int c = lane; c < 256; c += 32) S.counts[c] = 0;
                __syncwarp();
                for (u64 i = lane; i < n; i += 32) atomicAdd(&S.counts[bwt[i]], 1u);
                __syncwarp();
                // exclusive scan of 256 counters: 8 per lane
                u32 loc[8], sum = 0;
                for (int k = 0; k < 8; k++) { loc[k] = S.counts[lane * 8 + k]; sum += loc[k]; }
                u32 incl = sum;
                for (int d = 1; d < 32; d <<= 1) { u32 v = __shfl_up_sync(SWC_FULL, incl, d); if (lane >= (u32)d) incl += v; }
                u32 run = incl - sum;
                for (int k = 0; k < 8; k++) { S.counts[lane * 8 + k] = run; run += loc[k]; }
                __syncwarp();
                // stable scatter: successor[base[c]++] = i, in increasing i — 32 positions per round, ranked with match_any.
                // Blocks of < 2^20 bytes (every block a bzip2 encoder can produce: <= 900 000) carry bwt[i] in bits 20..27 of
                // the entry, so the chase below needs ONE dependent load per output byte instead of two.
                const bool packed = n < (1u << 20);
                for (u64 i0 = 0; i0 < n; i0 += 32) {
                    const u64 i = i0 + lane;
                    const bool act = i < n;
                    const u32 c = act ? bwt[i] : 0x100 + lane;
                    const u32 peers = __match_any_sync(SWC_FULL, c);
                    const u32 rank = __popc(peers & ((1u << lane) - 1));
                    if (act) succ[S.counts[c] + rank] = (u32)i | (packed ? c << 20 : 0u);   // entry = index i (+ bwt[i] when it fits)
                    __syncwarp();
                    if (act && rank == 0) S.counts[c] += __popc(peers);
                    __syncwarp();
                }
                __syncwarp();
#ifdef SWC_BZ_PROFILE
                long long t_sort = clock64();
#endif
                // ---- pointer chase: list ranking over NSEG splitters, NCH chains in flight per lane ----
                // The inverse BWT is one chain of n dependent loads (the reference walks it serially, BurrowsWheeler.swift:
                // 52-62).  NSEG indices are marked as splitters (index 0 of the list = orig_ptr, the chain's origin); the
                // chain pieces between splitters are independent, so lanes pull them from a queue — walk 1 measures each
                // piece and finds the splitter that ends it, one lane then strings the pieces together from orig_ptr and
                // gives each its output offset, walk 2 follows every piece again and writes its bytes.  Each lane keeps
                // NCH pieces going at once (NCH independent loads in flight).  With 32 fixed pieces (the previous form) the
                // longest piece was ~n/8 and ~6 lanes were busy on average (ncu source view).
                const u32 MARK = 0x80000000u;
                const u32 IDX = packed ? 0xFFFFFu : 0x7FFFFFFFu;
                u32 *seg_len = (u32 *)&S.syms[0][0];                 // the Huffman tables are dead until the next block
                u32 *seg_off = seg_len + NSEG;
                u16 *seg_next = (u16 *)&S.counts[0];                 // so are the bucket counters
                static_assert(sizeof(u32) * 2 * NSEG <= sizeof(S.syms) + sizeof(S.limit) + sizeof(S.base), "segment tables must fit the table area");
                static_assert(sizeof(u16) * NSEG <= sizeof(S.counts), "segment links must fit the counter area");
                const u32 nseg = n < 4096 ? 1u : (u32)NSEG;          // tiny blocks: one chain
                auto seg_start = [&](u32 j) -> u32 { return j == 0 ? orig_ptr : (u32)(((u64)j * n) / nseg); };
                // a regular splitter that coincides with orig_ptr is dropped (piece 0 owns that index); distinct j >= 1 give
                // distinct indices because n >= 4096 > nseg
                for (u32 j = lane; j < nseg; j += 32) {
                    const bool dup = j != 0 && seg_start(j) == orig_ptr;
                    seg_len[j] = dup ? 0xFFFFFFFFu : 0u;             // 0xFFFFFFFF = not a piece
                    seg_off[j] = 0xFFFFFFFFu;                        // not on the path from orig_ptr (yet)
                    seg_next[j] = 0xFFFF;
                    if (!dup) atomicOr(&succ[seg_start(j)], MARK);
                }
                if (lane == 0) S.stage[0] = 0;                       // piece queue head
                __syncwarp();
                __threadfence_block();
                auto end_to_seg = [&](u32 e) -> u32 {                // which piece starts at index e (e is a marked index)
                    if (e == orig_ptr) return 0;
                    const u32 j = (u32)(((u64)e * nseg + n - 1) / n);
                    return (j < nseg && seg_start(j) == e) ? j : 0xFFFFu;
                };
                // walk 1: piece lengths and links
                {
                    u32 id[NCH], cur[NCH], k[NCH];
#pragma unroll
                    for (int q = 0; q < NCH; q++) id[q] = 0xFFFFFFFEu; // needs a piece
                    bool more = true;
                    for (;;) {
                        bool any = false;
#pragma unroll
                        for (int q = 0; q < NCH; q++) {
                            while (id[q] == 0xFFFFFFFEu && more) {   // pull the next real piece
                                const u32 j = atomicAdd(&S.stage[0], 1u);
                                if (j >= nseg) { more = false; break; }
                                if (seg_len[j] != 0xFFFFFFFFu) { id[q] = j; cur[q] = seg_start(j); k[q] = 0; }
                            }
                            if (id[q] == 0xFFFFFFFEu) id[q] = 0xFFFFFFFFu;   // nothing left for this slot
                            any |= id[q] != 0xFFFFFFFFu;
                        }
                        if (!__any_sync(SWC_FULL, any)) break;     // vote-driven: the lanes stay converged
                        u32 v[NCH];
#pragma unroll
                        for (int q = 0; q < NCH; q++) v[q] = id[q] != 0xFFFFFFFFu ? succ[cur[q]] : 0u;
#pragma unroll
                        for (int q = 0; q < NCH; q++) {
                            if (id[q] == 0xFFFFFFFFu) continue;
                            if ((k[q] > 0 && (v[q] & MARK)) || k[q] >= n) {          // cur is the next splitter: piece complete
                                seg_len[id[q]] = k[q];
                                seg_next[id[q]] = (u16)end_to_seg(cur[q]);
                                id[q] = 0xFFFFFFFEu;
                            } else {
                                cur[q] = v[q] & IDX; k[q]++;
                            }
                        }
                    }
                }
                __syncwarp();
                // string the pieces together from orig_ptr (the path is a cycle of length C <= n; when C < n the output wraps)
                u64 cycle = 0;
                if (lane == 0) {
                    u32 j = 0; u64 off = 0;
                    for (u32 step = 0; step < nseg; step++) {
                        seg_off[j] = (u32)off;
                        off += seg_len[j];
                        const u32 nx = seg_next[j];
                        if (nx == 0 || nx >= nseg || seg_off[nx] != 0xFFFFFFFFu) break;
                        j = nx;
                    }
                    cycle = off;
                    S.stage[0] = 0;
                }
                cycle = __shfl_sync(SWC_FULL, cycle, 0);
                __syncwarp();
                // walk 2: emit.  The low half of the scratch after the successor array holds the text (RLE1 still has to
                // expand it): text = selectors + 32768 + 16.
                u8 *text = selectors + 32768 + 16;
                if (cycle > 0) {
                    u32 id[NCH], cur[NCH], k[NCH], len[NCH], off[NCH];
#pragma unroll
                    for (int q = 0; q < NCH; q++) id[q] = 0xFFFFFFFEu;
                    bool more = true;
                    for (;;) {
                        bool any = false;
#pragma unroll
                        for (int q = 0; q < NCH; q++) {
                            while (id[q] == 0xFFFFFFFEu && more) {
                                const u32 j = atomicAdd(&S.stage[0], 1u);
                                if (j >= nseg) { more = false; break; }
                                if (seg_len[j] != 0xFFFFFFFFu && seg_off[j] != 0xFFFFFFFFu && seg_len[j] != 0) {
                                    id[q] = j; cur[q] = seg_start(j); k[q] = 0; len[q] = seg_len[j]; off[q] = seg_off[j];
                                }
                            }
                            if (id[q] == 0xFFFFFFFEu) id[q] = 0xFFFFFFFFu;
                            any |= id[q] != 0xFFFFFFFFu;
                        }
                        if (!__any_sync(SWC_FULL, any)) break;     // vote-driven: the lanes stay converged
                        u32 v[NCH];
#pragma unroll
                        for (int q = 0; q < NCH; q++) v[q] = id[q] != 0xFFFFFFFFu ? succ[cur[q]] : 0u;
#pragma unroll
                        for (int q = 0; q < NCH; q++) {
                            if (id[q] == 0xFFFFFFFFu) continue;
                            cur[q] = v[q] & IDX;
                            const u8 ch = packed ? (u8)(v[q] >> 20) : bwt[cur[q]];
                            for (u64 pos = (u64)off[q] + k[q]; pos < n; pos += cycle) text[pos] = ch;
                            if (++k[q] == len[q]) id[q] = 0xFFFFFFFEu;
                        }
                    }
                }
                __syncwarp();
#ifdef SWC_BZ_PROFILE
                long long t_chase = clock64();
#endif
                // ------------------------------------------------ RLE1 undo :251-267, 32 text bytes per step
                // The reference walks i one byte at a time and, when text[i..i+3] are equal (and i < n-4), expands a run
                // and jumps 5 bytes.  Every step here starts at such a "fresh" position i: lane j tests whether a run would
                // start at i+j; all positions before the first run start are plain literals, so they are emitted together.
                u64 bop = op;
                {
                    u64 i = 0;
                    while (i < n) {
                        const u64 q = i + lane;
                        u32 b0 = 0; bool runs = false;
                        if (q < n) {
                            b0 = text[q];
                            if (n >= 5 && q < n - 4) runs = text[q + 1] == b0 && text[q + 2] == b0 && text[q + 3] == b0;
                        }
                        const u32 m = __ballot_sync(SWC_FULL, runs);
                        const u32 lits = m ? (u32)(__ffs(m) - 1) : (u32)(n - i < 32 ? n - i : 32);
                        if (lane < lits && bop + lane < cap) out[bop + lane] = (u8)b0;
                        bop += lits;
                        if (m) {
                            const u32 js = lits;
                            const u32 c0 = __shfl_sync(SWC_FULL, b0, js);
                            const u32 runl = (u32)text[i + js + 4] + 4;
                            for (u32 k = lane; k < runl; k += 32) if (bop + k < cap) out[bop + k] = (u8)c0;
                            bop += runl;
                            i += js + 5;
                        } else {
                            i += lits;
                        }
                    }
                }
                __syncwarp();
                // ------------------------------------------------ block CRC (CheckSums.swift:30-37), 32 segments + GF(2) combine
                u32 crc = 0;
                if (bop <= cap) {
                    for (int c = lane; c < 256; c += 32) S.counts[c] = c_bzcrc[c];
                    __syncwarp();
                    const u64 len = bop - op;
                    const u64 seg = (len + 31) / 32;
                    const u64 sb = lane * seg < len ? lane * seg : len, se = sb + seg < len ? sb + seg : len;
                    u32 part = 0xFFFFFFFFu;
                    const u8 *pdat = out + op;
                    for (u64 k = sb; k < se; k++) part = (part << 8) ^ S.counts[((part >> 24) ^ pdat[k]) & 0xFF];
                    part = ~part;
                    const u32 pw_full = xpow_bz(seg);
                    u32 acc = __shfl_sync(SWC_FULL, part, 0);
                    for (int l = 1; l < 32; l++) {
                        const u32 pl = __shfl_sync(SWC_FULL, part, l);
                        const u64 lb = (u64)l * seg < len ? (u64)l * seg : len, le = lb + seg < len ? lb + seg : len;
                        const u64 ll = le - lb;
                        if (ll == 0) continue;
                        acc = mulmod_bz(ll == seg ? pw_full : xpow_bz(ll), acc) ^ pl;
                    }
                    crc = acc;
                }
                op = bop;
#ifdef SWC_BZ_PROFILE
                if (unit == 0 && lane == 0) printf("bz2 block n=%llu: decode %lld  hist+scatter %lld  chase %lld  rle+crc %lld cycles\n", (unsigned long long)n, t_dec - t_hdr, t_sort - t_dec, t_chase - t_sort, clock64() - t_chase);
#endif
                if (op > cap) FAIL(SWC_ERR_OUTPUT_OVERFLOW);
                if (crc != block_crc) FAIL(SWC_BZIP2_WRONG_CRC);                         // :81 (payload includes this block)
            } else {
                if (block_crc != 0) FAIL(SWC_BZIP2_WRONG_CRC);                           // crc of the empty block is 0
            }
        }
        total_crc = ((total_crc << 1) | (total_crc >> 31)) ^ block_crc;                  // :83-84
    }
done:
#undef FAIL
    if (lane == 0) {
        a.out_len[unit] = op;
        a.consumed_bits[unit] = (u64)(total_bits - br.avail);
        a.status[unit] = status;
    }
}

size_t scratch_per_unit(u64 cap) {
    const u64 scr_cap = bwt_capacity(cap);
    // bwt | succ (u32) | selectors | text
    return (size_t)(scr_cap + 16 + scr_cap * 4 + 16 + 32768 + 16 + scr_cap + 256 + 255) & ~(size_t)255;
}

int launch(const Args &a, cudaStream_t stream) {
    if (a.n == 0) return SWC_OK;
    int st = configure_once(CFG_BZIP2_CRC, [](DeviceCtx &) {          // __constant__ memory is per device
        u32 tab[256];
        for (u32 i = 0; i < 256; i++) { u32 c = i << 24; for (int k = 0; k < 8; k++) c = (c & 0x80000000u) ? (c << 1) ^ 0x04C11DB7u : c << 1; tab[i] = c; }
        SWC_CUDA_TRY(cudaMemcpyToSymbol(c_bzcrc, tab, sizeof(tab)));
        return (int)SWC_OK;
    });
    if (st) return st;
    bzip2_kernel<<<(unsigned)((a.n + WARPS - 1) / WARPS), WARPS * 32, 0, stream>>>(a);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace bzip2
}  // namespace swc
