// inflate_warp.cu — K1w: Deflate Huffman stage, ONE WARP PER UNIT with speculative sub-stream decoding.
// Literals go to a packed stream, matches become records for lz_resolve_kernel (format in inflate.cuh),
// every reference error / trap case is reproduced (Deflate.swift:30-249).
//
// Why: with one thread per stream every lane needs private decode tables (536 B) and ~10 issue slots per symbol.  With
// one warp per stream the tables are shared, so a flat 2^11-entry lit/len LUT + 2^9-entry distance LUT fit in shared
// memory (one LDS per symbol), and the 32 lanes decode DIFFERENT 288-bit windows of the SAME block concurrently:
//   chunk = 32 windows.  Lane 0 starts at the known symbol boundary; lanes 1..31 guess their window start.
//   pass A (repeat until nothing changes): each lane whose start changed decodes its window and reports where its last
//          symbol ended (= the next lane's true start), plus byte / literal / record counts.  Huffman streams self-synchronise
//          within a few symbols, so a wrong start almost always yields the right end: typically 2 rounds.
//   scan : exclusive prefix sums of bytes, literals and records over the valid lanes give every lane its offsets.
//   pass B: every lane decodes its window once more from the now-proven start and emits literals + records.
// Block headers (code lengths, table build) and stored blocks are handled warp-uniformly / cooperatively.
// Code sets with Kraft sum > 1 are routed to inflate_slow_kernel exactly like in K1L.
#include "common.cuh"
#include "deflate_header.cuh"
#include "inflate.cuh"
#include "host_util.h"

namespace swc {
namespace inflate {

namespace w {

constexpr int WIN_WORDS = 19;                // window per lane in 32-bit words; odd stride = conflict-free initial reads
constexpr int WIN_BITS = WIN_WORDS * 32;
constexpr int STAGE_WORDS = 32 * WIN_WORDS + 8;
constexpr int LIT_BITS = 11, DST_BITS = 9;
constexpr int WARPS = 4;

// LUT entry: [3:0] code length (0 = no code) | [5:4] kind | [9:6] extra bits | [31:16] value
//   lit/len kinds: 0 literal (value = byte), 1 end of block, 2 length (value = base), 3 invalid symbol 286/287
//   special: length field 15 with kind... long codes are flagged by bit 10 (SLOW): decode with the canonical tables
constexpr u32 E_SLOW = 1u << 10;

struct Smem {
    u32 lit_lut[1 << LIT_BITS];
    u32 dst_lut[1 << DST_BITS];
    u32 stage[STAGE_WORDS];
    u16 lit_sym[288];            // canonical order (slow path + LUT construction)
    u8 dst_sym[32];
    u32 lit_bo[16], dst_bo[16];  // first left-justified code | first index << 16
    u32 cnt[2][16];
    u8 lens[320];
    u8 cl_lut[128];              // code-length alphabet: sym << 3 | len (0 = no code)
};

// ---- warp-uniform view of the unit's bitstream and the position of the true chain (header parsing reads it directly) ----
struct Stream {
    const u32 *wbase;     // 4-byte aligned word containing the unit's first byte
    u64 bit0;             // bit offset of the unit's first bit inside wbase (0..31+7)
    u64 total;            // unit length in bits counted from bit0 (the reference's initial bitsLeft)
    u64 nwords;           // words that may be read
    u64 pos;              // bits consumed from the unit start
    __device__ __forceinline__ u32 word(u64 i) const { return i < nwords ? __ldg(wbase + i) : 0u; }
    __device__ __forceinline__ u32 peek32() const {
        const u64 q = pos + bit0;
        const u64 wi = q >> 5;
        return __funnelshift_r(word(wi), word(wi + 1), (u32)(q & 31));
    }
    __device__ __forceinline__ void skip(int n) { pos += n; }
    __device__ __forceinline__ i64 avail() const { return (i64)(total - pos); }
};

// ---- per-lane bit cursor over the shared staging buffer ----
struct Cursor {
    u64 bb; int bc; u32 widx;
    __device__ __forceinline__ void init(const u32 *stage, u32 rel_bit) {      // rel_bit: bit offset inside stage
        const u32 wi = rel_bit >> 5, off = rel_bit & 31;
        bb = ((u64)stage[wi] | ((u64)stage[wi + 1] << 32)) >> off;
        bc = 64 - (int)off;
        widx = wi + 2;
    }
    __device__ __forceinline__ void need(const u32 *stage) {
        if (bc <= 32) { bb |= (u64)stage[widx < STAGE_WORDS ? widx : STAGE_WORDS - 1] << bc; bc += 32; widx++; }
    }
    __device__ __forceinline__ u32 peek(int n) const { return (u32)bb & ((1u << n) - 1); }
    __device__ __forceinline__ void skip(int n) { bb >>= n; bc -= n; }
};

struct Tables {
    Limits lit_lim, dst_lim;
};

// canonical (slow) decode of one symbol from a 15-bit peek; returns symbol or -1, length in L
template <int KIND>
__device__ __forceinline__ int canon_decode(const Smem &S, const Limits &lim, u32 peek15, int &L) {
    const u32 r15 = __brev(peek15) >> 17;
    L = code_length(r15, lim);
    if (L > 15) return -1;
    const u32 idx = canonical_index(r15, L, KIND == 0 ? S.lit_bo[L] : S.dst_bo[L]);
    return KIND == 0 ? (int)S.lit_sym[idx] : (int)S.dst_sym[idx];
}

// Result of decoding one window
struct WinResult {
    u32 end;        // bit position (relative to chunk base) after the last symbol decoded
    u32 nbytes;     // output bytes produced
    u32 nlit;       // literal bytes produced
    u32 nrec;       // records produced EXCLUDING a possible escape in front of the first match
    u32 head;       // literal bytes before the first match (== nbytes when no match)
    u32 tail;       // literal bytes after the last match
    u32 flags;      // bit0 has_match, bit1 eob, bits[31:8] error status (0 = none)
};

// Emission state of one lane in pass B
struct Emit {
    u8 *lits;        // unit literal stream
    u32 *rec;        // end of the unit's scratch region (records grow downward from here)
    u32 cap;
    u32 op;          // next output byte (absolute in unit)
    u32 li;          // next literal index (absolute in unit)
    u32 last_end;    // end of the previous match (absolute), for the literal-run field
    u32 ri;          // next record index (absolute in unit)
    __device__ __forceinline__ void literal(u32 byte) {
        if (op < cap) lits[li] = (u8)byte;
        li++;
        op++;
    }
    __device__ __forceinline__ void match(u32 len, u32 dist) {
        const u32 nop = op + len;
        if (nop <= cap) put_match(rec, ri, op - last_end, len, dist);
        last_end = nop;
        op = nop;
    }
};

// One match: length extra bits + distance symbol + distance extra bits (Deflate.swift:186-232). Returns an error or 0.
constexpr int KW_LIT = 4;               // lit/len steps per round before pending matches are serviced

template <bool EMIT>
__device__ __forceinline__ int window_match(const Smem &S, const Tables &T, const u32 *lens_tab, Cursor &c, u32 &p, u64 left,
                                            u32 value, int eb, Emit *em, u32 &length_out) {
    if ((u64)p + (u32)eb > left) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
    const u32 length = value + c.peek(eb);
    c.skip(eb); p += (u32)eb;
    c.need(S.stage);
    const u32 d = S.dst_lut[c.peek(DST_BITS)];
    int DL = (int)(d & 15);
    u32 dbase = d >> 16;
    int db = (int)((d >> 6) & 15);
    bool dbad = ((d >> 4) & 3) == 3;
    if (d & E_SLOW) {
        const int ds = canon_decode<1>(S, T.dst_lim, c.peek(15), DL);
        if (ds < 0) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
        dbad = ds > 29;
        const u32 de = lens_tab[32 + (ds & 31)];
        dbase = de & 0xFFFFu; db = (int)(de >> 16);
    }
    if ((u64)p + (u32)DL > left) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
    c.skip(DL); p += (u32)DL;
    if (dbad) return SWC_DEFLATE_WRONG_SYMBOL;
    if ((u64)p + (u32)db > left) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
    const u32 dist = dbase + c.peek(db);
    c.skip(db); p += (u32)db;
    if (EMIT) {
        if (dist > em->op) return SWC_ERR_REFERENCE_TRAP;                  // Deflate.swift:219 negative array index
        if ((u64)em->op + length > OUT_MAX) return SWC_ERR_UNSUPPORTED;
        em->match(length, dist);
    }
    length_out = length;
    return 0;
}

// Decode the window [start, hi) (bit offsets relative to the chunk base; symbols START below hi).
// EMIT=false: count only (pass A).  EMIT=true: also write literals / records through `em` (pass B).
// Called by ALL lanes (enable selects the working ones): the loop is driven by a warp vote so the lanes stay converged.
template <bool EMIT>
__device__ __forceinline__ WinResult decode_window(const Smem &S, const Tables &T, const u32 *lens_tab, bool enable, u32 start, u32 hi,
                                                  u64 left, u32 stage_bit0, Emit *em, WinResult prev) {
    WinResult r = prev;
    Cursor c; c.bb = 0; c.bc = 0; c.widx = 0;
    u32 p = start, run = 0;
    bool has_match = false;
    int err = 0;
    bool eob = false;
    bool active = enable;
    if (enable) { r.nbytes = 0; r.nlit = 0; r.nrec = 0; r.head = 0; r.tail = 0; r.flags = 0; c.init(S.stage, start + stage_bit0); }
    // A round = up to KW_LIT lit/len symbols per lane, then ONE pass of the (long, rare) match path for every lane that
    // parked a length symbol — the same scheme as K1L's parked phase (inflate_lut.cu): the match path used to run inside
    // every step with ~4 of 32 lanes (22 % of the issued instructions, ncu source view).
    bool pend = false;
    u32 pvalue = 0; int peb = 0;
    while (__any_sync(SWC_FULL, active)) {
#pragma unroll 1
        for (int k = 0; k < KW_LIT; k++) {
            if (active && !pend) {
                c.need(S.stage);
                const u32 e = S.lit_lut[c.peek(LIT_BITS)];
                int L = (int)(e & 15);
                int kind = (int)((e >> 4) & 3);
                u32 value = e >> 16;
                int eb = (int)((e >> 6) & 15);
                if (e & E_SLOW) {
                    const int sym = canon_decode<0>(S, T.lit_lim, c.peek(15), L);
                    if (sym < 0) err = SWC_DEFLATE_SYMBOL_NOT_FOUND;
                    else if (sym < 256) { kind = 0; value = (u32)sym; eb = 0; }
                    else if (sym == 256) { kind = 1; eb = 0; }
                    else if (sym > 285) { kind = 3; }
                    else { kind = 2; const u32 le = lens_tab[sym - 257]; value = le & 0xFFFFu; eb = (int)(le >> 16); }
                }
                if (!err && (u64)p + (u32)L > left) err = SWC_DEFLATE_SYMBOL_NOT_FOUND;
                if (!err) {
                    c.skip(L); p += (u32)L;
                    if (kind == 0) {
                        if (EMIT) em->literal(value);
                        r.nbytes++; r.nlit++; run++;
                    } else if (kind == 1) {
                        eob = true;
                    } else if (kind == 3) {
                        err = SWC_DEFLATE_WRONG_SYMBOL;
                    } else {
                        pend = true; pvalue = value; peb = eb;
                    }
                }
                if (err || eob || (!pend && p >= hi)) active = false;
            }
        }
        if (active && pend) {
            u32 length = 0;
            err = window_match<EMIT>(S, T, lens_tab, c, p, left, pvalue, peb, em, length);
            if (!err) {
                if (!has_match) { r.head = run; has_match = true; }
                else if (run > 255) r.nrec++;             // escape record in front of a later match of this window
                r.nrec++;
                r.nbytes += length;
                run = 0;
            }
            pend = false;
            if (err || p >= hi) active = false;
        }
    }
    if (enable) {
        r.end = p;
        r.tail = run;
        if (!has_match) r.head = run;
        r.flags = (has_match ? 1u : 0u) | (eob ? 2u : 0u) | ((u32)err << 8);
    }
    return r;
}

}  // namespace w

using namespace w;

__global__ void __launch_bounds__(WARPS * 32)
inflate_warp_kernel(BatchArgs a) {
    extern __shared__ __align__(16) u8 smem_raw[];
    __shared__ u32 lens_tab[64];
    if (threadIdx.x < 32) { lens_tab[threadIdx.x] = c_len_tab[threadIdx.x]; lens_tab[32 + threadIdx.x] = c_dist_tab[threadIdx.x]; }
    __syncthreads();
    const u32 lane = lane_id(), warp = threadIdx.x >> 5;
    Smem &S = *reinterpret_cast<Smem *>(smem_raw + (size_t)warp * sizeof(Smem));

    for (;;) {
        u64 unit = 0;
        if (lane == 0) unit = atomicAdd(a.ticket, 1ull);
        unit = __shfl_sync(SWC_FULL, (u32)unit, 0) | ((u64)__shfl_sync(SWC_FULL, (u32)(unit >> 32), 0) << 32);
        if (unit >= a.n) break;

        const u64 in_len = a.in_len[unit];
        const u64 cap64 = a.out_cap[unit];
        const u32 cap = cap64 > OUT_MAX ? OUT_MAX : (u32)cap64;
        u8 *lits = (u8 *)(a.rec_base + rec_start(a.out_off[unit]));
        u32 *rec = a.rec_base + rec_start(a.out_off[unit] + cap64);
        const u32 bitskip = a.start_bits ? a.start_bits[unit] : 0;
        int status = SWC_OK;
        u64 op = 0;                  // bytes produced
        u32 nlit = 0;                // literals produced
        u32 nrec = 0;
        u32 run_carry = 0;           // literal bytes since the last match
        Stream st;
        {
            const uintptr_t addr = (uintptr_t)(a.in_base + a.in_off[unit]);
            st.wbase = (const u32 *)(addr & ~(uintptr_t)3);
            st.bit0 = (addr & 3) * 8 + bitskip;
            st.total = in_len * 8 - bitskip;
            st.nwords = ((addr & 3) + in_len + 3) >> 2;
            st.pos = 0;
        }
        Tables T;
#define FAIL(c) do { status = (c); goto unit_done; } while (0)
#define TRY(e) do { status = (e); if (status != SWC_OK) goto unit_done; } while (0)
        if (in_len >= (1ull << 32)) FAIL(SWC_ERR_UNSUPPORTED);
        if (st.total < 10) FAIL(SWC_DEFLATE_WRONG_BLOCK_TYPE);                                   // Deflate.swift:36
        for (;;) {
            // ------------------------------------------------------------ block header (warp-uniform)
            bool is_last;
            u32 btype;
            TRY(hdr::block_start(st, is_last, btype));
            if (btype == 0) {
                u32 length;
                TRY(hdr::stored_length(st, length));
                const u8 *src = (const u8 *)st.wbase + ((st.pos + st.bit0) >> 3);
                if (op + length > OUT_MAX) FAIL(SWC_ERR_UNSUPPORTED);
                if (op + length <= cap) for (u32 i = lane; i < length; i += 32) lits[nlit + i] = src[i];
                op += length; nlit += length; run_carry += length;
                st.pos += (u64)length * 8;
                __syncwarp();
                if (is_last) break;
                continue;
            }
            // ---- code lengths -> S.lens[0..hlit+hdist)
            int hlit = 288, hdist = 32;
            if (btype == 1) {
                hdr::fixed_lengths([&](int n, int len, int reps) { for (int i = lane; i < reps; i += 32) S.lens[n + i] = (u8)len; });
            } else {
                u64 cl;
                TRY(hdr::dynamic_counts(st, hlit, hdist, cl));
                // canonical code of the 19-symbol alphabet -> 7-bit LUT (lane s handles symbol s)
                u32 cnt8[8];
#pragma unroll
                for (int L = 0; L < 8; L++) cnt8[L] = 0;
                for (int s = 0; s < 19; s++) { const u32 l = (u32)(cl >> (3 * s)) & 7;
#pragma unroll
                    for (int L = 1; L < 8; L++) cnt8[L] += (l == (u32)L); }
                u32 first[8]; u32 code = 0, kraft = 0;
#pragma unroll
                for (int L = 1; L < 8; L++) { first[L] = code; code = (code + cnt8[L]) << 1; kraft += cnt8[L] << (7 - L); }
                if (kraft > 128) FAIL(SWC_INTERNAL_NEEDS_SLOW);
                for (int i = lane; i < 128; i += 32) S.cl_lut[i] = 0;
                __syncwarp();
                if (lane < 19) {
                    const u32 l = (u32)(cl >> (3 * lane)) & 7;
                    if (l) {
                        u32 rank = 0;
                        for (int s = 0; s < (int)lane; s++) rank += (((u32)(cl >> (3 * s)) & 7) == l);
                        u32 cdw = 0;
#pragma unroll
                        for (int L = 1; L < 8; L++) if (l == (u32)L) cdw = first[L];
                        cdw += rank;
                        const u32 rc = __brev(cdw) >> (32 - l);
                        for (u32 k = rc; k < 128; k += 1u << l) S.cl_lut[k] = (u8)((lane << 3) | l);
                    }
                }
                __syncwarp();
                for (int i = lane; i < 320; i += 32) S.lens[i] = 0;
                __syncwarp();
                auto decode = [&](Stream &r, u32 pk) {                                          // uniform
                    const u32 ce = S.cl_lut[pk & 127], cll = ce & 7;
                    const bool ok = cll != 0 && r.avail() >= cll;
                    r.skip(ok ? cll : 0);
                    return ok ? (int)(ce >> 3) : -1;
                };
                // runs of at most 6: lane i writes length n + i
                TRY(hdr::code_lengths(st, hlit + hdist, decode, [&](int n, int len, int reps) { if ((int)lane < reps) S.lens[n + lane] = (u8)len; }));
            }
            __syncwarp();
            // ---- canonical tables for both alphabets
            for (int t = 0; t < 2; t++) {
                const int nsym = t == 0 ? hlit : hdist;
                const u8 *ln = S.lens + (t == 0 ? 0 : hlit);
                if (lane < 16) S.cnt[t][lane] = 0;
                __syncwarp();
                for (int s = lane; s < nsym; s += 32) if (ln[s]) atomicAdd(&S.cnt[t][ln[s]], 1u);
                __syncwarp();
                u32 code = 0, off = 0, lim[17];
                u32 *bo = t == 0 ? S.lit_bo : S.dst_bo;
#pragma unroll
                for (int L = 1; L <= 15; L++) {
                    const u32 c = S.cnt[t][L];
                    if (lane == 0) bo[L] = (code & 0xFFFFu) | (off << 16);
                    code += c << (15 - L); off += c;
                    lim[L] = code > 0x8000u ? 0x8000u : code;
                }
                lim[16] = 0x8000u;
                if (code > 0x8000u) FAIL(SWC_INTERNAL_NEEDS_SLOW);
                Limits &LM = t == 0 ? T.lit_lim : T.dst_lim;
#pragma unroll
                for (int k = 0; k < 8; k++) LM.p[k] = lim[2 * k + 1] | (lim[2 * k + 2] << 16);
                __syncwarp();
                // sorted symbol table: position = first_index[L] + rank among the symbols of length L
                for (int L = 1; L <= 15; L++) {
                    if (S.cnt[t][L] == 0) continue;
                    u32 running = bo[L] >> 16;
                    for (int s0 = 0; s0 < nsym; s0 += 32) {
                        const int s = s0 + lane;
                        const bool hit = s < nsym && ln[s] == L;
                        const u32 m = __ballot_sync(SWC_FULL, hit);
                        if (hit) { const u32 p2 = running + __popc(m & ((1u << lane) - 1)); if (t == 0) S.lit_sym[p2] = (u16)s; else S.dst_sym[p2] = (u8)s; }
                        running += __popc(m);
                    }
                }
                __syncwarp();
            }
            // ---- flat LUTs: entry e = canonical decode of the bit pattern e (exact when the code fits in the index)
            for (u32 e = lane; e < (1u << LIT_BITS); e += 32) {
                int L; const int sym = canon_decode<0>(S, T.lit_lim, e, L);
                u32 v;
                if (sym < 0 || L > LIT_BITS) v = E_SLOW;      // no code within 11 bits: resolve with the canonical tables at decode time
                else if (sym < 256) v = (u32)L | ((u32)sym << 16);
                else if (sym == 256) v = (u32)L | (1u << 4);
                else if (sym > 285) v = (u32)L | (3u << 4);
                else { const u32 le = lens_tab[sym - 257]; v = (u32)L | (2u << 4) | ((le >> 16) << 6) | ((le & 0xFFFFu) << 16); }
                S.lit_lut[e] = v;
            }
            for (u32 e = lane; e < (1u << DST_BITS); e += 32) {
                int L; const int sym = canon_decode<1>(S, T.dst_lim, e, L);
                u32 v;
                if (sym < 0 || L > DST_BITS) v = E_SLOW;
                else if (sym > 29) v = (u32)L | (3u << 4);
                else { const u32 de = lens_tab[32 + sym]; v = (u32)L | ((de >> 16) << 6) | ((de & 0xFFFFu) << 16); }
                S.dst_lut[e] = v;
            }
            __syncwarp();

            // ------------------------------------------------------------ symbol stream, chunk by chunk
            bool block_done = false;
            while (!block_done) {
                // stage the chunk: words covering bits [pos, pos + 32*WIN_BITS + margin)
                const u64 q = st.pos + st.bit0;
                const u64 w0 = q >> 5;
                const u32 stage_bit0 = (u32)(q & 31);
                for (int i = lane; i < STAGE_WORDS; i += 32) S.stage[i] = st.word(w0 + i);
                __syncwarp();
                const u64 left = st.total - st.pos;
                const u32 hi = (lane + 1) * WIN_BITS;
                u32 start = lane * WIN_BITS;
                bool dirty = true, valid = true;
                WinResult r; r.end = 0; r.nbytes = 0; r.nlit = 0; r.nrec = 0; r.head = 0; r.tail = 0; r.flags = 0;
                // pass A: iterate until every window starts where its predecessor ended
                for (int round = 0; round < 33; round++) {
                    r = decode_window<false>(S, T, lens_tab, dirty && valid, start, hi, left, stage_bit0, nullptr, r);
                    // propagate: lane i+1 starts at lane i's end, unless lane i stopped the block (eob / error) or is invalid
                    const bool stops = !valid || (r.flags & 2) || (r.flags >> 8);
                    const u32 pend = __shfl_up_sync(SWC_FULL, r.end, 1);
                    const u32 pstop = __shfl_up_sync(SWC_FULL, (u32)stops, 1);
                    bool nvalid = valid; u32 nstart = start;
                    if (lane > 0) { nvalid = !pstop; nstart = pend; }
                    // a window that begins at or beyond its own limit decodes nothing (can happen after a 48-bit symbol)
                    dirty = (nvalid != valid) || (nvalid && nstart != start);
                    valid = nvalid; start = nstart;
                    if (!__any_sync(SWC_FULL, dirty)) break;
                }
                // the first lane that stops the chain
                const bool stops = valid && ((r.flags & 2) || (r.flags >> 8));
                const u32 stopmask = __ballot_sync(SWC_FULL, stops);
                const u32 vmask = __ballot_sync(SWC_FULL, valid);
                const int last = stopmask ? __ffs(stopmask) - 1 : 31;              // last lane that contributes
                const bool contrib = valid && (int)lane <= last;
                (void)vmask;
                // literal-run carry into each lane, escapes in front of first matches, record counts
                u32 carry = run_carry;
                u32 my_carry = 0;
                for (int j = 0; j <= last; j++) {
                    const u32 fl = __shfl_sync(SWC_FULL, r.flags, j);
                    const u32 hd = __shfl_sync(SWC_FULL, r.head, j);
                    const u32 tl = __shfl_sync(SWC_FULL, r.tail, j);
                    if ((int)lane == j) my_carry = carry;
                    carry = (fl & 1) ? tl : carry + hd;
                }
                u32 myrec = contrib ? r.nrec : 0;
                if (contrib && (r.flags & 1) && my_carry + r.head > 255) myrec++;
                u32 mybytes = contrib ? r.nbytes : 0;
                u32 mylit = contrib ? r.nlit : 0;
                u32 ib = mybytes, il = mylit, ir = myrec;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const u32 vb = __shfl_up_sync(SWC_FULL, ib, d), vl = __shfl_up_sync(SWC_FULL, il, d), vr = __shfl_up_sync(SWC_FULL, ir, d);
                    if (lane >= (u32)d) { ib += vb; il += vl; ir += vr; }
                }
                const u32 tot_b = __shfl_sync(SWC_FULL, ib, 31), tot_l = __shfl_sync(SWC_FULL, il, 31), tot_r = __shfl_sync(SWC_FULL, ir, 31);
                if (op + tot_b > OUT_MAX) FAIL(SWC_ERR_UNSUPPORTED);
                // pass B: emit
                int my_err = 0;
                {
                    Emit em;
                    em.lits = lits; em.rec = rec; em.cap = cap;
                    em.op = (u32)op + (ib - mybytes);
                    em.li = nlit + (il - mylit);
                    em.last_end = em.op - my_carry;
                    em.ri = nrec + (ir - myrec);
                    const WinResult rb = decode_window<true>(S, T, lens_tab, contrib, start, hi, left, stage_bit0, &em, r);
                    if (contrib) my_err = (int)(rb.flags >> 8);
                }
                const u32 emask = __ballot_sync(SWC_FULL, my_err != 0);
                if (emask) FAIL(__shfl_sync(SWC_FULL, my_err, __ffs(emask) - 1));                 // earliest error in stream order
                // advance the true chain
                const u32 endbits = __shfl_sync(SWC_FULL, r.end, last);
                const u32 lflags = __shfl_sync(SWC_FULL, r.flags, last);
                op += tot_b; nlit += tot_l; nrec += tot_r; run_carry = carry;
                st.pos += endbits;
                __syncwarp();
                if (lflags & 2) block_done = true;
            }
            if (is_last) break;
        }
    unit_done:
#undef FAIL
#undef TRY
        __syncwarp();
        if (lane == 0) {
            if (status == SWC_OK && op > cap64) status = SWC_ERR_OUTPUT_OVERFLOW;
            // a unit of fewer than 8 literals may not fit its literals below its records (inflate.cuh)
            if (status == SWC_OK && (u64)nlit + 4ull * nrec > region_bytes(a.out_off[unit], cap64)) status = SWC_INTERNAL_NEEDS_SLOW;
            a.consumed[unit] = st.pos;
            a.out_len[unit] = op;
            a.status[unit] = status;
            a.rec_count[unit] = nrec;
        }
    }
}

int launch_warp(const BatchArgs &a, cudaStream_t stream) {
    const size_t smem = sizeof(Smem) * WARPS;
    static int per_sm_cached[64] = {};
    int dev = 0;
    SWC_CUDA_TRY(cudaGetDevice(&dev));
    int st = configure_once(CFG_INFLATE_K1W, [&](DeviceCtx &) {
        int per_sm = 1;
        SWC_CUDA_TRY(cudaFuncSetAttribute(inflate_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        SWC_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, inflate_warp_kernel, WARPS * 32, smem));
        per_sm_cached[dev & 63] = per_sm < 1 ? 1 : per_sm;
        return (int)SWC_OK;
    });
    if (st) return st;
    u64 grid = (a.n + WARPS - 1) / WARPS;
    const u64 resident = (u64)device_ctx().num_sms * per_sm_cached[dev & 63];
    if (grid > resident) grid = resident;
    inflate_warp_kernel<<<(unsigned)grid, WARPS * 32, smem, stream>>>(a);
    count_launch();
    return SWC_OK;
}

}  // namespace inflate
}  // namespace swc
