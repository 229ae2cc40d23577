// inflate_lut.cu — K1L: Deflate Huffman stage for large batches, table-lookup decode (one thread per unit).
// Replaces the walk of Deflate.decompress(_: LsbBitReader) (reference Sources/Deflate/Deflate.swift:30-249) and
// DecodingTree.findNextSymbol (Sources/Common/CodingTree/DecodingTree.swift:36-50) for the batched hot path.
// Literals go to a packed stream, every match becomes a record for lz_resolve_kernel (format in inflate.cuh).
//
// 32 different streams per warp, persistent lanes.  Units are handed out 32 at a time to a warp whose lanes are all idle, so the
// lanes of a warp run in phase (see the hand-out comment in the kernel).  A warp works in rounds that start with a full-mask vote:
//   top-up : every lane keeps an 8-word ring of its compressed stream in shared memory; a lane whose ring is half empty
//            stores the 16-byte chunk it prefetched a round earlier (one LDG.128 per lane) and issues the next
//            load — the only place global input is touched, so the load latency never sits on the decode chain.
//   fast   : up to KLIT table lookups per lane: peek (funnel shift of a 64-bit register window, refilled without a branch, the
//            next ring word already in a register) -> 2^7-entry 16-bit LUT in shared memory, halfword-interleaved across the
//            warp (entry h of lane l at halfword h*32+l: conflict-free) -> literal: shifted into the next 8-byte word of the
//            packed literal stream (the word that fills up is stored once, after the loop); anything else (length, end of block, code
//            longer than 7 bits) parks the lane, which leaves the loop.
//   parked : all parked lanes together: length extra bits, distance code (2^5-entry 8-bit LUT, canonical limit-compare decoder
//            for longer codes), reference checks (Deflate.swift:199-232), one record per match.
//   header : block headers (Deflate.swift:41-168) are parsed by the lanes that reached one (they wait for HDR_BATCH of them),
//            with a plain global-memory bit reader; short codes fill the LUTs, long ones go to sorted lists for the
//            canonical decoder.  Per-length counters / cursors live in local memory; shared memory keeps 12.3 KB per warp
//            (LUTs, 18 long-code base words, ring): 16 resident warps per SM.
// Input availability (the reference's bitsLeft guards) is checked lazily against an absolute bit position: reads past the
// unit return zero bits and the first field that crosses the end reports symbolNotFound exactly as the reference does.
// Code sets with Kraft sum > 1 go to inflate_slow_kernel via SWC_INTERNAL_NEEDS_SLOW.
// Variants that fused the LZ77 copy into this kernel were slower than this kernel followed by lz_resolve_kernel.
#include "common.cuh"
#include "deflate_header.cuh"
#include "inflate.cuh"
#include "host_util.h"

namespace swc {
namespace inflate {
namespace k1l {

constexpr int LB = 7;                       // lit/len LUT index bits
constexpr int DB = 5;                       // distance LUT index bits
// ---- per-lane shared memory: halfword area (entry h of lane l at H[h*32+l]), byte area (D[h*32+l]), word area (W[w*32+l]) ----
constexpr int H_LIT = 0;
constexpr int H_TOTAL = 1 << LB;            // lit/len LUT, 16-bit entries
constexpr int D_TOTAL = 1 << DB;            // distance LUT, 8-bit entries {code length:3 | symbol:5}, 0 = no code of <= DB bits
// word area in the symbol phase: for every code length the LUT does not cover, {first left-justified 15-bit code | index of its
// first symbol in the long-symbol list << 16}
constexpr int W_LONG_LIT = 0;               // lengths LB+1 .. 15
constexpr int W_LONG_DST = 15 - LB;         // lengths DB+1 .. 15
constexpr int W_TOTAL = (15 - LB) + (15 - DB);
// the same words while a header is parsed (the code-length alphabet is dead once the LUTs are filled)
constexpr int W_CL_BO = 0;                  // [1..7]
constexpr int W_CL_SYM = 8;                 // 19 x u8
static_assert(W_CL_SYM + 5 <= W_TOTAL, "code-length tables must fit the long-code words they alias");
constexpr int RING_BYTES = 8 * 32 * 4;      // per warp: 8 words of compressed input per lane; 1 KiB, 1 KiB-aligned (address wrap by mask)
constexpr int WARP_BYTES = H_TOTAL * 32 * 2 + D_TOTAL * 32 + W_TOTAL * 32 * 4;
constexpr int WARPS_PER_CTA = 4;
constexpr int CTAS_PER_SM = 4;              // 16 warps per SM with a 2^7-entry LUT (12.3 KB per warp)
constexpr int LUT_WORDS = 64;               // CTA-shared length / distance base+extra tables
// CTA layout: [rings: WARPS x 1 KiB][LUT_WORDS x 4][per-warp tables]
constexpr size_t SMEM_BYTES = (size_t)WARPS_PER_CTA * RING_BYTES + LUT_WORDS * 4 + (size_t)WARPS_PER_CTA * WARP_BYTES;

constexpr int KLIT = 8;                     // lookups a lane may do per round (<= 56 bits) before parked symbols are serviced
static_assert(KLIT <= 8, "at most one 8-byte literal word may fill up per round (deferred store)");

constexpr int PATIENCE_SHIFT = 3;           // an idle lane waits for its warp for at most 1/2^PATIENCE_SHIFT of its last unit's rounds
constexpr int HDR_BATCH = 6;                // lanes that gather at a block boundary before the warp parses their headers

constexpr u32 E_NONLIT = 0x8000u;           // LUT entry: bit15 = not a literal; [11:8] code length (0 = long / no code)
constexpr u32 CODE_EOB = 31;                //   non-literal low byte: 0..28 length symbol 257+k, 29/30 = 286/287, 31 = end of block

// The unit as seen by both readers: bit positions count from `origin`, the 16-byte aligned address at or below the unit's
// first byte.  Bytes outside [ubeg, uend) read as zero.
struct Span {
    const u8 *origin, *ubeg, *uend;
    u32 pos0;        // bit position of the unit's first bit
    u32 end;         // pos0 + unit length in bits  (the reference's bitsLeft == end - pos)
};

__device__ __noinline__ uint4 load_edge(const u8 *c, const u8 *ubeg, const u8 *uend) {   // chunk straddling an end of the unit
    u32 w[4] = {0, 0, 0, 0};
    if (c < uend && c + 16 > ubeg) {
        for (int k = 0; k < 16; k++) {
            const u8 *a = c + k;
            if (a >= ubeg && a < uend) w[k >> 2] |= (u32)__ldg(a) << ((k & 3) * 8);
        }
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ uint4 load_chunk(const Span &sp, u32 ch) {
    const u8 *c = sp.origin + (size_t)ch * 16;
    if (c >= sp.ubeg && c + 16 <= sp.uend) {
        uint4 v;
        // plain read-only 16-byte load.  (ld.global.nc.L1::no_allocate also makes the line evict-first in L2, so the second
        // 16-byte half of every sector comes from DRAM again.)
        v = __ldg((const uint4 *)c);
        return v;
    }
    return load_edge(c, sp.ubeg, sp.uend);
}

__device__ __forceinline__ u32 lds32(u32 saddr) { u32 v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr)); return v; }
__device__ __forceinline__ u32 lds16(u32 saddr) { u32 v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(saddr)); return v; }
// LUT entry address: base + index * 64 (halfword index*32 + lane), as one multiply-add
__device__ __forceinline__ u32 lut_addr(u32 index, u32 base) { u32 a; asm("mad.lo.u32 %0, %1, 64, %2;" : "=r"(a) : "r"(index), "r"(base)); return a; }

// ------------------------------------------------------------------------------------------------ symbol-phase bit reader
// Window (lo, hi) = stream words [wend/32 - 1, wend/32]; further words wait in the shared-memory ring (slot = word index & 7,
// slot k of lane l at ring + k*128 + l*4; the ring of a warp is 1 KiB-aligned so the slot address wraps with one LOP3).
struct Reader {
    u32 lo, hi;
    u32 nxt;          // stream word wend/32 + 1, popped one step early so that no shared-memory load sits on the decode chain
    u32 pos;          // absolute bit position of the next unread bit;  wend - 32 <= pos < wend + 32
    u32 wend;         // bit position where `hi` starts; the next word to pop from the ring has index wend/32 + 2
    u32 rptr;         // shared-memory address of that word's slot
    u32 wr;           // next word index to push into the ring
    u32 nextc;        // chunk index after `pre`
    uint4 pre;        // chunk wr/4, already loaded

    __device__ __forceinline__ u32 peek32() const { return __funnelshift_r(lo, hi, pos); }   // requires pos < wend
    __device__ __forceinline__ void advance() {                                                // requires pos >= wend
        lo = hi;
        hi = nxt;
        nxt = lds32(rptr);
        const u32 t = rptr + 128;
        rptr = (t & 0x380u) | (rptr & ~0x380u);
        wend += 32;
    }
    // `if (pos >= wend) advance()` without a branch: the slot is read either way
    __device__ __forceinline__ void refill() {
        const bool adv = pos >= wend;
        const u32 nw = lds32(rptr);
        const u32 t = rptr + 128;
        lo = adv ? hi : lo;
        hi = adv ? nxt : hi;
        nxt = adv ? nw : nxt;
        rptr = adv ? ((t & 0x380u) | (rptr & ~0x380u)) : rptr;
        wend = adv ? wend + 32 : wend;
    }
    __device__ __forceinline__ void topup(u32 *ring, const Span &sp) {
        if (wr - (wend >> 5) <= 6) {                                   // <= 4 unread words in the ring: chunk wr/4 - 2 is consumed
            u32 *s = ring + (wr & 4) * 32;
            s[0] = pre.x; s[32] = pre.y; s[64] = pre.z; s[96] = pre.w;
            wr += 4;
            pre = load_chunk(sp, nextc);
            nextc++;
        }
    }
    __device__ void seek(u32 *ring, const Span &sp, u32 bit) {
        const u32 w0 = bit >> 5, ch = w0 >> 2;
        const uint4 a = load_chunk(sp, ch), b = load_chunk(sp, ch + 1);
        pre = load_chunk(sp, ch + 2);
        nextc = ch + 3;
        u32 *s = ring + (ch & 1) * 4 * 32, *t = ring + ((ch + 1) & 1) * 4 * 32;
        s[0] = a.x; s[32] = a.y; s[64] = a.z; s[96] = a.w;
        t[0] = b.x; t[32] = b.y; t[64] = b.z; t[96] = b.w;
        wr = (ch + 2) * 4;
        lo = ring[(w0 & 7) * 32];
        hi = ring[((w0 + 1) & 7) * 32];
        nxt = ring[((w0 + 2) & 7) * 32];
        rptr = (u32)__cvta_generic_to_shared(ring + ((w0 + 3) & 7) * 32);
        wend = (w0 + 1) * 32;
        pos = bit;
    }
};

// ------------------------------------------------------------------------------------------------ header-phase bit reader
struct HeaderBits {
    Span sp;
    u32 pos;
    __device__ __forceinline__ u32 word(u32 i) const {
        const u8 *a = sp.origin + (size_t)i * 4;
        if (a >= sp.ubeg && a + 4 <= sp.uend) return __ldg((const u32 *)a);
        u32 v = 0;
        for (int k = 0; k < 4; k++)
            if (a + k >= sp.ubeg && a + k < sp.uend) v |= (u32)__ldg(a + k) << (8 * k);
        return v;
    }
    __device__ __forceinline__ u32 peek32() const { return __funnelshift_r(word(pos >> 5), word((pos >> 5) + 1), pos); }
    __device__ __forceinline__ void skip(int n) { pos += n; }
    __device__ __forceinline__ i64 avail() const { return (i64)sp.end - (i64)pos; }
};

// ------------------------------------------------------------------------------------------------ output side
// `acc` is a shift register of the last 8 literals, newest in the top byte.  Whenever `nlit` reaches a multiple of 8 the
// register is exactly the word [nlit-8, nlit) of the packed literal stream (inflate.cuh), so a literal costs two funnel
// shifts and the store needs no alignment arithmetic.  Literal words are stored as two 4-byte halves: the stream is only
// 4-byte aligned.
struct Emit {
    u8 *lits;       // unit literal stream
    u32 *rec;       // end of the unit's scratch region (records grow downward from here)
    u32 op;         // bytes produced so far
    u32 nlit;       // literals produced so far
    u32 cap;
    u32 last_end;   // end of the previous match (start of the current literal run)
    u32 nrec;
    u32 acc_lo, acc_hi;

    __device__ __forceinline__ void store_word(u32 lo, u32 hi) {          // the word that ends at nlit & ~7
        u32 *p = (u32 *)(lits + (nlit & ~7u) - 8);
        p[0] = lo; p[1] = hi;
    }
    __device__ __forceinline__ void literal(u32 e) {           // low byte of e
        acc_lo = __funnelshift_r(acc_lo, acc_hi, 8);
        acc_hi = __funnelshift_r(acc_hi, e, 8);
        op++;
        nlit++;
        if ((nlit & 7) == 0 && op <= cap) store_word(acc_lo, acc_hi);
    }
    // fast-loop form: the word that fills up (at most one per round, KLIT <= 8) is parked in (f_lo, f_hi) and stored after the
    // loop at a convergent point.  Only literals follow it in the round, so its last literal sat at output byte op - (nlit & 7) - 1.
    __device__ __forceinline__ void literal_deferred(u32 e, u32 &f_lo, u32 &f_hi, bool &full) {
        acc_lo = __funnelshift_r(acc_lo, acc_hi, 8);
        acc_hi = __funnelshift_r(acc_hi, e, 8);
        op++;
        nlit++;
        const bool fill = (nlit & 7) == 0;
        f_lo = fill ? acc_lo : f_lo;
        f_hi = fill ? acc_hi : f_hi;
        full = full || fill;
    }
    __device__ __forceinline__ void store_deferred(u32 f_lo, u32 f_hi) {
        if (op - (nlit & 7) <= cap) store_word(f_lo, f_hi);
    }
    __device__ __forceinline__ void match(u32 len, u32 dist) {
        const u32 nop = op + len;
        if (nop <= cap) put_match(rec, nrec, op - last_end, len, dist);
        last_end = nop;
        op = nop;
    }
    // stores the last, partial literal word when it fits below the records (inflate.cuh); false when it does not
    __device__ __forceinline__ bool finish(u64 region) {
        if (op > cap) return true;                             // overflow: K2 skips the unit, nothing to hand over
        if ((u64)nlit + 4ull * nrec > region) return false;
        const u32 k = nlit & 7;
        const u64 v = ((u64)acc_hi << 32) | acc_lo;
        for (u32 i = 0; i < k; i++) lits[(nlit & ~7u) + i] = (u8)(v >> (8 * (8 - k + i)));
        return true;
    }
    __device__ __forceinline__ void stored_byte(u32 b) { literal(b); }
};

// ------------------------------------------------------------------------------------------------ table construction
// finalize one alphabet: bo[L] holds count[L] on entry, {first_code_lj | first_long_index << 16} on exit; `lutbits` = codes of
// at most that many bits live in the LUT and are not indexed.  Returns the Kraft sum scaled to 2^15.
template <int STRIDE>
__device__ __forceinline__ u32 finalize_tables(u32 *bo, Limits &lim, int maxlen, int lutbits) {
    u32 code = 0, off = 0;
    u32 l[17];
#pragma unroll
    for (int L = 1; L <= 15; L++) {
        u32 c = L <= maxlen ? bo[L * STRIDE] : 0;
        if (L <= maxlen) bo[L * STRIDE] = (code & 0xFFFF) | (off << 16);
        code += c << (15 - L);
        if (L > lutbits) off += c;
        l[L] = code > 0x8000u ? 0x8000u : code;
    }
    l[16] = 0x8000u;
#pragma unroll
    for (int k = 0; k < 8; k++) lim.p[k] = l[2 * k + 1] | (l[2 * k + 2] << 16);
    return code;
}
// after the assignment pass bo[L] = {end code of length L | end index}: the canonical property makes that the first
// code / index of length L+1, so shifting the array up by one slot restores the "first" values
template <int STRIDE>
__device__ __forceinline__ void rewind_tables(u32 *bo, int maxlen) {
    u32 prev = 0;
#pragma unroll
    for (int L = 1; L <= 15; L++) {
        if (L <= maxlen) {
            const u32 w = bo[L * STRIDE];
            bo[L * STRIDE] = prev;
            prev = w;
        }
    }
}

struct LaneMem {
    u16 *H;        // this lane's halfword 0
    u8 *D;         // this lane's byte 0 of the distance LUT
    u32 *W;        // this lane's word 0
    u16 *longsym;  // lit/len symbols with codes longer than LB bits, in canonical order (local memory)
    u8 *longdst;   // distance symbols with codes longer than DB bits (local memory)
    u32 *bol, *bod; // header phase: per-length counters, then code / long-index cursors, [1..15] (local memory)
};

// code-length alphabet: canonical decode (<= 7-bit codes, 19 symbols) of the next symbol, its bits consumed; -1 if none
__device__ __forceinline__ int decode_cl(HeaderBits &hb, u32 peek, const Limits &lim, const LaneMem &M) {
    const u32 r15 = __brev(peek & 0x7FFFu) >> 17;
    const int L = code_length(r15, lim);
    if (L > 15 || hb.avail() < L) return -1;
    hb.skip(L);
    const u32 idx = canonical_index(r15, L, M.W[(W_CL_BO + L) * 32]);
    return ((const u8 *)(M.W + (W_CL_SYM + (idx >> 2)) * 32))[idx & 3];
}

// One pass over the code lengths of a block (hdr::code_lengths, or hdr::fixed_lengths for a fixed block).  PASS 0 counts
// lengths into the BO areas; PASS 1 assigns codes: short codes fill the LUTs, long ones are appended to the sorted symbol lists.
template <int PASS>
__device__ int run_lengths(HeaderBits &hb, const LaneMem &M, const Limits &cl_lim, bool dynamic, int hlit, int hdist) {
    auto sink = [&](int n, int len, int reps) {
        for (int r = 0; r < reps; r++, n++) {
            const bool is_lit = n < hlit;
            u32 *bo = (is_lit ? M.bol : M.bod) + len;
            if (PASS == 0) {
                *bo += 1;
            } else {
                const u32 w = *bo;
                const int lutbits = is_lit ? LB : DB;
                const u32 sym = is_lit ? (u32)n : (u32)(n - hlit);
                if (len <= lutbits) {
                    *bo = w + (1u << (15 - len));
                    const u32 step = 1u << len, lim = 1u << lutbits;
                    if (!is_lit) {
                        for (u32 k = __brev(w & 0xFFFFu) >> 17; k < lim; k += step) M.D[k * 32] = (u8)(((u32)len << 5) | sym);
                    } else {
                        u32 e;
                        if (sym < 256) e = ((u32)len << 8) | sym;
                        else e = E_NONLIT | ((u32)len << 8) | (sym == 256 ? CODE_EOB : sym - 257);
                        for (u32 k = __brev(w & 0xFFFFu) >> 17; k < lim; k += step) M.H[(H_LIT + k) * 32] = (u16)e;
                    }
                } else {
                    *bo = w + (1u << (15 - len)) + 0x10000u;
                    const u32 pos = w >> 16;
                    if (is_lit) M.longsym[pos] = (u16)sym;
                    else M.longdst[pos] = (u8)sym;
                }
            }
        }
    };
    if (!dynamic) {
        hdr::fixed_lengths(sink);
        return SWC_OK;
    }
    return hdr::code_lengths(hb, hlit + hdist, [&](HeaderBits &r, u32 pk) { return decode_cl(r, pk, cl_lim, M); }, sink);
}

enum { ST_HEADER = 0, ST_SYMBOLS = 1, ST_PARKED = 2, ST_DONE = 3 };

struct BlockCtx {
    Limits lit_lim, dst_lim;
    bool is_last;
};

// Block header (Deflate.swift:41-168): stored blocks are copied here; for Huffman blocks the per-lane tables are built.
// On entry hb.pos is the header's first bit; on SWC_OK exit it is the first bit after the header (or after the stored bytes).
__device__ __forceinline__ int begin_block(HeaderBits &hb, Emit &em, const LaneMem &M, BlockCtx &bc, int &next) {
    u32 btype, length;
    if (const int st = hdr::block_start(hb, bc.is_last, btype)) return st;
    if (btype == 0) {
        if (const int st = hdr::stored_length(hb, length)) return st;
        if ((u64)em.op + length > OUT_MAX) return SWC_ERR_UNSUPPORTED;
        const u8 *src = hb.sp.origin + (hb.pos >> 3);                                   // byte aligned here
        for (u32 i = 0; i < length; i++) em.stored_byte(__ldg(src + i));
        hb.skip(length * 8);
        next = bc.is_last ? ST_DONE : ST_HEADER;
        return SWC_OK;
    }
    const bool dynamic = btype == 2;
    int hlit = 288, hdist = 32;
    Limits cl_lim;
    u32 lens_pos = hb.pos;
#pragma unroll
    for (int L = 1; L <= 15; L++) { M.bol[L] = 0; M.bod[L] = 0; }
    if (dynamic) {
        u64 cl;                                     // 19 x 3-bit code lengths, indexed by symbol
        if (const int st = hdr::dynamic_counts(hb, hlit, hdist, cl)) return st;
        u64 cnt = 0;                                // 8 x 8-bit counters
        for (int s = 0; s < 19; s++) cnt += 1ull << (8 * ((cl >> (3 * s)) & 7));
#pragma unroll
        for (int L = 1; L <= 7; L++) M.W[(W_CL_BO + L) * 32] = (u32)(cnt >> (8 * L)) & 0xFF;
        const u32 kraft = finalize_tables<32>(M.W + W_CL_BO * 32, cl_lim, 7, 0);
        if (kraft > 0x8000u) return SWC_INTERNAL_NEEDS_SLOW;
        for (int s = 0; s < 19; s++) {
            const u32 l = (u32)(cl >> (3 * s)) & 7;
            if (l) {
                const u32 w = M.W[(W_CL_BO + l) * 32];
                M.W[(W_CL_BO + l) * 32] = w + (1u << (15 - l)) + 0x10000u;
                const u32 pos = w >> 16;
                ((u8 *)(M.W + (W_CL_SYM + (pos >> 2)) * 32))[pos & 3] = (u8)s;
            }
        }
        rewind_tables<32>(M.W + W_CL_BO * 32, 7);
        lens_pos = hb.pos;
    }
    const int st = run_lengths<0>(hb, M, cl_lim, dynamic, hlit, hdist);
    if (st) return st;
    const u32 k1 = finalize_tables<1>(M.bol, bc.lit_lim, 15, LB);
    const u32 k2 = finalize_tables<1>(M.bod, bc.dst_lim, 15, DB);
    if (k1 > 0x8000u || k2 > 0x8000u) return SWC_INTERNAL_NEEDS_SLOW;
    for (int k = 0; k < (1 << LB); k++) M.H[(H_LIT + k) * 32] = (u16)E_NONLIT;     // "no short code here": canonical decoder decides
    for (int k = 0; k < (1 << DB); k++) M.D[k * 32] = 0;
    hb.pos = lens_pos;
    run_lengths<1>(hb, M, cl_lim, dynamic, hlit, hdist);
    rewind_tables<1>(M.bol, 15);
    rewind_tables<1>(M.bod, 15);
    // the symbol phase only needs the lengths the LUTs do not cover: they replace the code-length tables in shared memory
#pragma unroll
    for (int L = LB + 1; L <= 15; L++) M.W[(W_LONG_LIT + L - LB - 1) * 32] = M.bol[L];
#pragma unroll
    for (int L = DB + 1; L <= 15; L++) M.W[(W_LONG_DST + L - DB - 1) * 32] = M.bod[L];
    next = ST_SYMBOLS;
    return SWC_OK;
}

// A symbol the LUT could not finish: long code, end of block, or a length + distance (Deflate.swift:171-232).
__device__ __forceinline__ int parked_step(Reader &br, Emit &em, const LaneMem &M, const BlockCtx &bc, const Span &sp,
                                           const u32 *lut, int &state, u32 e) {
    // br.pos < br.wend here: the window still holds the >= 32 bits the lookup saw
    const u32 w0 = br.peek32();                                                // lit/len code (<= 15) + extra bits (<= 5) lie in here
    u32 L = (e >> 8) & 15, code = e & 0xFF;
    if (L == 0) {                                                              // canonical decode of a long (or missing) code
        const u32 r15 = __brev(w0 & 0x7FFFu) >> 17;
        const int CL = code_length(r15, bc.lit_lim);
        if (CL > 15) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
        const u32 sym = M.longsym[canonical_index(r15, CL, M.W[(W_LONG_LIT + CL - LB - 1) * 32])];   // CL > LB: the LUT holds every shorter code
        br.pos += CL;
        L = (u32)CL;
        if (sym < 256) {
            if (br.pos > sp.end) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
            em.literal(sym);
            state = ST_SYMBOLS;
            return SWC_OK;
        }
        code = sym == 256 ? CODE_EOB : sym - 257;
    } else {
        br.pos += L;
    }
    if (br.pos > sp.end) return SWC_DEFLATE_SYMBOL_NOT_FOUND;                  // the code itself crossed the end of the input
    if (code == CODE_EOB) { state = bc.is_last ? ST_DONE : ST_HEADER; return SWC_OK; }
    if (code > 28) return SWC_DEFLATE_WRONG_SYMBOL;                            // 286 / 287
    const u32 le = lut[code];
    const u32 eb = le >> 16;
    const u32 length = (le & 0xFFFFu) + ((w0 >> L) & ((1u << eb) - 1));
    br.pos += eb;
    if (br.pos >= br.wend) br.advance();
    const u32 w32 = br.peek32();                                               // distance code (<= 15) + extra bits (<= 13)
    const u32 de = M.D[(w32 & ((1u << DB) - 1)) * 32];
    u32 DL = de >> 5, dsym = de & 31;
    if (DL == 0) {
        const u32 r15 = __brev(w32 & 0x7FFFu) >> 17;
        DL = (u32)code_length(r15, bc.dst_lim);
        if (DL > 15) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
        dsym = M.longdst[canonical_index(r15, DL, M.W[(W_LONG_DST + DL - DB - 1) * 32])];
    }
    br.pos += DL;
    if (br.pos > sp.end) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
    if (dsym > 29) return SWC_DEFLATE_WRONG_SYMBOL;
    const u32 dd = lut[32 + dsym];
    const u32 db = dd >> 16;
    const u32 dist = (dd & 0xFFFFu) + ((w32 >> DL) & ((1u << db) - 1));
    br.pos += db;
    if (br.pos > sp.end) return SWC_DEFLATE_SYMBOL_NOT_FOUND;
    if (dist > em.op) return SWC_ERR_REFERENCE_TRAP;                                     // :219 negative array index
    if ((u64)em.op + length > OUT_MAX) return SWC_ERR_UNSUPPORTED;
    em.match(length, dist);
    state = ST_SYMBOLS;
    return SWC_OK;
}

__global__ void __launch_bounds__(WARPS_PER_CTA * 32, CTAS_PER_SM)
inflate_lut_kernel(BatchArgs a) {
    extern __shared__ __align__(1024) u32 smem[];
    u32 *lut = smem + WARPS_PER_CTA * RING_BYTES / 4;  // [0,32) length table, [32,64) distance table
    if (threadIdx.x < 32) { lut[threadIdx.x] = c_len_tab[threadIdx.x]; lut[32 + threadIdx.x] = c_dist_tab[threadIdx.x]; }
    __syncthreads();
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u8 *wbase = (u8 *)(lut + LUT_WORDS) + (size_t)warp * WARP_BYTES;
    u16 longsym[288];
    u8 longdst[32];
    u32 bol[16], bod[16];
    LaneMem M;
    M.bol = bol;
    M.bod = bod;
    M.H = (u16 *)wbase + lane;
    M.D = wbase + H_TOTAL * 32 * 2 + lane;
    M.W = (u32 *)(wbase + H_TOTAL * 32 * 2 + D_TOTAL * 32) + lane;
    M.longsym = longsym;
    M.longdst = longdst;
    u32 *ring = smem + warp * (RING_BYTES / 4) + lane;
    const u32 hlit = (u32)__cvta_generic_to_shared(M.H + H_LIT * 32);

    int status = SWC_OK, state = ST_DONE;
    bool have_unit = false, exhausted = false;
    u64 unit = 0;
    Span sp;
    Reader br;
    Emit em;
    BlockCtx bc;
    u64 cap64 = 0;
    u32 pend = 0;
    sp.origin = sp.ubeg = sp.uend = nullptr; sp.pos0 = sp.end = 0;
    br.lo = br.hi = br.nxt = 0;
    br.pos = 0; br.wend = 32; br.rptr = 0; br.wr = 0; br.nextc = 0; br.pre = make_uint4(0, 0, 0, 0);
    em.lits = nullptr; em.rec = nullptr; em.op = 0; em.nlit = 0; em.cap = 0; em.last_end = 0; em.nrec = 0; em.acc_lo = em.acc_hi = 0;
    u32 rounds = 0, patience = 0;     // rounds spent on the current unit / rounds an idle lane still waits for its warp
    for (;;) {
        if (state == ST_DONE && have_unit) {                                             // retire the finished unit
            const bool fits = em.finish(region_bytes(a.out_off[unit], cap64));
            if (status == SWC_OK && em.op > OUT_MAX) status = SWC_ERR_UNSUPPORTED;
            if (status == SWC_OK && (u64)em.op > cap64) status = SWC_ERR_OUTPUT_OVERFLOW;
            if (status == SWC_OK && !fits) status = SWC_INTERNAL_NEEDS_SLOW;
            a.consumed[unit] = br.pos - sp.pos0;
            a.out_len[unit] = em.op;
            a.status[unit] = status;
            a.rec_count[unit] = em.nrec;
            have_unit = false;
            patience = rounds >> PATIENCE_SHIFT;
        }
        // Unit hand-out.  A unit keeps a lane busy for thousands of rounds, so WHEN lanes start matters: lanes that run in phase
        // share the header code (one pass serves all 32), finish together, and leave no tail of half-empty warps at the end of
        // the batch (with one lane-at-a-time ticket per finished lane, the units after the first of every lane took half as long
        // again, their lanes out of phase).  So a warp takes 32 consecutive units at once when all its lanes are idle; an idle lane
        // waits for that moment for at most 1/2^PATIENCE_SHIFT of the rounds its last unit took (units of similar size stay in
        // phase) and takes a unit of its own when its patience runs out (units of very different sizes).
        const bool idle = state == ST_DONE && !exhausted;                                // have_unit is false here
        const u32 idle_mask = __ballot_sync(SWC_FULL, idle);
        if (idle_mask) {
            const u32 working = __ballot_sync(SWC_FULL, state != ST_DONE);
            const bool take = idle && (working == 0 || patience == 0);
            if (idle && !take) patience--;
            const u32 take_mask = __ballot_sync(SWC_FULL, take);
            if (take_mask) {
                u64 first = 0;
                const u32 leader = __ffs(take_mask) - 1;
                if (lane == leader) first = atomicAdd(a.ticket + 1, (u64)__popc(take_mask));
                first = __shfl_sync(SWC_FULL, first, leader);
                if (take) {
                    unit = first + __popc(take_mask & ((1u << lane) - 1));
                    rounds = 0;
                    if (unit >= a.n) {
                        exhausted = true;
                    } else {
                        have_unit = true;
                        status = SWC_OK;
                        const u64 in_len = a.in_len[unit];
                        cap64 = a.out_cap[unit];
                        em.lits = (u8 *)(a.rec_base + rec_start(a.out_off[unit]));
                        em.rec = a.rec_base + rec_start(a.out_off[unit] + cap64);
                        em.cap = cap64 > OUT_MAX ? OUT_MAX : (u32)cap64;
                        em.op = 0; em.nlit = 0; em.last_end = 0; em.nrec = 0; em.acc_lo = em.acc_hi = 0;
                        const u32 bitskip = a.start_bits ? a.start_bits[unit] : 0;
                        sp.ubeg = a.in_base + a.in_off[unit];
                        sp.uend = sp.ubeg + in_len;
                        sp.origin = (const u8 *)((uintptr_t)sp.ubeg & ~(uintptr_t)15);
                        sp.pos0 = (u32)(sp.ubeg - sp.origin) * 8 + bitskip;
                        sp.end = sp.pos0 + (u32)(in_len * 8 - bitskip);
                        br.pos = sp.pos0;
                        if (in_len >= (1ull << 28)) status = SWC_ERR_UNSUPPORTED;        // bit positions are 32-bit here
                        else if (in_len * 8 - bitskip < 10) status = SWC_DEFLATE_WRONG_BLOCK_TYPE;  // Deflate.swift:36
                        else state = ST_HEADER;
                    }
                }
            }
        }
        rounds++;
        if (!__any_sync(SWC_FULL, state != ST_DONE || have_unit || !exhausted)) break;
        if (state == ST_SYMBOLS) {
            br.topup(ring, sp);
            if (br.pos > sp.end) { status = SWC_DEFLATE_SYMBOL_NOT_FOUND; state = ST_DONE; }
            // literals are not bounded one by one: a round adds at most KLIT + 1 of them, so em.op <= OUT_MAX at the
            // start of every round keeps the u32 from wrapping
            else if (em.op > OUT_MAX) { status = SWC_ERR_UNSUPPORTED; state = ST_DONE; }
        }
        // ---- fast: table lookups; a lane leaves the loop at its first non-literal ----
        u32 f_lo = 0, f_hi = 0;
        bool full = false;
        if (state == ST_SYMBOLS) {
#pragma unroll
            for (int k = 0; k < KLIT; k++) {
                br.refill();
                const u32 e = lds16(lut_addr(br.peek32() & ((1u << LB) - 1), hlit));
                if (e & E_NONLIT) { pend = e; state = ST_PARKED; break; }
                br.pos += e >> 8;
                em.literal_deferred(e, f_lo, f_hi, full);
            }
        }
        // Lanes leave the loop at different steps: re-converge them here, or the compiler threads each break edge straight into
        // the parked code and the warp executes it once per leaving group, several times per round with a few of 32 lanes active.
        __syncwarp();
        if (full) em.store_deferred(f_lo, f_hi);
        // ---- parked: lengths, distances, end of block, long codes ----
        if (state == ST_PARKED) {
            const int r = parked_step(br, em, M, bc, sp, lut, state, pend);
            if (r) { status = r; state = ST_DONE; }
        }
        __syncwarp();
        // ---- header: lanes at a block boundary ----
        // A header costs the warp ~100 K instructions whether one lane parses or all 32 do, and in steady state the lanes of a
        // warp reach their block boundaries one by one.  Lanes therefore wait at the boundary until HDR_BATCH of them have
        // gathered (or nobody is left decoding), so that one pass over the header code serves several streams.
        const u32 at_header = __ballot_sync(SWC_FULL, state == ST_HEADER);
        const u32 decoding = __ballot_sync(SWC_FULL, state == ST_SYMBOLS || state == ST_PARKED);
        if (state == ST_HEADER && (__popc(at_header) >= HDR_BATCH || decoding == 0)) {
            HeaderBits hb;
            hb.sp = sp; hb.pos = br.pos;
            int next = ST_DONE;
            const int r = begin_block(hb, em, M, bc, next);
            br.pos = hb.pos;
            if (r) { status = r; state = ST_DONE; }
            else {
                state = next;
                if (next == ST_SYMBOLS) br.seek(ring, sp, hb.pos);
            }
        }
    }
}

}  // namespace k1l

int launch_lut(const BatchArgs &a, cudaStream_t stream) {
    int st = configure_once(CFG_INFLATE_K1L, [](DeviceCtx &) {
        SWC_CUDA_TRY(cudaFuncSetAttribute(k1l::inflate_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1l::SMEM_BYTES));
        SWC_CUDA_TRY(cudaFuncSetAttribute(k1l::inflate_lut_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        return (int)SWC_OK;
    });
    if (st) return st;
    // Persistent lanes: one CTA per resident slot.  (Launching fewer, less crowded lanes so that n / lanes lands just under a
    // whole number of unit-times was slower than keeping every slot busy.)
    const u64 per_cta = k1l::WARPS_PER_CTA * 32;
    u64 grid = (a.n + per_cta - 1) / per_cta;
    const u64 resident = (u64)device_ctx().num_sms * k1l::CTAS_PER_SM;
    if (grid > resident) grid = resident;
    k1l::inflate_lut_kernel<<<(unsigned)grid, k1l::WARPS_PER_CTA * 32, k1l::SMEM_BYTES, stream>>>(a);
    count_launch();
    return SWC_OK;
}

}  // namespace inflate
}  // namespace swc
