// lzma_dec.cuh — the warp-per-stream LZMA decoder state (Dec) and the LZMA2 chunk loop, shared by lzma_kernel (lzma.cu) and
// xz_kernel (xz_batch.cu).  The library is built without relocatable device code, so the one copy lives in this header.
// Reference: LZMADecoder.swift:79-298, LZMARangeDecoder.swift:20-80, LZMABitTreeDecoder.swift, LZMALenDecoder.swift,
// LZMA2Decoder.swift:17-99.
#pragma once
#include "common.cuh"

namespace swc {
namespace lzma {

constexpr int OFF_PROBS = 0;        // 448: isMatch[192] | pad | isRep 193.. | isRepG0 205.. | G1 217.. | G2 229.. | isRep0Long 241..
constexpr int OFF_POSSLOT = 448;    // 4 x 64
constexpr int OFF_ALIGN = 704;      // 16
constexpr int OFF_POSDEC = 720;     // 115 (+1)
constexpr int OFF_LEN = 836;        // choice, choice2, low[16][8], mid[16][8], high[256]
constexpr int OFF_REPLEN = 1350;
constexpr int OFF_LIT = 1864;       // (1 << (lc+lp)) x 0x300
constexpr int LIT_SMEM_MAX = 16 * 0x300;
constexpr int SMEM_U16 = OFF_LIT + LIT_SMEM_MAX;           // 14152 u16 = 28304 B per warp
constexpr int WARPS = 2;
constexpr size_t SMEM_BYTES = (size_t)WARPS * SMEM_U16 * 2;
constexpr u32 TOP = 1u << 24;

struct Dec {
    // input window
    const u32 *chunkp; u64 end_addr; u32 cur, nxt; u64 addr;     // addr = absolute address of the next input byte
    bool trap;
    // range coder
    u32 range, code;
    // model
    u16 *P;            // shared-memory model base for this warp
    u16 *lit;          // literal coders (shared, or global scratch when lc+lp > 4)
    int lc, lp, pb;
    i64 dict_size, usize;
    // dictionary / output
    u8 *out; u64 cap;
    i64 dict_start, dict_end;        // dict_end == bytes produced
    i64 rep0, rep1, rep2, rep3;
    int state;
    bool ready;
    u32 prev_byte;

    // a fresh decoder (LZMADecoder.init / LZMA2Decoder.init) writing at `o`, model at `p`
    __device__ __forceinline__ void start(u16 *p, u8 *o, u64 c) {
        P = p; out = o; cap = c;
        dict_start = dict_end = 0;
        rep0 = rep1 = rep2 = rep3 = 0; state = 0; ready = false; lit = nullptr; prev_byte = 0;
        lc = 3; lp = 0; pb = 2; dict_size = 1 << 24; usize = -1;
    }

    __device__ __forceinline__ u32 load_chunk() {
        const u32 *p = chunkp + lane_id();
        chunkp += 32;
        return ((u64)(uintptr_t)p < end_addr) ? __ldg(p) : 0u;
    }
    __device__ void in_init(const u8 *p, u64 len) {
        addr = (u64)(uintptr_t)p; end_addr = addr + len;
        chunkp = (const u32 *)((uintptr_t)p & ~(uintptr_t)127);
        cur = load_chunk(); nxt = load_chunk();
        trap = false;
    }
    __device__ __forceinline__ u64 in_left() const { return end_addr - addr; }
    __device__ __forceinline__ u32 byte() {                       // BitByteData byte(): reading past the end traps
        if (addr >= end_addr) { trap = true; return 0; }
        const u32 w = __shfl_sync(SWC_FULL, cur, (int)((addr >> 2) & 31));
        const u32 b = (w >> ((addr & 3) * 8)) & 0xFF;
        addr++;
        if ((addr & 127) == 0) { cur = nxt; nxt = load_chunk(); }
        return b;
    }
    __device__ __forceinline__ int bit(u16 *prob) {               // LZMARangeDecoder.swift:65-80
        // select form (no branch on the decoded bit: the warp runs one dependent chain, a taken branch costs several issue slots)
        const u32 p = *prob;
        const u32 bound = (range >> 11) * p;
        const bool one = code >= bound;
        *prob = (u16)(one ? p - (p >> 5) : p + ((2048 - p) >> 5));
        range = one ? range - bound : bound;
        code = one ? code - bound : code;
        if (range < TOP) { range <<= 8; code = (code << 8) | byte(); }
        return one ? 1 : 0;
    }
    __device__ __forceinline__ int direct(int count) {            // LZMARangeDecoder.swift:46-62
        u32 res = 0;
        do {
            range >>= 1;
            code -= range;
            const u32 t = 0u - (code >> 31);
            code += range & t;
            if (range < TOP) { range <<= 8; code = (code << 8) | byte(); }
            res = (res << 1) + (t + 1);
        } while (--count > 0);
        return (int)res;
    }
    __device__ __forceinline__ int tree(u16 *probs, int nbits) {
        int m = 1;
        for (int i = 0; i < nbits; i++) m = (m << 1) + bit(&probs[m]);
        return m - (1 << nbits);
    }
    __device__ __forceinline__ int tree_rev(u16 *probs, int nbits) {
        int m = 1, sym = 0;
        for (int i = 0; i < nbits; i++) { int b = bit(&probs[m]); m = (m << 1) + b; sym |= b << i; }
        return sym;
    }
    __device__ __forceinline__ int len_decode(u16 *L, int pos_state) {   // LZMALenDecoder.swift:28-38
        if (bit(&L[0]) == 0) return tree(L + 2 + pos_state * 8, 3);
        if (bit(&L[1]) == 0) return 8 + tree(L + 2 + 128 + pos_state * 8, 3);
        return 16 + tree(L + 2 + 256, 8);
    }
    __device__ void reset_state(u16 *lit_global) {                // LZMADecoder.swift:79-100
        state = 0; rep0 = rep1 = rep2 = rep3 = 0;
        const int nlit = (1 << (lc + lp)) * 0x300;
        lit = nlit <= LIT_SMEM_MAX ? P + OFF_LIT : lit_global;
        __syncwarp();
        for (int i = lane_id(); i < OFF_LIT; i += 32) P[i] = 1024;
        if (lit) for (int i = lane_id(); i < nlit; i += 32) lit[i] = 1024;
        __syncwarp();
        ready = true;
    }
    __device__ __forceinline__ void put(u32 b) {                  // LZMADecoder.swift:288-294 (every lane stores the same byte)
        out[dict_end] = (u8)b;
        prev_byte = b;
        dict_end += 1;
        if (dict_end - dict_start == dict_size) dict_start += 1;
    }
    __device__ __forceinline__ u32 byte_at(i64 distance, bool &oob) {      // LZMADecoder.swift:296-298
        const i64 idx = distance <= dict_end ? dict_end - distance : dict_size - distance + dict_end;
        if (idx < 0 || idx >= dict_end) { oob = true; return 0; }
        return out[idx];
    }

    // LZMADecoder.decode()
    __device__ int decode() {
        if (in_left() < 5) return SWC_LZMA_RANGE_DECODER_INIT_ERROR;                 // LZMARangeDecoder.swift:22
        const u32 b0 = byte();
        code = byte() << 24; code |= byte() << 16; code |= byte() << 8; code |= byte();
        range = 0xFFFFFFFFu;
        if (b0 != 0) return SWC_LZMA_RANGE_DECODER_INIT_ERROR;
        if (!ready) return SWC_ERR_REFERENCE_TRAP;          // empty probability arrays in the reference
        if (!lit) return SWC_ERR_UNSUPPORTED;               // lc+lp > 4 without global literal scratch
        bool oob = false;
        const int pb_mask = (1 << pb) - 1, lp_mask = (1 << lp) - 1;
        u16 *probs = P + OFF_PROBS;
        for (;;) {
            if (trap || oob) return SWC_ERR_REFERENCE_TRAP;
            if (usize == 0 && code == 0) break;
            const int pos_state = (int)(dict_end & pb_mask);
            if (bit(&probs[(state << 4) + pos_state]) == 0) {                        // literal :119-172
                if (trap) return SWC_ERR_REFERENCE_TRAP;
                if (usize == 0) return SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE;
                const u32 prev = dict_end == dict_start ? 0 : prev_byte;
                int symbol = 1;
                u16 *lpz = lit + ((((u32)dict_end & lp_mask) << lc) + (prev >> (8 - lc))) * 0x300;
                if (state < 7) {                                                      // plain literal: exactly 8 tree levels
#pragma unroll
                    for (int i = 0; i < 8; i++) symbol = (symbol << 1) | bit(&lpz[symbol]);
                } else {
                    u32 match_byte = byte_at(rep0 + 1, oob);
                    if (oob) return SWC_ERR_REFERENCE_TRAP;
                    do {
                        const int match_bit = (match_byte >> 7) & 1;
                        match_byte = (match_byte << 1) & 0xFF;
                        const int b = bit(&lpz[((1 + match_bit) << 8) + symbol]);
                        symbol = (symbol << 1) | b;
                        if (match_bit != b) break;
                    } while (symbol < 0x100);
                    while (symbol < 0x100) symbol = (symbol << 1) | bit(&lpz[symbol]);
                }
                if (trap) return SWC_ERR_REFERENCE_TRAP;
                // capacity is checked once the literal is known to decode: a stream cut inside it traps in the reference
                if ((u64)dict_end >= cap) return SWC_ERR_OUTPUT_OVERFLOW;
                usize -= 1;
                put((u32)symbol - 0x100);
                state = state < 4 ? 0 : (state < 10 ? state - 3 : state - 6);
                continue;
            }
            i64 len;
            if (bit(&probs[193 + state]) != 0) {                                     // rep :176-215
                if (trap) return SWC_ERR_REFERENCE_TRAP;
                if (usize == 0) return SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE;
                if (dict_end == dict_start) return SWC_LZMA_WINDOW_IS_EMPTY;
                if (bit(&probs[205 + state]) == 0) {
                    const int idx = 241 + (state << 4) + pos_state;
                    if (idx >= 432) return SWC_ERR_REFERENCE_TRAP;                   // 432-entry array in the reference
                    if (bit(&probs[idx]) == 0) {
                        if (trap) return SWC_ERR_REFERENCE_TRAP;
                        state = state < 7 ? 9 : 11;
                        const u32 b = byte_at(rep0 + 1, oob);
                        if (oob) return SWC_ERR_REFERENCE_TRAP;
                        if ((u64)dict_end >= cap) return SWC_ERR_OUTPUT_OVERFLOW;
                        put(b);
                        usize -= 1;
                        continue;
                    }
                } else {
                    i64 dist;
                    if (bit(&probs[217 + state]) == 0) {
                        dist = rep1;
                    } else {
                        if (bit(&probs[229 + state]) == 0) dist = rep2;
                        else { dist = rep3; rep3 = rep2; }
                        rep2 = rep1;
                    }
                    rep1 = rep0;
                    rep0 = dist;
                }
                len = len_decode(P + OFF_REPLEN, pos_state);
                state = state < 7 ? 8 : 11;
            } else {                                                                 // match :216-272
                rep3 = rep2; rep2 = rep1; rep1 = rep0;
                len = len_decode(P + OFF_LEN, pos_state);
                state = state < 7 ? 7 : 10;
                const int len_state = len > 3 ? 3 : (int)len;
                const int pos_slot = tree(P + OFF_POSSLOT + len_state * 64, 6);
                if (pos_slot < 4) {
                    rep0 = pos_slot;
                } else {
                    const int nd = (pos_slot >> 1) - 1;
                    i64 dist = (i64)(2 | (pos_slot & 1)) << nd;
                    if (pos_slot < 14) {
                        dist += tree_rev(P + OFF_POSDEC + (dist - pos_slot), nd);
                    } else {
                        dist += (i64)direct(nd - 4) << 4;
                        dist += tree_rev(P + OFF_ALIGN, 4);
                    }
                    rep0 = dist;
                }
                if (trap) return SWC_ERR_REFERENCE_TRAP;
                if ((u32)rep0 == 0xFFFFFFFFu) {                                      // :260-264 end marker
                    if (code != 0) return SWC_LZMA_RANGE_DECODER_FINISH_ERROR;
                    break;
                }
                if (usize == 0) return SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE;
                if (rep0 >= dict_size || (rep0 > dict_end && dict_end < dict_size)) return SWC_LZMA_NOT_ENOUGH_TO_REPEAT;
            }
            if (trap) return SWC_ERR_REFERENCE_TRAP;
            len += 2;
            if (usize > -1 && usize < len) return SWC_LZMA_REPEAT_WILL_EXCEED;
            {   // copy :278-282 — first byte through byte_at (it carries the reference's index rule), rest cooperatively
                const i64 distance = rep0 + 1;
                (void)byte_at(distance, oob);
                if (oob) return SWC_ERR_REFERENCE_TRAP;
                if ((u64)(dict_end + len) > cap) return SWC_ERR_OUTPUT_OVERFLOW;
                // distance <= dict_end here (the wrapped branch of byte_at always lands out of range)
                const u8 *src = out + dict_end - distance;
                u8 *dst = out + dict_end;
                __syncwarp();
                for (i64 i = lane_id(); i < len; i += 32) dst[i] = src[distance >= len ? i : i % distance];
                __syncwarp();
                prev_byte = dst[len - 1];
                // dictStart bookkeeping of `len` put() calls
                // (closed form of: repeat len times { dict_end += 1; if (dict_end - dict_start == dict_size) dict_start += 1; } —
                // the gap climbs to dict_size-1 and then every further byte advances dict_start; a gap that is already
                // >= dict_size never meets the equality again)
                {
                    const i64 gap = dict_end - dict_start;
                    if (gap < (i64)dict_size) { const i64 adv = gap + len - ((i64)dict_size - 1); if (adv > 0) dict_start += adv; }
                    dict_end += len;
                }
                usize -= len;
            }
        }
        return SWC_OK;
    }
};

// LZMA2Decoder.init + decode()  LZMA2Decoder.swift:17-99: `db` is the dictionary-size byte, the chunks are read from d's
// input window and appended at d.out + d.dict_end.  On return d.dict_end is the output produced and d.addr the next byte.
__device__ __forceinline__ int lzma2_decode(Dec &d, u32 db, u16 *lit_global) {
    if (db & 0xC0) return SWC_LZMA2_WRONG_DICTIONARY_SIZE;
    if ((db & 0x3F) >= 40) return SWC_LZMA2_WRONG_DICTIONARY_SIZE;
    const u32 bits = db & 0x3F;
    const u32 ds = (2 | (bits & 1)) << (bits / 2 + 11);
    d.dict_size = ds < 4096 ? 4096 : ds;
#define NEED(k) if (d.in_left() < (u64)(k)) return SWC_ERR_REFERENCE_TRAP
    for (;;) {
        NEED(1);
        const u32 control = d.byte();
        if (control == 0) return SWC_OK;
        if (control == 1 || control == 2) {                                 // :84-89
            if (control == 1) d.dict_start = d.dict_end;
            NEED(2);
            u64 size = (u64)d.byte() << 8; size += d.byte(); size += 1;
            NEED(size);
            if ((u64)d.dict_end + size > d.cap) return SWC_ERR_OUTPUT_OVERFLOW;
            // stored chunk: cooperative copy straight from the input
            const u8 *src = (const u8 *)(uintptr_t)d.addr;
            u8 *dst = d.out + d.dict_end;
            for (u64 i = lane_id(); i < size; i += 32) dst[i] = src[i];
            __syncwarp();
            d.prev_byte = dst[size - 1];
            for (u64 i = 0; i < size; i++) { d.dict_end += 1; if (d.dict_end - d.dict_start == d.dict_size) d.dict_start += 1; }
            // re-seat the input window after the skipped bytes
            d.in_init((const u8 *)(uintptr_t)(d.addr + size), d.end_addr - (d.addr + size));
            continue;
        }
        if (control < 0x80) return SWC_LZMA2_WRONG_CONTROL_BYTE;
        const int reset = (control & 0x60) >> 5;                            // :56-82
        NEED(4);
        i64 unpack = ((i64)(control & 0x1F) << 16); unpack += (i64)d.byte() << 8; unpack += d.byte(); unpack += 1;
        i64 comp = (i64)d.byte() << 8; comp += d.byte(); comp += 1;
        if (reset == 1) {
            d.reset_state(lit_global);
        } else if (reset >= 2) {
            NEED(1);
            const u32 b = d.byte();
            if (b >= 225) return SWC_LZMA_WRONG_PROPERTIES;
            d.lc = b % 9; d.pb = (b / 9) / 5; d.lp = (b / 9) % 5;
            d.reset_state(lit_global);
            if (reset == 3) d.dict_start = d.dict_end;
        }
        d.usize = unpack;
        const i64 out_start = d.dict_end;
        const u64 in_start = d.addr;
        const int st = d.decode();
        if (st) return st;
        if (!(unpack == d.dict_end - out_start && (i64)(d.addr - in_start) == comp)) return SWC_LZMA2_WRONG_SIZES;
    }
#undef NEED
}

}  // namespace lzma
}  // namespace swc
