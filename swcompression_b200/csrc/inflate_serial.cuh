// inflate_serial.cuh — the generic serial Deflate decoder, one thread per stream: inflate_slow_kernel's body, shared with the
// fallback walk of the multi-member gzip batch (gzip_member_batch.cu).  The library is built without relocatable device code,
// so the one copy lives in this header.  Over-subscribed code sets follow the reference's heap-slot overwrites (see
// inflate_slow.cu).
#pragma once
#include "common.cuh"
#include "deflate_header.cuh"
#include "inflate.cuh"

namespace swc {
namespace inflate {

struct SlowBits {
    const u8 *p;
    u64 nbits, pos;
    __device__ i64 avail() const { return (i64)(nbits - pos); }
    __device__ u32 bit() { u32 b = (p[pos >> 3] >> (pos & 7)) & 1; pos++; return b; }
    __device__ u32 bits(int n) { u32 v = 0; for (int i = 0; i < n; i++) v |= bit() << i; return v; }
    __device__ u32 peek32() const {      // zero past the end
        SlowBits c = *this;
        u32 v = 0;
        for (int i = 0; i < 32 && c.avail() > 0; i++) v |= c.bit() << i;
        return v;
    }
    __device__ void skip(int n) { pos += n; }
};

template <int N>
struct SlowTree {
    u16 sym[N];
    u32 code[N];        // canonical counter value (may exceed `len` bits for over-subscribed sets)
    u16 first[17], count[17];
    int max_bits;

    __device__ void build(const u8 *lens, int n) {
        max_bits = 0;
        for (int L = 0; L <= 16; L++) { first[L] = 0; count[L] = 0; }
        for (int i = 0; i < n; i++) if (lens[i] > max_bits) max_bits = lens[i];
        int k = 0, loop_bits = -1;
        long long counter = -1;
        for (int L = 1; L <= max_bits; L++) {
            first[L] = (u16)k;
            for (int s = 0; s < n; s++) {
                if (lens[s] != L) continue;
                counter += 1;                                      // Code.swift:27
                if (L != loop_bits) { counter <<= (L - loop_bits); loop_bits = L; }   // :30-33
                sym[k] = (u16)s; code[k] = (u32)counter; k++;
            }
            count[L] = (u16)(k - first[L]);
        }
    }
    // DecodingTree.findNextSymbol
    __device__ int next(SlowBits &r) const {
        i64 left = r.avail();
        u32 v = 0;
        for (int d = 1; left > 0; d++) {
            v = (v << 1) | r.bit();
            left--;
            if (d > max_bits) return -1;                           // index >= leafCount
            int hit = -1;
            const u32 mask = (1u << d) - 1;
            for (int k = first[d]; k < first[d] + count[d]; k++)
                if ((code[k] & mask) == v) hit = sym[k];           // the last writer of the heap slot wins
            if (hit >= 0) return hit;
        }
        return -1;
    }
};

// Deflate.decompress from bit `skip` of p[0, nbits / 8) into out[0, cap): returns the status, *produced = the bytes the
// stream decodes to (counted past cap: only bytes below cap are stored, and a match reads only bytes below cap) and
// *used = the bits read from `skip` on.
__device__ __forceinline__ int inflate_serial(const u8 *p, u64 nbits, u32 skip, u8 *out, u64 cap, u64 *produced, u64 *used) {
    SlowBits r;
    r.p = p;
    r.nbits = nbits;
    r.pos = skip;
    u64 op = 0;
    int status = SWC_OK;
    SlowTree<288> lit;
    SlowTree<32> dist;
    SlowTree<19> cl;
    u8 lens[320];
#define FAIL(c) do { status = (c); goto done; } while (0)
#define TRY(e) do { status = (e); if (status != SWC_OK) goto done; } while (0)
    if (r.avail() < 10) FAIL(SWC_DEFLATE_WRONG_BLOCK_TYPE);
    for (;;) {
        bool is_last;
        u32 btype;
        TRY(hdr::block_start(r, is_last, btype));
        if (btype == 0) {
            u32 length;
            TRY(hdr::stored_length(r, length));
            for (u32 i = 0; i < length; i++) { u8 b = (u8)r.bits(8); if (op < cap) out[op] = b; op++; }
        } else {
            int hlit = 288, hdist = 32;
            auto sink = [&](int n, int len, int reps) { for (int i = 0; i < reps; i++) lens[n + i] = (u8)len; };
            if (btype == 1) {
                hdr::fixed_lengths(sink);
            } else {
                u64 cl_lens;
                TRY(hdr::dynamic_counts(r, hlit, hdist, cl_lens));
                u8 cll[19];
                for (int s = 0; s < 19; s++) cll[s] = (u8)((cl_lens >> (3 * s)) & 7);
                cl.build(cll, 19);
                for (int i = 0; i < hlit + hdist; i++) lens[i] = 0;
                TRY(hdr::code_lengths(r, hlit + hdist, [&](SlowBits &b, u32) { return cl.next(b); }, sink));
            }
            lit.build(lens, hlit);
            dist.build(lens + hlit, hdist);
            for (;;) {
                const int s = lit.next(r);
                if (s < 0) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                if (s < 256) { if (op < cap) out[op] = (u8)s; op++; continue; }
                if (s == 256) break;
                if (s > 285) FAIL(SWC_DEFLATE_WRONG_SYMBOL);
                const u32 le = c_len_tab[s - 257];
                const int eb = (int)(le >> 16);
                if (r.avail() < eb) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                const u32 length = (le & 0xFFFFu) + r.bits(eb);
                const int dc = dist.next(r);
                if (dc < 0) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                if (dc > 29) FAIL(SWC_DEFLATE_WRONG_SYMBOL);
                const u32 de = c_dist_tab[dc];
                const int db = (int)(de >> 16);
                if (r.avail() < db) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                const u64 d = (u64)(de & 0xFFFFu) + r.bits(db);
                if (d > op) FAIL(SWC_ERR_REFERENCE_TRAP);
                for (u32 i = 0; i < length; i++) { if (op < cap) out[op] = out[op - d]; op++; }
            }
        }
        if (is_last) break;
    }
done:
#undef FAIL
#undef TRY
    if (status == SWC_OK && op > OUT_MAX) status = SWC_ERR_UNSUPPORTED;            // the Huffman stages' limit (inflate.cuh)
    if (status == SWC_OK && op > cap) status = SWC_ERR_OUTPUT_OVERFLOW;
    *produced = op;
    *used = r.pos - skip;
    return status;
}

}  // namespace inflate
}  // namespace swc
