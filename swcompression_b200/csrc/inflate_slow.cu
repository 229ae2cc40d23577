// inflate_slow.cu — generic serial Deflate decoder, one thread per unit, for the (malformed) streams the fast path
// cannot take: Huffman code sets whose Kraft sum exceeds 1.  The reference accepts those: Code.huffmanCodes never
// validates (Sources/Common/CodingTree/Code.swift:15-39), DecodingTree.init overwrites heap slots
// (DecodingTree.swift:22-32) and findNextSymbol returns at the first leaf on the path (:36-50) — so "shortest prefix
// wins, and among equal paths the code assigned last wins".  That rule is emulated here directly on the sorted code
// list (no 2^16-slot heap per tree).  Only units the Huffman stage (K1L / K1w) flagged SWC_INTERNAL_NEEDS_SLOW are touched.
#include "common.cuh"
#include "deflate_tables.cuh"
#include "inflate.cuh"

namespace swc {
namespace inflate {

struct SlowBits {
    const u8 *p;
    u64 nbits, pos;
    __device__ u64 left() const { return nbits - pos; }
    __device__ u32 bit() { u32 b = (p[pos >> 3] >> (pos & 7)) & 1; pos++; return b; }
    __device__ u32 bits(int n) { u32 v = 0; for (int i = 0; i < n; i++) v |= bit() << i; return v; }
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
        u64 left = r.left();
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

__global__ void __launch_bounds__(64) inflate_slow_kernel(BatchArgs a) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= a.n) return;
    if (a.status[unit] != SWC_INTERNAL_NEEDS_SLOW) return;
    SlowBits r;
    const u32 skip = a.start_bits ? a.start_bits[unit] : 0;
    r.p = a.in_base + a.in_off[unit];
    r.nbits = a.in_len[unit] * 8;
    r.pos = skip;
    u8 *out = a.out_base + a.out_off[unit];
    const u64 cap = a.out_cap[unit];
    u64 op = 0;
    int status = SWC_OK;
    SlowTree<288> lit;
    SlowTree<32> dist;
    SlowTree<19> cl;
    u8 lens[320];
#define FAIL(c) do { status = (c); goto done; } while (0)
    if (r.left() < 10) FAIL(SWC_DEFLATE_WRONG_BLOCK_TYPE);
    for (;;) {
        if (r.left() < 3) FAIL(SWC_ERR_REFERENCE_TRAP);
        const u32 is_last = r.bit();
        const u32 btype = r.bits(2);
        if (btype == 0) {
            r.pos = (r.pos + 7) & ~7ull;
            if (r.left() < 32) FAIL(SWC_DEFLATE_WRONG_UNCOMPRESSED_BLOCK_LENGTHS);
            const u32 length = r.bits(16), nlength = r.bits(16);
            if (length & nlength) FAIL(SWC_DEFLATE_WRONG_UNCOMPRESSED_BLOCK_LENGTHS);
            if ((r.left() >> 3) < length) FAIL(SWC_DEFLATE_WRONG_UNCOMPRESSED_BLOCK_LENGTHS);
            for (u32 i = 0; i < length; i++) { u8 b = (u8)r.bits(8); if (op < cap) out[op] = b; op++; }
        } else if (btype == 3) {
            FAIL(SWC_DEFLATE_WRONG_BLOCK_TYPE);
        } else {
            int hlit = 288, hdist = 32;
            if (btype == 1) {
                for (int i = 0; i < 320; i++) lens[i] = (u8)static_len(i);
            } else {
                if (r.left() < 14) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                hlit = (int)r.bits(5) + 257;
                if (hlit > 286) FAIL(SWC_DEFLATE_WRONG_SYMBOL);
                hdist = (int)r.bits(5) + 1;
                const int hclen = (int)r.bits(4) + 4;
                if (r.left() < (u64)(3 * hclen)) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                u8 cll[19];
                for (int i = 0; i < 19; i++) cll[i] = 0;
                for (int i = 0; i < hclen; i++) cll[c_cl_order[i]] = (u8)r.bits(3);
                cl.build(cll, 19);
                const int count = hlit + hdist;
                for (int i = 0; i < count; i++) lens[i] = 0;
                int n = 0;
                while (n < count) {
                    const int s = cl.next(r);
                    if (s < 0) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                    if (s <= 15) { lens[n++] = (u8)s; }
                    else if (s == 16 && n > 0) {
                        if (r.left() < 2) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                        const int c = (int)r.bits(2) + 3;
                        if (n + c > count) FAIL(SWC_DEFLATE_WRONG_SYMBOL);
                        for (int i = 0; i < c; i++) lens[n + i] = lens[n - 1];
                        n += c;
                    } else if (s == 17) {
                        if (r.left() < 3) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                        n += (int)r.bits(3) + 3;
                    } else if (s == 18) {
                        if (r.left() < 7) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                        n += (int)r.bits(7) + 11;
                    } else FAIL(SWC_DEFLATE_WRONG_SYMBOL);
                }
                if (n != count) FAIL(SWC_DEFLATE_WRONG_SYMBOL);
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
                if (r.left() < (u64)eb) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                const u32 length = (le & 0xFFFFu) + r.bits(eb);
                const int dc = dist.next(r);
                if (dc < 0) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                if (dc > 29) FAIL(SWC_DEFLATE_WRONG_SYMBOL);
                const u32 de = c_dist_tab[dc];
                const int db = (int)(de >> 16);
                if (r.left() < (u64)db) FAIL(SWC_DEFLATE_SYMBOL_NOT_FOUND);
                const u64 d = (u64)(de & 0xFFFFu) + r.bits(db);
                if (d > op) FAIL(SWC_ERR_REFERENCE_TRAP);
                for (u32 i = 0; i < length; i++) { if (op < cap) out[op] = out[op - d]; op++; }
            }
        }
        if (is_last) break;
    }
done:
#undef FAIL
    if (status == SWC_OK && op > cap) status = SWC_ERR_OUTPUT_OVERFLOW;
    a.out_len[unit] = op;
    a.consumed_bits[unit] = r.pos - skip;
    a.status[unit] = status;
    a.rec_count[unit] = REC_DIRECT;      // the output is written: K2 leaves the unit alone
}

void launch_slow(const BatchArgs &a, cudaStream_t stream) {
    inflate_slow_kernel<<<(unsigned)((a.n + 63) / 64), 64, 0, stream>>>(a);
    count_launch();
}

}  // namespace inflate
}  // namespace swc
