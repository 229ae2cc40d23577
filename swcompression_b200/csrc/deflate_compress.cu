// deflate_compress.cu — batched Deflate compression for sm_90a.  Replaces Deflate.compress(data:) (reference
// Sources/Deflate/Deflate+Compress.swift:22-197) and reproduces its output byte for byte: one block, stored or static
// Huffman, from the reference's greedy parse over an exact 3-byte key table.
//
// Like the LZ4 compressor (lz4_compress.cu) the parse is split into parallel work and a cheap serial walk (DESIGN §4.10):
//   link_kernel   — ONE WARP PER TILE of TILE positions, with REACH positions of halo in front: link[p] = distance to the
//      nearest earlier position with the same 3-byte key, 0 if there is none within REACH.  Keys come from aligned word
//      loads.  A forward pass over the halo and the tile threads every position onto a hash-bucket chain whose entries
//      carry the rest of the key (the bucket and that tag are a bijection of the key), so the walk to the nearest equal
//      key compares tags in the chain and never goes back to the input.
//   parse_kernel  — ONE THREAD PER UNIT: the reference's loop with the table lookup replaced by a walk down link[] to the
//      first visited position.  Writes {literal run : 32 | length : 9 | distance : 16} records, the exact static bit
//      count, the stored/static choice, out_len and status, and a checkpoint every CHUNK input bytes.
//   emit_kernel   — ONE WARP PER CHUNK: from its checkpoint the warp places 32 symbols at a time with warp scans, gathers
//      their bits in shared memory and stores every aligned 32-bit word that lies wholly inside the chunk once.  The word
//      a chunk shares with its neighbour goes to a seam slot.
//   seam_kernel   — ONE THREAD PER CHUNK: ORs the two halves of each shared word and stores it, clipping the unit's last
//      word to out_len.
// Every result depends only on the unit's bytes, never on the grid, the tiling or the slicing.
#include "common.cuh"
#include "deflate_compress.cuh"
#include "deflate_tables.cuh"

namespace swc {
namespace deflatec {

namespace {

constexpr u32 EMPTY = 0xFFFFFFFFu;
constexpr int HBITS = 12;                       // 4096 buckets: 16 KiB of shared memory per warp, 2 warps per CTA

struct Checkpoint { u32 rec, off, pos, pad; u64 bit; };   // first symbol at or after the chunk's first byte
static_assert(sizeof(Checkpoint) == CHECKPOINT_BYTES, "unit_scratch counts checkpoints of this size");

// ---- the link builder (a template over key width and reach, so other LZ77 parses can share it) ----

// the KB bytes at p as an integer (byte p lowest), from aligned words: any alignment, and no byte outside [p, p + KB)
// is read except inside the aligned words that hold those bytes
template <int KB> __device__ __forceinline__ u32 key_at(const u8 *p) {
    const uintptr_t a = (uintptr_t)p;
    const u32 *w = (const u32 *)(a & ~(uintptr_t)3);
    const u32 sh = (u32)(a & 3) * 8;
    const u32 lo = w[0];
    const u32 v = sh + 8 * KB > 32 ? __funnelshift_r(lo, w[1], sh) : lo >> sh;
    return KB == 4 ? v : v & ((1u << (8 * KB)) - 1u);
}

template <int KB> struct Keying {
    static constexpr int KBITS = 8 * KB, TBITS = KBITS - HBITS;
    // chain entry: distance to the previous position of the same bucket (16 bits) | tag << 16
    typedef typename std::conditional<(TBITS + 16 <= 32), u32, u64>::type Entry;
    // k -> k * odd (mod 2^KBITS) is a bijection, so (bucket, tag) identifies the key
    __device__ __forceinline__ static u32 mix(u32 k) {
        const u32 x = k * 0x9E3779B1u;
        return KB == 4 ? x : x & ((1u << KBITS) - 1u);
    }
};

// link[p] for p in [t0, t1): the nearest earlier position with the same KB-byte key, at most R back (0: none).  One warp;
// `chain` holds one entry per position of [r0, t1) with r0 = max(0, t0 - R); `head` has 1 << HBITS entries.
template <int KB, u32 R>
__device__ __forceinline__ void build_links(const u8 *src, u32 t0, u32 t1, u16 *link,
                                            typename Keying<KB>::Entry *chain, u32 *head) {
    static_assert(R <= 65535, "distances are 16-bit");
    typedef typename Keying<KB>::Entry Entry;
    constexpr u32 HSIZE = 1u << HBITS;
    const u32 lane = lane_id();
    for (u32 i = lane; i < HSIZE; i += 32) head[i] = EMPTY;
    __syncwarp();
    const u32 r0 = t0 > R ? t0 - R : 0;
    for (u32 base = r0; base < t1; base += 32) {
        const u32 p = base + lane;
        const bool valid = p < t1;
        const u32 x = valid ? Keying<KB>::mix(key_at<KB>(src + p)) : 0;
        const u32 h = valid ? x >> Keying<KB>::TBITS : HSIZE + lane;
        const u32 tag = x & ((1u << Keying<KB>::TBITS) - 1u);
        const u32 m = __match_any_sync(SWC_FULL, h);
        const u32 lower = m & ((1u << lane) - 1u);
        u32 bd = 0;
        if (valid) {
            const u32 q = lower ? base + 31 - __clz(lower) : head[h];
            if (q != EMPTY && p - q <= R) bd = p - q;
            chain[p - r0] = (Entry)bd | (Entry)tag << 16;
        }
        __syncwarp();
        if (valid && (m >> lane) == 1u) head[h] = p;     // the group's last position becomes the bucket head
        if (valid && p >= t0) {
            // down the bucket chain to the first entry with the same tag; every same-key position within R is on it
            u32 q = p, d = 0;
            while (bd) {
                q -= bd;
                if (p - q > R) break;
                const Entry e = chain[q - r0];
                if ((u32)(e >> 16) == tag) { d = p - q; break; }
                bd = (u32)e & 0xFFFFu;
            }
            link[p] = (u16)d;
        }
        __syncwarp();
    }
}

typedef Keying<3>::Entry Entry3;
static_assert(sizeof(Entry3) == CHAIN_ENTRY_BYTES, "unit_scratch counts chain entries of this size");

// scratch of one unit: header | link (u16 per keyed position) | visited bitmap | checkpoints | seam words |
// link-builder chains, later reused for the records
struct Scr {
    u64 *hdr;                 // [0] records, [1] stream bits including the end-of-block code, [2] stored
    u16 *link; u32 *vis; Checkpoint *cp; u32 *seam; u8 *big;
    __device__ __forceinline__ Scr(u8 *base, u64 n) {
        hdr = (u64 *)base;
        link = (u16 *)(base + 256);
        vis = (u32 *)((u8 *)link + a256(2 * keyed(n)));
        cp = (Checkpoint *)((u8 *)vis + a256(4 * ((keyed(n) + 31) / 32)));
        seam = (u32 *)((u8 *)cp + a256(sizeof(Checkpoint) * (unit_chunks(n) + 1)));
        big = (u8 *)seam + a256(8 * unit_chunks(n));
    }
    __device__ __forceinline__ u64 *rec() const { return (u64 *)big; }
};

// tile t reads its chain from entry t * TILE + (t - 1) * REACH (tile 0 has no halo)
__device__ __forceinline__ u64 chain_off(u32 t) { return (u64)t * TILE + (t ? (u64)(t - 1) * REACH : 0); }

// the unit j of a slice whose range of `start` (count + 1 prefix sums) holds g
__device__ __forceinline__ u64 locate(const u64 *start, u64 count, u64 g) {
    u64 lo = 0, hi = count;
    while (hi - lo > 1) {
        const u64 mid = (lo + hi) >> 1;
        if (start[mid] <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// fixed-code symbols (RFC 1951 3.2.6), with the bit counts of staticHuffmanBitSize (Deflate+Compress.swift:44-72)
__device__ __forceinline__ u32 len_sym(u32 len) {                 // index into c_len_tab: code 257 + index
    u32 s = 0;
#pragma unroll
    for (u32 b = 16; b; b >>= 1)
        if (s + b <= 28 && (inflate::c_len_tab[s + b] & 0xFFFFu) <= len) s += b;
    return s;
}
__device__ __forceinline__ u32 dist_sym(u32 dist) {
    u32 s = 0;
#pragma unroll
    for (u32 b = 16; b; b >>= 1)
        if (s + b <= 29 && (inflate::c_dist_tab[s + b] & 0xFFFFu) <= dist) s += b;
    return s;
}
__device__ __forceinline__ u32 lit_bits(u32 v) { return v < 144 ? 8u : 9u; }
__device__ __forceinline__ u32 match_bits(u32 len, u32 dist) {
    const u32 ls = len_sym(len), ds = dist_sym(dist);
    return (ls <= 22 ? 7u : 8u) + (inflate::c_len_tab[ls] >> 16) + 5u + (inflate::c_dist_tab[ds] >> 16);
}
// the bits of one symbol in stream order (Huffman codes reversed, extra bits as numbers): value, and count in *nb
__device__ __forceinline__ u32 lit_code(u32 v, u32 *nb) {
    const u32 c = v < 144 ? 0x30u + v : 0x190u + (v - 144u);
    *nb = lit_bits(v);
    return __brev(c) >> (32 - *nb);
}
__device__ __forceinline__ u32 match_code(u32 len, u32 dist, u32 *nb) {
    const u32 ls = len_sym(len), ds = dist_sym(dist);
    const u32 code = 257u + ls;
    const u32 cl = code <= 279 ? 7u : 8u;
    const u32 cv = code <= 279 ? code - 256u : 0xC0u + (code - 280u);
    const u32 lt = inflate::c_len_tab[ls], dt = inflate::c_dist_tab[ds];
    const u32 lx = lt >> 16, dx = dt >> 16;
    u32 v = __brev(cv) >> (32 - cl);
    u32 at = cl;
    v |= (len - (lt & 0xFFFFu)) << at; at += lx;
    v |= (__brev(ds) >> 27) << at; at += 5;
    v |= (dist - (dt & 0xFFFFu)) << at; at += dx;
    *nb = at;
    return v;
}

struct Unit {
    const u8 *src;
    u64 n;
    __device__ __forceinline__ Unit(const Args &a, u64 u) : src(a.in_base + a.in_off[u]), n(a.in_len[u]) {}
};

// [S_c, S_{c+1}): the bits chunk c writes (chunk 0 starts with the block header, the last chunk ends with end-of-block)
__device__ __forceinline__ u64 chunk_begin(const Scr &s, u32 c) { return c ? s.cp[c].bit : 0; }
__device__ __forceinline__ u64 chunk_end(const Scr &s, u32 c, u32 nch) { return c + 1 == nch ? s.hdr[1] : s.cp[c + 1].bit; }

}  // namespace

__global__ void __launch_bounds__(64) link_kernel(Args a, u64 first, u64 count, u8 *scr, Plan p) {
    __shared__ u32 heads[2][1u << HBITS];
    const u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (g >= p.tile_start[count]) return;
    const u64 j = locate(p.tile_start, count, g);
    const u32 t = (u32)(g - p.tile_start[j]);
    const Unit un(a, first + j);
    const Scr s(scr + p.scr_off[j], un.n);
    const u32 nk = (u32)keyed(un.n);
    const u32 t0 = t * TILE, t1 = nk - t0 < TILE ? nk : t0 + TILE;
    // the parse's visited bitmap starts empty: each tile clears its own words
    const u32 w1 = t1 == nk ? (nk + 31) / 32 : t1 / 32;
    for (u32 w = t0 / 32 + lane_id(); w < w1; w += 32) s.vis[w] = 0;
    build_links<3, REACH>(un.src, t0, t1, s.link, (Entry3 *)s.big + chain_off(t), heads[(threadIdx.x >> 5) & 1]);
}

__global__ void __launch_bounds__(128) parse_kernel(Args a, u64 first, u64 count, u8 *scr, Plan p) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const u64 u = first + j;
    const Unit un(a, u);
    if (un.n >= MAX_UNIT) { a.out_len[u] = 0; a.status[u] = SWC_ERR_UNSUPPORTED; return; }
    const Scr s(scr + p.scr_off[j], un.n);
    const u8 *d = un.src;
    const u32 n = (u32)un.n, nch = (u32)unit_chunks(n);
    u64 *rec = s.rec();
    u64 bits = 3;                                                                 // BFINAL, BTYPE (:96-97)
    u32 i = 0, lit = 0, nrec = 0, next = 1;
    s.cp[0] = Checkpoint{0, 0, 0, 0, bits};
    auto mark = [&](u32 off) {
        while (next < nch && i >= next * CHUNK) s.cp[next++] = Checkpoint{nrec, off, i, 0, bits};
    };
    while (i + 2 < n) {                                                           // :143
        mark(lit);
        // the table's entry for key(i) is the nearest earlier visited position with that key (DESIGN §4.10)
        u32 q = i, dd = s.link[i];
        bool found = false;
        while (dd) {
            q -= dd;
            if (i - q > REACH) break;                                             // :166 (no nearer visited one exists)
            if ((s.vis[q >> 5] >> (q & 31)) & 1u) { found = true; break; }
            dd = s.link[q];
        }
        s.vis[i >> 5] |= 1u << (i & 31);                                          // :151 / :158
        if (!found) { bits += lit_bits(d[i]); lit++; i++; continue; }
        u32 len = 3;                                                              // :161-175
        while (i + len < n && len < 258 && d[i + len] == d[q + len]) len++;
        rec[nrec++] = (u64)lit | (u64)len << 32 | (u64)(i - q) << 41;
        bits += match_bits(len, i - q);
        i += len;                                                                 // :181
        lit = 0;
    }
    for (; i < n; i++, lit++) { mark(lit); bits += lit_bits(d[i]); }              // :186-191
    if (lit) rec[nrec++] = lit;
    while (next <= nch) s.cp[next++] = Checkpoint{nrec, 0, n, 0, bits};
    bits += 7;                                                                    // end of block (:194)
    const u64 static_bytes = (bits + 7) / 8;
    const bool stored = (u64)n + 5 <= static_bytes && (u64)n + 5 <= 65535;        // :35
    s.hdr[0] = nrec; s.hdr[1] = bits; s.hdr[2] = stored;
    const u64 size = stored ? (u64)n + 5 : static_bytes;
    a.out_len[u] = size;
    a.status[u] = size > a.out_cap[u] ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
}

__global__ void __launch_bounds__(128) emit_kernel(Args a, u64 first, u64 count, u8 *scr, Plan p) {
    __shared__ u32 stage[4][64];
    const u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (g >= p.chunk_start[count]) return;
    const u64 j = locate(p.chunk_start, count, g);
    const u64 u = first + j;
    if (a.status[u] != SWC_OK) return;
    const u32 c = (u32)(g - p.chunk_start[j]);
    const u32 lane = lane_id();
    const Unit un(a, u);
    const u32 n = (u32)un.n, nch = (u32)unit_chunks(n);
    const Scr s(scr + p.scr_off[j], n);
    u8 *out = a.out_base + a.out_off[u];
    if (s.hdr[2]) {                                                               // createUncompressedBlock :74-83
        if (c == 0 && lane < 5) {
            const u32 nl = n ^ 0xFFFFu;
            out[lane] = (u8)(lane == 0 ? 1u : lane == 1 ? n : lane == 2 ? n >> 8 : lane == 3 ? nl : nl >> 8);
        }
        const u32 e = n - c * CHUNK < CHUNK ? n : (c + 1) * CHUNK;
        for (u32 k = c * CHUNK + lane; k < e; k += 32) out[5 + k] = un.src[k];
        return;
    }
    u32 *buf = stage[(threadIdx.x >> 5) & 3];
    buf[lane] = 0; buf[lane + 32] = 0;
    __syncwarp();
    const u64 sb = chunk_begin(s, c), eb = chunk_end(s, c, nch);
    const u64 wbase = sb >> 5;
    u32 *out32 = (u32 *)out;
    u64 flushed = wbase;
    auto put = [&](u64 at, u32 v) {
        const u64 x = (u64)v << (at & 31);
        const u64 w = at >> 5;
        if ((u32)x) atomicOr(&buf[(w - wbase) & 63], (u32)x);
        if ((u32)(x >> 32)) atomicOr(&buf[(w + 1 - wbase) & 63], (u32)(x >> 32));
    };
    // words below `lim` are complete: whole ones go out, the first one goes to the seam if the previous chunk shares it
    auto flush = [&](u64 lim) {
        __syncwarp();
        for (u64 w = flushed + lane; w < lim; w += 32) {
            u32 &slot = buf[(w - wbase) & 63];
            if (w == wbase && (sb & 31)) s.seam[2 * c] = slot;
            else out32[w] = slot;
            slot = 0;
        }
        if (lim > flushed) flushed = lim;
        __syncwarp();
    };
    const u64 *rec = s.rec();
    const u32 nrec = (u32)s.hdr[0];
    const Checkpoint cb = s.cp[c], ce = s.cp[c + 1];
    u32 r = cb.rec, o = cb.off, pos = cb.pos;
    u64 cur = cb.bit;
    if (c == 0 && lane == 0) put(0, 3u);                                          // BFINAL 1, BTYPE 01
    while (r < ce.rec || (r == ce.rec && o < ce.off)) {
        const u32 k = r + lane;
        const u64 rv = k < nrec && k <= ce.rec ? rec[k] : 0;
        const u32 lit = (u32)rv, len = (u32)(rv >> 32) & 511u, dist = (u32)(rv >> 41);
        const u32 so = lane == 0 ? o : 0;
        const u32 full = lit + (len ? 1u : 0u);
        const u32 lim = k < ce.rec ? full : k == ce.rec ? ce.off : 0u;
        const u32 nsym = k < nrec && lim > so ? lim - so : 0u;
        const u32 adv = lit - so + len;
        u32 cs = nsym, ca = adv;
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
            const u32 vs = __shfl_up_sync(SWC_FULL, cs, dd), va = __shfl_up_sync(SWC_FULL, ca, dd);
            if (lane >= (u32)dd) { cs += vs; ca += va; }
        }
        const u32 total = __shfl_sync(SWC_FULL, cs, 31);
        const u32 take = total < 32 ? total : 32;
        // lane l places the l-th symbol: its record is the first whose running symbol count exceeds l
        u32 idx = 0;
#pragma unroll
        for (u32 b = 16; b; b >>= 1)
            if (__shfl_sync(SWC_FULL, cs, idx + b - 1) <= lane) idx += b;
        idx = idx > 31 ? 31 : idx;
        const u32 r_cs = __shfl_sync(SWC_FULL, cs, idx), r_ns = __shfl_sync(SWC_FULL, nsym, idx);
        const u32 r_so = __shfl_sync(SWC_FULL, so, idx), r_lit = __shfl_sync(SWC_FULL, lit, idx);
        const u32 r_len = __shfl_sync(SWC_FULL, len, idx), r_dist = __shfl_sync(SWC_FULL, dist, idx);
        const u32 r_pos = pos + __shfl_sync(SWC_FULL, ca, idx) - __shfl_sync(SWC_FULL, adv, idx);
        const u32 off = r_so + lane - (r_cs - r_ns);
        const bool is_lit = off < r_lit;
        const u32 at = r_pos + (off - r_so);                                      // input position of the symbol
        u32 nb = 0, v = 0;
        if (lane < take) v = is_lit ? lit_code(un.src[at], &nb) : match_code(r_len, r_dist, &nb);
        u32 bo = nb;
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
            const u32 t = __shfl_up_sync(SWC_FULL, bo, dd);
            if (lane >= (u32)dd) bo += t;
        }
        if (nb) put(cur + bo - nb, v);
        cur += __shfl_sync(SWC_FULL, bo, 31);
        // the cursor moves past the last placed symbol
        const u32 l_idx = __shfl_sync(SWC_FULL, idx, take - 1), l_off = __shfl_sync(SWC_FULL, off, take - 1);
        const u32 l_at = __shfl_sync(SWC_FULL, at, take - 1), l_lit = __shfl_sync(SWC_FULL, r_lit, take - 1);
        const u32 l_len = __shfl_sync(SWC_FULL, r_len, take - 1);
        pos = l_off < l_lit ? l_at + 1 : l_at + l_len;
        r += l_idx;
        o = l_off + 1;
        if (o >= l_lit + (l_len ? 1u : 0u)) { r++; o = 0; }
        flush(cur >> 5);
    }
    flush(eb >> 5);
    if (eb & 31) {
        const u32 v = buf[((eb >> 5) - wbase) & 63];
        if (lane == 0) s.seam[2 * c + ((eb >> 5) == wbase && (sb & 31) ? 0 : 1)] = v;
    }
}

__global__ void __launch_bounds__(256) seam_kernel(Args a, u64 first, u64 count, u8 *scr, Plan p) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= p.chunk_start[count]) return;
    const u64 j = locate(p.chunk_start, count, g);
    const u64 u = first + j;
    if (a.status[u] != SWC_OK) return;
    const u32 c = (u32)(g - p.chunk_start[j]);
    const u64 n = a.in_len[u];
    const u32 nch = (u32)unit_chunks(n);
    const Scr s(scr + p.scr_off[j], n);
    if (s.hdr[2]) return;
    const u64 sb = chunk_begin(s, c), eb = chunk_end(s, c, nch);
    // chunk c owns the word holding its last bits unless they all sit in the word it shares with chunk c - 1
    if (!(eb & 31) || ((eb >> 5) == (sb >> 5) && (sb & 31))) return;
    const u64 w = eb >> 5;
    u32 v = s.seam[2 * c + 1];
    if (c + 1 < nch) v |= s.seam[2 * (c + 1)];
    u8 *out = a.out_base + a.out_off[u];
    const u64 len = a.out_len[u];
    if (4 * w + 4 <= len) { ((u32 *)out)[w] = v; return; }
    for (u64 b = 4 * w; b < len; b++) out[b] = (u8)(v >> (8 * (b - 4 * w)));
}

int run(const Args &a, u64 first, u64 count, u8 *scr, const Plan &p, cudaStream_t s) {
    if (count == 0) return SWC_OK;
    timing_mark(s);
    if (p.tiles) link_kernel<<<(unsigned)((p.tiles * 32 + 63) / 64), 64, 0, s>>>(a, first, count, scr, p);
    timing_mark(s);
    parse_kernel<<<(unsigned)((count + 127) / 128), 128, 0, s>>>(a, first, count, scr, p);
    timing_mark(s);
    if (p.chunks) {
        emit_kernel<<<(unsigned)((p.chunks * 32 + 127) / 128), 128, 0, s>>>(a, first, count, scr, p);
        timing_mark(s);
        seam_kernel<<<(unsigned)((p.chunks + 255) / 256), 256, 0, s>>>(a, first, count, scr, p);
        timing_mark(s);
    }
    count_launch(p.tiles ? 4 : 3);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace deflatec
}  // namespace swc
