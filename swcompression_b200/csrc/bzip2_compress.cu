// bzip2_compress.cu — batched BZip2 compression that writes the streams of BZip2.compress(data:blockSize:)
// (BZip2+Compress.swift:44-262) byte for byte.  Every raw block of every unit of a slice is one work item; DESIGN §4.11
// proves the stages equal to the reference.
//   rle_kernel     — ONE THREAD PER BLOCK: initialRle (:265-283), the block's bzip2 CRC and its used-byte map.
//   sort_kernel    — ONE CTA PER BLOCK: sorts the cyclic rotations of the RLE1 bytes by prefix doubling (8-byte keys,
//                    then (rank[i], rank[i + h]) pairs) with a stable CTA-wide radix sort, and stops after a round that
//                    splits no group.  Writes the BWT bytes and the pointer (the rank of rotation 0).
//   mtf_kernel     — ONE WARP PER BLOCK: mtfRle (:299-349).  The 256-entry list lives 8 bytes per lane.
//   group_kernel   — ONE THREAD PER 50-SYMBOL GROUP: the candidate table of BZip2.lengths(from:), built with a heap keyed
//                    (frequency ascending, symbol descending), kept as its length histogram.
//   select_kernel  — ONE WARP PER BLOCK: the greedy table choice (:93-148), each group's data bit offset, and the block's
//                    exact bit count.
//   layout_kernel  — ONE THREAD PER UNIT: block bit offsets, stream CRC, out_len and status; writes stream header and EOS.
//   header_kernel  — ONE THREAD PER BLOCK: the block header (:150-221).
//   emit_kernel    — ONE THREAD PER GROUP: the group's codes (:223-240).
//   copy_kernel    — ONE CTA PER UNIT AND 64 KiB CHUNK: staging words to the caller's output region for units that fit.
// Blocks are not byte aligned, so every stage writes into zero-filled 32-bit staging words with atomicOr; bit ranges of
// different writers never overlap.
#include "bzip2_compress.cuh"

namespace swc {
namespace bzip2c {

namespace {

constexpr int SORT_WARPS = 16;

struct BlockMeta {
    u32 crc, n, ptr, nsym, maxsym, ntab, nsel, hbits;
    u32 used[8];
    u64 bit_off, dbits;
    u16 tab[6][12];                      // each table as its length histogram (index = code length)
};

struct Blk {
    u8 *rle; u64 *key[2]; u32 *idx[2]; u32 *rank; u8 *bwt; u16 *sym;
    __device__ Blk(const Slice &sl, const BlockPlan &bp) {
        const u64 c = (bp.cap + 8 + 255) & ~255ull;
        u8 *b = (u8 *)(uintptr_t)bp.scr;
        rle = b; key[0] = (u64 *)(b + c); key[1] = (u64 *)(b + 9 * c);
        idx[0] = (u32 *)(b + 17 * c); idx[1] = (u32 *)(b + 21 * c); rank = (u32 *)(b + 25 * c);
        bwt = (u8 *)key[0]; sym = (u16 *)key[1];
    }
};

__device__ __forceinline__ BlockMeta *meta_of(const Slice &sl, u64 b) { return (BlockMeta *)sl.meta + b; }
__device__ __forceinline__ u16 *cand_of(const Slice &sl, u64 g) { return (u16 *)sl.groups + 12 * g; }
__device__ __forceinline__ u8 *sel_of(const Slice &sl) { return sl.groups + 24 * sl.ngroups; }
__device__ __forceinline__ u32 *goff_of(const Slice &sl) { return (u32 *)(sl.groups + ((25 * sl.ngroups + 255) & ~255ull)); }

// MSB-first bit writer into zero-filled staging words: whole words are ORed in once
struct BitW {
    u32 *w; u64 word; u64 acc; int fill;
    __device__ BitW(u32 *words, u64 pos) : w(words), word(pos >> 5), acc(0), fill((int)(pos & 31)) {}
    __device__ void flush() { const u32 v = (u32)(acc >> 32); if (v) atomicOr(w + word, __byte_perm(v, 0, 0x0123)); }
    __device__ void put(u32 v, int n) {  // n <= 32
        if (!n) return;
        acc |= (u64)v << (64 - fill - n);
        fill += n;
        if (fill >= 32) { flush(); word++; acc <<= 32; fill -= 32; }
    }
    __device__ void put64(u64 v, int n) { if (n > 32) { put((u32)(v >> 32), n - 32); n = 32; } put((u32)v, n); }
    __device__ void finish() { if (fill) flush(); }
};

__device__ __forceinline__ u64 block_of_group(const Slice &sl, u64 g) {
    u64 lo = 0, hi = sl.nblocks;         // the last block whose group0 <= g
    while (hi - lo > 1) { const u64 mid = (lo + hi) / 2; if (sl.blocks[mid].group0 <= g) lo = mid; else hi = mid; }
    return lo;
}

// ---- stage 1 ----
__global__ void __launch_bounds__(128) rle_kernel(Args a, u64 first, Slice sl) {
    __shared__ u32 tab[256];
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) {
        u32 c = i << 24;
        for (int k = 0; k < 8; k++) c = (c & 0x80000000u) ? (c << 1) ^ 0x04C11DB7u : c << 1;
        tab[i] = c;
    }
    __syncthreads();
    const u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= sl.nblocks) return;
    const BlockPlan bp = sl.blocks[b];
    const u64 unit = first + bp.unit;
    const u8 *src = a.in_base + a.in_off[unit] + (u64)bp.index * RAW_PER_LEVEL * a.level;
    Blk k(sl, bp);
    u32 crc = 0xFFFFFFFFu, o = 0, used[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (u32 i = 0; i < bp.raw;) {
        const u8 v = src[i];
        crc = (crc << 8) ^ tab[(crc >> 24) ^ v];
        u32 run = 1;
        while (i + run < bp.raw && run < 255 && src[i + run] == v) { crc = (crc << 8) ^ tab[(crc >> 24) ^ v]; run++; }
        for (u32 r = 0; r < run && r < 4; r++) k.rle[o++] = v;
        used[v >> 5] |= 1u << (v & 31);
        if (run >= 4) { const u32 x = run - 4; k.rle[o++] = (u8)x; used[x >> 5] |= 1u << (x & 31); }
        i += run;
    }
    BlockMeta *m = meta_of(sl, b);
    m->crc = ~crc; m->n = o;
    for (int j = 0; j < 8; j++) m->used[j] = used[j];
}

// ---- stage 2: rotation sort ----
struct SortShared {
    u32 hist[SORT_WARPS][256];
    u32 tot[256];
    u32 seg_max[SORT_WARPS], seg_cnt[SORT_WARPS];
    int uniform;
    u32 groups;
};

__device__ __forceinline__ void seg_bounds(u32 n, u32 &lo, u32 &hi) {
    const u32 seg = ((n + SORT_WARPS - 1) / SORT_WARPS + 31) & ~31u, w = threadIdx.x >> 5;
    lo = min(n, w * seg); hi = min(n, lo + seg);
}

// one stable pass over the 8-bit digit at `shift`; false (and nothing moved) when every key has the same digit
__device__ bool radix_pass(SortShared &sh, const u64 *kin, const u32 *iin, u64 *kout, u32 *iout, u32 n, int shift) {
    const u32 w = threadIdx.x >> 5, lane = lane_id();
    u32 lo, hi;
    seg_bounds(n, lo, hi);
    for (u32 t = threadIdx.x; t < SORT_WARPS * 256; t += blockDim.x) (&sh.hist[0][0])[t] = 0;
    if (threadIdx.x == 0) sh.uniform = 0;
    __syncthreads();
    for (u32 j = lo + lane; j < hi; j += 32) atomicAdd(&sh.hist[w][(kin[j] >> shift) & 255], 1u);
    __syncthreads();
    if (threadIdx.x < 256) {
        u32 run = 0;
        for (int v = 0; v < SORT_WARPS; v++) { const u32 t = sh.hist[v][threadIdx.x]; sh.hist[v][threadIdx.x] = run; run += t; }
        sh.tot[threadIdx.x] = run;
        if (run == n) sh.uniform = 1;
    }
    __syncthreads();
    const bool uniform = sh.uniform;
    __syncthreads();
    if (uniform) return false;
    if (w == 0) {                        // exclusive scan of the 256 digit totals, 8 per lane
        u32 v[8], s = 0;
        for (int k = 0; k < 8; k++) { v[k] = sh.tot[8 * lane + k]; s += v[k]; }
        u32 inc = s;
        for (int d = 1; d < 32; d <<= 1) { const u32 t = __shfl_up_sync(SWC_FULL, inc, d); if (lane >= (u32)d) inc += t; }
        u32 p = inc - s;
        for (int k = 0; k < 8; k++) { sh.tot[8 * lane + k] = p; p += v[k]; }
    }
    __syncthreads();
    if (threadIdx.x < 256)
        for (int v = 0; v < SORT_WARPS; v++) sh.hist[v][threadIdx.x] += sh.tot[threadIdx.x];
    __syncthreads();
    for (u32 base = lo; base < hi; base += 32) {
        const u32 j = base + lane;
        const bool valid = j < hi;
        u64 key = 0; u32 id = 0;
        if (valid) { key = kin[j]; id = iin[j]; }
        const u32 d = valid ? (u32)((key >> shift) & 255) : 256 + lane;
        const u32 peers = __match_any_sync(SWC_FULL, d);
        if (valid) {
            const u32 pos = sh.hist[w][d] + __popc(peers & ((1u << lane) - 1));
            kout[pos] = key; iout[pos] = id;
        }
        __syncwarp();
        if (valid && lane == 31 - __clz(peers)) sh.hist[w][d] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    return true;
}

// rank[idx[j]] = the first sorted position whose key equals key[j]; returns the number of groups
__device__ u32 rank_groups(SortShared &sh, const u64 *key, const u32 *idx, u32 *rank, u32 n) {
    const u32 w = threadIdx.x >> 5, lane = lane_id();
    u32 lo, hi;
    seg_bounds(n, lo, hi);
    u32 mx = 0, cnt = 0;
    for (u32 j = lo + lane; j < hi; j += 32)
        if (j == 0 || key[j] != key[j - 1]) { mx = max(mx, j); cnt++; }
    for (int d = 16; d; d >>= 1) { mx = max(mx, __shfl_xor_sync(SWC_FULL, mx, d)); cnt += __shfl_xor_sync(SWC_FULL, cnt, d); }
    if (lane == 0) { sh.seg_max[w] = mx; sh.seg_cnt[w] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 run = 0, total = 0;
        for (int v = 0; v < SORT_WARPS; v++) { const u32 t = sh.seg_max[v]; sh.seg_max[v] = run; run = max(run, t); total += sh.seg_cnt[v]; }
        sh.groups = total;
    }
    __syncthreads();
    u32 carry = sh.seg_max[w];
    for (u32 base = lo; base < hi; base += 32) {
        const u32 j = base + lane;
        u32 g = (j < hi && (j == 0 || key[j] != key[j - 1])) ? j : 0;
        for (int d = 1; d < 32; d <<= 1) { const u32 t = __shfl_up_sync(SWC_FULL, g, d); if (lane >= (u32)d) g = max(g, t); }
        g = max(g, carry);
        if (j < hi) rank[idx[j]] = g;
        carry = __shfl_sync(SWC_FULL, g, 31);
    }
    __syncthreads();
    const u32 groups = sh.groups;
    __syncthreads();
    return groups;
}

__global__ void __launch_bounds__(SORT_WARPS * 32) sort_kernel(Slice sl) {
    __shared__ SortShared sh;
    const u64 b = blockIdx.x;
    Blk k(sl, sl.blocks[b]);
    BlockMeta *m = meta_of(sl, b);
    const u32 n = m->n;
    for (u32 i = threadIdx.x; i < n; i += blockDim.x) {
        u64 v = 0;
        for (u32 t = 0, p = i; t < 8; t++) { v = (v << 8) | k.rle[p]; p = p + 1 == n ? 0 : p + 1; }
        k.key[0][i] = v; k.idx[0][i] = i;
    }
    __syncthreads();
    int cur = 0;
    for (int shift = 0; shift < 64; shift += 8)
        if (radix_pass(sh, k.key[cur], k.idx[cur], k.key[cur ^ 1], k.idx[cur ^ 1], n, shift)) cur ^= 1;
    u32 groups = rank_groups(sh, k.key[cur], k.idx[cur], k.rank, n);
    const int rbits = n > 1 ? 32 - __clz(n - 1) : 1;
    for (u64 h = 8; groups < n; h *= 2) {
        const u32 hm = (u32)(h % n);
        for (u32 j = threadIdx.x; j < n; j += blockDim.x) {
            const u32 i = k.idx[cur][j];
            const u32 i2 = i + hm >= n ? i + hm - n : i + hm;
            k.key[cur][j] = ((u64)k.rank[i] << 32) | k.rank[i2];
        }
        __syncthreads();
        for (int half = 0; half < 64; half += 32)
            for (int shift = 0; shift < rbits; shift += 8)
                if (radix_pass(sh, k.key[cur], k.idx[cur], k.key[cur ^ 1], k.idx[cur ^ 1], n, half + shift)) cur ^= 1;
        const u32 g2 = rank_groups(sh, k.key[cur], k.idx[cur], k.rank, n);
        if (g2 == groups) break;                 // no group split: the partition is final (DESIGN §4.11, lemma 2)
        groups = g2;
    }
    // the key buffers are free now; bwt aliases key[0], so read idx first
    for (u32 j = threadIdx.x; j < n; j += blockDim.x) {
        const u32 i = k.idx[cur][j];
        k.bwt[j] = k.rle[i == 0 ? n - 1 : i - 1];
    }
    if (threadIdx.x == 0) m->ptr = k.rank[0];
}

// ---- stage 3: MTF + RUNA/RUNB ----
__global__ void __launch_bounds__(32) mtf_kernel(Slice sl) {
    __shared__ u8 perm[256];
    const u64 b = blockIdx.x;
    const u32 lane = lane_id();
    Blk k(sl, sl.blocks[b]);
    BlockMeta *m = meta_of(sl, b);
    const u32 n = m->n;
    if (lane == 0) {                     // the used bytes in order, then the unused ones (which never move)
        u32 o = 0;
        for (int pass = 0; pass < 2; pass++)
            for (u32 c = 0; c < 256; c++)
                if (((m->used[c >> 5] >> (c & 31)) & 1) == (pass == 0 ? 1u : 0u)) perm[o++] = (u8)c;
    }
    __syncwarp();
    u64 word = 0;
    for (int t = 7; t >= 0; t--) word = (word << 8) | perm[8 * lane + t];
    u32 o = 0, zrun = 0, maxsym = 1;
    auto put = [&](u32 s) { if (lane == 0) k.sym[o] = (u16)s; o++; };
    for (u32 i0 = 0; i0 < n; i0 += 32) {
        const u32 mine = i0 + lane < n ? k.bwt[i0 + lane] : 0;
        const u32 lim = min(32u, n - i0);
        for (u32 t = 0; t < lim; t++) {
            const u32 c = __shfl_sync(SWC_FULL, mine, t);
            const u32 c4 = c * 0x01010101u;
            const u64 eq = (u64)__vcmpeq4((u32)word, c4) | ((u64)__vcmpeq4((u32)(word >> 32), c4) << 32);
            const u32 ball = __ballot_sync(SWC_FULL, eq != 0);
            const u32 L = __ffs(ball) - 1;
            const u32 bpos = __shfl_sync(SWC_FULL, eq ? (u32)(__ffsll((long long)eq) - 1) >> 3 : 0u, L);
            const u32 idx = 8 * L + bpos;
            u64 carry = __shfl_up_sync(SWC_FULL, word >> 56, 1);
            if (lane == 0) carry = c;
            if (lane < L) word = (word << 8) | carry;
            else if (lane == L) {
                const u64 low = bpos == 7 ? ~0ull : ((1ull << (8 * (bpos + 1))) - 1);
                word = (word & ~low) | (((word << 8) | carry) & low);
            }
            const u32 i = i0 + t;
            if (idx == 0) zrun++;
            if ((idx == 0 && i == n - 1) || idx != 0) {
                for (u32 rem = zrun; rem > 0;) {       // bijective base 2, low digit first: RUNA = 1, RUNB = 2
                    const u32 q = (rem + 1) / 2 - 1;
                    put(rem - 2 * q == 1 ? 0 : 1);
                    rem = q;
                }
                zrun = 0;
            }
            if (idx != 0) { put(idx + 1); maxsym = max(maxsym, idx + 1); }
        }
    }
    put(maxsym + 1);
    if (lane == 0) { m->nsym = o; m->maxsym = maxsym; }
}

// ---- stage 4: one candidate table per group ----
__global__ void __launch_bounds__(128) group_kernel(Slice sl) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= sl.ngroups) return;
    const u64 b = block_of_group(sl, g);
    Blk k(sl, sl.blocks[b]);
    const BlockMeta *m = meta_of(sl, b);
    const u32 s0 = (u32)(g - sl.blocks[b].group0) * 50, nsym = m->nsym;
    if (s0 >= nsym) return;
    const u32 A = m->maxsym + 2, s1 = min(nsym, s0 + 50);
    u16 stats[MAX_SYMBOLS];
    u32 heap[MAX_SYMBOLS];
    u8 cl[MAX_SYMBOLS];
    int16_t others[MAX_SYMBOLS];
    for (u32 s = 0; s < A; s++) { stats[s] = 1; cl[s] = 0; others[s] = -1; }
    for (u32 i = s0; i < s1; i++) stats[k.sym[i]]++;
    // BZip2+Lengths.swift:36-76 picks c1 = (least frequency, last index), then c2 the same among the rest, and keeps
    // the merged weight under c1: a min-heap on (frequency, 0xFFFF - symbol) pops them in that order
    u32 hn = 0;
    auto down = [&](u32 i) {
        for (;;) {
            u32 l = 2 * i + 1, s = i;
            if (l < hn && heap[l] < heap[s]) s = l;
            if (l + 1 < hn && heap[l + 1] < heap[s]) s = l + 1;
            if (s == i) return;
            const u32 t = heap[i]; heap[i] = heap[s]; heap[s] = t; i = s;
        }
    };
    for (u32 s = 0; s < A; s++) heap[hn++] = ((u32)stats[s] << 16) | (0xFFFFu - s);
    for (int i = (int)hn / 2 - 1; i >= 0; i--) down((u32)i);
    while (hn >= 2) {
        const u32 k1 = heap[0]; heap[0] = heap[--hn]; down(0);
        const u32 k2 = heap[0];
        u32 c1 = 0xFFFFu - (k1 & 0xFFFFu), c2 = 0xFFFFu - (k2 & 0xFFFFu);
        heap[0] = (((k1 >> 16) + (k2 >> 16)) << 16) | (0xFFFFu - c1); down(0);
        cl[c1]++;
        while (others[c1] >= 0) { c1 = (u32)others[c1]; cl[c1]++; }
        others[c1] = (int16_t)c2;
        cl[c2]++;
        while (others[c2] >= 0) { c2 = (u32)others[c2]; cl[c2]++; }
    }
    u16 hist[12] = {0};
    for (u32 s = 0; s < A; s++) hist[min((u32)cl[s], MAX_LEN)]++;
    u16 *out = cand_of(sl, g);
    for (int l = 0; l < 12; l++) out[l] = hist[l];
}

// ---- stage 5: table choice ----
__device__ __forceinline__ u32 warp_sum(u32 v) {
    for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(SWC_FULL, v, d);
    return v;
}

// lengths of symbols 0..A-1 from a histogram (non-decreasing in the symbol); returns their sum
__device__ u32 expand(const u16 *hist, u8 *len, u32 A) {
    u32 sum = 0;
    for (u32 s = lane_id(); s < A; s += 32) {
        u32 cum = 0, l = 1;
        for (; l <= MAX_LEN; l++) { cum += hist[l]; if (s < cum) break; }
        len[s] = (u8)l;
        sum += l;
    }
    __syncwarp();
    return warp_sum(sum);
}

__global__ void __launch_bounds__(32) select_kernel(Slice sl) {
    __shared__ u8 len[7][264];
    __shared__ u32 sumlen[7];
    const u64 b = blockIdx.x;
    const u32 lane = lane_id();
    const BlockPlan bp = sl.blocks[b];
    Blk k(sl, bp);
    BlockMeta *m = meta_of(sl, b);
    const u32 A = m->maxsym + 2, nsym = m->nsym, ng = (nsym + 49) / 50;
    u8 *sel = sel_of(sl) + bp.group0;
    u32 *goff = goff_of(sl) + bp.group0;
    u32 ntab = 0, hsel = 0, mtf = 0x543210;   // selector MTF list, 4 bits per entry
    u64 bits = 0;
    for (u32 g = 0; g < ng; g++) {
        const u32 base = 50 * g, end = min(nsym, base + 50);
        const int a0 = base + lane < end ? (int)k.sym[base + lane] : -1;
        const int a1 = lane < 18 && base + 32 + lane < end ? (int)k.sym[base + 32 + lane] : -1;
        u32 best = 0xFFFFFFFFu, bsel = 0, bdata = 0;
        for (u32 t = 0; t < ntab; t++) {
            const u32 p = warp_sum((a0 >= 0 ? len[t][a0] : 0) + (a1 >= 0 ? len[t][a1] : 0));
            if (sumlen[t] + p < best) { best = sumlen[t] + p; bsel = t; bdata = p; }
        }
        if (ntab < 6) {
            const u16 *cand = cand_of(sl, bp.group0 + g);
            const u32 sl_ = expand(cand, len[ntab], A);
            const u32 p = warp_sum((a0 >= 0 ? len[ntab][a0] : 0) + (a1 >= 0 ? len[ntab][a1] : 0));
            if (sl_ + p < best) {
                if (lane < 12) m->tab[ntab][lane] = cand[lane];
                if (lane == 0) sumlen[ntab] = sl_;
                bsel = ntab; bdata = p; ntab++;
            }
            __syncwarp();
        }
        if (lane == 0) { sel[g] = (u8)bsel; goff[g] = (u32)bits; }
        bits += bdata;
        u32 idx = 0;
        while (((mtf >> (4 * idx)) & 15) != bsel) idx++;
        hsel += idx + 1;
        const u32 low = (1u << (4 * idx)) - 1;     // move entry idx to the front
        mtf = (mtf & ~((low << 4) | 15u) & ~(15u << (4 * idx))) | ((mtf & low) << 4) | bsel;
    }
    __syncwarp();
    if (ntab == 1) { if (lane < 12) m->tab[1][lane] = m->tab[0][lane]; ntab = 2; }
    __syncwarp();
    if (lane == 0) {
        u32 maps = 0;
        for (int j = 0; j < 16; j++) maps += ((m->used[j >> 1] >> (16 * (j & 1))) & 0xFFFFu) != 0;
        u32 h = 48 + 32 + 1 + 24 + 16 + 16 * maps + 3 + 15 + hsel;
        for (u32 t = 0; t < ntab; t++) {
            u32 lo = 0, hi = 0;
            for (u32 l = 1; l <= MAX_LEN; l++) if (m->tab[t][l]) { if (!lo) lo = l; hi = l; }
            h += 5 + A + 2 * (hi - lo);            // delta coding: lengths only rise, by hi - lo in all
        }
        m->ntab = ntab; m->nsel = ng; m->hbits = h; m->dbits = bits;
    }
}

// ---- stage 6: layout, stream header and EOS ----
__global__ void __launch_bounds__(128) layout_kernel(Args a, u64 first, u64 count, Slice sl) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const UnitPlan up = sl.units[j];
    u64 bits = 32;
    u32 crc = 0;
    for (u32 b = up.block0; b < up.block0 + up.blocks; b++) {
        BlockMeta *m = meta_of(sl, b);
        m->bit_off = bits;
        bits += m->hbits + m->dbits;
        crc = ((crc << 1) | (crc >> 31)) ^ m->crc;
    }
    const u64 len = (bits + 80 + 7) / 8;
    a.out_len[first + j] = len;
    a.status[first + j] = len > a.out_cap[first + j] ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
    u32 *w = (u32 *)(sl.stage + up.stage);
    BitW h(w, 0);
    h.put(0x425A6830u + a.level, 32);           // 'B' 'Z' 'h' '0' + k
    h.finish();
    BitW e(w, bits);
    e.put64(0x177245385090ull, 48);
    e.put(crc, 32);
    e.finish();
}

// ---- stage 7: block headers and codes ----
__global__ void __launch_bounds__(128) header_kernel(Slice sl) {
    const u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= sl.nblocks) return;
    const BlockPlan bp = sl.blocks[b];
    const BlockMeta *m = meta_of(sl, b);
    BitW w((u32 *)(sl.stage + sl.units[bp.unit].stage), m->bit_off);
    w.put64(0x314159265359ull, 48);
    w.put(m->crc, 32);
    w.put(0, 1);
    w.put(m->ptr, 24);
    u32 maps = 0;
    for (int j = 0; j < 16; j++) maps |= (((m->used[j >> 1] >> (16 * (j & 1))) & 0xFFFFu) != 0) << (15 - j);
    w.put(maps, 16);
    for (int j = 0; j < 16; j++) {
        if (!((maps >> (15 - j)) & 1)) continue;
        const u32 v = (m->used[j >> 1] >> (16 * (j & 1))) & 0xFFFFu;
        w.put(__brev(v) >> 16, 16);              // byte 16 j + i is bit 15 - i
    }
    w.put(m->ntab, 3);
    w.put(m->nsel, 15);
    const u8 *sel = sel_of(sl) + bp.group0;
    u32 mtf = 0x543210;
    for (u32 g = 0; g < m->nsel; g++) {
        const u32 s = sel[g];
        u32 idx = 0;
        while (((mtf >> (4 * idx)) & 15) != s) idx++;
        w.put(((1u << idx) - 1) << 1, idx + 1);  // idx ones, then a zero
        const u32 low = (1u << (4 * idx)) - 1;
        mtf = (mtf & ~((low << 4) | 15u) & ~(15u << (4 * idx))) | ((mtf & low) << 4) | s;
    }
    const u32 A = m->maxsym + 2;
    for (u32 t = 0; t < m->ntab; t++) {
        u32 prev = 0, cum = 0, l = 1;
        for (u32 s = 0; s < A; s++) {
            while (s >= cum + m->tab[t][l] && l < MAX_LEN) { cum += m->tab[t][l]; l++; }
            if (s == 0) { prev = l; w.put(l, 5); }
            for (; prev < l; prev++) w.put(2, 2);    // "10": one longer
            w.put(0, 1);
        }
    }
    w.finish();
}

__global__ void __launch_bounds__(128) emit_kernel(Slice sl) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= sl.ngroups) return;
    const u64 b = block_of_group(sl, g);
    const BlockPlan bp = sl.blocks[b];
    Blk k(sl, bp);
    const BlockMeta *m = meta_of(sl, b);
    const u32 local = (u32)(g - bp.group0), s0 = local * 50, nsym = m->nsym;
    if (s0 >= nsym) return;
    const u16 *hist = m->tab[sel_of(sl)[g]];
    u32 first_code[MAX_LEN + 2], first_sym[MAX_LEN + 2];
    u32 code = 0, sym = 0;
    for (u32 l = 1; l <= MAX_LEN; l++) { first_code[l] = code; first_sym[l] = sym; code = (code + hist[l]) << 1; sym += hist[l]; }
    first_sym[MAX_LEN + 1] = sym;
    BitW w((u32 *)(sl.stage + sl.units[bp.unit].stage), m->bit_off + m->hbits + goff_of(sl)[g]);
    for (u32 i = s0; i < min(nsym, s0 + 50); i++) {
        const u32 s = k.sym[i];
        u32 l = 1;
        while (s >= first_sym[l + 1]) l++;
        w.put(first_code[l] + (s - first_sym[l]), l);
    }
    w.finish();
}

// blockIdx.x = unit, blockIdx.y = chunk of sl.copy_chunk bytes: a large unit is copied by many CTAs
__global__ void __launch_bounds__(256) copy_kernel(Args a, u64 first, Slice sl) {
    const u64 j = blockIdx.x, u = first + j;
    if (a.status[u] != SWC_OK) return;
    const u64 len = a.out_len[u], beg = (u64)blockIdx.y * sl.copy_chunk;
    if (beg >= len) return;
    const u64 end = min(len, beg + sl.copy_chunk);
    const u8 *src = sl.stage + sl.units[j].stage;
    u8 *dst = a.out_base + a.out_off[u];
    for (u64 i = beg + threadIdx.x; i < end; i += blockDim.x) dst[i] = src[i];
}

}  // namespace

u64 unit_blocks(u64 n, u32 level) { const u64 raw = (u64)RAW_PER_LEVEL * level; return (n + raw - 1) / raw; }

u64 max_stream_bytes(u64 n, u32 level) {
    const u64 raw = (u64)RAW_PER_LEVEL * level;
    u64 bits = 32 + 80;
    for (u64 at = 0; at < n; at += raw) {
        const u32 r = rle_cap((u32)(n - at < raw ? n - at : raw));
        const u64 groups = ((u64)r + 1 + 49) / 50;
        bits += 395 + 6 * groups + 6 * (5 + MAX_SYMBOLS + 2 * (MAX_LEN - 1)) + (u64)MAX_LEN * (r + 1);
    }
    return (bits + 7) / 8;
}

u64 unit_scratch(u64 n, u32 level) {
    const u64 raw = (u64)RAW_PER_LEVEL * level;
    u64 s = a256(max_stream_bytes(n, level) + 8);
    for (u64 at = 0; at < n; at += raw) {
        const u32 r = (u32)(n - at < raw ? n - at : raw);
        s += block_scratch(r) + a256(sizeof(BlockMeta) + sizeof(BlockPlan)) + 32 * group_slots(r);
    }
    return s + 256;
}

int run(const Args &a, u64 first, u64 count, const Slice &sl, cudaStream_t s) {
    // one timing mark in front and one after every stage, whether or not the slice has blocks: 8 intervals per slice
    timing_mark(s);
    SWC_CUDA_TRY(cudaMemsetAsync(sl.stage, 0, sl.stage_bytes, s));
    const unsigned bb = (unsigned)((sl.nblocks + 127) / 128), gb = (unsigned)((sl.ngroups + 127) / 128);
    const unsigned nb = (unsigned)sl.nblocks;
    if (sl.nblocks) { rle_kernel<<<bb, 128, 0, s>>>(a, first, sl); count_launch(); }
    timing_mark(s);
    if (sl.nblocks) { sort_kernel<<<nb, SORT_WARPS * 32, 0, s>>>(sl); count_launch(); }
    timing_mark(s);
    if (sl.nblocks) { mtf_kernel<<<nb, 32, 0, s>>>(sl); count_launch(); }
    timing_mark(s);
    if (sl.nblocks) { group_kernel<<<gb, 128, 0, s>>>(sl); count_launch(); }
    timing_mark(s);
    if (sl.nblocks) { select_kernel<<<nb, 32, 0, s>>>(sl); count_launch(); }
    timing_mark(s);
    layout_kernel<<<(unsigned)((count + 127) / 128), 128, 0, s>>>(a, first, count, sl);
    count_launch();
    timing_mark(s);
    if (sl.nblocks) {
        header_kernel<<<bb, 128, 0, s>>>(sl);
        emit_kernel<<<gb, 128, 0, s>>>(sl);
        count_launch(2);
    }
    timing_mark(s);
    const dim3 cg((unsigned)count, (unsigned)((sl.max_stage + sl.copy_chunk - 1) / sl.copy_chunk));
    copy_kernel<<<cg, 256, 0, s>>>(a, first, sl);
    count_launch();
    timing_mark(s);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace bzip2c
}  // namespace swc
