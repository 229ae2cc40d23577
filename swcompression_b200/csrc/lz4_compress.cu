// lz4_compress.cu — batched LZ4 block compression for sm_90a.  Replaces LZ4.compress(block:_:) (reference
// Sources/LZ4/LZ4+Compress.swift:156-298) and reproduces its output byte for byte.
//
// The reference's parse is greedy and serial: at every position it visits it looks up the exact 4-byte key in a table
// holding the last VISITED position with that key, records the current position, and takes the match if it is at most
// 65 535 bytes back.  Three kernels split it into a parallel, parse-independent part and a cheap serial walk
// (DESIGN §4.9 proves that the walk makes the reference's decisions):
//   lz4c_chain_kernel — ONE WARP PER UNIT: for every position p of the window (dictionary + block), link[p] = distance to
//      the nearest earlier position with the same exact key, 0 if there is none within 65 535 bytes.  A forward pass
//      builds hash-bucket chains (a per-warp head table in shared memory, __match_any_sync for same-bucket lanes); a
//      backward pass follows each bucket chain to the first position whose key is equal.  It also seeds the visited
//      bitmap with the dictionary positions the reference's table starts with.
//   lz4c_parse_kernel — ONE THREAD PER UNIT: the reference's loop, with the table lookup replaced by a walk down link[]
//      to the first visited position.  Writes one 8-byte record per sequence and the exact compressed size.
//   lz4c_emit_kernel  — ONE WARP PER UNIT: warp scans over 32 records at a time place each sequence; a lane writes its
//      token, length bytes and offset, the warp copies the literals.
// The parse result depends only on the unit's bytes, never on the grid or on the order in which units run.
#include "common.cuh"
#include "lz4_compress.cuh"

namespace swc {
namespace lz4c {

namespace {

constexpr int HBITS = 12;                       // 4096 buckets: 16 KiB per warp, 2 warps per CTA
constexpr u32 HSIZE = 1u << HBITS;
constexpr u32 EMPTY = 0xFFFFFFFFu;
constexpr u32 MAX_DIST = 65535;                 // LZ4+Compress.swift:195

__host__ __device__ __forceinline__ u64 a256(u64 v) { return (v + 255) & ~(u64)255; }

// one unit's window: the dictionary bytes at positions [0, d), the block at [d, w)
struct Geo {
    const u8 *dict, *blk;
    u32 d, l, w;
    int st;
    __device__ __forceinline__ u32 at(u32 p) const { return p < d ? dict[p] : blk[p - d]; }
    // combine(_:from:) :290-298 (byte order only matters for equality here)
    __device__ __forceinline__ u32 key(u32 p) const { return at(p) << 24 | at(p + 1) << 16 | at(p + 2) << 8 | at(p + 3); }
};

__device__ __forceinline__ Geo geo(const Args &a, u64 u) {
    Geo g;
    const u64 l = a.in_len[u];
    u64 d = a.dict_off ? a.dict_len[u] : 0;
    g.blk = a.in_base + a.in_off[u];
    g.dict = a.dict_off ? a.in_base + a.dict_off[u] + (d > MAX_DICT ? d - MAX_DICT : 0) : nullptr;
    g.st = l > MAX_BLOCK ? SWC_ERR_UNSUPPORTED : (d >= 1 && d <= 3) ? SWC_ERR_REFERENCE_TRAP : SWC_OK;   // :283 traps
    if (d > MAX_DICT) d = MAX_DICT;
    g.d = (u32)d; g.l = g.st ? 0u : (u32)l; g.w = g.d + g.l;
    return g;
}

// scratch of one unit: link (u16 per position) | visited bitmap | records ([0] = count)
struct Scr {
    u16 *link; u32 *vis; u64 *rec;
    __device__ __forceinline__ Scr(u8 *base, const Geo &g) {
        link = (u16 *)base;
        vis = (u32 *)(base + a256(2ull * (g.w + 1)));
        rec = (u64 *)((u8 *)vis + a256(4ull * ((g.w + 31) / 32)));
    }
};

__device__ __forceinline__ u32 hash4(u32 k) { return (k * 2654435761u) >> (32 - HBITS); }
__device__ __forceinline__ u32 ext_bytes(u32 v /* length minus its base */) { return v < 15 ? 0u : 1u + (v - 15u) / 255u; }
// the length bytes of :222-230 / :240-248 for a field value v >= 15
__device__ __forceinline__ u8 *put_len(u8 *o, u32 rest) {
    while (rest >= 255) { *o++ = 255; rest -= 255; }
    *o++ = (u8)rest;
    return o;
}

}  // namespace

__global__ void __launch_bounds__(64) lz4c_chain_kernel(Args a, u64 first, u64 count, u8 *scr, const u64 *scr_off) {
    __shared__ u32 heads[2][HSIZE];
    const u64 j = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= count) return;
    const u32 lane = lane_id();
    const Geo g = geo(a, first + j);
    if (g.st) return;
    u32 *head = heads[(threadIdx.x >> 5) & 1];
    Scr s(scr + scr_off[j], g);
    for (u32 i = lane; i < HSIZE; i += 32) head[i] = EMPTY;
    // the reference's table starts with dictionary positions 0 ..< d-4 (populateMatchStorage :279-288): they count as visited
    const u32 dict_vis = g.d >= 4 ? g.d - 4 : 0;
    for (u32 w = lane; w < (g.w + 31) / 32; w += 32) {
        const u32 lo = w * 32;
        s.vis[w] = lo + 32 <= dict_vis ? ~0u : lo >= dict_vis ? 0u : (1u << (dict_vis - lo)) - 1u;
    }
    __syncwarp();
    const u32 nk = g.w >= 4 ? g.w - 3 : 0;       // positions with a full key
    // forward: nearest earlier position in the same hash bucket
    for (u32 base = 0; base < nk; base += 32) {
        const u32 p = base + lane;
        const bool valid = p < nk;
        const u32 h = valid ? hash4(g.key(p)) : HSIZE + lane;
        const u32 m = __match_any_sync(SWC_FULL, h);
        const u32 lower = m & ((1u << lane) - 1u);
        u32 d = 0;
        if (valid) {
            const u32 q = lower ? base + 31 - __clz(lower) : head[h];
            if (q != EMPTY && p - q <= MAX_DIST) d = p - q;
        }
        __syncwarp();
        if (valid && (m >> lane) == 1u) head[h] = p;     // the group's last position becomes the bucket head
        if (valid) s.link[p] = (u16)d;
        __syncwarp();
    }
    // backward: follow the bucket chain to the nearest position with the same exact key.  Chunks go from the end, so every
    // link[q] read here (q < p) is still a bucket link; a chunk's lanes read before any of them writes.
    for (u32 base = nk ? (nk - 1) & ~31u : 0; nk; base -= 32) {
        const u32 p = base + lane;
        u32 d = 0;
        if (p < nk && (d = s.link[p]) != 0) {
            const u32 k = g.key(p);
            u32 q = p - d;
            for (;;) {
                if (g.key(q) == k) { d = p - q; break; }
                const u32 dd = s.link[q];
                if (dd == 0 || p - (q - dd) > MAX_DIST) { d = 0; break; }
                q -= dd;
            }
        }
        __syncwarp();
        if (p < nk) s.link[p] = (u16)d;
        __syncwarp();
        if (base == 0) break;
    }
}

__global__ void __launch_bounds__(128, 8) lz4c_parse_kernel(Args a, u64 first, u64 count, u8 *scr, const u64 *scr_off) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const u64 u = first + j;
    const Geo g = geo(a, u);
    if (g.st) { a.out_len[u] = 0; a.status[u] = g.st; return; }
    Scr s(scr + scr_off[j], g);
    u32 i = g.d, lit = 0, nrec = 0;                                               // :161
    u64 size = 0;
    while ((i64)i < (i64)g.w - 9) {                                               // :176
        // the table's entry for key(i) is the nearest earlier visited position with that key (DESIGN §4.9)
        u32 q = i, d = s.link[i];
        bool found = false;
        while (d) {
            q -= d;
            if (i - q > MAX_DIST) break;                                          // :195 (nearer visited ones do not exist)
            if ((s.vis[q >> 5] >> (q & 31)) & 1u) { found = true; break; }
            d = s.link[q];
        }
        s.vis[i >> 5] |= 1u << (i & 31);                                          // :181 / :187
        if (!found) { lit++; i++; continue; }
        u32 len = 4;                                                              // :190-208
        while ((i64)(i + len) < (i64)g.w - 5 && g.at(i + len) == g.at(q + len)) len++;
        if (g.w - i < 12) break;                                                  // :210-214
        s.rec[1 + nrec++] = (u64)lit | (u64)len << 24 | (u64)(i - q) << 48;
        size += 1 + ext_bytes(lit) + lit + 2 + ext_bytes(len - 4);
        i += len;                                                                 // :239
        lit = 0;
    }
    lit += g.w - i;                                                               // :254-257
    s.rec[1 + nrec++] = lit;
    size += 1 + ext_bytes(lit) + lit;                                             // :262-274
    s.rec[0] = nrec;
    a.out_len[u] = size;
    a.status[u] = size > a.out_cap[u] ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
}

__global__ void __launch_bounds__(256) lz4c_emit_kernel(Args a, u64 first, u64 count, const u8 *scr, const u64 *scr_off) {
    const u64 j = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= count) return;
    const u64 u = first + j;
    if (a.status[u] != SWC_OK) return;
    const u32 lane = lane_id();
    const Geo g = geo(a, u);
    u8 *out = a.out_base + a.out_off[u];
    if (a.stored && a.stored[u]) {                                                // LZ4+Compress.swift:112-118
        for (u32 k = lane; k < g.l; k += 32) out[k] = g.blk[k];
        return;
    }
    const Scr s((u8 *)scr + scr_off[j], g);
    const u32 nrec = (u32)s.rec[0];
    u32 ipos = 0, opos = 0;
    for (u32 g0 = 0; g0 < nrec; g0 += 32) {
        const bool have = g0 + lane < nrec;
        const u64 r = have ? s.rec[1 + g0 + lane] : 0ull;
        const u32 lit = (u32)r & 0xFFFFFFu, mlen = (u32)(r >> 24) & 0xFFFFFFu, off = (u32)(r >> 48);
        const u32 enc = have ? 1u + ext_bytes(lit) + lit + (mlen ? 2u + ext_bytes(mlen - 4u) : 0u) : 0u;
        const u32 adv = lit + mlen;
        u32 ie = enc, ia = adv;
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
            const u32 ve = __shfl_up_sync(SWC_FULL, ie, dd), va = __shfl_up_sync(SWC_FULL, ia, dd);
            if (lane >= (u32)dd) { ie += ve; ia += va; }
        }
        const u32 src = ipos + ia - adv;
        u32 dst = 0;
        if (have) {                                                               // :218-248
            u8 *o = out + opos + ie - enc;
            *o++ = (u8)((lit < 15 ? lit : 15) << 4 | (mlen ? (mlen - 4 < 15 ? mlen - 4 : 15) : 0));
            if (lit >= 15) o = put_len(o, lit - 15);
            dst = (u32)(o - out);
            o += lit;
            if (mlen) {
                o[0] = (u8)(off & 0xFF); o[1] = (u8)(off >> 8);
                if (mlen - 4 >= 15) put_len(o + 2, mlen - 19);
            }
        }
        for (int k = 0; k < 32; k++) {                                            // literals, one record at a time
            const u32 n = __shfl_sync(SWC_FULL, lit, k);
            if (n == 0) continue;
            const u32 sk = __shfl_sync(SWC_FULL, src, k), dk = __shfl_sync(SWC_FULL, dst, k);
            for (u32 x = lane; x < n; x += 32) out[dk + x] = g.blk[sk + x];
        }
        opos += __shfl_sync(SWC_FULL, ie, 31);
        ipos += __shfl_sync(SWC_FULL, ia, 31);
    }
}

u64 unit_scratch(u64 w, u64 l) { return a256(2 * (w + 1)) + a256(4 * ((w + 31) / 32)) + a256(8 * (l / 4 + 3)); }

int parse(const Args &a, u64 first, u64 count, u8 *scr, const u64 *scr_off, cudaStream_t s) {
    if (count == 0) return SWC_OK;
    timing_mark(s);
    lz4c_chain_kernel<<<(unsigned)((count * 32 + 63) / 64), 64, 0, s>>>(a, first, count, scr, scr_off);
    timing_mark(s);
    lz4c_parse_kernel<<<(unsigned)((count + 127) / 128), 128, 0, s>>>(a, first, count, scr, scr_off);
    timing_mark(s);
    count_launch(2);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

int emit(const Args &a, u64 first, u64 count, const u8 *scr, const u64 *scr_off, cudaStream_t s) {
    if (count == 0) return SWC_OK;
    lz4c_emit_kernel<<<(unsigned)((count * 32 + 255) / 256), 256, 0, s>>>(a, first, count, scr, scr_off);
    timing_mark(s);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace lz4c
}  // namespace swc
