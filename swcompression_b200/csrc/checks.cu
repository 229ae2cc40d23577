// checks.cu — device-side checksums used by the wrappers (reference: Sources/Common/CheckSums.swift:12-57,
// Sources/LZ4/XxHash32.swift:24-83, Sources/XZ/Sha256.swift).
//
// CRC-32 / CRC-32(bzip2) / CRC-64 are linear over GF(2): every thread folds one 4 KiB chunk with a byte table held in
// shared memory, then one thread chains the chunk values with x^(8*len) multiplications (zlib's crc32_combine
// identity, which holds for the conditioned CRC values).  Adler-32 splits the same way.  xxHash32 and SHA-256 have no
// combine operator, so they run one thread per buffer (many buffers in parallel for LZ4 block checksums).
#include "common.cuh"
#include <algorithm>
#include <vector>
#include "checks.cuh"
#include "checks_device.cuh"
#include "host_util.h"

namespace swc {
namespace checks {

constexpr u32 CHUNK = 4096;

// GF(2) helpers, the warp CRC and SHA-256: checks_device.cuh

// ---------------------------------------------------------------- chunk kernels
// The bytes a chunk pass covers: n bytes at data, or, when len is set, one unit of a batch read on the device: *len bytes at
// data + *off, none when *status is not OK (Deflate reports the size it WOULD need on overflow), and then the result is 0.
struct Span {
    const u8 *data;
    u64 n;
    const u64 *off, *len;
    const int32_t *status;
    __device__ bool skipped() const { return len && *status != SWC_OK; }
    __device__ u64 size() const { return !len ? n : skipped() ? 0 : *len; }
};

template <int KIND>   // 0 crc32, 1 bzip2 crc32, 2 crc64, 3 adler32
__global__ void __launch_bounds__(128) chunk_kernel(Span sp, u64 *partial) {
    __shared__ u64 tab[256];
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) {
        if (KIND == 0) { u32 c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1; tab[i] = c; }
        if (KIND == 1) { u32 c = i << 24; for (int k = 0; k < 8; k++) c = (c & 0x80000000u) ? (c << 1) ^ 0x04C11DB7u : c << 1; tab[i] = c; }
        if (KIND == 2) { u64 c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? 0xC96C5795D7870F42ull ^ (c >> 1) : c >> 1; tab[i] = c; }
    }
    __syncthreads();
    const u8 *data = sp.len ? sp.data + *sp.off : sp.data;
    const u64 n = sp.size();
    const u64 chunk = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 beg = chunk * CHUNK;
    if (beg >= n) return;
    const u64 end = beg + CHUNK < n ? beg + CHUNK : n;
    if (KIND == 0) {
        u32 c = 0xFFFFFFFFu;
        for (u64 i = beg; i < end; i++) c = (u32)tab[(c ^ data[i]) & 0xFF] ^ (c >> 8);
        partial[chunk] = ~c;
    } else if (KIND == 1) {
        u32 c = 0xFFFFFFFFu;
        for (u64 i = beg; i < end; i++) c = (c << 8) ^ (u32)tab[((c >> 24) ^ data[i]) & 0xFF];
        partial[chunk] = ~c;
    } else if (KIND == 2) {
        u64 c = ~0ull;
        for (u64 i = beg; i < end; i++) c = tab[(c ^ data[i]) & 0xFF] ^ (c >> 8);
        partial[chunk] = ~c;
    } else {
        u32 s1 = 0, s2 = 0;                       // sums of this chunk alone (s1 without the leading 1)
        for (u64 i = beg; i < end; i++) { s1 += data[i]; s2 += s1; }   // 4096*255 and 4096*4097/2*255 fit in u32
        partial[chunk] = (u64)(s1 % 65521u) | ((u64)(s2 % 65521u) << 32);
    }
}

template <int KIND, typename R>
__global__ void combine_kernel(Span sp, const u64 *partial, R *result) {
    const u64 n = sp.size();
    const u64 nchunks = (n + CHUNK - 1) / CHUNK;
    if (sp.skipped()) { *result = 0; return; }
    if (KIND == 3) {
        u64 a = 1, b = 0;                         // CheckSums.swift:48-57
        for (u64 c = 0; c < nchunks; c++) {
            u64 len = (c + 1) * CHUNK <= n ? CHUNK : n - c * CHUNK;
            u64 s1 = partial[c] & 0xFFFFFFFFu, s2 = partial[c] >> 32;
            b = (b + (len % 65521u) * a + s2) % 65521u;
            a = (a + s1) % 65521u;
        }
        *result = (R)((b << 16) + a);
        return;
    }
    if (nchunks == 0) { *result = 0; return; }    // CRC of the empty string is 0 in all three variants
    u64 acc = partial[0];
    const u32 p32r = KIND == 0 ? xpow32r(CHUNK) : 0;
    const u32 p32n = KIND == 1 ? xpow32n(CHUNK) : 0;
    const u64 p64r = KIND == 2 ? xpow64r(CHUNK) : 0;
    for (u64 c = 1; c < nchunks; c++) {
        const bool full = (c + 1) * CHUNK <= n;
        const u64 len = full ? CHUNK : n - c * CHUNK;
        if (KIND == 0) acc = mulmod32r(full ? p32r : xpow32r(len), (u32)acc) ^ (u32)partial[c];
        if (KIND == 1) acc = mulmod32n(full ? p32n : xpow32n(len), (u32)acc) ^ (u32)partial[c];
        if (KIND == 2) acc = mulmod64r(full ? p64r : xpow64r(len), acc) ^ partial[c];
    }
    *result = (R)acc;
}

// the grid covers `cap` bytes, at least the span's size
template <int KIND, typename R>
static int run(const Span &sp, u64 cap, R *d_result, u64 *d_partial, cudaStream_t s) {
    const u64 nchunks = (cap + CHUNK - 1) / CHUNK;
    if (nchunks) {
        chunk_kernel<KIND><<<(unsigned)((nchunks + 127) / 128), 128, 0, s>>>(sp, d_partial);
        count_launch();
    }
    combine_kernel<KIND><<<1, 1, 0, s>>>(sp, d_partial, d_result);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

size_t partial_bytes(u64 n) { return (size_t)(((n + CHUNK - 1) / CHUNK) + 1) * 8; }

int crc32(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s) { return run<0>(Span{d, n}, n, d_result, d_partial, s); }
int bzip2_crc32(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s) { return run<1>(Span{d, n}, n, d_result, d_partial, s); }
int crc64(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s) { return run<2>(Span{d, n}, n, d_result, d_partial, s); }
int adler32(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s) { return run<3>(Span{d, n}, n, d_result, d_partial, s); }
int unit_check(Kind k, const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u64 cap, u32 *result, u64 *d_partial,
               cudaStream_t s) {
    const Span u{base, 0, off, len, status};
    return k == CRC32 ? run<0>(u, cap, result, d_partial, s) : run<3>(u, cap, result, d_partial, s);
}

// ---------------------------------------------------------------- CRC-32 of many buffers: one warp per buffer
// warp_crc (checks_device.cuh): each lane folds one of 32 contiguous segments (a multiple of 16 bytes, read with 16-byte
// loads) four bytes per step with four byte tables in shared memory ("slicing by 4": 2.8 instead of 6 instructions per byte),
// then the 32 conditioned values are chained with x^(8*len) multiplications — the same identity as above, inside one warp.
__global__ void __launch_bounds__(256) crc32_units_kernel(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u32 *result, u64 n) {
    __shared__ u32 tab[4][256];
    crc_tables<Crc32R>(tab, threadIdx.x, blockDim.x);
    __syncthreads();
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= n) return;
    // a unit that did not decode cleanly has no defined extent (Deflate reports the size it WOULD need on overflow): skip it
    const u64 L = (status && status[unit] != SWC_OK) ? 0 : len[unit];
    const u32 c = warp_crc<Crc32R, true>(tab, base + off[unit], L);
    if (lane_id() == 0) result[unit] = c;
}

int crc32_units(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u32 *result, u64 n, cudaStream_t s) {
    if (!n) return SWC_OK;
    crc32_units_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(base, off, len, status, result, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// ---------------------------------------------------------------- CRC-64 of many buffers: one warp per buffer
// warp_crc (checks_device.cuh), the segment scheme of crc32_units_kernel in 64 bits; 8 KiB of slicing tables per CTA
__global__ void __launch_bounds__(256) crc64_units_kernel(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u64 *result, u64 n) {
    __shared__ u64 tab[4][256];
    crc_tables<Crc64R>(tab, threadIdx.x, blockDim.x);
    __syncthreads();
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= n) return;
    const u64 L = (status && status[unit] != SWC_OK) ? 0 : len[unit];
    const u64 c = warp_crc<Crc64R, true>(tab, base + off[unit], L);
    if (lane_id() == 0) result[unit] = c;
}

int crc64_units(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u64 *result, u64 n, cudaStream_t s) {
    if (!n) return SWC_OK;
    crc64_units_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(base, off, len, status, result, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// ---------------------------------------------------------------- Adler-32 of many buffers: one warp per buffer
// The same 32 segments as crc32_units_kernel.  A lane sums its segment from a = b = 0 (s1 = sum of bytes, s2 = sum of
// (bytes left including this one) x byte), 16 bytes per step with byte dot products, in 64-bit sums reduced mod 65 521
// every 4 KiB; the lanes are then chained with the concatenation rule a' = a + s1, b' = b + len x a + s2 (CheckSums.swift:
// 48-57 over the whole buffer gives the same value).  64-bit sums cannot overflow for any byte values between reductions.
constexpr u32 ADLER_MOD = 65521;
__global__ void __launch_bounds__(256) adler32_units_kernel(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u32 *result, u64 n) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= n) return;
    const u32 lane = threadIdx.x & 31;
    const bool skip = status && status[unit] != SWC_OK;
    const u8 *p = base + off[unit];
    const u64 L = skip ? 0 : len[unit];
    const u64 seg = (((L + 31) / 32) + 15) & ~(u64)15;
    const u64 sb = lane * seg < L ? lane * seg : L, se = sb + seg < L ? sb + seg : L;
    u64 s1 = 0, s2 = 0;
    u64 i = sb;
    for (; i < se && ((uintptr_t)(p + i) & 15); i++) { s1 += p[i]; s2 += s1; }
    u32 steps = 0;
    for (; i + 16 <= se; i += 16) {
        const uint4 v = __ldg((const uint4 *)(p + i));
        // byte j of the 16 weighs 16 - j in s2
        const u32 sum = __dp4a(v.x, 0x01010101u, __dp4a(v.y, 0x01010101u, __dp4a(v.z, 0x01010101u, __dp4a(v.w, 0x01010101u, 0u))));
        const u32 wsum = __dp4a(v.x, 0x0D0E0F10u, __dp4a(v.y, 0x090A0B0Cu, __dp4a(v.z, 0x05060708u, __dp4a(v.w, 0x01020304u, 0u))));
        s2 += 16 * s1 + wsum;
        s1 += sum;
        if (++steps == 256) { s1 %= ADLER_MOD; s2 %= ADLER_MOD; steps = 0; }
    }
    for (; i < se; i++) { s1 += p[i]; s2 += s1; }
    s1 %= ADLER_MOD; s2 %= ADLER_MOD;
    u64 a = 1, b = 0;
    for (int l = 0; l < 32; l++) {
        const u64 p1 = __shfl_sync(SWC_FULL, s1, l), p2 = __shfl_sync(SWC_FULL, s2, l);
        const u64 lb = (u64)l * seg < L ? (u64)l * seg : L, le = lb + seg < L ? lb + seg : L;
        b = (b + ((le - lb) % ADLER_MOD) * a + p2) % ADLER_MOD;
        a = (a + p1) % ADLER_MOD;
    }
    if (lane == 0) result[unit] = skip ? 0u : (u32)((b << 16) | a);
}

int adler32_units(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u32 *result, u64 n, cudaStream_t s) {
    if (!n) return SWC_OK;
    adler32_units_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(base, off, len, status, result, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// gzip member signature scan over unit ranges (GzipHeader.swift:70-81: magic 1f 8b, method 8, reserved flag bits clear):
// position p of unit u is a candidate when the signature starts there and p + 20 <= in_len[u] (a shorter member fails
// the 20-byte guard), or when p = 0 and s.with_zero (a multi-member walk always starts at 0).  Grid: blockIdx.y strides
// the units, the x-threads stride the unit's 16-byte groups of positions, so the launch shape depends on n alone.  Each
// candidate takes slot = atomicAdd(&count[u], 1): with `first` set (and first[u] != ~0) it goes to list[first[u] + slot],
// with list alone (one unit) to list[slot] while slot < cap, and with neither it is only counted.  Positions come in any
// order.  Units may be unaligned: a thread loads the aligned 16-byte lines that hold its 16 positions and the 3 bytes
// behind them, skipping a line that starts past the unit, and no byte outside the unit is matched.
__global__ void __launch_bounds__(256) gzip_scan_kernel(GzipScan s) {
    for (u64 u = blockIdx.y; u < s.n; u += gridDim.y) {
        if (s.first && s.first[u] == ~0ull) continue;
        const u8 *p = s.base + s.off[u];
        const u64 L = s.len[u];
        for (u64 base = ((u64)blockIdx.x * blockDim.x + threadIdx.x) * 16; base < L; base += (u64)gridDim.x * blockDim.x * 16) {
            const u8 *at = p + base, *stop = p + L;
            const uint4 *line = (const uint4 *)((uintptr_t)at & ~(uintptr_t)15);
            u32 v[12];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const uint4 x = (const u8 *)(line + k) < stop ? __ldg(line + k) : make_uint4(0, 0, 0, 0);
                v[4 * k] = x.x; v[4 * k + 1] = x.y; v[4 * k + 2] = x.z; v[4 * k + 3] = x.w;
            }
            const u32 r = (u32)((uintptr_t)at & 15), q = r >> 2, sh = (r & 3) * 8;
            u32 w[5];                                        // bytes base .. base + 19 of the unit
#pragma unroll
            for (int k = 0; k < 5; k++) {
                const u32 a0 = q == 0 ? v[k] : q == 1 ? v[k + 1] : q == 2 ? v[k + 2] : v[k + 3];
                const u32 a1 = q == 0 ? v[k + 1] : q == 1 ? v[k + 2] : q == 2 ? v[k + 3] : v[k + 4];
                w[k] = __funnelshift_r(a0, a1, sh);
            }
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const u32 x = __funnelshift_r(w[i >> 2], w[(i >> 2) + 1], (i & 3) * 8);
                const u64 pos = base + i;
                if (((x & 0xE0FFFFFFu) == 0x00088B1Fu && pos + 20 <= L) || (pos == 0 && s.with_zero)) {
                    const u64 slot = atomicAdd(&s.count[u], 1ull);
                    if (s.first) s.list[s.first[u] + slot] = pos;
                    else if (s.list && slot < s.cap) s.list[slot] = pos;
                }
            }
        }
    }
}

int gzip_scan(const GzipScan &s, cudaStream_t stream) {
    if (!s.n) return SWC_OK;
    const unsigned y = (unsigned)(s.n < 65535 ? s.n : 65535), x = y >= 2048 ? 1u : 2048u / y;
    gzip_scan_kernel<<<dim3(x, y), 256, 0, stream>>>(s);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

int find_gzip_members(const u8 *d_in, u64 n, std::vector<size_t> &pos) {
    pos.clear();
    if (n < 20) return SWC_OK;
    const u64 cap = 1u << 22;
    void *p = nullptr;
    int st = arena_get(2, 256 + cap * 8, &p, 0);
    if (st) return st;
    unsigned long long *count = (unsigned long long *)p;
    u64 *range = (u64 *)p + 1;                                        // the one unit: offset 0, length n
    u64 *list = (u64 *)((u8 *)p + 256);
    const u64 head[3] = {0, 0, n};
    SWC_CUDA_TRY(cudaMemcpy(p, head, sizeof head, cudaMemcpyHostToDevice));
    if ((st = gzip_scan(GzipScan{d_in, range, range + 1, 1, count, nullptr, list, cap, false}, 0))) return st;
    unsigned long long h = 0;
    SWC_CUDA_TRY(cudaMemcpy(&h, count, 8, cudaMemcpyDeviceToHost));
    if (h > cap) return SWC_OK;                                       // absurd candidate count: caller walks sequentially
    std::vector<u64> tmp(h);
    if (h) SWC_CUDA_TRY(cudaMemcpy(tmp.data(), list, h * 8, cudaMemcpyDeviceToHost));
    std::sort(tmp.begin(), tmp.end());
    pos.assign(tmp.begin(), tmp.end());
    return SWC_OK;
}

// bzip2 block / end-of-stream magics at EVERY bit offset (blocks are not byte aligned: BZip2.swift:71-90 reads 48 bits from
// wherever the previous block ended).  Entry = bit position << 1 | (1 for the end-of-stream magic).
__global__ void __launch_bounds__(256) bzip2_magic_scan_kernel(const u8 *d, u64 begin, u64 n, u64 *list, unsigned long long *count, u64 cap) {
    const u64 i = begin + (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i + 6 > n) return;                                            // a magic needs 48 bits
    u64 w = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) w = (w << 8) | (i + k < n ? d[i + k] : 0);   // bits of bytes i..i+6, MSB first
    u32 blk, eos;
    bzip2_magics_in_byte(w, (int)min((n - i) * 8 - 47, (u64)8), &blk, &eos);
    for (u32 m = blk | eos; m; m &= m - 1) {
        const u32 b = __ffs(m) - 1;
        const u64 slot = atomicAdd(count, 1ull);
        if (slot < cap) list[slot] = ((i * 8 + b) << 1) | ((eos >> b) & 1u);
    }
}

int find_bzip2_magics(const u8 *d_in, u64 begin, u64 n, std::vector<u64> &entries) {
    entries.clear();
    if (n < begin + 6) return SWC_OK;
    const u64 cap = 1u << 20;
    void *p = nullptr;
    int st = arena_get(2, 256 + cap * 8, &p, 0);
    if (st) return st;
    unsigned long long *count = (unsigned long long *)p;
    u64 *list = (u64 *)((u8 *)p + 256);
    SWC_CUDA_TRY(cudaMemsetAsync(count, 0, 8, 0));
    const u64 threads = n - begin;
    bzip2_magic_scan_kernel<<<(unsigned)((threads + 255) / 256), 256>>>(d_in, begin, n, list, count, cap);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    unsigned long long h = 0;
    SWC_CUDA_TRY(cudaMemcpy(&h, count, 8, cudaMemcpyDeviceToHost));
    if (h > cap) return SWC_OK;                                       // caller decodes sequentially
    entries.resize(h);
    if (h) SWC_CUDA_TRY(cudaMemcpy(entries.data(), list, h * 8, cudaMemcpyDeviceToHost));
    std::sort(entries.begin(), entries.end());
    return SWC_OK;
}

// gather: unit i's bytes [src_off[i], +len[i]) -> dst[dst_off[i] ...), one warp per unit
__global__ void __launch_bounds__(256) gather_units_kernel(const u8 *src, const u64 *src_off, const u64 *len, u8 *dst, const u64 *dst_off, u64 n) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= n) return;
    const u32 lane = threadIdx.x & 31;
    const u8 *s = src + src_off[unit];
    u8 *d = dst + dst_off[unit];
    const u64 L = len[unit];
    for (u64 i = lane; i < L; i += 32) d[i] = s[i];
}

int gather_units(const u8 *src, const u64 *src_off, const u64 *len, u8 *dst, const u64 *dst_off, u64 n, cudaStream_t s) {
    if (!n) return SWC_OK;
    gather_units_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(src, src_off, len, dst, dst_off, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// ---------------------------------------------------------------- xxHash32 (seed 0), one thread per buffer
#define XP1 0x9E3779B1u
#define XP2 0x85EBCA77u
#define XP3 0xC2B2AE3Du
#define XP4 0x27D4EB2Fu
#define XP5 0x165667B1u
__device__ __forceinline__ u32 rotl32(u32 v, int s) { return __funnelshift_l(v, v, s); }
__device__ __forceinline__ u32 rd32(const u8 *p) { return (u32)p[0] | (u32)p[1] << 8 | (u32)p[2] << 16 | (u32)p[3] << 24; }

// One WARP per buffer.  The four accumulators of xxHash32 (XxHash32.swift:39-57) are four serial chains over the 16-byte
// stripes — nothing to parallelise there — but a single thread spends most of its time waiting for its own loads.  Here the
// 32 lanes fetch 32 stripes (512 B, coalesced) one chunk ahead into shared memory and lanes 0..3 run one chain each out of
// shared memory: ~1 byte per cycle per buffer instead of ~0.1.
__global__ void __launch_bounds__(128) xxh32_warp_kernel(const u8 *base, const u64 *off, const u64 *len, u32 *result, u64 n) {
    __shared__ u32 stripes[4][2][128];
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u64 unit = (u64)blockIdx.x * 4 + warp;
    if (unit >= n) return;
    const u8 *p = base + (off ? off[unit] : 0);
    const u64 bytes = len[unit] & ~(1ull << 63);
    const u64 nstripes = bytes / 16;
    const bool aligned = (((uintptr_t)p) & 15) == 0;
    auto fetch = [&](u64 s) -> uint4 {                                  // stripe s (caller guarantees s < nstripes)
        const u8 *q = p + s * 16;
        if (aligned) return __ldg((const uint4 *)q);
        return make_uint4(rd32(q), rd32(q + 4), rd32(q + 8), rd32(q + 12));
    };
    u32 acc = lane == 0 ? XP1 + XP2 : lane == 1 ? XP2 : lane == 2 ? 0u : 0u - XP1;
    uint4 next = make_uint4(0, 0, 0, 0);
    if (lane < nstripes) next = fetch(lane);
    int buf = 0;
    for (u64 s0 = 0; s0 < nstripes; s0 += 32, buf ^= 1) {
        u32 *st = stripes[warp][buf];
        *(uint4 *)(st + lane * 4) = next;
        if (s0 + 32 + lane < nstripes) next = fetch(s0 + 32 + lane);   // the next chunk travels while this one is hashed
        __syncwarp();
        const u32 cnt = nstripes - s0 < 32 ? (u32)(nstripes - s0) : 32u;
        if (lane < 4)
            for (u32 k = 0; k < cnt; k++) acc = rotl32(acc + st[k * 4 + lane] * XP2, 13) * XP1;
        __syncwarp();
    }
    const u32 a0 = __shfl_sync(SWC_FULL, acc, 0), a1 = __shfl_sync(SWC_FULL, acc, 1), a2 = __shfl_sync(SWC_FULL, acc, 2), a3 = __shfl_sync(SWC_FULL, acc, 3);
    if (lane == 0) {
        u32 h = bytes < 16 ? XP5 : rotl32(a0, 1) + rotl32(a1, 7) + rotl32(a2, 12) + rotl32(a3, 18);
        h += (u32)bytes;
        u64 i = nstripes * 16;
        for (; bytes - i >= 4; i += 4) h = rotl32(h + rd32(p + i) * XP3, 17) * XP4;
        for (; bytes - i >= 1; i += 1) h = rotl32(h + (u32)p[i] * XP5, 11) * XP1;
        h ^= h >> 15; h *= XP2; h ^= h >> 13; h *= XP3; h ^= h >> 16;
        result[unit] = h;
    }
}

int xxh32_batch(const u8 *base, const u64 *off, const u64 *len, u32 *result, u64 n, cudaStream_t s) {
    if (!n) return SWC_OK;
    xxh32_warp_kernel<<<(unsigned)((n + 3) / 4), 128, 0, s>>>(base, off, len, result, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// ---------------------------------------------------------------- SHA-256, one thread
__global__ void sha256_kernel(const u8 *p, u64 n, u8 *digest) { sha256_buffer(p, n, digest); }

int sha256(const u8 *d, u64 n, u8 *d_digest, cudaStream_t s) {
    sha256_kernel<<<1, 1, 0, s>>>(d, n, d_digest);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// ---- host convenience ----
int check_device(Kind k, const u8 *d, u64 n, u64 *value) {
    DevBuf res, part;
    int st;
    {   // result slot + chunk partials live in a grow-only arena: per-block checks of big archives do no cudaMalloc
        void *a = nullptr;
        if ((st = arena_get(3, 64 + partial_bytes(n), &a, 0))) return st;
        res.borrow(a, 32);
        part.borrow((u8 *)a + 64, partial_bytes(n));
    }
    if (k == XXH32) {
        SWC_CUDA_TRY(cudaMemcpy(res.p, &n, 8, cudaMemcpyHostToDevice));
        if ((st = xxh32_batch(d, nullptr, res.as<u64>(), (u32 *)(res.as<u8>() + 8), 1, 0))) return st;
        u32 v = 0;
        SWC_CUDA_TRY(cudaMemcpy(&v, res.as<u8>() + 8, 4, cudaMemcpyDeviceToHost));
        *value = v;
        return SWC_OK;
    }
    switch (k) {
    case CRC32: st = crc32(d, n, res.as<u64>(), part.as<u64>(), 0); break;
    case BZIP2_CRC32: st = bzip2_crc32(d, n, res.as<u64>(), part.as<u64>(), 0); break;
    case CRC64: st = crc64(d, n, res.as<u64>(), part.as<u64>(), 0); break;
    default: st = adler32(d, n, res.as<u64>(), part.as<u64>(), 0); break;
    }
    if (st) return st;
    SWC_CUDA_TRY(cudaMemcpy(value, res.p, 8, cudaMemcpyDeviceToHost));
    return SWC_OK;
}

}  // namespace checks
}  // namespace swc
