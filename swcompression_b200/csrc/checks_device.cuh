// checks_device.cuh — device pieces of the checksums shared by checks.cu and xz_batch.cu (the library is built without
// relocatable device code, so the one copy lives in this header): the GF(2) helpers of the CRC combine, the warp-per-buffer
// CRC-32 / CRC-64 and the one-thread SHA-256.
// Reference: Sources/Common/CheckSums.swift:12-45, Sources/XZ/Sha256.swift.
#pragma once
#include "common.cuh"

namespace swc {
namespace checks {

// ---------------------------------------------------------------- BZip2 magics at every bit offset
// BZip2.swift:71-90 reads the 48-bit block magic 0x314159265359 or end-of-stream magic 0x177245385090 from wherever the
// previous block ended, so a magic may start at any bit.  w holds bytes i .. i+6 MSB first (byte i in bits 55..48); a magic
// starts at bit b (0 = the byte's most significant bit) of byte i when the 48 bits from there match.  Only the first
// `limit` offsets are tested (fewer than 8 where the data ends inside the 48 bits).  Bit b of *blk / *eos = a match at b.
__device__ __forceinline__ void bzip2_magics_in_byte(u64 w, int limit, u32 *blk, u32 *eos) {
    u32 mb = 0, me = 0;
#pragma unroll
    for (int b = 0; b < 8; b++) {
        const u64 v = (w >> (8 - b)) & 0xFFFFFFFFFFFFull;
        if (b < limit) {
            mb |= (u32)(v == 0x314159265359ull) << b;
            me |= (u32)(v == 0x177245385090ull) << b;
        }
    }
    *blk = mb; *eos = me;
}

// ---------------------------------------------------------------- GF(2) helpers
// reflected 32-bit: bit 31 = x^0
__device__ inline u32 mulmod32r(u32 a, u32 b) {
    u32 m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
__device__ inline u64 mulmod64r(u64 a, u64 b) {
    u64 m = 1ull << 63, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xC96C5795D7870F42ull : b >> 1;
    }
    return p;
}
// normal (MSB-first) 32-bit: bit 0 = x^0, poly 0x04C11DB7
__device__ inline u32 mulmod32n(u32 a, u32 b) {
    u32 p = 0;
    while (a) {
        if (a & 1) p ^= b;
        a >>= 1;
        b = (b & 0x80000000u) ? (b << 1) ^ 0x04C11DB7u : b << 1;
    }
    return p;
}
// x^(8*nbytes) mod P in each representation
__device__ inline u32 xpow32r(u64 nbytes) {
    u32 p = 1u << 31, sq = 1u << 23;           // x^0, x^8
    while (nbytes) { if (nbytes & 1) p = mulmod32r(sq, p); sq = mulmod32r(sq, sq); nbytes >>= 1; }
    return p;
}
__device__ inline u64 xpow64r(u64 nbytes) {
    u64 p = 1ull << 63, sq = 1ull << 55;
    while (nbytes) { if (nbytes & 1) p = mulmod64r(sq, p); sq = mulmod64r(sq, sq); nbytes >>= 1; }
    return p;
}
__device__ inline u32 xpow32n(u64 nbytes) {
    u32 p = 1, sq = 1u << 8;
    while (nbytes) { if (nbytes & 1) p = mulmod32n(sq, p); sq = mulmod32n(sq, sq); nbytes >>= 1; }
    return p;
}

// ---------------------------------------------------------------- warp-per-buffer reflected CRC (CRC-32 and CRC-64)
struct Crc32R {
    typedef u32 T;
    static constexpr u32 POLY = 0xEDB88320u;
    __device__ static u32 mul(u32 a, u32 b) { return mulmod32r(a, b); }
    __device__ static u32 xpow(u64 n) { return xpow32r(n); }
    __device__ static u32 high(u32) { return 0; }
};
struct Crc64R {
    typedef u64 T;
    static constexpr u64 POLY = 0xC96C5795D7870F42ull;
    __device__ static u64 mul(u64 a, u64 b) { return mulmod64r(a, b); }
    __device__ static u64 xpow(u64 n) { return xpow64r(n); }
    __device__ static u64 high(u64 c) { return c >> 32; }
};

// the four slicing tables: tab[t][i] is the register after byte i and then t zero bytes.  Entries are independent, so
// threads first, first + stride, ... fill them without a barrier between the tables (the caller synchronises afterwards).
template <class K>
__device__ __forceinline__ void crc_tables(typename K::T (*tab)[256], u32 first, u32 stride) {
    for (u32 i = first; i < 1024; i += stride) {
        typename K::T c = i & 255;
        for (u32 k = 0, steps = 8 * ((i >> 8) + 1); k < steps; k++) c = (c & 1) ? K::POLY ^ (c >> 1) : c >> 1;
        tab[i >> 8][i & 255] = c;
    }
}

template <class K>
__device__ __forceinline__ typename K::T crc_word(const typename K::T (*tab)[256], typename K::T c, u32 w) {
    c ^= w;
    return tab[3][c & 0xFF] ^ tab[2][(c >> 8) & 0xFF] ^ tab[1][(c >> 16) & 0xFF] ^ tab[0][(u32)c >> 24] ^ K::high(c);
}

// CRC of p[0, L), every lane of the warp taking part and receiving it.  Each lane folds one of 32 contiguous segments (a
// multiple of 16 bytes, read with 16-byte loads, four bytes per table step), then the 32 conditioned values are chained with
// x^(8*len) multiplications (zlib's crc32_combine identity).  LDG: the buffer is read-only for the whole kernel and goes
// through the non-coherent path; without it, plain loads (the buffer may have been written by this warp).
template <class K, bool LDG = false>
__device__ __forceinline__ typename K::T warp_crc(const typename K::T (*tab)[256], const u8 *p, u64 L) {
    typedef typename K::T T;
    const u32 lane = lane_id();
    const u64 seg = (((L + 31) / 32) + 15) & ~(u64)15;
    const u64 sb = lane * seg < L ? lane * seg : L, se = sb + seg < L ? sb + seg : L;
    T c = ~(T)0;
    u64 i = sb;
    for (; i < se && ((uintptr_t)(p + i) & 15); i++) c = tab[0][(c ^ p[i]) & 0xFF] ^ (c >> 8);
    for (; i + 16 <= se; i += 16) {
        const uint4 v = LDG ? __ldg((const uint4 *)(p + i)) : *(const uint4 *)(p + i);
        c = crc_word<K>(tab, c, v.x); c = crc_word<K>(tab, c, v.y); c = crc_word<K>(tab, c, v.z); c = crc_word<K>(tab, c, v.w);
    }
    for (; i < se; i++) c = tab[0][(c ^ p[i]) & 0xFF] ^ (c >> 8);
    c = ~c;
    const T pw = K::xpow(seg);
    T acc = __shfl_sync(SWC_FULL, c, 0);
    for (int l = 1; l < 32; l++) {
        const T pl = __shfl_sync(SWC_FULL, c, l);
        const u64 lb = (u64)l * seg < L ? (u64)l * seg : L, le = lb + seg < L ? lb + seg : L;
        if (le == lb) continue;
        acc = K::mul(le - lb == seg ? pw : K::xpow(le - lb), acc) ^ pl;
    }
    return acc;
}

// ---------------------------------------------------------------- SHA-256, one thread (the round constants are read at a
// uniform index, so constant memory serves them)
static __constant__ u32 c_k256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
__device__ __forceinline__ u32 rotr32(u32 v, int s) { return __funnelshift_r(v, v, s); }

__device__ inline void sha256_block(u32 h[8], const u8 *b) {
    u32 w[64];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = (u32)b[4 * i] << 24 | (u32)b[4 * i + 1] << 16 | (u32)b[4 * i + 2] << 8 | b[4 * i + 3];
#pragma unroll
    for (int i = 16; i < 64; i++) {
        u32 s0 = rotr32(w[i - 15], 7) ^ rotr32(w[i - 15], 18) ^ (w[i - 15] >> 3);
        u32 s1 = rotr32(w[i - 2], 17) ^ rotr32(w[i - 2], 19) ^ (w[i - 2] >> 10);
        w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    u32 a = h[0], bb = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        u32 t1 = hh + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ((e & f) ^ (~e & g)) + c_k256[i] + w[i];
        u32 t2 = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + ((a & bb) ^ (a & c) ^ (bb & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = bb; bb = a; a = t1 + t2;
    }
    h[0] += a; h[1] += bb; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// Sha256.hash of p[0, n) into digest[32]
__device__ inline void sha256_buffer(const u8 *p, u64 n, u8 *digest) {
    u32 h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    u64 i = 0;
    for (; i + 64 <= n; i += 64) sha256_block(h, p + i);
    u8 tail[128];
    for (int k = 0; k < 128; k++) tail[k] = 0;
    u64 rem = n - i;
    for (u64 k = 0; k < rem; k++) tail[k] = p[i + k];
    tail[rem] = 0x80;
    int tl = rem + 9 <= 64 ? 64 : 128;
    u64 bits = n * 8;
    for (int k = 0; k < 8; k++) tail[tl - 1 - k] = (u8)(bits >> (8 * k));
    sha256_block(h, tail);
    if (tl == 128) sha256_block(h, tail + 64);
    for (int k = 0; k < 8; k++) { digest[4 * k] = (u8)(h[k] >> 24); digest[4 * k + 1] = (u8)(h[k] >> 16); digest[4 * k + 2] = (u8)(h[k] >> 8); digest[4 * k + 3] = (u8)h[k]; }
}

}  // namespace checks
}  // namespace swc
