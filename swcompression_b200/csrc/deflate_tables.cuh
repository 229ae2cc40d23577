// deflate_tables.cuh — Deflate constants and the canonical limit-compare decoder shared by the Huffman-stage kernels
// (inflate_lut.cu, inflate_warp.cu) and the generic decoder (inflate_slow.cu); their block-header grammar is deflate_header.cuh.
// The library is built without relocatable device code, so every translation unit gets its own module: the tables are
// `static` to give each one a private copy (a plain __constant__ here would define the host shadow symbols twice).
#pragma once
#include "common.cuh"

namespace swc {
namespace inflate {

// RFC 1951 3.2.5 tables as {base | extra_bits << 16}; Deflate+Constants.swift:179-186 + Deflate.swift:188-189,206
static __constant__ u32 c_len_tab[32] = {
    3, 4, 5, 6, 7, 8, 9, 10, 11 | 1 << 16, 13 | 1 << 16, 15 | 1 << 16, 17 | 1 << 16, 19 | 2 << 16, 23 | 2 << 16, 27 | 2 << 16,
    31 | 2 << 16, 35 | 3 << 16, 43 | 3 << 16, 51 | 3 << 16, 59 | 3 << 16, 67 | 4 << 16, 83 | 4 << 16, 99 | 4 << 16,
    115 | 4 << 16, 131 | 5 << 16, 163 | 5 << 16, 195 | 5 << 16, 227 | 5 << 16, 258, 0, 0, 0};
static __constant__ u32 c_dist_tab[32] = {
    1, 2, 3, 4, 5 | 1 << 16, 7 | 1 << 16, 9 | 2 << 16, 13 | 2 << 16, 17 | 3 << 16, 25 | 3 << 16, 33 | 4 << 16, 49 | 4 << 16,
    65 | 5 << 16, 97 | 5 << 16, 129 | 6 << 16, 193 | 6 << 16, 257 | 7 << 16, 385 | 7 << 16, 513 | 8 << 16, 769 | 8 << 16,
    1025 | 9 << 16, 1537 | 9 << 16, 2049 | 10 << 16, 3073 | 10 << 16, 4097 | 11 << 16, 6145 | 11 << 16, 8193 | 12 << 16,
    12289 | 12 << 16, 16385 | 13 << 16, 24577 | 13 << 16, 0, 0};
// order of the code-length code lengths in a dynamic block header (RFC 1951 3.2.7)
static __constant__ u8 c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct Limits {
    u32 p[8];   // p[k] = limit[2k+1] | limit[2k+2] << 16 ; limit[L] = left-justified end of the length-L code range
};

// Length of the canonical code at the head of r15 (the next 15 input bits, first bit most significant); 16 if no code matches.
__device__ __forceinline__ int code_length(u32 r15, const Limits &lim) {
    // count the limits that r15 has reached; limits are non-decreasing so this is the code length - 1
    const u32 X = (r15 | (r15 << 16)) + 0x80008000u;
    u32 t[8];
#pragma unroll
    for (int k = 0; k < 8; k++) t[k] = X - lim.p[k];       // bit15 / bit31 = (r15 >= limit)
    // gather the 16 flag bytes (byte1/byte3 of each t) into 4 words, fold, one popc
    u32 a = __byte_perm(t[0], t[1], 0x7531), b = __byte_perm(t[2], t[3], 0x7531);
    u32 c = __byte_perm(t[4], t[5], 0x7531), d = __byte_perm(t[6], t[7], 0x7531);
    u32 v = (a & 0x80808080u) | ((b & 0x80808080u) >> 1) | ((c & 0x80808080u) >> 2) | ((d & 0x80808080u) >> 3);
    return 1 + __popc(v);                                    // 16 => no code matches (incomplete set)
}

// Index in the canonically sorted symbol list of the length-L code at the head of r15, given
// w = {first left-justified code of length L | index of its first symbol << 16}.
__device__ __forceinline__ u32 canonical_index(u32 r15, int L, u32 w) {
    return (w >> 16) + ((r15 - (w & 0xFFFFu)) >> (15 - L));
}

}  // namespace inflate
}  // namespace swc
