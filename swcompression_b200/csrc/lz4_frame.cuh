// lz4_frame.cuh — pieces of the LZ4 frame format shared by the frame layers: the decoders (api_lz4.cu, lz4_frame_batch.cu)
// and the encoder (lz4_frame_compress.cu).
#pragma once
#include "common.cuh"

namespace swc {
namespace lz4f {

// FLG bits of the frame descriptor (LZ4.swift:198-214, LZ4+Compress.swift:57-81)
constexpr u32 FLG_DICT_ID = 0x01, FLG_CONTENT_CK = 0x04, FLG_CONTENT_SIZE = 0x08, FLG_BLOCK_CK = 0x10, FLG_INDEPENDENT = 0x20;

// xxHash32 of the <= 14-byte frame descriptor (XxHash32.swift:24-83 with n < 16); with n = 0 it is the hash of no bytes
__host__ __device__ __forceinline__ u32 xxh32_descriptor(const u8 *p, u32 n) {
    auto rotl = [](u32 v, int s) { return (v << s) | (v >> (32 - s)); };
    auto rd32 = [](const u8 *q) { return (u32)q[0] | (u32)q[1] << 8 | (u32)q[2] << 16 | (u32)q[3] << 24; };
    u32 acc = 0x165667B1u + n, i = 0;
    for (; n - i >= 4; i += 4) acc = rotl(acc + rd32(p + i) * 0xC2B2AE3Du, 17) * 0x27D4EB2Fu;
    for (; i < n; i++) acc = rotl(acc + (u32)p[i] * 0x165667B1u, 11) * 0x9E3779B1u;
    acc ^= acc >> 15; acc *= 0x85EBCA77u; acc ^= acc >> 13; acc *= 0xC2B2AE3Du; acc ^= acc >> 16;
    return acc;
}

}  // namespace lz4f
}  // namespace swc
