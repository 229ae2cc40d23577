// lzma.cuh — argument block of the LZMA / LZMA2 kernel.
#pragma once
#include "common.cuh"

namespace swc {
namespace lzma {

enum { MODE_LZMA2 = 0, MODE_RAW = 1 };

struct Args : DecodeIO {
    int mode;
    const u8 *dict_bytes;      // MODE_LZMA2: per-unit dictionary-size byte
    const u32 *props;          // MODE_RAW: lc | lp << 8 | pb << 16
    const i64 *dict_size;      // MODE_RAW
    const i64 *usize;          // MODE_RAW: < 0 = unknown (end marker required)
    u16 *lit_scratch;          // optional: n x 4096 x 0x300 u16 for streams with lc+lp > 4 (else those units are refused)
};

inline size_t lit_scratch_bytes(u64 n) { return (size_t)n * 4096 * 0x300 * 2; }
int launch(const Args &a, cudaStream_t stream);
int occupancy_blocks(int *blocks);   // resident lzma_kernel CTAs per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor)

}  // namespace lzma
}  // namespace swc
