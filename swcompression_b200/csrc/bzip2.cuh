// bzip2.cuh — argument block of the BZip2 kernel.
#pragma once
#include "common.cuh"

namespace swc {
namespace bzip2 {

struct Args : DecodeIO {
    u8 *scratch;
    const u64 *scr_off;      // per unit, bytes into scratch
    const u8 *start_bits = nullptr;   // block mode: bit offset (0..7) of the block magic inside the unit's first byte
    int32_t block_mode = 0;           // 1: every unit is one block (magic first), decode it and stop; 0: whole streams
};

size_t scratch_per_unit(u64 out_cap);
int launch(const Args &a, cudaStream_t stream);

}  // namespace bzip2
}  // namespace swc
