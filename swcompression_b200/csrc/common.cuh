// common.cuh — shared device/host helpers for libswcgpu (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/swc_status.h"

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int64_t i64;

#define SWC_WARP 32
#define SWC_FULL 0xFFFFFFFFu

// internal status: unit needs the generic (slow) decoder — never escapes the library
#define SWC_INTERNAL_NEEDS_SLOW 9001

namespace swc {

__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }

// the unit table of a batched kernel: unit i reads in_base[in_off[i], in_off[i] + in_len[i]) and writes
// out_base[out_off[i], out_off[i] + out_cap[i]); out_len[i] and status[i] are its results.  Each codec's Args extends it.
struct UnitIO {
    const u8 *in_base;
    const u64 *in_off, *in_len;
    u8 *out_base;
    const u64 *out_off, *out_cap;
    u64 *out_len;
    int32_t *status;
    u64 n;
};
// the unit table of a batched decoder: consumed[i] is how much of its input unit i read, in bits for Deflate and BZip2,
// in bytes for LZMA
struct DecodeIO : UnitIO {
    u64 *consumed;
};

// launch bookkeeping (swc_kernel_launches)
void count_launch(int n = 1);
// record a CUDA failure; returns SWC_ERR_CUDA
int cuda_fail(cudaError_t e, const char *where);

#define SWC_CUDA_TRY(expr)                                                     \
    do {                                                                       \
        cudaError_t _e = (expr);                                               \
        if (_e != cudaSuccess) return swc::cuda_fail(_e, #expr);               \
    } while (0)

// optional per-kernel timing: when enabled, launchers drop a CUDA event on `stream` between their kernels
void timing_mark(cudaStream_t stream);

// scratch pool: grow-only per-device buffer, used when the caller passes no scratch
int scratch_get(size_t bytes, void **p, cudaStream_t stream);
// grow-only arenas reused across calls: slot 0 = kernel scratch, 1..3 = device staging of the *_batch_host paths
int arena_get(int slot, size_t bytes, void **p, cudaStream_t stream);

}  // namespace swc
