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

// The contiguous run [b, e) of n units that thread threadIdx.x of a 1024-thread CTA takes: ceil(n / 1024) of them, in order.
__device__ __forceinline__ void cta_unit_run(u64 n, u64 &b, u64 &e) {
    const u64 per = (n + 1023) / 1024;
    b = threadIdx.x * per < n ? threadIdx.x * per : n;
    e = b + per < n ? b + per : n;
}

// the inclusive prefix sum of part[k][0..1024) in place (one CTA of 1024 threads)
template <int K> __device__ __forceinline__ void cta_scan(u64 (*part)[1024]) {
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
        u64 v[K];
#pragma unroll
        for (int k = 0; k < K; k++) v[k] = threadIdx.x >= (u32)d ? part[k][threadIdx.x - d] : 0;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < K; k++) part[k][threadIdx.x] += v[k];
        __syncthreads();
    }
}

// One CTA: entries [0, cnt) in launch order by a counting sort on key(j) in 0..64, the leading zeros of a size, so the
// largest come first.  put(j, at) gives entry j launch position `at`.
template <typename Key, typename Put> __device__ __forceinline__ void clz_order(u64 cnt, Key key, Put put) {
    __shared__ u32 start[65];
    if (threadIdx.x < 65) start[threadIdx.x] = 0;
    __syncthreads();
    for (u64 j = threadIdx.x; j < cnt; j += blockDim.x) atomicAdd(&start[key(j)], 1u);
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 at = 0;
        for (int k = 0; k < 65; k++) { const u32 h = start[k]; start[k] = at; at += h; }
    }
    __syncthreads();
    for (u64 j = threadIdx.x; j < cnt; j += blockDim.x) put(j, atomicAdd(&start[key(j)], 1u));
}

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
int scratch_get(size_t bytes, void **p, cudaStream_t stream, bool *kept = nullptr);
// grow-only arenas reused across calls: slot 0 = kernel scratch, 1..3 = device staging of the *_batch_host paths.
// *kept (optional): the arena was large enough, so it still holds what the last call left in it.
int arena_get(int slot, size_t bytes, void **p, cudaStream_t stream, bool *kept = nullptr);

}  // namespace swc
