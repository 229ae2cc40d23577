// host_util.h — host-side helpers shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <vector>
#include "common.cuh"

#include <mutex>

namespace swc {

int ensure_device();

// ---- per-device library context (runtime.cu) -----------------------------------------------------------------------------
// The reference is re-entrant; here the mutable state is one lazily created context per device: scratch arenas, the streams /
// pinned result buffer of the *_batch_host paths, one-time kernel configuration flags.  Every C-ABI entry point that touches it
// holds the device's API mutex for the duration of the call (ApiLock), so any number of host threads may call into the library
// concurrently on the same or on different devices; calls on one device are serialised, calls on different devices are not.
struct DeviceCtx {
    std::recursive_mutex api_mu;
    std::mutex cfg_mu;
    bool configured[16] = {};
    cudaStream_t streams[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t tables_ready = nullptr;
    uint8_t *h_res = nullptr;
    size_t h_res_bytes = 0;
    int num_sms = 0;
};
DeviceCtx &device_ctx();                 // context of the CURRENT device
struct ApiLock {
    std::unique_lock<std::recursive_mutex> lk;
    ApiLock() : lk(device_ctx().api_mu) {}
};
enum { CFG_INFLATE_K1W = 0, CFG_INFLATE_K1L = 1, CFG_LZMA = 2, CFG_BZIP2_CRC = 3, CFG_LZ4 = 4 };
// runs `f` (returning an swc status) once per device, thread-safe; a failing `f` is retried by the next caller
template <typename F> int configure_once(int slot, F f) {
    DeviceCtx &c = device_ctx();
    std::lock_guard<std::mutex> g(c.cfg_mu);
    if (c.configured[slot]) return SWC_OK;
    if (!c.num_sms) {
        int dev = 0;
        SWC_CUDA_TRY(cudaGetDevice(&dev));
        SWC_CUDA_TRY(cudaDeviceGetAttribute(&c.num_sms, cudaDevAttrMultiProcessorCount, dev));
    }
    const int st = f(c);
    if (st == SWC_OK) c.configured[slot] = true;
    return st;
}

// RAII device allocation (single-unit paths; the batch paths use caller memory + the scratch pool)
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    bool owned = true;          // false: a view into memory owned elsewhere (never freed here)
    DevBuf() {}
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    void release() { if (p && owned) cudaFree(p); p = nullptr; bytes = 0; owned = true; }
    void borrow(void *ptr, size_t n) { release(); p = ptr; bytes = n; owned = false; }
    void take(DevBuf &o) { release(); p = o.p; bytes = o.bytes; owned = o.owned; o.p = nullptr; o.bytes = 0; o.owned = true; }
    int alloc(size_t n) {
        release();
        cudaError_t e = cudaMalloc(&p, n ? n : 16);
        if (e != cudaSuccess) { p = nullptr; return cuda_fail(e, "cudaMalloc"); }
        bytes = n;
        return SWC_OK;
    }
    template <typename T> T *as() const { return (T *)p; }
};

// result of decoding ONE unit that is already resident on the device
struct UnitResult {
    DevBuf out;            // decoded bytes (device)
    size_t out_len = 0;
    size_t consumed = 0;   // bits (Deflate/BZip2) or bytes (LZ4/LZMA)
    int status = 0;
};

// Deflate stream starting at byte `start` + `start_bit` bits inside d_in[0..in_len)
int deflate_unit_device(const u8 *d_in, size_t in_len, size_t start_bit_abs, UnitResult &r, size_t hint = 0);

// batched Deflate on device-resident tables (api_deflate.cu); scratch == nullptr -> library pool
int deflate_batch_impl(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, const uint8_t *start_bits,
                       uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t out_total,
                       uint64_t *out_len, uint64_t *consumed_bits, int32_t *status, uint64_t n,
                       void *scratch, size_t scratch_bytes, cudaStream_t stream);

inline size_t round16(size_t v) { return (v + 15) & ~(size_t)15; }

// large transfers between pageable host memory and the device: T threads x (stream + two pinned bounce buffers) (runtime.cu)
int copy_pageable(void *dst, const void *src, size_t bytes, bool to_device);

// hand a device buffer back to a C caller as swc_alloc'ed host memory
int to_host_alloc(const void *d, size_t n, uint8_t **out, size_t *out_len);

}  // namespace swc
