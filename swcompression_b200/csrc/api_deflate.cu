// api_deflate.cu — C ABI for Deflate (include/swcgpu.h): batched device call, batched host call, single unit.
#include <cstdlib>
#include <cstring>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "inflate.cuh"

namespace swc {

int to_host_alloc(const void *d, size_t n, uint8_t **out, size_t *out_len) {
    uint8_t *h = (uint8_t *)swc_alloc(n);
    if (!h) return SWC_ERR_OUTPUT_OVERFLOW;
    if (n) {
        int st = copy_pageable(h, d, n, false);
        if (st) { swc_free(h); return st; }
    }
    *out = h;
    *out_len = n;
    return SWC_OK;
}

int deflate_batch_impl(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, const uint8_t *start_bits,
                              uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t out_total,
                              uint64_t *out_len, uint64_t *consumed_bits, int32_t *status, uint64_t n,
                              void *scratch, size_t scratch_bytes, cudaStream_t stream) {
    if (n == 0) return SWC_OK;
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !consumed_bits || !status)
        return SWC_ERR_INVALID_ARG;
    const size_t need = inflate::scratch_bytes(n, out_total);
    if (!scratch) {
        int st = scratch_get(need, &scratch, stream);
        if (st) return st;
    } else if (scratch_bytes < need) {
        return SWC_ERR_INVALID_ARG;
    }
    inflate::BatchArgs a;
    a.in_base = in_base; a.in_off = in_off; a.in_len = in_len; a.start_bits = start_bits;
    a.out_base = out_base; a.out_off = out_off; a.out_cap = out_cap;
    a.out_len = out_len; a.consumed_bits = consumed_bits; a.status = status; a.n = n;
    a.ticket = (unsigned long long *)scratch;                       // 8 bytes (256 reserved)
    a.rec_count = (u32 *)((u8 *)scratch + 256);                     // n entries
    a.rec_base = (u32 *)((u8 *)scratch + 256 + ((n * 4 + 255) & ~(size_t)255));
    return inflate::launch(a, stream);
}

// Decode one Deflate stream that already sits on the device; grows the output buffer until it fits.
int deflate_unit_device(const u8 *d_in, size_t in_len, size_t start_bit_abs, UnitResult &r, size_t hint) {
    size_t start_byte = start_bit_abs >> 3;
    if (start_byte > in_len) start_byte = in_len;
    u8 sb = (u8)(start_bit_abs & 7);
    size_t cap = hint ? hint : (in_len - start_byte) * 4 + 65536;
    DevBuf meta;
    int st = meta.alloc(256);
    if (st) return st;
    for (int attempt = 0; attempt < 3; attempt++) {
        cap = round16(cap);
        if ((st = r.out.alloc(cap))) return st;
        // meta layout: in_off, in_len, out_off, out_cap, out_len, consumed (u64 each) | status (i32) | start_bits (u8)
        u64 h[6] = {start_byte, in_len - start_byte, 0, cap, 0, 0};
        SWC_CUDA_TRY(cudaMemcpy(meta.p, h, sizeof(h), cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy((u8 *)meta.p + 64, &sb, 1, cudaMemcpyHostToDevice));
        u64 *m = meta.as<u64>();
        st = deflate_batch_impl(d_in, m + 0, m + 1, (u8 *)meta.p + 64, r.out.as<u8>(), m + 2, m + 3, cap, m + 4, m + 5,
                                (int32_t *)((u8 *)meta.p + 48), 1, nullptr, 0, 0);
        if (st) return st;
        SWC_CUDA_TRY(cudaStreamSynchronize(0));
        u64 res[7];
        SWC_CUDA_TRY(cudaMemcpy(res, meta.p, 56, cudaMemcpyDeviceToHost));
        r.out_len = (size_t)res[4];
        r.consumed = (size_t)res[5];
        int32_t st32; memcpy(&st32, &res[6], 4);
        r.status = st32;
        if (r.status != SWC_ERR_OUTPUT_OVERFLOW) break;
        cap = r.out_len;          // exact size reported by the counting pass
    }
    if (r.status == SWC_INTERNAL_NEEDS_SLOW) r.status = SWC_ERR_UNSUPPORTED;
    return SWC_OK;
}

}  // namespace swc

using namespace swc;

extern "C" {

size_t swc_deflate_batch_scratch_bytes(uint64_t n, uint64_t out_capacity_total) {
    return inflate::scratch_bytes(n, out_capacity_total);
}

int32_t swc_deflate_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     const uint8_t *start_bits,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t out_capacity_total,
                                     uint64_t *out_len, uint64_t *consumed_bits, int32_t *status,
                                     uint64_t n, void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    return deflate_batch_impl(in_base, in_off, in_len, start_bits, out_base, out_off, out_cap, out_capacity_total,
                              out_len, consumed_bits, status, n, scratch, scratch_bytes, (cudaStream_t)cuda_stream);
}

// Host-buffer batch: the units are cut into slices that flow through three CUDA streams, so the host->device copy of
// slice k+1, the kernels of slice k and the device->host copy of slice k-1 overlap (PCIe is full duplex). Device staging
// buffers come from grow-only arenas, so steady-state calls do no cudaMalloc.
int32_t swc_deflate_decompress_batch_host(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                          uint64_t in_total,
                                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                          uint64_t out_total,
                                          uint64_t *out_len, uint64_t *consumed_bits, int32_t *status, uint64_t n) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !consumed_bits || !status) return SWC_ERR_INVALID_ARG;
    DeviceCtx &ctx = device_ctx();                                       // streams / event / pinned result buffer of THIS device
    cudaStream_t *streams = ctx.streams;
    if (!streams[0]) {
        for (int i = 0; i < 3; i++) SWC_CUDA_TRY(cudaStreamCreateWithFlags(&streams[i], cudaStreamNonBlocking));
        SWC_CUDA_TRY(cudaEventCreateWithFlags(&ctx.tables_ready, cudaEventDisableTiming));
    }
    cudaEvent_t tables_ready = ctx.tables_ready;
    // every unit must lie inside the two arenas (checked for ALL units, without overflowing sums); slices additionally need
    // monotone offsets so that a slice is one contiguous byte range on both sides
    bool monotone = true;
    for (uint64_t i = 0; i < n; i++) {
        if (in_off[i] > in_total || in_len[i] > in_total - in_off[i] || out_off[i] > out_total || out_cap[i] > out_total - out_off[i])
            return SWC_ERR_INVALID_ARG;
        if (out_off[i] & 15) return SWC_ERR_INVALID_ARG;
        if (i && (in_off[i] < in_off[i - 1] + in_len[i - 1] || out_off[i] < out_off[i - 1] + out_cap[i - 1])) monotone = false;
    }
    static const int s_env = [] { const char *e = getenv("SWC_HOST_SLICES"); return e ? atoi(e) : 0; }();
    // slice count: ~2048 units per slice keeps the warp-per-unit decoder's grid full while the first device->host copy can
    // start after 1/32 of the batch
    uint64_t S = 1;
    if (monotone && n >= 4096) { S = s_env > 0 ? (uint64_t)s_env : n / 2048; if (S > 32) S = 32; if (S > 64) S = 64; }
    void *p_in = nullptr, *p_out = nullptr, *p_meta = nullptr, *p_scr = nullptr;
    int st;
    const size_t tb = n * 8;
    const size_t hdr = 256 * 64 + ((n * 4 + 255) & ~(size_t)255);      // up to 64 slices, one ticket block each
    if ((st = arena_get(1, round16(in_total) + 64, &p_in, 0))) return st;
    if ((st = arena_get(2, round16(out_total) + 64, &p_out, 0))) return st;
    if ((st = arena_get(3, tb * 6 + n * 4 + 256, &p_meta, 0))) return st;
    if ((st = arena_get(0, hdr + (out_total / 3 + 2) * 4 + 256, &p_scr, 0))) return st;
    // result tables come back through a library-owned pinned buffer: a D2H into pageable caller memory would block the
    // host thread inside the slice loop and serialise the whole pipeline
    const size_t res_bytes = n * 20;
    if (ctx.h_res_bytes < res_bytes) {
        if (ctx.h_res) cudaFreeHost(ctx.h_res);
        ctx.h_res = nullptr; ctx.h_res_bytes = 0;
        SWC_CUDA_TRY(cudaMallocHost((void **)&ctx.h_res, res_bytes + (res_bytes >> 2)));
        ctx.h_res_bytes = res_bytes + (res_bytes >> 2);
    }
    u8 *h_res = ctx.h_res;
    u64 *h_out_len = (u64 *)h_res, *h_cons = h_out_len + n;
    int32_t *h_status = (int32_t *)(h_cons + n);
    u8 *m = (u8 *)p_meta;
    u64 *d_in_off = (u64 *)(m + 0 * tb), *d_in_len = (u64 *)(m + 1 * tb), *d_out_off = (u64 *)(m + 2 * tb), *d_out_cap = (u64 *)(m + 3 * tb);
    u64 *d_out_len = (u64 *)(m + 4 * tb), *d_cons = (u64 *)(m + 5 * tb);
    int32_t *d_status = (int32_t *)(m + 6 * tb);
    SWC_CUDA_TRY(cudaMemcpyAsync(d_in_off, in_off, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaMemcpyAsync(d_in_len, in_len, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaMemcpyAsync(d_out_off, out_off, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaMemcpyAsync(d_out_cap, out_cap, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaEventRecord(tables_ready, streams[0]));
    for (uint64_t k = 0; k < S; k++) {
        const uint64_t b = n * k / S, e = n * (k + 1) / S;
        if (b == e) continue;
        cudaStream_t s = streams[k % 3];
        SWC_CUDA_TRY(cudaStreamWaitEvent(s, tables_ready, 0));
        const uint64_t i0 = S == 1 ? 0 : in_off[b], i1 = S == 1 ? in_total : in_off[e - 1] + in_len[e - 1];
        SWC_CUDA_TRY(cudaMemcpyAsync((u8 *)p_in + i0, in_base + i0, i1 - i0, cudaMemcpyHostToDevice, s));
        inflate::BatchArgs a;
        a.in_base = (const u8 *)p_in; a.in_off = d_in_off + b; a.in_len = d_in_len + b; a.start_bits = nullptr;
        a.out_base = (u8 *)p_out; a.out_off = d_out_off + b; a.out_cap = d_out_cap + b;
        a.out_len = d_out_len + b; a.consumed_bits = d_cons + b; a.status = d_status + b; a.n = e - b;
        a.ticket = (unsigned long long *)((u8 *)p_scr + 256 * k);
        a.rec_count = (u32 *)((u8 *)p_scr + 256 * 64) + b;
        a.rec_base = (u32 *)((u8 *)p_scr + hdr);
        if ((st = inflate::launch(a, s))) return st;
        // only the output regions come back: the caller's bytes between and around them are not ours to overwrite
        // (regions that touch are merged, so a densely packed slice is still one copy)
        for (uint64_t i = b; i < e;) {
            const uint64_t r0 = out_off[i];
            uint64_t r1 = r0 + out_cap[i++];
            while (i < e && out_off[i] == r1) r1 += out_cap[i++];
            if (r1 > r0) SWC_CUDA_TRY(cudaMemcpyAsync(out_base + r0, (u8 *)p_out + r0, r1 - r0, cudaMemcpyDeviceToHost, s));
        }
        SWC_CUDA_TRY(cudaMemcpyAsync(h_out_len + b, d_out_len + b, (e - b) * 8, cudaMemcpyDeviceToHost, s));
        SWC_CUDA_TRY(cudaMemcpyAsync(h_cons + b, d_cons + b, (e - b) * 8, cudaMemcpyDeviceToHost, s));
        SWC_CUDA_TRY(cudaMemcpyAsync(h_status + b, d_status + b, (e - b) * 4, cudaMemcpyDeviceToHost, s));
    }
    for (int i = 0; i < 3; i++) SWC_CUDA_TRY(cudaStreamSynchronize(streams[i]));
    memcpy(out_len, h_out_len, n * 8);
    memcpy(consumed_bits, h_cons, n * 8);
    memcpy(status, h_status, n * 4);
    return SWC_OK;
}

int32_t swc_deflate_decompress(const uint8_t *in, size_t in_len, size_t start_bit,
                               uint8_t **out, size_t *out_len, size_t *consumed_bits) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bits) *consumed_bits = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    int st = d_in.alloc(round16(in_len) + 16);
    if (st) return st;
    { int cst = copy_pageable(d_in.p, in, in_len, true); if (cst) return cst; }
    UnitResult r;
    if ((st = deflate_unit_device(d_in.as<u8>(), in_len, start_bit, r))) return st;
    if (consumed_bits) *consumed_bits = r.consumed;
    if (r.status != SWC_OK) return r.status;
    return to_host_alloc(r.out.p, r.out_len, out, out_len);
}

}  // extern "C"
