// api_deflate.cu — C ABI for Deflate (include/swcgpu.h): batched device call, batched host call, single unit.
#include <cstdlib>
#include <cstring>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "inflate.cuh"

namespace swc {

int deflate_batch_impl(const DecodeIO &io, const uint8_t *start_bits, uint64_t out_total, void *scratch, size_t scratch_bytes,
                       cudaStream_t stream) {
    if (io.n == 0) return SWC_OK;
    if (missing(io)) return SWC_ERR_INVALID_ARG;
    const size_t need = inflate::scratch_bytes(io.n, out_total);
    if (!scratch) {
        int st = scratch_get(need, &scratch, stream);
        if (st) return st;
    } else if (scratch_bytes < need) {
        return SWC_ERR_INVALID_ARG;
    }
    inflate::BatchArgs a{io, start_bits};
    inflate::seat_scratch(a, scratch, io.n, 0, 1, 0);
    return inflate::launch(a, stream);
}

// Decode one Deflate stream that already sits on the device; retries once more at the exact size the counting pass reports.
static int deflate_unit_device(const u8 *d_in, size_t in_len, size_t start_bit_abs, UnitResult &r) {
    size_t start_byte = start_bit_abs >> 3;
    if (start_byte > in_len) start_byte = in_len;
    UnitTable t;
    UnitCols c(t, 1);
    const Col<u8> sb = t.in<u8>(1);
    *t.host(sb) = (u8)(start_bit_abs & 7);
    int st = decode_unit(t, c, d_in, start_byte, in_len, (in_len - start_byte) * 4 + 65536, 3, [](size_t, size_t need) { return need; },
                         [&](const DecodeIO &io, size_t cap) { return deflate_batch_impl(io, t.dev(sb), cap, nullptr, 0, 0); }, r);
    if (st) return st;
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
    const DecodeIO io{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bits};
    return deflate_batch_impl(io, start_bits, out_capacity_total, scratch, scratch_bytes, (cudaStream_t)cuda_stream);
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
    if (missing(DecodeIO{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bits}))
        return SWC_ERR_INVALID_ARG;
    DeviceCtx &ctx = device_ctx();                                       // streams / event / pinned result buffer of THIS device
    cudaStream_t *streams = ctx.streams;
    if (!streams[0]) {
        for (int i = 0; i < 3; i++) SWC_CUDA_TRY(cudaStreamCreateWithFlags(&streams[i], cudaStreamNonBlocking));
        SWC_CUDA_TRY(cudaEventCreateWithFlags(&ctx.tables_ready, cudaEventDisableTiming));
    }
    cudaEvent_t tables_ready = ctx.tables_ready;
    // slices additionally need monotone offsets so that a slice is one contiguous byte range on both sides
    bool monotone = true;
    int st = check_host_units(in_off, in_len, in_total, out_off, out_cap, out_total, n, &monotone);
    if (st) return st;
    static const int s_env = [] { const char *e = getenv("SWC_HOST_SLICES"); return e ? atoi(e) : 0; }();
    // slice count: ~2048 units per slice keeps the warp-per-unit decoder's grid full while the first device->host copy can
    // start after 1/32 of the batch
    uint64_t S = 1;
    if (monotone && n >= 4096) { S = s_env > 0 ? (uint64_t)s_env : n / 2048; if (S > 32) S = 32; if (S > 64) S = 64; }
    // the unit table lives in an arena; its columns are filled straight from the caller's arrays
    UnitTable t;
    const UnitCols c(t, n, false);
    void *p_in = nullptr, *p_out = nullptr, *p_meta = nullptr, *p_scr = nullptr;
    const size_t tb = n * 8;
    const int tickets = 64;                                              // up to 64 slices, one ticket block each
    if ((st = arena_get(1, round16(in_total) + 64, &p_in, 0))) return st;
    if ((st = arena_get(2, round16(out_total) + 64, &p_out, 0))) return st;
    if ((st = arena_get(3, t.bytes(), &p_meta, 0))) return st;
    if ((st = arena_get(0, inflate::scratch_header(n, tickets) + (out_total / 3 + 2) * 4 + 256, &p_scr, 0))) return st;
    t.place(p_meta);
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
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(c.in_off), in_off, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(c.in_len), in_len, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(c.out_off), out_off, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(c.out_cap), out_cap, tb, cudaMemcpyHostToDevice, streams[0]));
    SWC_CUDA_TRY(cudaEventRecord(tables_ready, streams[0]));
    for (uint64_t k = 0; k < S; k++) {
        const uint64_t b = n * k / S, e = n * (k + 1) / S;
        if (b == e) continue;
        cudaStream_t s = streams[k % 3];
        SWC_CUDA_TRY(cudaStreamWaitEvent(s, tables_ready, 0));
        const uint64_t i0 = S == 1 ? 0 : in_off[b], i1 = S == 1 ? in_total : in_off[e - 1] + in_len[e - 1];
        SWC_CUDA_TRY(cudaMemcpyAsync((u8 *)p_in + i0, in_base + i0, i1 - i0, cudaMemcpyHostToDevice, s));
        inflate::BatchArgs a{c.bind(t, (const u8 *)p_in, (u8 *)p_out, b, e - b), nullptr};
        inflate::seat_scratch(a, p_scr, n, b, tickets, (int)k);
        if ((st = inflate::launch(a, s))) return st;
        if ((st = copy_back_regions(out_base, (const u8 *)p_out, out_off, out_cap, b, e, s))) return st;
        SWC_CUDA_TRY(cudaMemcpyAsync(h_out_len + b, a.out_len, (e - b) * 8, cudaMemcpyDeviceToHost, s));
        SWC_CUDA_TRY(cudaMemcpyAsync(h_cons + b, a.consumed, (e - b) * 8, cudaMemcpyDeviceToHost, s));
        SWC_CUDA_TRY(cudaMemcpyAsync(h_status + b, a.status, (e - b) * 4, cudaMemcpyDeviceToHost, s));
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
    int st = upload_input(d_in, in, in_len);
    if (st) return st;
    UnitResult r;
    if ((st = deflate_unit_device(d_in.as<u8>(), in_len, start_bit, r))) return st;
    if (consumed_bits) *consumed_bits = r.consumed;
    if (r.status != SWC_OK) return r.status;
    return to_host_alloc(r.out.p, r.out_len, out, out_len);
}

}  // extern "C"
