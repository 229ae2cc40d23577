// api_deflate_compress.cu — C ABI for raw Deflate compression: batches in device memory, and the single call
// Deflate.compress (Deflate+Compress.swift:22-42).  The gzip and zlib archives are archive_compress.cu.
#include <vector>
#include "../../include/swcgpu.h"
#include "compress_host.h"
#include "deflate_compress.cuh"

using namespace swc;

namespace {

inline u64 meta_bytes(u64 count) { return (3 * count + 2) * 8 + 3 * 256; }

// the batch on device-resident tables; `lens` is the host copy of in_len
int batch_impl(const deflatec::Args &a, const std::vector<u64> &lens, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    std::vector<u64> plan;
    return run_in_slices(a.n, [&](u64 i) { return deflatec::unit_scratch(lens[i]); }, meta_bytes, scratch, scratch_bytes, s,
                         [&](u64 first, u64 count, u8 *scr, size_t) -> int {
        // the slice's plan first (scratch offsets, tile and chunk prefix sums), then each unit's region
        plan.assign(3 * count + 2, 0);
        u64 *off = plan.data(), *tiles = off + count, *chunks = tiles + count + 1;
        u64 at = meta_bytes(count);
        for (u64 j = 0; j < count; j++) {
            const u64 l = lens[first + j];
            off[j] = at; at += deflatec::unit_scratch(l);
            tiles[j + 1] = tiles[j] + deflatec::unit_tiles(l);
            chunks[j + 1] = chunks[j] + deflatec::unit_chunks(l);
        }
        // a copy from pageable memory has read `plan` when it returns, so the next slice may refill it
        SWC_CUDA_TRY(cudaMemcpyAsync(scr, plan.data(), plan.size() * 8, cudaMemcpyHostToDevice, s));
        deflatec::Plan p;
        p.scr_off = (const u64 *)scr; p.tile_start = p.scr_off + count; p.chunk_start = p.tile_start + count + 1;
        p.tiles = tiles[count]; p.chunks = chunks[count];
        return deflatec::run(a, first, count, scr, p, s);
    });
}

}  // namespace

extern "C" {

size_t swc_deflate_compress_batch_scratch_bytes(uint64_t n, uint64_t in_bytes_total) {
    // unit_scratch(l) <= 9 l + 2048 (link 2 l, chains 6 l, visited, checkpoints and alignment), plus the slice's plan
    return (size_t)(in_bytes_total * 9 + n * (2048 + 24) + 4096);
}

int32_t swc_deflate_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                   uint64_t *out_len, int32_t *status, uint64_t n,
                                   void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !status) return SWC_ERR_INVALID_ARG;
    const cudaStream_t s = (cudaStream_t)cuda_stream;
    // the scratch layout is planned on the host from the unit sizes (n x 8 bytes)
    std::vector<u64> lens;
    int st = read_lens(in_len, n, s, lens);
    if (st) return st;
    const deflatec::Args a{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}};
    return batch_impl(a, lens, scratch, scratch_bytes, s);
}

// Deflate.compress(data:) Deflate+Compress.swift:22-42
int32_t swc_deflate_compress(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (in_len >= deflatec::MAX_UNIT) return SWC_ERR_UNSUPPORTED;
    // (9 n + 17) / 8: the largest stream Deflate.compress writes for n bytes
    return compress_one(deflatec::Args{}, batch_impl, (9 * (u64)in_len + 17) / 8, in, in_len, out, out_len);
}

}  // extern "C"
