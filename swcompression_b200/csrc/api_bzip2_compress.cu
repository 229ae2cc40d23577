// api_bzip2_compress.cu — C ABI for BZip2 compression: .bz2 stream batches in device memory, and the single call
// BZip2.compress(data:blockSize:) (BZip2+Compress.swift:44-74).
#include <vector>
#include "../../include/swcgpu.h"
#include "compress_host.h"
#include "bzip2_compress.cuh"

using namespace swc;

namespace {

int batch_impl(const bzip2c::Args &a, const std::vector<u64> &lens, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    using namespace bzip2c;
    const u64 raw = (u64)RAW_PER_LEVEL * a.level;
    std::vector<u8> plan;
    return run_in_slices(a.n, [&](u64 i) { return unit_scratch(lens[i], a.level); }, [](u64) { return (u64)4096; }, scratch,
                         scratch_bytes, s, [&](u64 first, u64 count, u8 *scr, size_t cap) -> int {
        // plans first, then per-block results, per-group results, block scratch and the units' staging words
        std::vector<BlockPlan> bl;
        std::vector<UnitPlan> un(count);
        u64 groups = 0, stage = 0;
        for (u64 j = 0; j < count; j++) {
            const u64 l = lens[first + j];
            un[j].block0 = (u32)bl.size();
            un[j].blocks = (u32)unit_blocks(l, a.level);
            un[j].stage = stage;
            un[j].stage_bytes = a256(max_stream_bytes(l, a.level) + 8);
            stage += un[j].stage_bytes;
            for (u32 b = 0; b < un[j].blocks; b++) {
                BlockPlan p{};
                p.unit = (u32)j; p.index = b;
                p.raw = (u32)(l - b * raw < raw ? l - b * raw : raw);
                p.cap = rle_cap(p.raw);
                p.group0 = groups;
                groups += group_slots(p.raw);
                bl.push_back(p);
            }
        }
        const u64 nb = bl.size();
        const u64 o_units = a256(nb * sizeof(BlockPlan)), o_meta = o_units + a256(count * sizeof(UnitPlan));
        const u64 o_groups = o_meta + a256(nb * 256), o_blocks = o_groups + a256(a256(25 * groups) + 4 * groups);
        u64 at = o_blocks;
        for (auto &p : bl) { p.scr = (u64)(uintptr_t)(scr + at); at += block_scratch(p.raw); }
        const u64 o_stage = at;
        if (o_stage + stage > cap) return SWC_ERR_INVALID_ARG;          // never: unit_scratch covers every region
        plan.assign(o_meta, 0);
        if (nb) memcpy(plan.data(), bl.data(), nb * sizeof(BlockPlan));
        memcpy(plan.data() + o_units, un.data(), count * sizeof(UnitPlan));
        // a copy from pageable memory has read `plan` when it returns, so the next slice may refill it
        SWC_CUDA_TRY(cudaMemcpyAsync(scr, plan.data(), plan.size(), cudaMemcpyHostToDevice, s));
        Slice sl;
        sl.blocks = (const BlockPlan *)scr; sl.units = (const UnitPlan *)(scr + o_units);
        sl.nblocks = nb; sl.ngroups = groups;
        sl.meta = scr + o_meta; sl.groups = scr + o_groups;
        sl.stage = scr + o_stage; sl.stage_bytes = stage;
        sl.max_stage = 1;
        for (const UnitPlan &u : un) sl.max_stage = u.stage_bytes > sl.max_stage ? u.stage_bytes : sl.max_stage;
        sl.copy_chunk = 64 << 10;                                         // at most 65 535 chunks per unit
        while ((sl.max_stage + sl.copy_chunk - 1) / sl.copy_chunk > 65535) sl.copy_chunk *= 2;
        return run(a, first, count, sl, s);
    });
}

}  // namespace

extern "C" {

size_t swc_bzip2_compress_max_bytes(uint64_t in_len, int32_t block_size) {
    if (block_size < 1 || block_size > 9) return 0;
    return (size_t)bzip2c::max_stream_bytes(in_len, (u32)block_size);
}

size_t swc_bzip2_compress_batch_scratch_bytes(uint64_t n, uint64_t in_bytes_total, int32_t block_size) {
    if (block_size < 1 || block_size > 9) return 0;
    // bzip2c::unit_scratch, bounded term by term: per raw byte 29 x 1.25 bytes of block scratch, 11 x 1.25 / 8 bits of
    // staging and 32 / 50 x 1.25 of group results (under 40 bytes in all); per block 29 x 264 bytes of rounding, 256 of
    // plan and results, 32 x 2 of group slots and 2 110 / 8 of header staging (under 9 KiB); per unit 1 KiB of
    // staging rounding and padding.  A unit of n bytes has at most n / raw + 1 blocks.
    const u64 blocks = n + in_bytes_total / (bzip2c::RAW_PER_LEVEL * (u64)block_size);
    return (size_t)(in_bytes_total * 40 + blocks * 9216 + n * 1024 + 4096);
}

int32_t swc_bzip2_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, int32_t block_size,
                                 uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                 uint64_t *out_len, int32_t *status, uint64_t n,
                                 void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (block_size < 1 || block_size > 9) return SWC_ERR_INVALID_ARG;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !status) return SWC_ERR_INVALID_ARG;
    const cudaStream_t s = (cudaStream_t)cuda_stream;
    std::vector<u64> lens;
    int st = read_lens(in_len, n, s, lens);
    if (st) return st;
    for (u64 l : lens)
        if (l >= (1ull << 40)) return SWC_ERR_UNSUPPORTED;
    const bzip2c::Args a{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, (u32)block_size};
    return batch_impl(a, lens, scratch, scratch_bytes, s);
}

// BZip2.compress(data:blockSize:) BZip2+Compress.swift:44-74
int32_t swc_bzip2_compress(const uint8_t *in, size_t in_len, int32_t block_size, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (block_size < 1 || block_size > 9) return SWC_ERR_INVALID_ARG;
    if ((u64)in_len >= (1ull << 40)) return SWC_ERR_UNSUPPORTED;
    return compress_one(bzip2c::Args{{}, (u32)block_size}, batch_impl, bzip2c::max_stream_bytes(in_len, (u32)block_size), in,
                        in_len, out, out_len);
}

}  // extern "C"
