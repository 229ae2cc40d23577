// api_bzip2_compress.cu — C ABI for BZip2 compression: .bz2 stream batches in device memory, and the single call
// BZip2.compress(data:blockSize:) (BZip2+Compress.swift:44-74).
#include <cstring>
#include <vector>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "bzip2_compress.cuh"

using namespace swc;

namespace {

constexpr u64 kCompressPoolLimit = 16ull << 30;      // library-pool scratch per slice of a compress batch

int batch_impl(const bzip2c::Args &a, const std::vector<uint64_t> &lens, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    using namespace bzip2c;
    const u64 n = a.n, raw = (u64)RAW_PER_LEVEL * a.level;
    u64 total = 4096, biggest = 0;
    for (u64 i = 0; i < n; i++) {
        const u64 need = unit_scratch(lens[i], a.level);
        total += need;
        if (need > biggest) biggest = need;
    }
    size_t cap = scratch_bytes;
    if (!scratch) {
        cap = (size_t)(total < kCompressPoolLimit ? total : kCompressPoolLimit);
        if (cap < 4096 + biggest) cap = (size_t)(4096 + biggest);
        int st = scratch_get(cap, &scratch, s);
        if (st) return st;
    }
    u8 *scr = (u8 *)scratch;
    std::vector<u8> plan;
    for (u64 first = 0; first < n;) {
        u64 count = 0, used = 4096;
        while (first + count < n) {
            const u64 need = unit_scratch(lens[first + count], a.level);
            if (used + need > cap) break;
            used += need;
            count++;
        }
        if (count == 0) return SWC_ERR_INVALID_ARG;                       // caller scratch smaller than one unit needs
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
        int st = run(a, first, count, sl, s);
        if (st) return st;
        first += count;
    }
    return SWC_OK;
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
    std::vector<uint64_t> lens(n);
    SWC_CUDA_TRY(cudaMemcpyAsync(lens.data(), in_len, n * 8, cudaMemcpyDeviceToHost, s));
    SWC_CUDA_TRY(cudaStreamSynchronize(s));
    for (u64 l : lens)
        if (l >= (1ull << 40)) return SWC_ERR_UNSUPPORTED;
    bzip2c::Args a;
    a.in_base = in_base; a.in_off = in_off; a.in_len = in_len;
    a.out_base = out_base; a.out_off = out_off; a.out_cap = out_cap; a.out_len = out_len; a.status = status; a.n = n;
    a.level = (u32)block_size;
    return batch_impl(a, lens, scratch, scratch_bytes, s);
}

// BZip2.compress(data:blockSize:) BZip2+Compress.swift:44-74
int32_t swc_bzip2_compress(const uint8_t *in, size_t in_len, int32_t block_size, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (block_size < 1 || block_size > 9) return SWC_ERR_INVALID_ARG;
    if ((u64)in_len >= (1ull << 40)) return SWC_ERR_UNSUPPORTED;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in, d_out;
    int st;
    if ((st = upload_input(d_in, in, in_len))) return st;
    const u64 cap = round16(bzip2c::max_stream_bytes(in_len, (u32)block_size));
    UnitTable t;
    const Col<u64> in_off = t.in<u64>(1), c_len = t.in<u64>(1), out_off = t.in<u64>(1), out_cap = t.in<u64>(1);
    const Col<u64> r_len = t.out<u64>(1);
    const Col<int32_t> r_st = t.out<int32_t>(1);
    if ((st = t.alloc()) || (st = d_out.alloc(cap))) return st;
    *t.host(c_len) = in_len; *t.host(out_cap) = cap;
    if ((st = t.upload())) return st;
    bzip2c::Args a;
    a.in_base = d_in.as<u8>(); a.in_off = t.dev(in_off); a.in_len = t.dev(c_len);
    a.out_base = d_out.as<u8>(); a.out_off = t.dev(out_off); a.out_cap = t.dev(out_cap);
    a.out_len = t.dev(r_len); a.status = t.dev(r_st); a.n = 1; a.level = (u32)block_size;
    const std::vector<uint64_t> lens(1, in_len);
    if ((st = batch_impl(a, lens, nullptr, 0, 0))) return st;
    std::vector<u64> len;
    std::vector<int32_t> status;
    if ((st = t.fetch(r_len, len)) || (st = t.fetch(r_st, status))) return st;
    if (status[0] != SWC_OK) return status[0];
    uint8_t *host = (uint8_t *)swc_alloc((size_t)len[0]);
    if (!host) return SWC_ERR_OUTPUT_OVERFLOW;
    if ((st = copy_pageable(host, d_out.p, (size_t)len[0], false))) { swc_free(host); return st; }
    *out = host; *out_len = (size_t)len[0];
    return SWC_OK;
}

}  // extern "C"
