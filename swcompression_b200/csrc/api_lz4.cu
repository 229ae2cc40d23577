// api_lz4.cu — C ABI for LZ4: raw block batches (device / host) and the single calls LZ4.decompress /
// LZ4.multiDecompress (reference Sources/LZ4/LZ4.swift:73-146).  A frame is one unit of the frame batch
// (lz4_frame_batch.cu), which walks descriptors and block marks on the device and reports the reference's statuses;
// only multiDecompress's loop over frames (skippable frames, the next magic) stays on the host.
// The compress half here is the raw block batch; frames (LZ4.compress, LZ4+Compress.swift:16-154) are laid out on the
// device by lz4_frame_compress.cu.
#include <algorithm>
#include <vector>
#include "../../include/swcgpu.h"
#include "compress_host.h"
#include "lz4.cuh"
#include "lz4_compress.cuh"

using namespace swc;

namespace {

// LZ4.decompress(data:dictionary:dictionaryID:) of d_in[start, in_len) as a one-unit swc_lz4_frame_decompress_batch;
// r.consumed counts from `start`.  d_dict is NULL for `dictionary: nil`.
int frame_unit(const u8 *d_in, size_t in_len, size_t start, const u8 *d_dict, size_t dict_len, int32_t has_dict_id,
               uint32_t dict_id, UnitResult &r) {
    const u64 len = in_len - start;
    UnitTable t;
    const UnitCols c(t, 1);
    const Col<swc_lz4_frame_info> info = t.out<swc_lz4_frame_info>(1);
    // the walk alone first: it sizes the block table and the first output attempt
    std::vector<swc_lz4_frame_info> f;
    int st = t.alloc();
    if (st) return st;
    *t.host(c.in_off) = start;
    *t.host(c.in_len) = len;
    if ((st = t.upload()) || (st = swc_lz4_frame_info_batch(d_in, t.dev(c.in_off), t.dev(c.in_len), d_dict != nullptr, has_dict_id,
                                                            dict_id, t.dev(info), 1, 0)) || (st = t.fetch(info, f)))
        return st;
    // every block could be full, but no input byte decodes to more than 255 bytes; a legacy frame's blocks are guessed at
    // 8 MiB.  A unit that needs more reports its exact size, and the one rerun at that size is final.
    const u64 nb = f[0].n_blocks, max_block = f[0].max_block_size ? f[0].max_block_size : 8u << 20;
    u64 cap = std::min(nb * max_block, 255 * (len - f[0].frame_start) + 64 * nb);
    if (f[0].content_size != UINT64_MAX) cap = std::min(cap, f[0].content_size);
    const u64 max_blocks = nb ? nb : 1;
    const size_t scratch_bytes = swc_lz4_frame_batch_scratch_bytes(1, len, max_blocks);
    void *scratch = nullptr;
    if ((st = scratch_get(scratch_bytes, &scratch, 0))) return st;
    return decode_unit(t, c, d_in, start, in_len, cap, 2, [](size_t, size_t need) { return need; }, [&](const DecodeIO &io, size_t) {
        return swc_lz4_frame_decompress_batch(io.in_base, io.in_off, io.in_len, d_dict, dict_len, has_dict_id, dict_id, io.out_base,
                                              io.out_off, io.out_cap, io.out_len, io.consumed, io.status, 1, max_blocks, scratch,
                                              scratch_bytes, 0);
    }, r);
}

// the input, and the dictionary unless it is nil (an empty one is still a device pointer)
int upload(DevBuf &d_in, DevBuf &d_dict, const uint8_t *in, size_t in_len, const uint8_t *dict, size_t dict_len) {
    const int st = upload_input(d_in, in, in_len);
    return st || !dict ? st : upload_input(d_dict, dict, dict_len);
}

}  // namespace

extern "C" {

int32_t swc_lz4_block_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                       const uint8_t *dict, uint64_t dict_len,
                                       uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, int32_t *status, uint64_t n, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    lz4::Args a{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, nullptr, nullptr, dict, dict ? dict_len : 0, nullptr};
    if (missing(a)) return SWC_ERR_INVALID_ARG;
    // two-phase path needs a record scratch sized from the compressed lengths: fetch them once (n x 8 bytes)
    {
        std::vector<u64> lens;
        int st = read_lens(in_len, n, (cudaStream_t)cuda_stream, lens);
        if (st) return st;
        uint64_t total = 0;
        for (uint64_t i = 0; i < n; i++) total += lens[i] & ~(1ull << 63);
        void *scratch = nullptr;
        st = scratch_get(lz4::two_phase_scratch_bytes(n, total), &scratch, (cudaStream_t)cuda_stream);
        if (st) return st;
        a.scratch = scratch;
    }
    return lz4::launch(a, (cudaStream_t)cuda_stream);
}

int32_t swc_lz4_block_decompress_batch_host(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                            uint64_t in_total,
                                            uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                            uint64_t out_total,
                                            uint64_t *out_len, int32_t *status, uint64_t n) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    if (missing(UnitIO{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n})) return SWC_ERR_INVALID_ARG;
    bool monotone;
    int st = check_host_units(in_off, in_len, in_total, out_off, out_cap, out_total, n, &monotone);
    if (st) return st;
    // the unit table's columns are filled straight from the caller's arrays
    UnitTable t;
    const Col<u64> d_in_off = t.out<u64>(n), d_in_len = t.out<u64>(n), d_out_off = t.out<u64>(n), d_out_cap = t.out<u64>(n);
    const Col<u64> d_out_len = t.out<u64>(n);
    const Col<int32_t> d_status = t.out<int32_t>(n);
    DevBuf d_in, d_out;
    if ((st = d_in.alloc(round16(in_total) + 32))) return st;
    if ((st = d_out.alloc(round16(out_total)))) return st;
    if ((st = t.alloc())) return st;
    const size_t tb = n * 8;
    cudaStream_t s = 0;
    SWC_CUDA_TRY(cudaMemcpyAsync(d_in.p, in_base, in_total, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(d_in_off), in_off, tb, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(d_in_len), in_len, tb, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(d_out_off), out_off, tb, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(t.dev(d_out_cap), out_cap, tb, cudaMemcpyHostToDevice, s));
    st = swc_lz4_block_decompress_batch(d_in.as<u8>(), t.dev(d_in_off), t.dev(d_in_len), nullptr, 0, d_out.as<u8>(), t.dev(d_out_off),
                                        t.dev(d_out_cap), t.dev(d_out_len), t.dev(d_status), n, s);
    if (st) return st;
    if ((st = copy_back_regions(out_base, d_out.as<u8>(), out_off, out_cap, 0, n, s))) return st;
    SWC_CUDA_TRY(cudaMemcpyAsync(out_len, t.dev(d_out_len), tb, cudaMemcpyDeviceToHost, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(status, t.dev(d_status), n * 4, cudaMemcpyDeviceToHost, s));
    SWC_CUDA_TRY(cudaStreamSynchronize(s));
    return SWC_OK;
}

// LZ4.decompress(data:dictionary:dictionaryID:) LZ4.swift:73-91
int32_t swc_lz4_decompress(const uint8_t *in, size_t in_len, const uint8_t *dict, size_t dict_len,
                           int32_t has_dict_id, uint32_t dict_id, uint8_t **out, size_t *out_len, size_t *consumed_bytes) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bytes) *consumed_bytes = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in, d_dict;
    UnitResult r;
    int st = upload(d_in, d_dict, in, in_len, dict, dict_len);
    if (st || (st = frame_unit(d_in.as<u8>(), in_len, 0, d_dict.as<u8>(), dict_len, has_dict_id, dict_id, r))) return st;
    if (consumed_bytes) *consumed_bytes = r.consumed;
    if (r.status != SWC_OK && r.status != SWC_DATA_CHECKSUM_MISMATCH) return r.status;
    return (st = to_host_alloc(r.out.p, r.out_len, out, out_len)) ? st : r.status;
}

// LZ4.multiDecompress LZ4.swift:116-146: the frame loop on the host, each frame one unit of the frame batch
int32_t swc_lz4_multi_decompress(const uint8_t *in, size_t in_len, const uint8_t *dict, size_t dict_len,
                                 int32_t has_dict_id, uint32_t dict_id,
                                 uint8_t **out, size_t *out_len, size_t **frame_ends, size_t *n_frames) {
    if (!out || !out_len || !frame_ends || !n_frames) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0; *frame_ends = nullptr; *n_frames = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in, d_dict;
    int st = upload(d_in, d_dict, in, in_len, dict, dict_len);
    if (st) return st;
    HostOut o;
    std::vector<size_t> ends;
    size_t next = 0;
    int result = SWC_OK;
    do {
        if (in_len - next < 4) { result = SWC_DATA_TRUNCATED; break; }
        const uint32_t magic = le32(in + next);
        if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) {       // skipped here; unlike decompress(data:), the dictionary stays
            if (in_len - next - 4 < 4) { result = SWC_DATA_TRUNCATED; break; }
            const size_t size = le32(in + next + 4);
            if (in_len - next - 8 < size) { result = SWC_DATA_TRUNCATED; break; }
            next += 8 + size;
            continue;
        }
        if (magic != 0x184D2204u && magic != 0x184C2102u) { result = SWC_DATA_CORRUPTED; break; }
        UnitResult r;
        if ((st = frame_unit(d_in.as<u8>(), in_len, next, d_dict.as<u8>(), dict_len, has_dict_id, dict_id, r))) return st;
        result = r.status;
        if (result != SWC_OK && result != SWC_DATA_CHECKSUM_MISMATCH) break;
        uint8_t *dst = o.grow(r.out_len);
        if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
        if ((st = copy_pageable(dst, r.out.p, r.out_len, false))) return st;
        ends.push_back(o.len);
        next += r.consumed;
    } while (result == SWC_OK && next < in_len);
    if (result != SWC_OK && result != SWC_DATA_CHECKSUM_MISMATCH) return result;
    int g;
    if ((g = o.release_to(out, out_len)) || (g = give_sizes(ends, frame_ends, out, out_len))) return g;
    *n_frames = ends.size();
    return result;
}

}  // extern "C"

// ---- compression ----------------------------------------------------------------------------------------------------

namespace {

inline u64 window_of(u64 in_len, u64 dict_len) {
    if (in_len > lz4c::MAX_BLOCK || (dict_len >= 1 && dict_len <= 3)) return 0;       // rejected units need no scratch
    return in_len + (dict_len > lz4c::MAX_DICT ? lz4c::MAX_DICT : dict_len);
}
inline u64 need_of(u64 in_len, u64 dict_len) {
    const u64 w = window_of(in_len, dict_len);
    return lz4c::unit_scratch(w, w ? in_len : 0);
}
inline u64 meta_bytes(u64 count) { return (count * 8 + 255) & ~(u64)255; }

}  // namespace

extern "C" {

size_t swc_lz4_compress_batch_scratch_bytes(uint64_t n, uint64_t window_bytes_total) {
    // unit_scratch(w, l) <= 33 w / 8 + 795 for l <= w, plus 8 bytes of offsets per unit and the alignment of that table
    return (size_t)(window_bytes_total / 8 * 33 + 33 + n * 1040 + 4096);
}

int32_t swc_lz4_block_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     const uint64_t *dict_off, const uint64_t *dict_len,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t *out_len, int32_t *status, uint64_t n,
                                     void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !status) return SWC_ERR_INVALID_ARG;
    if ((dict_off == nullptr) != (dict_len == nullptr)) return SWC_ERR_INVALID_ARG;
    const cudaStream_t s = (cudaStream_t)cuda_stream;
    // the scratch layout is planned on the host from the unit sizes (n x 16 bytes)
    std::vector<u64> lens, dlens(n, 0), offs(n);
    int st = read_lens(in_len, n, s, lens);
    if (!st && dict_len) st = read_lens(dict_len, n, s, dlens);
    if (st) return st;
    const lz4c::Args a{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, dict_off, dict_len, nullptr};
    auto need = [&](u64 i) { return need_of(lens[i], dlens[i]); };
    return run_in_slices(n, need, meta_bytes, scratch, scratch_bytes, s, [&](u64 first, u64 count, u8 *scr, size_t) -> int {
        // the slice's table of offsets first, then each unit's region
        u64 at = meta_bytes(count);
        for (u64 j = 0; j < count; j++) { offs[first + j] = at; at += need(first + j); }
        SWC_CUDA_TRY(cudaMemcpyAsync(scr, offs.data() + first, count * 8, cudaMemcpyHostToDevice, s));
        int st = lz4c::parse(a, first, count, scr, (const u64 *)scr, s);
        return st ? st : lz4c::emit(a, first, count, scr, (const u64 *)scr, s);
    });
}

}  // extern "C"
