// api_bzip2.cu — C ABI for BZip2 (include/swcgpu.h): batched device call, single stream, multi-stream.
#include <cstring>
#include <vector>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "bzip2.cuh"
#include "checks.cuh"

using namespace swc;

namespace {

// Lays the scratch out for units of output capacity caps[0, a.n) (host): a table of a.n offsets rounded up to 256 bytes,
// then scratch_per_unit(cap) bytes per unit.  Uploads the table into the front of the scratch and launches.  When the pool
// cannot supply the scratch, *no_scratch is set and its status returned without a launch.
int launch_with_scratch(bzip2::Args a, const u64 *caps, cudaStream_t stream, bool *no_scratch = nullptr) {
    std::vector<u64> soff(a.n);
    size_t total = (a.n * 8 + 255) & ~(size_t)255;
    for (u64 i = 0; i < a.n; i++) { soff[i] = total; total += bzip2::scratch_per_unit(caps[i]); }
    void *scratch = nullptr;
    int st = scratch_get(total, &scratch, stream);
    if (no_scratch) *no_scratch = st != SWC_OK;
    if (st) return st;
    SWC_CUDA_TRY(cudaMemcpyAsync(scratch, soff.data(), a.n * 8, cudaMemcpyHostToDevice, stream));
    SWC_CUDA_TRY(cudaStreamSynchronize(stream));     // soff lives on this stack frame
    a.scratch = (u8 *)scratch; a.scr_off = (const u64 *)scratch;
    return bzip2::launch(a, stream);
}

// whole streams; the per-unit scratch sizes depend on the capacities: fetch them (n x 8 bytes)
int bzip2_batch_impl(const DecodeIO &io, cudaStream_t stream) {
    if (io.n == 0) return SWC_OK;
    if (missing(io)) return SWC_ERR_INVALID_ARG;
    std::vector<u64> caps;
    int st = read_lens(io.out_cap, io.n, stream, caps);
    return st ? st : launch_with_scratch(bzip2::Args{io}, caps.data(), stream);
}

// 32 bits at an arbitrary bit position of the host copy, MSB first (BZip2's reader order)
uint32_t bits32_at(const uint8_t *in, size_t in_len, uint64_t bitpos) {
    uint64_t w = 0;
    const size_t b0 = (size_t)(bitpos >> 3);
    for (int k = 0; k < 5; k++) w = (w << 8) | (b0 + k < in_len ? in[b0 + k] : 0);
    return (uint32_t)(w >> (8 - (bitpos & 7)));
}

// Block-parallel decode of ONE stream.  The blocks of a stream are independent once their starts are known, and the starts
// are marked by a 48-bit magic — at any bit offset.  All magics are found by a device scan, every block candidate is decoded
// as its own unit of one batched launch (block mode of the kernel), and the reference's sequential walk (BZip2.swift:66-95)
// is kept as the validator: block k is accepted iff it decoded cleanly (including its CRC) and ended exactly at the next
// magic; the walk must end on the end-of-stream magic with the right combined CRC.  Anything else (a look-alike magic, an
// overflowing block, damage) leaves *done == false and the caller decodes the stream the sequential way, which also
// produces the reference's error.  `in` is the host copy of the archive, d_in the device copy.
int bzip2_stream_by_blocks(const uint8_t *in, const u8 *d_in, size_t in_len, size_t start, UnitResult &r, bool *done) {
    *done = false;
    if (in_len < start + 14) return SWC_OK;
    if (in[start] != 'B' || in[start + 1] != 'Z' || in[start + 2] != 'h' || in[start + 3] < '1' || in[start + 3] > '9') return SWC_OK;
    const size_t level = (size_t)(in[start + 3] - '0');
    std::vector<u64> mags;
    int st = checks::find_bzip2_magics(d_in, start + 4, in_len, mags);
    if (st) return st;
    // blocks from the first magic (which must sit right behind the header) up to the first end-of-stream magic
    std::vector<u64> pos;
    u64 end_pos = 0; bool have_end = false;
    for (u64 e : mags) {
        if (e & 1) { end_pos = e >> 1; have_end = true; break; }
        pos.push_back(e >> 1);
    }
    if (!have_end || pos.size() < 2 || pos[0] != (u64)(start + 4) * 8) return SWC_OK;
    const size_t nb = pos.size();
    const size_t cap = round16(level * 100000 * 2 + 65536);          // RLE1 can expand a block further: then the sequential path takes over
    UnitTable t;
    UnitCols c(t, nb);
    const Col<u8> sb = t.in<u8>(nb);
    for (size_t k = 0; k < nb; k++) {
        t.host(c.in_off)[k] = pos[k] >> 3; t.host(c.in_len)[k] = in_len - (pos[k] >> 3);
        t.host(c.out_off)[k] = k * cap; t.host(c.out_cap)[k] = cap;
        t.host(sb)[k] = (u8)(pos[k] & 7);
    }
    // the block-parallel attempt needs nb x (cap + ~6 x cap of scratch); when that does not fit, the sequential decoder (which
    // holds one block at a time) takes over instead of failing the call
    {
        size_t free_b = 0, total_b = 0;
        SWC_CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        const size_t need = nb * (cap + bzip2::scratch_per_unit(cap)) + ((size_t)64 << 20);
        if (need > free_b / 2) return SWC_OK;
    }
    DevBuf d_out;
    if (d_out.alloc(nb * cap + 64)) return SWC_OK;
    if (t.alloc()) return SWC_OK;
    if ((st = t.upload())) return st;
    const std::vector<u64> caps(nb, cap);
    bool no_scratch = false;
    if ((st = launch_with_scratch(bzip2::Args{c.bind(t, d_in, d_out.as<u8>(), 0, nb), nullptr, nullptr, t.dev(sb), 1}, caps.data(), 0,
                                  &no_scratch)))
        return no_scratch ? SWC_OK : st;
    UnitCols::Results res;
    if ((st = c.fetch(t, res))) return st;
    // the in-order walk: every block must end where the next magic starts, the last one at the end-of-stream magic
    uint32_t total_crc = 0;
    UnitTable g;
    const Col<u64> dst = g.in<u64>(nb);
    u64 *g_dst = g.host(dst);
    u64 out_total = 0;
    for (size_t k = 0; k < nb; k++) {
        const u64 ends_at = (pos[k] & ~7ull) + res.consumed[k];            // consumed is counted from the unit's first byte
        const u64 next = k + 1 < nb ? pos[k + 1] : end_pos;
        if (res.status[k] != SWC_OK || ends_at != next) return SWC_OK;
        const uint32_t block_crc = bits32_at(in, in_len, pos[k] + 48);
        total_crc = ((total_crc << 1) | (total_crc >> 31)) ^ block_crc;  // BZip2.swift:83-84
        g_dst[k] = out_total;
        out_total += res.out_len[k];
    }
    if (end_pos + 80 > (u64)in_len * 8) return SWC_OK;
    if (bits32_at(in, in_len, end_pos + 48) != total_crc) return SWC_OK;   // the sequential path reports wrongCRC with its payload
    // contiguous result
    if ((st = r.out.alloc(round16((size_t)out_total) + 64))) return st;
    if ((st = g.alloc()) || (st = g.upload())) return st;
    if ((st = checks::gather_units(d_out.as<u8>(), t.dev(c.out_off), t.dev(c.out_len), r.out.as<u8>(), g.dev(dst), nb, 0))) return st;
    SWC_CUDA_TRY(cudaStreamSynchronize(0));
    r.out_len = (size_t)out_total;
    r.consumed = (size_t)(end_pos + 80 - (u64)start * 8);
    r.status = SWC_OK;
    *done = true;
    return SWC_OK;
}

// one stream starting at byte `start` of d_in; output grows until it fits.  `in` (optional) = host copy of the archive:
// with it, multi-block streams are first tried block-parallel.
int bzip2_unit_device(const u8 *d_in, size_t in_len, size_t start, UnitResult &r, const uint8_t *in = nullptr) {
    if (in) {
        bool done = false;
        int bst = bzip2_stream_by_blocks(in, d_in, in_len, start, r, &done);
        if (bst) return bst;
        if (done) return SWC_OK;
    }
    UnitTable t;
    UnitCols c(t, 1);
    // BZip2 cannot report the final size before it has decoded everything: x4 per attempt
    return decode_unit(t, c, d_in, start, in_len, (in_len - start) * 16 + (1u << 20), 8,
                       [](size_t cap, size_t) { return cap >= ((size_t)1 << 32) ? 0 : cap * 4; },
                       [](const DecodeIO &io, size_t) { return bzip2_batch_impl(io, 0); }, r);
}

}  // namespace

extern "C" {

int32_t swc_bzip2_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                   uint64_t *out_len, uint64_t *consumed_bits, int32_t *status,
                                   uint64_t n, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    const DecodeIO io{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bits};
    return bzip2_batch_impl(io, (cudaStream_t)cuda_stream);
}

// BZip2.decompress(data:) BZip2.swift:22-26 (+ reader form :50)
int32_t swc_bzip2_decompress(const uint8_t *in, size_t in_len, size_t start_bit,
                             uint8_t **out, size_t *out_len, size_t *consumed_bits) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bits) *consumed_bits = 0;
    if (start_bit & 7) return SWC_ERR_UNSUPPORTED;      // the reference's byte reads require an aligned reader (BZip2.swift:59)
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    int st = upload_input(d_in, in, in_len);
    if (st) return st;
    UnitResult r;
    if ((st = bzip2_unit_device(d_in.as<u8>(), in_len, start_bit >> 3, r, in))) return st;
    if (consumed_bits) *consumed_bits = r.consumed;
    if (r.status != SWC_OK && r.status != SWC_BZIP2_WRONG_CRC) return r.status;
    if ((st = to_host_alloc(r.out.p, r.out_len, out, out_len))) return st;
    return r.status;
}

// BZip2.multiDecompress(data:) BZip2.swift:40-48
int32_t swc_bzip2_multi_decompress(const uint8_t *in, size_t in_len,
                                   uint8_t **out, size_t *out_len, size_t **stream_ends, size_t *n_streams) {
    if (!out || !out_len || !stream_ends || !n_streams) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0; *stream_ends = nullptr; *n_streams = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    int st = upload_input(d_in, in, in_len);
    if (st) return st;
    HostOut o;
    std::vector<size_t> ends;
    size_t off = 0;
    int result = SWC_OK;
    // ---- fast path: discover the streams up front and decode them as ONE batch ------------------------------------
    // A stream starts byte-aligned with 'B' 'Z' 'h' '1'..'9' followed by a block magic (or the end magic of an empty
    // stream).  Candidates found by scanning for that 10-byte signature are decoded in parallel; a candidate is accepted
    // only if the previous stream ended exactly there (consumed bytes == distance to the next candidate).  The first
    // stream that does not validate — or fails — hands over to the sequential loop below, which IS the reference's
    // order of events (BZip2.swift:40-48), so results and errors are the same with or without the fast path.
    {
        std::vector<size_t> cand;
        static const uint8_t blk[6] = {0x31, 0x41, 0x59, 0x26, 0x53, 0x59}, eos[6] = {0x17, 0x72, 0x45, 0x38, 0x50, 0x90};
        for (size_t i = 0; i + 10 <= in_len; i++) {
            if (in[i] != 'B' || in[i + 1] != 'Z' || in[i + 2] != 'h' || in[i + 3] < '1' || in[i + 3] > '9') continue;
            if (memcmp(in + i + 4, blk, 6) == 0 || memcmp(in + i + 4, eos, 6) == 0) cand.push_back(i);
        }
        if (cand.size() >= 2 && cand[0] == 0) {
            const size_t n = cand.size();
            auto len_of = [&](size_t k) { return (k + 1 < n ? cand[k + 1] : in_len) - cand[k]; };
            auto cap_of = [&](size_t k) { return round16(len_of(k) * 12 + (1u << 20)); };
            // groups bounded by a scratch budget (the BWT working set is ~6x the output capacity of a unit)
            const size_t budget = (size_t)24 << 30;
            size_t k0 = 0;
            bool handed_over = false;
            while (k0 < n && !handed_over) {
                size_t k1 = k0, need = 0;
                while (k1 < n) {
                    const size_t add = bzip2::scratch_per_unit(cap_of(k1)) + cap_of(k1);
                    if (k1 > k0 && need + add > budget) break;
                    need += add; k1++;
                }
                const size_t g = k1 - k0;
                UnitTable t;
                UnitCols c(t, g);
                u64 *h_len = t.host(c.in_len), *h_ooff = t.host(c.out_off);
                size_t out_total = 0;
                for (size_t j = 0; j < g; j++) {
                    t.host(c.in_off)[j] = cand[k0 + j]; h_len[j] = len_of(k0 + j);
                    h_ooff[j] = out_total; t.host(c.out_cap)[j] = cap_of(k0 + j);
                    out_total += cap_of(k0 + j);
                }
                DevBuf d_out;
                if ((st = d_out.alloc(out_total + 64))) return st;
                if ((st = t.alloc()) || (st = t.upload())) return st;
                if ((st = bzip2_batch_impl(c.bind(t, d_in.as<u8>(), d_out.as<u8>(), 0, g), 0))) return st;
                UnitCols::Results res;
                if ((st = c.fetch(t, res))) return st;
                for (size_t j = 0; j < g; j++) {
                    const u64 r_len = res.out_len[j];
                    const bool ok = res.status[j] == SWC_OK && (res.consumed[j] + 7) / 8 == h_len[j];
                    if (!ok) { off = cand[k0 + j]; handed_over = true; break; }   // sequential loop re-decodes this stream
                    uint8_t *dst = o.grow(r_len);
                    if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
                    if (r_len) SWC_CUDA_TRY(cudaMemcpy(dst, d_out.as<u8>() + h_ooff[j], r_len, cudaMemcpyDeviceToHost));
                    ends.push_back(o.len);
                    off = cand[k0 + j] + h_len[j];
                }
                k0 = k1;
            }
        }
    }
    while (off < in_len) {                               // !reader.isFinished
        UnitResult r;
        if ((st = bzip2_unit_device(d_in.as<u8>(), in_len, off, r, in))) return st;
        if (r.status != SWC_OK && r.status != SWC_BZIP2_WRONG_CRC) return r.status;
        if (r.status == SWC_BZIP2_WRONG_CRC) { o.len = 0; ends.clear(); }   // payload = the failing archive only
        uint8_t *dst = o.grow(r.out_len);
        if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
        if (r.out_len) SWC_CUDA_TRY(cudaMemcpy(dst, r.out.p, r.out_len, cudaMemcpyDeviceToHost));
        ends.push_back(o.len);
        if (r.status) { result = r.status; break; }
        off += (r.consumed + 7) / 8;                     // reader.align()
    }
    if ((st = o.release_to(out, out_len)) || (st = give_sizes(ends, stream_ends, out, out_len))) return st;
    *n_streams = ends.size();
    return result;
}

}  // extern "C"
