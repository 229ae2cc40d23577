// api_lz4.cu — C ABI for LZ4: raw block batches (device / host) and the frame layer of
// LZ4.decompress / LZ4.multiDecompress (reference Sources/LZ4/LZ4.swift:73-330).  Frame descriptors and block marks
// are walked on the host (a few bytes per block); block decode, block checksums and the content checksum run on the
// device.  Errors are reported in the order the reference's sequential loop would meet them.
// The compress half (LZ4.compress, LZ4+Compress.swift:16-154) writes its frame the other way round: every block is
// compressed on the device, the host lays out the frame from the compressed sizes, the device writes the payloads and
// checksums in place, and the host adds the header, block marks and EndMark.
#include <cstring>
#include <vector>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "lz4.cuh"
#include "lz4_compress.cuh"
#include "checks.cuh"

using namespace swc;

namespace {

inline uint32_t rd32(const uint8_t *p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
inline uint64_t rd64(const uint8_t *p) { return (uint64_t)rd32(p) | (uint64_t)rd32(p + 4) << 32; }
inline bool is_magic(uint32_t v) { return v == 0x184D2204u || v == 0x184C2102u || (v >= 0x184D2A50u && v <= 0x184D2A5Fu); }

// xxHash32 of the <= 14-byte frame descriptor (framing, not payload) — XxHash32.swift:24-83 with n < 16
uint32_t xxh32_descriptor(const uint8_t *p, size_t n) {
    auto rotl = [](uint32_t v, int s) { return (v << s) | (v >> (32 - s)); };
    uint32_t acc = 0x165667B1u + (uint32_t)n;
    size_t i = 0;
    for (; n - i >= 4; i += 4) acc = rotl(acc + rd32(p + i) * 0xC2B2AE3Du, 17) * 0x27D4EB2Fu;
    for (; n - i >= 1; i += 1) acc = rotl(acc + (uint32_t)p[i] * 0x165667B1u, 11) * 0x9E3779B1u;
    acc ^= acc >> 15; acc *= 0x85EBCA77u; acc ^= acc >> 13; acc *= 0xC2B2AE3Du; acc ^= acc >> 16;
    return acc;
}

struct Block { uint64_t off, len; bool stored; uint32_t stored_ck; bool has_ck; };

struct DeviceInput {      // compressed input + optional dictionary, resident on the device for one API call
    DevBuf in, dict;
    size_t in_len = 0, dict_len = 0;
    bool have_dict = false;
};

// Decode `blocks` (offsets into dev.in) as `units` on the device and append the result to `host_out`.
// mode: 0 = every block is its own unit (independent / legacy), 1 = one chain (dependent blocks).
// `pending_error` is the framing error the host scan stopped at (0 if it reached the EndMark).
int run_blocks(DeviceInput &dev, const std::vector<Block> &blocks, int mode, bool use_dict, size_t max_block,
               bool check_blocks, int pending_error, std::vector<uint8_t> &host_out, DevBuf &d_out_keep, size_t &d_out_len) {
    const size_t nb = blocks.size();
    d_out_len = 0;
    if (nb == 0) return pending_error;
    const size_t nunits = mode == 0 ? nb : 1;
    std::vector<uint64_t> h_off(nb), h_len(nb), u_off(nunits), u_cap(nunits);
    std::vector<uint32_t> h_first(nunits), h_cnt(nunits);
    for (size_t i = 0; i < nb; i++) { h_off[i] = blocks[i].off; h_len[i] = blocks[i].len | (blocks[i].stored ? 1ull << 63 : 0); }
    // first-attempt capacity: the frame's block size, but never more than an LZ4 block of that many bytes can expand to
    // (each input byte adds at most 255 output bytes) — frames made of many tiny flushed blocks would otherwise ask for
    // nb x 4 MiB; a block that decodes to more than this reports the size it needs and is redone (overflow retry below)
    auto cap_of = [&](size_t i) {
        if (blocks[i].stored) return round16(blocks[i].len);
        const size_t expand = blocks[i].len < (max_block / 255 + 1) ? blocks[i].len * 255 + 64 : max_block;
        return round16(expand < max_block ? expand : max_block);
    };
    size_t total = 0;
    if (mode == 0) {
        for (size_t i = 0; i < nb; i++) { u_off[i] = total; u_cap[i] = cap_of(i); total += u_cap[i]; h_first[i] = (uint32_t)i; h_cnt[i] = 1; }
    } else {
        for (size_t i = 0; i < nb; i++) total += cap_of(i);
        u_off[0] = 0; u_cap[0] = total; h_first[0] = 0; h_cnt[0] = (uint32_t)nb;
    }
    DevBuf d_meta, d_ck;
    std::vector<uint64_t> r_len(nunits);
    std::vector<int32_t> r_st(nunits);
    std::vector<uint32_t> r_ck(nb);
    int st;
    for (int attempt = 0; attempt < 2; attempt++) {
        if ((st = d_out_keep.alloc(total))) return st;
        const size_t mbytes = nb * 16 + nunits * (8 * 3 + 4 * 3) + 64;
        if ((st = d_meta.alloc(mbytes))) return st;
        uint8_t *m = d_meta.as<uint8_t>();
        uint64_t *d_boff = (uint64_t *)m, *d_blen = d_boff + nb, *d_uoff = d_blen + nb, *d_ucap = d_uoff + nunits, *d_ulen = d_ucap + nunits;
        uint32_t *d_first = (uint32_t *)(d_ulen + nunits), *d_cnt = d_first + nunits;
        int32_t *d_st = (int32_t *)(d_cnt + nunits);
        SWC_CUDA_TRY(cudaMemcpy(d_boff, h_off.data(), nb * 8, cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy(d_blen, h_len.data(), nb * 8, cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy(d_uoff, u_off.data(), nunits * 8, cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy(d_ucap, u_cap.data(), nunits * 8, cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy(d_first, h_first.data(), nunits * 4, cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy(d_cnt, h_cnt.data(), nunits * 4, cudaMemcpyHostToDevice));
        lz4::Args a;
        a.in_base = dev.in.as<u8>(); a.blk_off = d_boff; a.blk_len = d_blen; a.first_blk = d_first; a.n_blk = d_cnt;
        a.dict = use_dict && dev.have_dict ? dev.dict.as<u8>() : nullptr;
        a.dict_len = use_dict && dev.have_dict ? dev.dict_len : 0;
        if (mode == 1 && a.dict_len > 65536) { a.dict += a.dict_len - 65536; a.dict_len = 65536; }    // LZ4.swift:309
        a.out_base = d_out_keep.as<u8>(); a.out_off = d_uoff; a.out_cap = d_ucap; a.out_len = d_ulen; a.status = d_st; a.n = nunits;
        a.scratch = nullptr;
        if (mode == 0) {               // one block per unit: take the two-phase (parse + 8-wide execute) path
            uint64_t tot = 0;
            for (size_t i = 0; i < nb; i++) tot += blocks[i].len;
            void *scr = nullptr;
            if ((st = scratch_get(lz4::two_phase_scratch_bytes(nb, tot), &scr, 0))) return st;
            a.first_blk = nullptr; a.n_blk = nullptr; a.scratch = scr;
        }
        if ((st = lz4::launch(a, 0))) return st;
        if (check_blocks && attempt == 0) {
            if ((st = d_ck.alloc(nb * 4))) return st;
            if ((st = checks::xxh32_batch(dev.in.as<u8>(), d_boff, d_blen, d_ck.as<u32>(), nb, 0))) return st;
            SWC_CUDA_TRY(cudaMemcpy(r_ck.data(), d_ck.p, nb * 4, cudaMemcpyDeviceToHost));
        }
        SWC_CUDA_TRY(cudaMemcpy(r_len.data(), d_ulen, nunits * 8, cudaMemcpyDeviceToHost));
        SWC_CUDA_TRY(cudaMemcpy(r_st.data(), d_st, nunits * 4, cudaMemcpyDeviceToHost));
        bool overflow = false;
        for (size_t u = 0; u < nunits; u++) if (r_st[u] == SWC_ERR_OUTPUT_OVERFLOW) overflow = true;
        if (!overflow) break;
        // a block decoded to more than the frame's block size (the reference does not forbid it): redo with exact sizes
        total = 0;
        for (size_t u = 0; u < nunits; u++) {
            if (r_st[u] == SWC_ERR_OUTPUT_OVERFLOW || r_st[u] == SWC_OK) u_cap[u] = round16((size_t)r_len[u]);
            u_off[u] = total; total += u_cap[u];
        }
    }
    // report in the reference's sequential order: block k checksum (LZ4.swift:300), then block k decode (:305-313)
    if (mode == 0) {
        for (size_t i = 0; i < nb; i++) {
            if (check_blocks && blocks[i].has_ck && r_ck[i] != blocks[i].stored_ck) return SWC_DATA_CORRUPTED;
            if (r_st[i] != SWC_OK) return r_st[i];
        }
    } else {
        size_t fail_blk = r_st[0] != SWC_OK ? (size_t)r_len[0] : nb;
        for (size_t i = 0; i < nb; i++) {
            if (check_blocks && blocks[i].has_ck && r_ck[i] != blocks[i].stored_ck) return SWC_DATA_CORRUPTED;
            if (i == fail_blk) return r_st[0];
        }
        if (r_st[0] != SWC_OK) return r_st[0];
    }
    if (pending_error) return pending_error;
    // gather
    size_t produced = 0;
    for (size_t u = 0; u < nunits; u++) produced += (size_t)r_len[u];
    size_t base = host_out.size();
    host_out.resize(base + produced);
    bool contiguous = true;
    { size_t run = 0; for (size_t u = 0; u < nunits; u++) { if (u_off[u] != run) contiguous = false; run += (size_t)r_len[u]; } }
    if (contiguous) {
        if (produced) SWC_CUDA_TRY(cudaMemcpy(host_out.data() + base, d_out_keep.p, produced, cudaMemcpyDeviceToHost));
    } else {
        size_t w = base;
        for (size_t u = 0; u < nunits; u++) {
            if (r_len[u]) SWC_CUDA_TRY(cudaMemcpy(host_out.data() + w, d_out_keep.as<u8>() + u_off[u], (size_t)r_len[u], cudaMemcpyDeviceToHost));
            w += (size_t)r_len[u];
        }
    }
    d_out_len = contiguous ? produced : 0;     // 0 = the device copy is not one contiguous run
    return SWC_OK;
}

// process(frame:) LZ4.swift:188-330; `p` is the whole input, `pos` points right after the magic.
int frame(DeviceInput &dev, const uint8_t *p, size_t n_total, size_t pos, bool have_dict, bool has_ext_id, uint32_t ext_id,
          std::vector<uint8_t> &out, size_t *next) {
    const uint8_t *in = p + pos;
    const size_t n = n_total - pos;
    if (n < 7) return SWC_DATA_TRUNCATED;
    size_t off = 0;
    const unsigned flg = in[off++];
    if (!(((flg & 0xC0) >> 6) == 1 && (flg & 0x2) == 0)) return SWC_DATA_CORRUPTED;
    const bool independent = flg & 0x20, block_ck = flg & 0x10, csize_p = flg & 0x8, cck = flg & 0x4, dictid_p = flg & 1;
    const unsigned bd = in[off++];
    size_t max_block;
    switch (bd) {
    case 0x40: max_block = 64u << 10; break;
    case 0x50: max_block = 256u << 10; break;
    case 0x60: max_block = 1u << 20; break;
    case 0x70: max_block = 4u << 20; break;
    default: return SWC_DATA_CORRUPTED;
    }
    uint64_t content_size = 0;
    if (csize_p) {
        if (n - off < 13) return SWC_DATA_TRUNCATED;
        content_size = rd64(in + off); off += 8;
        if (content_size > (uint64_t)INT64_MAX) return SWC_DATA_UNSUPPORTED_FEATURE;
    }
    if (dictid_p) {
        if (!have_dict) return SWC_DATA_CORRUPTED;
        if (n - off < 9) return SWC_DATA_TRUNCATED;
        uint32_t id = rd32(in + off); off += 4;
        if (has_ext_id && ext_id != id) return SWC_DATA_CORRUPTED;
    }
    const uint8_t hc = (uint8_t)((xxh32_descriptor(in, off) >> 8) & 0xFF);
    if (hc != in[off]) return SWC_DATA_CORRUPTED;
    off++;

    std::vector<Block> blocks;
    int pending = SWC_OK;
    for (;;) {                                                     // LZ4.swift:278-318 framing only
        if (n - off < 4) { pending = SWC_DATA_TRUNCATED; break; }
        uint32_t mark = rd32(in + off); off += 4;
        if (mark == 0) break;
        size_t bs = mark & 0x7FFFFFFFu;
        if (bs > max_block) { pending = SWC_DATA_CORRUPTED; break; }
        if (n - off < bs + (block_ck ? 4 : 0) + 4) { pending = SWC_DATA_TRUNCATED; break; }
        Block b; b.off = pos + off; b.len = bs; b.stored = (mark & 0x80000000u) != 0; b.has_ck = block_ck; b.stored_ck = 0;
        off += bs;
        if (block_ck) { b.stored_ck = rd32(in + off); off += 4; }
        blocks.push_back(b);
    }
    const size_t fstart = out.size();
    DevBuf d_out; size_t d_out_len = 0;
    int st = run_blocks(dev, blocks, independent ? 0 : 1, have_dict, max_block, block_ck, pending, out, d_out, d_out_len);
    if (st) return st;
    if (csize_p && (uint64_t)(out.size() - fstart) != content_size) return SWC_DATA_CORRUPTED;
    if (cck) {                                                     // :323-328
        if (n - off < 4) return SWC_DATA_TRUNCATED;
        uint32_t stored = rd32(in + off); off += 4;
        // content checksum over the decoded frame, on the device
        DevBuf d_res; uint64_t len64 = d_out_len; uint32_t got = 0;
        bool whole = (d_out_len == out.size() - fstart);
        DevBuf d_tmp;
        const u8 *d_data = d_out.as<u8>();
        if (!whole || d_out_len == 0) {        // output was gathered from non-contiguous regions (or is empty): re-upload
            if ((st = d_tmp.alloc(out.size() - fstart + 16))) return st;
            if (out.size() > fstart) SWC_CUDA_TRY(cudaMemcpy(d_tmp.p, out.data() + fstart, out.size() - fstart, cudaMemcpyHostToDevice));
            d_data = d_tmp.as<u8>(); len64 = out.size() - fstart;
        }
        if ((st = d_res.alloc(16))) return st;
        SWC_CUDA_TRY(cudaMemcpy(d_res.p, &len64, 8, cudaMemcpyHostToDevice));
        if ((st = checks::xxh32_batch(d_data, nullptr, d_res.as<u64>(), (u32 *)(d_res.as<u8>() + 8), 1, 0))) return st;
        SWC_CUDA_TRY(cudaMemcpy(&got, d_res.as<u8>() + 8, 4, cudaMemcpyDeviceToHost));
        *next = pos + off;
        if (got != stored) return SWC_DATA_CHECKSUM_MISMATCH;
    }
    *next = pos + off;
    return SWC_OK;
}

// process(legacyFrame:) LZ4.swift:160-186
int legacy_frame(DeviceInput &dev, const uint8_t *p, size_t n_total, size_t pos, std::vector<uint8_t> &out, size_t *next) {
    size_t off = pos;
    std::vector<Block> blocks;
    int pending = SWC_OK;
    while (off < n_total) {
        if (n_total - off < 4) { pending = SWC_DATA_TRUNCATED; break; }
        uint32_t raw = rd32(p + off); off += 4;
        if (is_magic(raw)) { off -= 4; break; }
        if (n_total - off < raw) { pending = SWC_DATA_TRUNCATED; break; }
        Block b; b.off = off; b.len = raw; b.stored = false; b.has_ck = false; b.stored_ck = 0;
        blocks.push_back(b);
        off += raw;
    }
    DevBuf d_out; size_t d_out_len = 0;
    int st = run_blocks(dev, blocks, 0, false, 8u << 20, false, pending, out, d_out, d_out_len);
    if (st) return st;
    *next = off;
    return SWC_OK;
}

int upload(DeviceInput &dev, const uint8_t *in, size_t in_len, const uint8_t *dict, size_t dict_len) {
    int st;
    if ((st = dev.in.alloc(round16(in_len) + 32))) return st;
    { int cst = copy_pageable(dev.in.p, in, in_len, true); if (cst) return cst; }
    dev.in_len = in_len;
    dev.have_dict = dict != nullptr;
    dev.dict_len = dict ? dict_len : 0;
    if (dict && dict_len) {
        if ((st = dev.dict.alloc(dict_len))) return st;
        SWC_CUDA_TRY(cudaMemcpy(dev.dict.p, dict, dict_len, cudaMemcpyHostToDevice));
    }
    return SWC_OK;
}

int give(const std::vector<uint8_t> &v, uint8_t **out, size_t *out_len) {
    uint8_t *h = (uint8_t *)swc_alloc(v.size());
    if (!h) return SWC_ERR_OUTPUT_OVERFLOW;
    if (!v.empty()) memcpy(h, v.data(), v.size());
    *out = h; *out_len = v.size();
    return SWC_OK;
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
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !status) return SWC_ERR_INVALID_ARG;
    lz4::Args a;
    a.in_base = in_base; a.blk_off = in_off; a.blk_len = in_len; a.first_blk = nullptr; a.n_blk = nullptr;
    a.dict = dict; a.dict_len = dict ? dict_len : 0;
    a.out_base = out_base; a.out_off = out_off; a.out_cap = out_cap; a.out_len = out_len; a.status = status; a.n = n;
    // two-phase path needs a record scratch sized from the compressed lengths: fetch them once (n x 8 bytes)
    {
        std::vector<uint64_t> lens(n);
        SWC_CUDA_TRY(cudaMemcpyAsync(lens.data(), in_len, n * 8, cudaMemcpyDeviceToHost, (cudaStream_t)cuda_stream));
        SWC_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)cuda_stream));
        uint64_t total = 0;
        for (uint64_t i = 0; i < n; i++) total += lens[i] & ~(1ull << 63);
        void *scratch = nullptr;
        int st = scratch_get(lz4::two_phase_scratch_bytes(n, total), &scratch, (cudaStream_t)cuda_stream);
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
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !status) return SWC_ERR_INVALID_ARG;
    for (uint64_t i = 0; i < n; i++)                                       // every unit inside the two arenas, overflow-safe
        if (in_off[i] > in_total || in_len[i] > in_total - in_off[i] || out_off[i] > out_total || out_cap[i] > out_total - out_off[i] || (out_off[i] & 15))
            return SWC_ERR_INVALID_ARG;
    DevBuf d_in, d_out, d_meta;
    int st;
    if ((st = d_in.alloc(round16(in_total) + 32))) return st;
    if ((st = d_out.alloc(round16(out_total)))) return st;
    const size_t tb = n * 8;
    if ((st = d_meta.alloc(tb * 5 + n * 4))) return st;
    u8 *m = d_meta.as<u8>();
    cudaStream_t s = 0;
    SWC_CUDA_TRY(cudaMemcpyAsync(d_in.p, in_base, in_total, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(m + 0 * tb, in_off, tb, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(m + 1 * tb, in_len, tb, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(m + 2 * tb, out_off, tb, cudaMemcpyHostToDevice, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(m + 3 * tb, out_cap, tb, cudaMemcpyHostToDevice, s));
    st = swc_lz4_block_decompress_batch(d_in.as<u8>(), (u64 *)(m + 0 * tb), (u64 *)(m + 1 * tb), nullptr, 0, d_out.as<u8>(),
                                        (u64 *)(m + 2 * tb), (u64 *)(m + 3 * tb), (u64 *)(m + 4 * tb), (int32_t *)(m + 5 * tb), n, s);
    if (st) return st;
    for (uint64_t i = 0; i < n;) {                         // only the output regions come back (touching ones as one copy)
        const uint64_t r0 = out_off[i];
        uint64_t r1 = r0 + out_cap[i++];
        while (i < n && out_off[i] == r1) r1 += out_cap[i++];
        if (r1 > r0) SWC_CUDA_TRY(cudaMemcpyAsync(out_base + r0, d_out.as<u8>() + r0, r1 - r0, cudaMemcpyDeviceToHost, s));
    }
    SWC_CUDA_TRY(cudaMemcpyAsync(out_len, m + 4 * tb, tb, cudaMemcpyDeviceToHost, s));
    SWC_CUDA_TRY(cudaMemcpyAsync(status, m + 5 * tb, n * 4, cudaMemcpyDeviceToHost, s));
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
    size_t base = 0;
    bool have_dict = dict != nullptr;
    for (;;) {
        if (in_len - base < 4) return SWC_DATA_TRUNCATED;
        const uint32_t magic = rd32(in + base);
        if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) {           // :148-155, then recursion without dictionary (:85)
            if (in_len - base - 4 < 4) return SWC_DATA_TRUNCATED;
            size_t size = rd32(in + base + 4);
            if (in_len - base - 4 < size + 4) return SWC_DATA_TRUNCATED;
            base += 4 + size + 4;
            have_dict = false; has_dict_id = 0;
            continue;
        }
        if (magic != 0x184D2204u && magic != 0x184C2102u) return SWC_DATA_CORRUPTED;
        DeviceInput dev;
        int st = upload(dev, in, in_len, have_dict ? dict : nullptr, dict_len);
        if (st) return st;
        std::vector<uint8_t> o;
        size_t next = base + 4;
        if (magic == 0x184D2204u) st = frame(dev, in, in_len, base + 4, have_dict, has_dict_id != 0, dict_id, o, &next);
        else st = legacy_frame(dev, in, in_len, base + 4, o, &next);
        if (consumed_bytes) *consumed_bytes = next;
        if (st != SWC_OK && st != SWC_DATA_CHECKSUM_MISMATCH) return st;
        int g = give(o, out, out_len);
        return g ? g : st;
    }
}

// LZ4.multiDecompress LZ4.swift:116-146
int32_t swc_lz4_multi_decompress(const uint8_t *in, size_t in_len, const uint8_t *dict, size_t dict_len,
                                 int32_t has_dict_id, uint32_t dict_id,
                                 uint8_t **out, size_t *out_len, size_t **frame_ends, size_t *n_frames) {
    if (!out || !out_len || !frame_ends || !n_frames) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0; *frame_ends = nullptr; *n_frames = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DeviceInput dev;
    bool uploaded = false;
    std::vector<uint8_t> o;
    std::vector<size_t> ends;
    size_t next = 0;
    int result = SWC_OK;
    do {
        if (next + 4 > in_len) { result = SWC_DATA_TRUNCATED; break; }
        const uint32_t magic = rd32(in + next); next += 4;
        int st = SWC_OK; bool produced = false;
        if (magic == 0x184D2204u || magic == 0x184C2102u) {
            if (!uploaded) { if ((st = upload(dev, in, in_len, dict, dict_len))) return st; uploaded = true; }
            size_t nn = next;
            if (magic == 0x184D2204u) st = frame(dev, in, in_len, next, dict != nullptr, has_dict_id != 0, dict_id, o, &nn);
            else st = legacy_frame(dev, in, in_len, next, o, &nn);
            next = nn; produced = true;
        } else if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) {
            if (in_len - next < 4) { result = SWC_DATA_TRUNCATED; break; }
            size_t size = rd32(in + next);
            if (in_len - next < size + 4) { result = SWC_DATA_TRUNCATED; break; }
            next += size + 4;
        } else { result = SWC_DATA_CORRUPTED; break; }
        if (produced && (st == SWC_OK || st == SWC_DATA_CHECKSUM_MISMATCH)) ends.push_back(o.size());
        if (st) { result = st; break; }
    } while (next < in_len);
    if (result != SWC_OK && result != SWC_DATA_CHECKSUM_MISMATCH) return result;
    int g = give(o, out, out_len);
    if (g) return g;
    *frame_ends = (size_t *)swc_alloc(sizeof(size_t) * (ends.size() + 1));
    for (size_t i = 0; i < ends.size(); i++) (*frame_ends)[i] = ends[i];
    *n_frames = ends.size();
    return result;
}

}  // extern "C"

// ---- compression ----------------------------------------------------------------------------------------------------

namespace {

constexpr u64 kCompressPoolLimit = 16ull << 30;      // library-pool scratch per slice of a compress batch

inline u64 window_of(u64 in_len, u64 dict_len) {
    if (in_len > lz4c::MAX_BLOCK || (dict_len >= 1 && dict_len <= 3)) return 0;       // rejected units need no scratch
    return in_len + (dict_len > lz4c::MAX_DICT ? lz4c::MAX_DICT : dict_len);
}
inline u64 need_of(u64 in_len, u64 dict_len) {
    const u64 w = window_of(in_len, dict_len);
    return lz4c::unit_scratch(w, w ? in_len : 0);
}
inline u64 meta_bytes(u64 count) { return (count * 8 + 255) & ~(u64)255; }

inline void put32(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

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
    std::vector<uint64_t> lens(n), dlens(n, 0), offs(n);
    SWC_CUDA_TRY(cudaMemcpyAsync(lens.data(), in_len, n * 8, cudaMemcpyDeviceToHost, s));
    if (dict_len) SWC_CUDA_TRY(cudaMemcpyAsync(dlens.data(), dict_len, n * 8, cudaMemcpyDeviceToHost, s));
    SWC_CUDA_TRY(cudaStreamSynchronize(s));
    u64 total = meta_bytes(n), biggest = 0;
    for (uint64_t i = 0; i < n; i++) {
        const u64 need = need_of(lens[i], dlens[i]);
        total += need;
        if (need > biggest) biggest = need;
    }
    size_t cap = scratch_bytes;
    if (!scratch) {
        cap = (size_t)(total < kCompressPoolLimit ? total : kCompressPoolLimit);
        if (cap < meta_bytes(1) + biggest) cap = (size_t)(meta_bytes(1) + biggest);
        int st = scratch_get(cap, &scratch, s);
        if (st) return st;
    }
    lz4c::Args a;
    a.in_base = in_base; a.in_off = in_off; a.in_len = in_len; a.dict_off = dict_off; a.dict_len = dict_len;
    a.out_base = out_base; a.out_off = out_off; a.out_cap = out_cap; a.out_len = out_len; a.status = status;
    a.stored = nullptr; a.n = n;
    u8 *scr = (u8 *)scratch;
    // units go in slices whose scratch fits: a slice's table of offsets first, then each unit's region
    for (uint64_t first = 0; first < n;) {
        uint64_t count = 0;
        u64 used = 0;
        while (first + count < n) {
            const u64 need = need_of(lens[first + count], dlens[first + count]);
            if (meta_bytes(count + 1) + used + need > cap) break;
            offs[first + count] = used;
            used += need;
            count++;
        }
        if (count == 0) return SWC_ERR_INVALID_ARG;                       // caller scratch smaller than one unit needs
        const u64 mb = meta_bytes(count);
        for (uint64_t j = 0; j < count; j++) offs[first + j] += mb;
        SWC_CUDA_TRY(cudaMemcpyAsync(scr, offs.data() + first, count * 8, cudaMemcpyHostToDevice, s));
        int st = lz4c::parse(a, first, count, scr, (const u64 *)scr, s);
        if (!st) st = lz4c::emit(a, first, count, scr, (const u64 *)scr, s);
        if (st) return st;
        first += count;
    }
    return SWC_OK;
}

// LZ4.compress(data:independentBlocks:blockChecksums:contentChecksum:contentSize:blockSize:dictionary:dictionaryID:)
// LZ4+Compress.swift:47-154
int32_t swc_lz4_compress(const uint8_t *in, size_t in_len, int32_t independent_blocks, int32_t block_checksums,
                         int32_t content_checksum, int32_t content_size, int64_t block_size,
                         const uint8_t *dict, size_t dict_len, int32_t has_dict_id, uint32_t dict_id,
                         uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (!(block_size <= (int64_t)lz4c::MAX_BLOCK && block_size > 0)) return SWC_ERR_REFERENCE_TRAP;     // :51
    const u64 bs = (u64)block_size;
    const u64 nb = (in_len + bs - 1) / bs;
    const u64 D = dict ? (dict_len > lz4c::MAX_DICT ? lz4c::MAX_DICT : dict_len) : 0;                    // :95-101
    // compress(block:_:) traps on a 1-3 byte dictionary (:283): the user's, or a short previous block (:106-110)
    if (nb > 0 && D >= 1 && D <= 3) return SWC_ERR_REFERENCE_TRAP;
    if (nb > 1 && !independent_blocks && bs <= 3) return SWC_ERR_REFERENCE_TRAP;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;

    uint8_t hdr[19];                                                                                     // :54-93
    size_t h = 0;
    hdr[h++] = 0x04; hdr[h++] = 0x22; hdr[h++] = 0x4D; hdr[h++] = 0x18;
    hdr[h++] = (uint8_t)(0x40 | (independent_blocks ? 0x20 : 0) | (block_checksums ? 0x10 : 0) | (content_size ? 0x8 : 0) |
                         (content_checksum ? 0x4 : 0) | (has_dict_id ? 0x1 : 0));
    hdr[h++] = bs <= (64u << 10) ? 0x40 : bs <= (256u << 10) ? 0x50 : bs <= (1u << 20) ? 0x60 : 0x70;
    if (content_size) for (int k = 0; k < 8; k++) hdr[h++] = (uint8_t)((uint64_t)in_len >> (8 * k));
    if (has_dict_id) for (int k = 0; k < 4; k++) hdr[h++] = (uint8_t)(dict_id >> (8 * k));
    hdr[h] = (uint8_t)((xxh32_descriptor(hdr + 4, h - 4) >> 8) & 0xFF);
    h++;

    int st;
    // device input: the dictionary window, then the data
    DevBuf d_in;
    if ((st = d_in.alloc(D + in_len + 16))) return st;
    if (D) SWC_CUDA_TRY(cudaMemcpy(d_in.p, dict + (dict_len - D), D, cudaMemcpyHostToDevice));
    if (in_len) { int cst = copy_pageable(d_in.as<u8>() + D, in, in_len, true); if (cst) return cst; }

    // per block: in_off, in_len, dict_off, dict_len, out_off, out_cap, then out_len, status, payload length, stored flag
    std::vector<uint64_t> meta(nb * 6);
    uint64_t *h_in_off = meta.data(), *h_in_len = h_in_off + nb, *h_doff = h_in_len + nb, *h_dlen = h_doff + nb;
    uint64_t *h_out_off = h_dlen + nb, *h_out_cap = h_out_off + nb;
    std::vector<uint64_t> scr_off(nb);
    u64 scr_total = 0;
    for (u64 k = 0; k < nb; k++) {
        const u64 o = k * bs, l = in_len - o < bs ? in_len - o : bs;
        h_in_off[k] = D + o; h_in_len[k] = l;
        if (independent_blocks || k == 0) { h_doff[k] = 0; h_dlen[k] = D; }                               // :105
        else { const u64 pl = bs < lz4c::MAX_DICT ? bs : lz4c::MAX_DICT; h_doff[k] = D + o - pl; h_dlen[k] = pl; }   // :106-110
        h_out_off[k] = 0; h_out_cap[k] = ~0ull;
        scr_off[k] = scr_total;
        scr_total += need_of(l, h_dlen[k]);
    }
    DevBuf d_meta, d_scr;
    const size_t mb = nb * 8;
    if ((st = d_meta.alloc(mb * 10 + 64))) return st;
    u8 *m = d_meta.as<u8>();
    u64 *d_res_len = (u64 *)(m + 6 * mb), *d_scr_off = (u64 *)(m + 7 * mb);
    int32_t *d_status = (int32_t *)(m + 8 * mb);
    u8 *d_stored = m + 9 * mb;
    u32 *d_ck = (u32 *)(m + 9 * mb + ((nb + 15) & ~(u64)15));
    if ((st = d_scr.alloc(scr_total + 256))) return st;
    std::vector<uint64_t> res_len(nb);
    std::vector<int32_t> res_st(nb);
    std::vector<uint8_t> stored(nb);
    std::vector<uint32_t> cks(nb);
    u64 frame_len = h;
    std::vector<u64> pay_off(nb), pay_len(nb);
    lz4c::Args a;
    if (nb) {
        SWC_CUDA_TRY(cudaMemcpy(m, meta.data(), 6 * mb, cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy(d_scr_off, scr_off.data(), mb, cudaMemcpyHostToDevice));
        a.in_base = d_in.as<u8>(); a.in_off = (u64 *)m; a.in_len = (u64 *)(m + mb);
        a.dict_off = (u64 *)(m + 2 * mb); a.dict_len = (u64 *)(m + 3 * mb);
        a.out_base = nullptr; a.out_off = (u64 *)(m + 4 * mb); a.out_cap = (u64 *)(m + 5 * mb);
        a.out_len = d_res_len; a.status = d_status; a.stored = nullptr; a.n = nb;
        if ((st = lz4c::parse(a, 0, nb, d_scr.as<u8>(), d_scr_off, 0))) return st;
        SWC_CUDA_TRY(cudaMemcpy(res_len.data(), d_res_len, mb, cudaMemcpyDeviceToHost));
        SWC_CUDA_TRY(cudaMemcpy(res_st.data(), d_status, nb * 4, cudaMemcpyDeviceToHost));
        for (u64 k = 0; k < nb; k++) {
            if (res_st[k] != SWC_OK) return res_st[k];
            stored[k] = res_len[k] > h_in_len[k];                                                        // :112
            pay_len[k] = stored[k] ? h_in_len[k] : res_len[k];
            pay_off[k] = frame_len + 4;
            frame_len += 4 + pay_len[k] + (block_checksums ? 4 : 0);
        }
    }
    const u64 payload_end = frame_len;
    frame_len += 4 + (content_checksum ? 4 : 0);                                                         // :143-151
    DevBuf d_frame;
    if ((st = d_frame.alloc(frame_len + 16))) return st;
    if (nb) {
        // the payloads go straight to their frame offsets; out_cap keeps the parse's "unbounded" fence
        memcpy(h_out_off, pay_off.data(), mb);
        SWC_CUDA_TRY(cudaMemcpy(m + 4 * mb, h_out_off, mb, cudaMemcpyHostToDevice));
        SWC_CUDA_TRY(cudaMemcpy(d_stored, stored.data(), nb, cudaMemcpyHostToDevice));
        a.out_base = d_frame.as<u8>(); a.stored = d_stored;
        if ((st = lz4c::emit(a, 0, nb, d_scr.as<u8>(), d_scr_off, 0))) return st;
        if (block_checksums) {                                                                           // :120-125, :133-138
            SWC_CUDA_TRY(cudaMemcpy(d_res_len, pay_len.data(), mb, cudaMemcpyHostToDevice));
            if ((st = checks::xxh32_batch(d_frame.as<u8>(), a.out_off, d_res_len, d_ck, nb, 0))) return st;
            SWC_CUDA_TRY(cudaMemcpy(cks.data(), d_ck, nb * 4, cudaMemcpyDeviceToHost));
        }
    }
    uint32_t content_ck = xxh32_descriptor(nullptr, 0);
    if (content_checksum && in_len) {                                                                    // :146-151
        DevBuf d_res;
        if ((st = d_res.alloc(16))) return st;
        const u64 len64 = in_len;
        SWC_CUDA_TRY(cudaMemcpy(d_res.p, &len64, 8, cudaMemcpyHostToDevice));
        if ((st = checks::xxh32_batch(d_in.as<u8>() + D, nullptr, d_res.as<u64>(), (u32 *)(d_res.as<u8>() + 8), 1, 0))) return st;
        SWC_CUDA_TRY(cudaMemcpy(&content_ck, d_res.as<u8>() + 8, 4, cudaMemcpyDeviceToHost));
    }
    uint8_t *host = (uint8_t *)swc_alloc(frame_len);
    if (!host) return SWC_ERR_OUTPUT_OVERFLOW;
    if (payload_end > h) {
        int cst = copy_pageable(host + h, d_frame.as<u8>() + h, payload_end - h, false);
        if (cst) { swc_free(host); return cst; }
    }
    memcpy(host, hdr, h);
    for (u64 k = 0; k < nb; k++) {                                                                       // :113-139
        put32(host + pay_off[k] - 4, (stored[k] ? 0x80000000u : 0u) | (uint32_t)pay_len[k]);
        if (block_checksums) put32(host + pay_off[k] + pay_len[k], cks[k]);
    }
    put32(host + payload_end, 0);
    if (content_checksum) put32(host + payload_end + 4, content_ck);
    *out = host; *out_len = frame_len;
    return SWC_OK;
}

}  // extern "C"
