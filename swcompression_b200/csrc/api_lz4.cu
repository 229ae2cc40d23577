// api_lz4.cu — C ABI for LZ4: raw block batches (device / host) and the frame layer of
// LZ4.decompress / LZ4.multiDecompress (reference Sources/LZ4/LZ4.swift:73-330).  Frame descriptors and block marks
// are walked on the host (a few bytes per block); block decode, block checksums and the content checksum run on the
// device.  Errors are reported in the order the reference's sequential loop would meet them.
// The compress half here is the raw block batch; frames (LZ4.compress, LZ4+Compress.swift:16-154) are laid out on the
// device by lz4_frame_compress.cu.
#include <cstring>
#include <vector>
#include "../../include/swcgpu.h"
#include "compress_host.h"
#include "lz4.cuh"
#include "lz4_compress.cuh"
#include "lz4_frame.cuh"

using namespace swc;

namespace {

inline uint64_t rd64(const uint8_t *p) { return (uint64_t)le32(p) | (uint64_t)le32(p + 4) << 32; }
inline bool is_magic(uint32_t v) { return v == 0x184D2204u || v == 0x184C2102u || (v >= 0x184D2A50u && v <= 0x184D2A5Fu); }

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
               bool check_blocks, int pending_error, HostOut &host_out, DevBuf &d_out_keep, size_t &d_out_len) {
    const size_t nb = blocks.size();
    d_out_len = 0;
    if (nb == 0) return pending_error;
    const size_t nunits = mode == 0 ? nb : 1;
    // block columns, then unit columns (a unit is one block, or the whole chain of a dependent frame)
    UnitTable t;
    const Col<u64> blk_off = t.in<u64>(nb), blk_len = t.in<u64>(nb), unit_off = t.in<u64>(nunits), unit_cap = t.in<u64>(nunits);
    const Col<uint32_t> first = t.in<uint32_t>(nunits), count = t.in<uint32_t>(nunits);
    const Col<u64> unit_len = t.out<u64>(nunits);
    const Col<int32_t> status = t.out<int32_t>(nunits);
    const Col<uint32_t> ck = t.out<uint32_t>(nb);
    u64 *u_off = t.host(unit_off), *u_cap = t.host(unit_cap);
    uint32_t *h_first = t.host(first), *h_cnt = t.host(count);
    for (size_t i = 0; i < nb; i++) { t.host(blk_off)[i] = blocks[i].off; t.host(blk_len)[i] = blocks[i].len | (blocks[i].stored ? 1ull << 63 : 0); }
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
    std::vector<uint64_t> r_len;
    std::vector<int32_t> r_st;
    std::vector<uint32_t> r_ck;
    int st = t.alloc();
    if (st) return st;
    for (int attempt = 0; attempt < 2; attempt++) {
        if ((st = d_out_keep.alloc(total))) return st;
        if ((st = t.upload())) return st;
        lz4::Args a{{dev.in.as<u8>(), t.dev(blk_off), t.dev(blk_len), d_out_keep.as<u8>(), t.dev(unit_off), t.dev(unit_cap),
                     t.dev(unit_len), t.dev(status), nunits},
                    t.dev(first), t.dev(count), use_dict && dev.have_dict ? dev.dict.as<u8>() : nullptr,
                    use_dict && dev.have_dict ? dev.dict_len : 0, nullptr};
        if (mode == 1 && a.dict_len > 65536) { a.dict += a.dict_len - 65536; a.dict_len = 65536; }    // LZ4.swift:309
        if (mode == 0) {               // one block per unit: take the two-phase (parse + 8-wide execute) path
            uint64_t tot = 0;
            for (size_t i = 0; i < nb; i++) tot += blocks[i].len;
            void *scr = nullptr;
            if ((st = scratch_get(lz4::two_phase_scratch_bytes(nb, tot), &scr, 0))) return st;
            a.first_blk = nullptr; a.n_blk = nullptr; a.scratch = scr;
        }
        if ((st = lz4::launch(a, 0))) return st;
        if (check_blocks && attempt == 0) {
            if ((st = checks::xxh32_batch(dev.in.as<u8>(), t.dev(blk_off), t.dev(blk_len), t.dev(ck), nb, 0))) return st;
            if ((st = t.fetch(ck, r_ck))) return st;
        }
        if ((st = t.fetch(unit_len, r_len)) || (st = t.fetch(status, r_st))) return st;
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
    uint8_t *dst = host_out.grow(produced);
    if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
    bool contiguous = true;
    { size_t run = 0; for (size_t u = 0; u < nunits; u++) { if (u_off[u] != run) contiguous = false; run += (size_t)r_len[u]; } }
    if (contiguous) {
        if (produced) SWC_CUDA_TRY(cudaMemcpy(dst, d_out_keep.p, produced, cudaMemcpyDeviceToHost));
    } else {
        for (size_t u = 0; u < nunits; u++) {
            if (r_len[u]) SWC_CUDA_TRY(cudaMemcpy(dst, d_out_keep.as<u8>() + u_off[u], (size_t)r_len[u], cudaMemcpyDeviceToHost));
            dst += (size_t)r_len[u];
        }
    }
    d_out_len = contiguous ? produced : 0;     // 0 = the device copy is not one contiguous run
    return SWC_OK;
}

// process(frame:) LZ4.swift:188-330; `p` is the whole input, `pos` points right after the magic.
int frame(DeviceInput &dev, const uint8_t *p, size_t n_total, size_t pos, bool have_dict, bool has_ext_id, uint32_t ext_id,
          HostOut &out, size_t *next) {
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
        uint32_t id = le32(in + off); off += 4;
        if (has_ext_id && ext_id != id) return SWC_DATA_CORRUPTED;
    }
    const uint8_t hc = (uint8_t)((lz4f::xxh32_descriptor(in, (u32)off) >> 8) & 0xFF);
    if (hc != in[off]) return SWC_DATA_CORRUPTED;
    off++;

    std::vector<Block> blocks;
    int pending = SWC_OK;
    for (;;) {                                                     // LZ4.swift:278-318 framing only
        if (n - off < 4) { pending = SWC_DATA_TRUNCATED; break; }
        uint32_t mark = le32(in + off); off += 4;
        if (mark == 0) break;
        size_t bs = mark & 0x7FFFFFFFu;
        if (bs > max_block) { pending = SWC_DATA_CORRUPTED; break; }
        if (n - off < bs + (block_ck ? 4 : 0) + 4) { pending = SWC_DATA_TRUNCATED; break; }
        Block b; b.off = pos + off; b.len = bs; b.stored = (mark & 0x80000000u) != 0; b.has_ck = block_ck; b.stored_ck = 0;
        off += bs;
        if (block_ck) { b.stored_ck = le32(in + off); off += 4; }
        blocks.push_back(b);
    }
    const size_t fstart = out.len;
    DevBuf d_out; size_t d_out_len = 0;
    int st = run_blocks(dev, blocks, independent ? 0 : 1, have_dict, max_block, block_ck, pending, out, d_out, d_out_len);
    if (st) return st;
    const size_t flen = out.len - fstart;
    if (csize_p && (uint64_t)flen != content_size) return SWC_DATA_CORRUPTED;
    if (cck) {                                                     // :323-328
        if (n - off < 4) return SWC_DATA_TRUNCATED;
        uint32_t stored = le32(in + off); off += 4;
        // content checksum over the decoded frame, on the device
        DevBuf d_tmp;
        const u8 *d_data = d_out.as<u8>();
        if (d_out_len != flen || d_out_len == 0) {  // output was gathered from non-contiguous regions (or is empty): re-upload
            if ((st = d_tmp.alloc(flen + 16))) return st;
            if (flen) SWC_CUDA_TRY(cudaMemcpy(d_tmp.p, out.p + fstart, flen, cudaMemcpyHostToDevice));
            d_data = d_tmp.as<u8>();
        }
        u64 got = 0;
        if ((st = checks::check_device(checks::XXH32, d_data, flen, &got))) return st;
        *next = pos + off;
        if ((uint32_t)got != stored) return SWC_DATA_CHECKSUM_MISMATCH;
    }
    *next = pos + off;
    return SWC_OK;
}

// process(legacyFrame:) LZ4.swift:160-186
int legacy_frame(DeviceInput &dev, const uint8_t *p, size_t n_total, size_t pos, HostOut &out, size_t *next) {
    size_t off = pos;
    std::vector<Block> blocks;
    int pending = SWC_OK;
    while (off < n_total) {
        if (n_total - off < 4) { pending = SWC_DATA_TRUNCATED; break; }
        uint32_t raw = le32(p + off); off += 4;
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
    if ((st = upload_input(dev.in, in, in_len))) return st;
    dev.in_len = in_len;
    dev.have_dict = dict != nullptr;
    dev.dict_len = dict ? dict_len : 0;
    if (dict && dict_len && (st = upload_input(dev.dict, dict, dict_len))) return st;
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
    size_t base = 0;
    bool have_dict = dict != nullptr;
    for (;;) {
        if (in_len - base < 4) return SWC_DATA_TRUNCATED;
        const uint32_t magic = le32(in + base);
        if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) {           // :148-155, then recursion without dictionary (:85)
            if (in_len - base - 4 < 4) return SWC_DATA_TRUNCATED;
            size_t size = le32(in + base + 4);
            if (in_len - base - 4 < size + 4) return SWC_DATA_TRUNCATED;
            base += 4 + size + 4;
            have_dict = false; has_dict_id = 0;
            continue;
        }
        if (magic != 0x184D2204u && magic != 0x184C2102u) return SWC_DATA_CORRUPTED;
        DeviceInput dev;
        int st = upload(dev, in, in_len, have_dict ? dict : nullptr, dict_len);
        if (st) return st;
        HostOut o;
        size_t next = base + 4;
        if (magic == 0x184D2204u) st = frame(dev, in, in_len, base + 4, have_dict, has_dict_id != 0, dict_id, o, &next);
        else st = legacy_frame(dev, in, in_len, base + 4, o, &next);
        if (consumed_bytes) *consumed_bytes = next;
        if (st != SWC_OK && st != SWC_DATA_CHECKSUM_MISMATCH) return st;
        int g = o.release_to(out, out_len);
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
    HostOut o;
    std::vector<size_t> ends;
    size_t next = 0;
    int result = SWC_OK;
    do {
        if (next + 4 > in_len) { result = SWC_DATA_TRUNCATED; break; }
        const uint32_t magic = le32(in + next); next += 4;
        int st = SWC_OK; bool produced = false;
        if (magic == 0x184D2204u || magic == 0x184C2102u) {
            if (!uploaded) { if ((st = upload(dev, in, in_len, dict, dict_len))) return st; uploaded = true; }
            size_t nn = next;
            if (magic == 0x184D2204u) st = frame(dev, in, in_len, next, dict != nullptr, has_dict_id != 0, dict_id, o, &nn);
            else st = legacy_frame(dev, in, in_len, next, o, &nn);
            next = nn; produced = true;
        } else if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) {
            if (in_len - next < 4) { result = SWC_DATA_TRUNCATED; break; }
            size_t size = le32(in + next);
            if (in_len - next < size + 4) { result = SWC_DATA_TRUNCATED; break; }
            next += size + 4;
        } else { result = SWC_DATA_CORRUPTED; break; }
        if (produced && (st == SWC_OK || st == SWC_DATA_CHECKSUM_MISMATCH)) ends.push_back(o.len);
        if (st) { result = st; break; }
    } while (next < in_len);
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
