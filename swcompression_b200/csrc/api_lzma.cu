// api_lzma.cu — C ABI for LZMA / LZMA2 / XZ (include/swcgpu.h).
// Reference: Sources/LZMA/LZMA.swift:25-73, LZMAProperties.swift:49-64, Sources/LZMA2/LZMA2.swift:25-36,
// Sources/XZ/XZArchive.swift:27-218, XZBlock.swift:18-97, XZStreamHeader.swift:33-57,
// LittleEndianByteReader+XZ.swift:10-30, Sources/Common/DeltaFilter.swift:11-32.
// Container framing (tens of bytes per stream/block) is walked on the host; LZMA2 decode, the delta filter and the
// CRC-32 / CRC-64 / SHA-256 checks over the payload run on the device.
#include <cstring>
#include <unordered_map>
#include <vector>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "lzma.cuh"
#include "checks.cuh"
#include "xz_framing.cuh"

using namespace swc;

namespace {

struct LzmaJob {           // one unit, resident on the device
    int mode;              // lzma::MODE_*
    u8 dict_byte;
    u32 props; i64 dict_size, usize;
};

// d_in[start..in_len) holds the stream; grows the output until it fits.
int lzma_unit_device(const u8 *d_in, size_t in_len, size_t start, const LzmaJob &job, size_t cap_hint, UnitResult &r) {
    DevBuf lit;
    int st = lit.alloc(lzma::lit_scratch_bytes(1));
    if (st) return st;
    UnitTable t;
    UnitCols c(t, 1);
    const Col<u8> dict_byte = t.in<u8>(1);
    const Col<u32> props = t.in<u32>(1);
    const Col<i64> dict_size = t.in<i64>(1), usize = t.in<i64>(1);
    *t.host(dict_byte) = job.dict_byte; *t.host(props) = job.props; *t.host(dict_size) = job.dict_size; *t.host(usize) = job.usize;
    // LZMA cannot size its output without decoding it (the dictionary IS the output): x4 per attempt
    return decode_unit(t, c, d_in, start, in_len, cap_hint ? cap_hint : (in_len - start) * 8 + (1u << 20), 8,
                       [](size_t cap, size_t) { return cap >= ((size_t)1 << 33) ? 0 : cap * 4; }, [&](const DecodeIO &io, size_t) {
        const lzma::Args a{io, job.mode, t.dev(dict_byte), t.dev(props), t.dev(dict_size), t.dev(usize), lit.as<u16>()};
        return lzma::launch(a, 0);
    }, r);
}

// ---- delta filter (DeltaFilter.swift:11-32): out[i] = in[i] + out[i - distance], one thread per residue class ----
__global__ void delta_kernel(const u8 *in, u8 *out, u64 n, u32 distance) {
    const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= distance) return;
    u8 acc = 0;
    for (u64 i = j; i < n; i += distance) { acc = (u8)(acc + in[i]); out[i] = acc; }
}

// ---- XZ framing: xz_framing.cuh ----
using xz::Rd;

// ---- speculative batch decode of every LZMA2 block of a (multi-stream / multi-block) .xz file ------------------------
// XZArchive walks streams and blocks strictly in order, but the stream footers + indexes at the END of each stream
// (XZArchive.swift:132-192) tell where every block starts and how large it decodes.  xz_prefetch() reads them backwards,
// decodes all blocks as ONE batch (lzma_kernel, one warp per block) and files the results by input offset.  The in-order
// parser below stays the single source of truth: when it reaches a block it takes the cached result only if the offset,
// the dictionary byte and an OK status match — otherwise it decodes the block itself, exactly as without the cache.
struct PrefetchEntry { size_t out_off, out_len, consumed; u8 dict_byte; };
struct Prefetch {
    DevBuf out;
    std::unordered_map<size_t, PrefetchEntry> by_offset;
};
thread_local Prefetch *g_prefetch = nullptr;

// XZBlock.init XZBlock.swift:18-97. Block data ends up in `blk` (device) with length blk_len.
int xz_block(Rd &r, const u8 *d_in, unsigned hsize_byte, int csize, DevBuf &blk, size_t &blk_len, int64_t *unpadded) {
    xz::BlockHeader h;
    int st = xz::block_header(r, hsize_byte, h);
    if (st) return st;
    const int nfilters = h.nfilters;
    const int64_t uncomp_size = h.uncomp_size;
    const int *kinds = h.kind, *params = h.param;
    const size_t data_start = r.off;
    // filters.reversed().reduce(byteReader): the LAST filter reads the archive, earlier ones read its output
    DevBuf cur; size_t cur_len = 0; bool have_cur = false;
    for (int f = nfilters - 1; f >= 0; f--) {
        DevBuf next; size_t next_len = 0;
        const u8 *src = have_cur ? cur.as<u8>() : d_in;
        const size_t src_n = have_cur ? cur_len : r.n, src_start = have_cur ? 0 : r.off;
        if (kinds[f] == 0x21) {
            const PrefetchEntry *pe = nullptr;
            if (!have_cur && g_prefetch) {
                auto it = g_prefetch->by_offset.find(r.off);
                if (it != g_prefetch->by_offset.end() && it->second.dict_byte == (u8)params[f]) pe = &it->second;
            }
            if (pe) {                                                            // decoded ahead of time by xz_prefetch()
                next.borrow(g_prefetch->out.as<u8>() + pe->out_off, pe->out_len);
                r.off += pe->consumed;
                next_len = pe->out_len;
            } else {
                UnitResult u;
                LzmaJob job; job.mode = lzma::MODE_LZMA2; job.dict_byte = (u8)params[f]; job.props = 0; job.dict_size = 0; job.usize = -1;
                const size_t hint = uncomp_size >= 0 && f == 0 ? (size_t)uncomp_size + 16 : 0;
                if ((st = lzma_unit_device(src, src_n, src_start, job, hint, u))) return st;
                if (u.status != SWC_OK) return u.status;
                if (!have_cur) r.off += u.consumed;
                next_len = u.out_len;
                next.take(u.out);
            }
        } else {
            const size_t n = src_n - src_start;
            if ((st = next.alloc(n + 16))) return st;
            if (n) { delta_kernel<<<1, 256, 0, 0>>>(src + src_start, next.as<u8>(), n, (u32)params[f]); count_launch(); }
            SWC_CUDA_TRY(cudaGetLastError());
            if (!have_cur) r.off += n;
            next_len = n;
        }
        cur.take(next);
        cur_len = next_len; have_cur = true;
    }
    if ((st = xz::block_tail(r, h, data_start, (int64_t)cur_len, csize, unpadded))) return st;
    blk.take(cur);
    blk_len = cur_len;
    return SWC_OK;
}

// processStream XZArchive.swift:90-130 (+ processIndex, processFooter); stream data is appended to `out` (host)
int xz_stream(Rd &r, const u8 *d_in, HostOut &out, bool *check_error) {
    int ctype = 0;
    int st = xz::stream_header(r, &ctype);
    if (st) return st;
    std::vector<std::pair<int64_t, int64_t>> infos;
    int64_t index_size = -1;
    *check_error = false;
    for (;;) {
        if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
        const unsigned hs = r.p[r.off++];
        if (hs == 0) {                                               // processIndex
            st = xz::index(r, (int64_t)infos.size(), [&](int64_t k, int64_t *unp, int64_t *unc) {
                *unp = infos[(size_t)k].first; *unc = infos[(size_t)k].second;
            }, &index_size);
            if (st) return st;
            break;
        }
        DevBuf blk; size_t blk_len = 0; int64_t unp = 0;
        if ((st = xz_block(r, d_in, hs, xz::check_size(ctype), blk, blk_len, &unp))) return st;
        uint8_t *dst = out.grow(blk_len);
        if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
        if (blk_len) SWC_CUDA_TRY(cudaMemcpy(dst, blk.p, blk_len, cudaMemcpyDeviceToHost));
        const uint8_t *stored = nullptr;
        if ((st = xz::check_field(r, ctype, &stored))) return st;
        if (ctype == 1) {
            u64 got = 0;
            if ((st = checks::check_device(checks::CRC32, blk.as<u8>(), blk_len, &got))) return st;
            if ((uint32_t)got != le32(stored)) { *check_error = true; return SWC_OK; }
        } else if (ctype == 4) {
            u64 got = 0;
            if ((st = checks::check_device(checks::CRC64, blk.as<u8>(), blk_len, &got))) return st;
            if (got != ((uint64_t)le32(stored) | (uint64_t)le32(stored + 4) << 32)) { *check_error = true; return SWC_OK; }
        } else if (ctype == 0x0A) {
            DevBuf dg; uint8_t h[32];
            if ((st = dg.alloc(32))) return st;
            if ((st = checks::sha256(blk.as<u8>(), blk_len, dg.as<u8>(), 0))) return st;
            SWC_CUDA_TRY(cudaMemcpy(h, dg.p, 32, cudaMemcpyDeviceToHost));
            if (memcmp(h, stored, 32) != 0) { *check_error = true; return SWC_OK; }
        }
        infos.emplace_back(unp, (int64_t)blk_len);
    }
    return xz::footer(r, ctype, index_size);
}

// Walk the stream footers / indexes backwards (xz::back_stream) and batch-decode every single-filter LZMA2 block. Any
// inconsistency simply ends the discovery (the in-order parser will then report it in the reference's order); only a CUDA
// error is returned.
int xz_prefetch(const uint8_t *in, size_t n, const u8 *d_in, Prefetch &pf) {
    struct Blk { size_t data_off, comp_len, uncomp; u8 dict_byte; };
    std::vector<Blk> blks;
    size_t pos = n;
    while (pos >= 32) {
        xz::BackStream s;
        if (!xz::back_stream(in, pos, s)) break;
        const size_t csize = (size_t)xz::check_size(s.ctype), istart = s.istart;
        Rd ir{in, s.foot, s.rec_off};                                   // the records back_stream checked
        size_t boff = s.start + 12;
        bool bad = false;
        for (int64_t k = 0; k < s.count; k++) {
            int64_t unp = 0, unc = 0;
            xz::multibyte(ir, &unp); xz::multibyte(ir, &unc);          // read and checked by back_stream
            if (boff + 2 > istart) { bad = true; break; }
            const size_t hsz = ((size_t)in[boff] + 1) * 4;
            if (hsz > istart - boff) { bad = true; break; }
            // single LZMA2 filter, optional size fields: flags, [comp], [uncomp], id 0x21, props size 1, dict byte
            Rd hr{in, boff + hsz, boff + 1};
            const unsigned flags = in[boff + 1]; hr.off = boff + 2;
            int64_t tmp; bool ok = (flags & 0x3F) == 0;
            if (ok && (flags & 0x40)) ok = xz::multibyte(hr, &tmp) == 0;
            if (ok && (flags & 0x80)) ok = xz::multibyte(hr, &tmp) == 0;
            if (ok && hr.off + 3 <= boff + hsz && in[hr.off] == 0x21 && in[hr.off + 1] == 1 && (size_t)unp > hsz + csize) {
                blks.push_back({boff + hsz, (size_t)unp - hsz - csize, (size_t)unc, in[hr.off + 2]});
            }
            boff += ((size_t)unp + 3) & ~(size_t)3;
        }
        if (bad) break;
        pos = s.start;
    }
    if (blks.size() < 2) return SWC_OK;                   // nothing to gain
    uint64_t total = 0;
    for (auto &b : blks) {
        if (b.uncomp > ((uint64_t)48 << 30)) return SWC_OK;
        total += round16(b.uncomp + 16);
    }
    if (total > ((uint64_t)48 << 30)) return SWC_OK;
    const size_t nb = blks.size();
    UnitTable t;
    UnitCols c(t, nb);
    const Col<u8> dict = t.in<u8>(nb);
    u64 *h_off = t.host(c.in_off), *h_len = t.host(c.in_len), *o_off = t.host(c.out_off), *o_cap = t.host(c.out_cap);
    uint64_t run = 0;
    for (size_t i = 0; i < nb; i++) {
        h_off[i] = blks[i].data_off; h_len[i] = blks[i].comp_len; o_off[i] = run; o_cap[i] = round16(blks[i].uncomp + 16); run += o_cap[i];
        t.host(dict)[i] = blks[i].dict_byte;
    }
    if (pf.out.alloc(run + 64) || t.alloc()) return SWC_OK;       // no room: the in-order parser decodes block by block
    int st = t.upload();
    if (st) return st;
    const lzma::Args a{c.bind(t, d_in, pf.out.as<u8>(), 0, nb), lzma::MODE_LZMA2, t.dev(dict), nullptr, nullptr, nullptr, nullptr};
    if ((st = lzma::launch(a, 0))) return st;
    UnitCols::Results res;
    if ((st = c.fetch(t, res))) return st;
    for (size_t i = 0; i < nb; i++)
        if (res.status[i] == SWC_OK)
            pf.by_offset[blks[i].data_off] = PrefetchEntry{(size_t)o_off[i], (size_t)res.out_len[i], (size_t)res.consumed[i], blks[i].dict_byte};
    return SWC_OK;
}

int xz_all(const uint8_t *in, size_t n, HostOut &out, std::vector<size_t> &ends) {
    DevBuf d_in;
    int st = upload_input(d_in, in, n);
    if (st) return st;
    Prefetch pf;
    if ((st = xz_prefetch(in, n, d_in.as<u8>(), pf))) return st;
    struct Guard { Guard(Prefetch *p) { g_prefetch = p; } ~Guard() { g_prefetch = nullptr; } } guard(pf.by_offset.empty() ? nullptr : &pf);
    Rd r{in, n, 0};
    while (r.off < r.n) {
        if (r.n - r.off < 32) return SWC_XZ_WRONG_MAGIC;
        bool check_error = false;
        if ((st = xz_stream(r, d_in.as<u8>(), out, &check_error))) return st;
        ends.push_back(out.len);
        if (check_error) return SWC_XZ_WRONG_CHECK;
        if ((st = xz::padding(r))) return st;
    }
    return SWC_OK;
}

int single(const uint8_t *in, size_t in_len, size_t start, const LzmaJob &job, size_t hint,
           uint8_t **out, size_t *out_len, size_t *consumed, size_t header_bytes) {
    DevBuf d_in;
    int st = upload_input(d_in, in, in_len);
    if (st) return st;
    UnitResult r;
    if ((st = lzma_unit_device(d_in.as<u8>(), in_len, start, job, hint, r))) return st;
    if (consumed) *consumed = header_bytes + r.consumed;
    if (r.status != SWC_OK) return r.status;
    return to_host_alloc(r.out.p, r.out_len, out, out_len);
}

}  // namespace

extern "C" {

// LZMA.decompress(data:) LZMA.swift:25-34
int32_t swc_lzma_decompress(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, size_t *consumed_bytes) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bytes) *consumed_bytes = 0;
    if (in_len < 13) return SWC_LZMA_WRONG_PROPERTIES;
    const unsigned b = in[0];
    if (b >= 225) return SWC_LZMA_WRONG_PROPERTIES;                  // LZMAProperties.swift:50
    LzmaJob job; job.mode = lzma::MODE_RAW; job.dict_byte = 0;
    job.props = (b % 9) | (((b / 9) % 5) << 8) | (((b / 9) / 5) << 16);
    job.dict_size = (i64)in[1] | (i64)in[2] << 8 | (i64)in[3] << 16 | (i64)in[4] << 24;     // no clamp in init
    uint64_t us = 0;
    for (int i = 0; i < 8; i++) us |= (uint64_t)in[5 + i] << (8 * i);
    job.usize = (i64)us;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    const size_t hint = job.usize >= 0 && job.usize < ((i64)1 << 36) ? (size_t)job.usize + 16 : 0;
    return single(in, in_len, 13, job, hint, out, out_len, consumed_bytes, 13);
}

// LZMA.decompress(data:properties:uncompressedSize:) LZMA.swift:56-61
int32_t swc_lzma_decompress_raw(const uint8_t *in, size_t in_len, int32_t lc, int32_t lp, int32_t pb,
                                int64_t dictionary_size, int64_t uncompressed_size,
                                uint8_t **out, size_t *out_len, size_t *consumed_bytes) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bytes) *consumed_bytes = 0;
    // properties no properties byte can express: the reference decodes some such streams and traps on others (DESIGN §6)
    if (lc < 0 || lp < 0 || pb < 0 || lc > 8 || lp > 4 || pb > 4) return SWC_ERR_UNSUPPORTED;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    LzmaJob job; job.mode = lzma::MODE_RAW; job.dict_byte = 0;
    job.props = (u32)lc | ((u32)lp << 8) | ((u32)pb << 16);
    job.dict_size = dictionary_size; job.usize = uncompressed_size < 0 ? -1 : uncompressed_size;
    const size_t hint = job.usize >= 0 && job.usize < ((i64)1 << 36) ? (size_t)job.usize + 16 : 0;
    return single(in, in_len, 0, job, hint, out, out_len, consumed_bytes, 0);
}

// LZMA2.decompress(data:) LZMA2.swift:25-30
int32_t swc_lzma2_decompress(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, size_t *consumed_bytes) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bytes) *consumed_bytes = 0;
    if (in_len < 1) return SWC_LZMA_RANGE_DECODER_INIT_ERROR;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    LzmaJob job; job.mode = lzma::MODE_LZMA2; job.dict_byte = in[0]; job.props = 0; job.dict_size = 0; job.usize = -1;
    return single(in, in_len, 1, job, 0, out, out_len, consumed_bytes, 1);
}

int32_t swc_lzma_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                  const uint32_t *props, const int64_t *dict_size, const int64_t *uncompressed_size,
                                  uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                  uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                  uint64_t n, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    // no lit_scratch: lc + lp > 4 would need 6 MB of literal coders per unit, such units are refused here
    const lzma::Args a{{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bytes},
                       lzma::MODE_RAW, nullptr, props, (const i64 *)dict_size, (const i64 *)uncompressed_size, nullptr};
    if (missing(a) || !props || !dict_size || !uncompressed_size) return SWC_ERR_INVALID_ARG;
    return lzma::launch(a, (cudaStream_t)cuda_stream);
}

int32_t swc_lzma2_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                   const uint8_t *dict_bytes,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                   uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                   uint64_t n, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    // no lit_scratch: a chunk with lc + lp > 4 would need 6 MB of literal coders, such units are refused here
    const lzma::Args a{{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bytes},
                       lzma::MODE_LZMA2, dict_bytes, nullptr, nullptr, nullptr, nullptr};
    if (missing(a) || !dict_bytes) return SWC_ERR_INVALID_ARG;
    return lzma::launch(a, (cudaStream_t)cuda_stream);
}

int32_t swc_xz_unarchive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    HostOut o; std::vector<size_t> ends;
    int st = xz_all(in, in_len, o, ends);
    if (st != SWC_OK && st != SWC_XZ_WRONG_CHECK) return st;
    int g = o.release_to(out, out_len);
    return g ? g : st;
}

int32_t swc_xz_split_unarchive(const uint8_t *in, size_t in_len,
                               uint8_t **out, size_t *out_len, size_t **stream_ends, size_t *n_streams) {
    if (!out || !out_len || !stream_ends || !n_streams) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0; *stream_ends = nullptr; *n_streams = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    HostOut o; std::vector<size_t> ends;
    int st = xz_all(in, in_len, o, ends);
    if (st != SWC_OK && st != SWC_XZ_WRONG_CHECK) return st;
    int g;
    if ((g = o.release_to(out, out_len)) || (g = give_sizes(ends, stream_ends, out, out_len))) return g;
    *n_streams = ends.size();
    return st;
}

}  // extern "C"
