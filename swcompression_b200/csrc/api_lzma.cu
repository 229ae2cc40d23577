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
    return decode_unit(t, c, start, in_len, cap_hint ? cap_hint : (in_len - start) * 8 + (1u << 20), 8,
                       [](size_t cap, size_t) { return cap >= ((size_t)1 << 33) ? 0 : cap * 4; }, [&](u8 *out, size_t) {
        lzma::Args a;
        a.mode = job.mode; a.in_base = d_in; a.in_off = t.dev(c.in_off); a.in_len = t.dev(c.in_len);
        a.dict_bytes = t.dev(dict_byte); a.props = t.dev(props); a.dict_size = t.dev(dict_size); a.usize = t.dev(usize);
        a.out_base = out; a.out_off = t.dev(c.out_off); a.out_cap = t.dev(c.out_cap); a.out_len = t.dev(c.out_len);
        a.consumed = t.dev(c.consumed); a.status = t.dev(c.status); a.n = 1; a.lit_scratch = lit.as<u16>();
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

// ---- XZ framing ----
struct Rd {
    const uint8_t *p; size_t n, off;
    bool need(size_t k) const { return n - off >= k; }
};
int multibyte(Rd &r, int64_t *val) {                          // LittleEndianByteReader+XZ.swift:10-30
    if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
    int i = 1;
    int64_t result = r.p[r.off++];
    if (result <= 127) { *val = result; return SWC_OK; }
    result &= 0x7F;
    for (;;) {
        if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
        unsigned b = r.p[r.off++];
        if (i >= 9 || b == 0) return SWC_XZ_MULTI_BYTE_INTEGER_ERROR;
        result += (int64_t)(b & 0x7F) << (7 * i);
        i++;
        if ((b & 0x80) == 0) break;
    }
    *val = result;
    return SWC_OK;
}
int check_size(int t) { return t == 0 ? 0 : t == 1 ? 4 : t == 4 ? 8 : 32; }

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
    const size_t hstart = r.off - 1;
    const size_t real = ((size_t)hsize_byte + 1) * 4;
    if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
    const unsigned flags = r.p[r.off++];
    const int nfilters = (flags & 0x03) + 1;
    if (flags & 0x3C) return SWC_XZ_WRONG_FIELD;
    int64_t comp_size = -1, uncomp_size = -1;
    int st;
    if (flags & 0x40) { if ((st = multibyte(r, &comp_size))) return st; }
    if (flags & 0x80) { if ((st = multibyte(r, &uncomp_size))) return st; }
    int kinds[4], params[4];
    for (int f = 0; f < nfilters; f++) {
        int64_t id, psz;
        if ((st = multibyte(r, &id))) return st;
        if ((uint64_t)id >= 0x4000000000000000ull) return SWC_XZ_WRONG_FILTER_ID;
        if (id == 0x21) {
            if ((st = multibyte(r, &psz))) return st;
            if (psz != 1) return SWC_LZMA2_WRONG_DICTIONARY_SIZE;
            if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
            kinds[f] = 0x21; params[f] = r.p[r.off++];
        } else if (id == 0x03) {
            if ((st = multibyte(r, &psz))) return st;
            if (psz != 1) return SWC_XZ_WRONG_FIELD;
            if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
            kinds[f] = 0x03; params[f] = (r.p[r.off++] + 1) & 0xFF;
        } else return SWC_XZ_WRONG_FILTER_ID;
    }
    while ((int64_t)(r.off - hstart) < (int64_t)real - 4) {
        if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
        if (r.p[r.off++] != 0) return SWC_XZ_WRONG_PADDING;
    }
    if (!r.need(4)) return SWC_ERR_REFERENCE_TRAP;
    const uint32_t hcrc = le32(r.p + r.off);
    if (r.n - hstart < real - 4) return SWC_ERR_REFERENCE_TRAP;
    if (crc32_framing(r.p + hstart, real - 4) != hcrc) return SWC_XZ_WRONG_INFO_CRC;
    r.off = hstart + real;

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
            if (n) { delta_kernel<<<1, 256, 0, 0>>>(src + src_start, next.as<u8>(), n, (u32)(params[f] == 0 ? 256 : params[f])); count_launch(); }
            SWC_CUDA_TRY(cudaGetLastError());
            if (!have_cur) r.off += n;
            next_len = n;
        }
        cur.take(next);
        cur_len = next_len; have_cur = true;
    }
    if (!((comp_size < 0 || comp_size == (int64_t)(r.off - data_start)) && (uncomp_size < 0 || uncomp_size == (int64_t)cur_len)))
        return SWC_XZ_WRONG_DATA_SIZE;
    const int64_t unp = (int64_t)(r.off - hstart);
    if (unp % 4 != 0) {
        for (int i = 0, pad = 4 - (int)(unp % 4); i < pad; i++) {
            if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
            if (r.p[r.off++] != 0) return SWC_XZ_WRONG_PADDING;
        }
    }
    *unpadded = unp + csize;
    blk.take(cur);
    blk_len = cur_len;
    return SWC_OK;
}

// processStream XZArchive.swift:90-130 (+ processIndex, processFooter); stream data is appended to `out` (host)
int xz_stream(Rd &r, const u8 *d_in, HostOut &out, bool *check_error) {
    static const uint8_t magic[6] = {0xFD, 0x37, 0x7A, 0x58, 0x5A, 0x00};
    if (!r.need(12)) return SWC_ERR_REFERENCE_TRAP;
    if (memcmp(r.p + r.off, magic, 6) != 0) return SWC_XZ_WRONG_MAGIC;
    const uint8_t *fl = r.p + r.off + 6;
    if (crc32_framing(fl, 2) != le32(r.p + r.off + 8)) return SWC_XZ_WRONG_INFO_CRC;
    if (!(fl[0] == 0 && (fl[1] & 0xF0) == 0)) return SWC_XZ_WRONG_FIELD;
    const int ctype = fl[1] & 0xF;
    if (!(ctype == 0 || ctype == 1 || ctype == 4 || ctype == 0x0A)) return SWC_XZ_WRONG_FIELD;
    r.off += 12;
    std::vector<std::pair<int64_t, int64_t>> infos;
    int64_t index_size = -1;
    *check_error = false;
    for (;;) {
        if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
        const unsigned hs = r.p[r.off++];
        if (hs == 0) {                                               // processIndex
            const size_t istart = r.off - 1;
            int64_t v; int st;
            if ((st = multibyte(r, &v))) return st;
            if (v != (int64_t)infos.size()) return SWC_XZ_WRONG_FIELD;
            for (auto &bi : infos) {
                if ((st = multibyte(r, &v))) return st;
                if (v != bi.first) return SWC_XZ_WRONG_FIELD;
                if ((st = multibyte(r, &v))) return st;
                if (v != bi.second) return SWC_XZ_WRONG_DATA_SIZE;
            }
            int64_t isz = (int64_t)(r.off - istart);
            if (isz % 4 != 0) {
                for (int i = 0, pad = 4 - (int)(isz % 4); i < pad; i++) {
                    if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
                    if (r.p[r.off++] != 0) return SWC_XZ_WRONG_PADDING;
                    isz++;
                }
            }
            if (!r.need(4)) return SWC_ERR_REFERENCE_TRAP;
            if (crc32_framing(r.p + istart, (size_t)isz) != le32(r.p + r.off)) return SWC_XZ_WRONG_INFO_CRC;
            r.off = istart + (size_t)isz + 4;
            index_size = isz + 4;
            break;
        }
        DevBuf blk; size_t blk_len = 0; int64_t unp = 0;
        int st = xz_block(r, d_in, hs, check_size(ctype), blk, blk_len, &unp);
        if (st) return st;
        uint8_t *dst = out.grow(blk_len);
        if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
        if (blk_len) SWC_CUDA_TRY(cudaMemcpy(dst, blk.p, blk_len, cudaMemcpyDeviceToHost));
        if (ctype == 1) {
            if (!r.need(4)) return SWC_ERR_REFERENCE_TRAP;
            const uint32_t c = le32(r.p + r.off); r.off += 4;
            u64 got = 0;
            if ((st = checks::check_device(checks::CRC32, blk.as<u8>(), blk_len, &got))) return st;
            if ((uint32_t)got != c) { *check_error = true; return SWC_OK; }
        } else if (ctype == 4) {
            if (!r.need(8)) return SWC_ERR_REFERENCE_TRAP;
            const uint64_t c = (uint64_t)le32(r.p + r.off) | (uint64_t)le32(r.p + r.off + 4) << 32; r.off += 8;
            u64 got = 0;
            if ((st = checks::check_device(checks::CRC64, blk.as<u8>(), blk_len, &got))) return st;
            if (got != c) { *check_error = true; return SWC_OK; }
        } else if (ctype == 0x0A) {
            if (!r.need(32)) return SWC_ERR_REFERENCE_TRAP;
            DevBuf dg; uint8_t h[32];
            if ((st = dg.alloc(32))) return st;
            if ((st = checks::sha256(blk.as<u8>(), blk_len, dg.as<u8>(), 0))) return st;
            SWC_CUDA_TRY(cudaMemcpy(h, dg.p, 32, cudaMemcpyDeviceToHost));
            const bool bad = memcmp(h, r.p + r.off, 32) != 0; r.off += 32;
            if (bad) { *check_error = true; return SWC_OK; }
        }
        infos.emplace_back(unp, (int64_t)blk_len);
    }
    if (!r.need(12)) return SWC_ERR_REFERENCE_TRAP;                  // processFooter
    const uint32_t fcrc = le32(r.p + r.off);
    const int64_t backward = ((int64_t)le32(r.p + r.off + 4) + 1) * 4;
    const unsigned fflags = r.p[r.off + 8] | r.p[r.off + 9] << 8;
    if (crc32_framing(r.p + r.off + 4, 6) != fcrc) return SWC_XZ_WRONG_INFO_CRC;
    if (backward != index_size) return SWC_XZ_WRONG_FIELD;
    if (!((fflags & 0xFF) == 0 && ((fflags & 0xF00) >> 8) == (unsigned)ctype && (fflags & 0xF000) == 0)) return SWC_XZ_WRONG_FIELD;
    if (!(r.p[r.off + 10] == 0x59 && r.p[r.off + 11] == 0x5A)) return SWC_XZ_WRONG_MAGIC;
    r.off += 12;
    return SWC_OK;
}

int xz_padding(Rd &r) {                                               // processPadding XZArchive.swift:194-218
    if (r.off >= r.n) return SWC_OK;
    int padding = 0;
    for (;;) {
        const unsigned b = r.p[r.off++];
        if (b != 0) { if (padding % 4 != 0) return SWC_XZ_WRONG_PADDING; break; }
        if (r.off >= r.n) { if (padding % 4 != 3) return SWC_XZ_WRONG_PADDING; return SWC_OK; }
        padding++;
    }
    r.off -= 1;
    return SWC_OK;
}

// Walk the stream footers / indexes backwards and batch-decode every single-filter LZMA2 block. Any inconsistency simply
// ends the discovery (the in-order parser will then report it in the reference's order); only a CUDA error is returned.
int xz_prefetch(const uint8_t *in, size_t n, const u8 *d_in, Prefetch &pf) {
    struct Blk { size_t data_off, comp_len, uncomp; u8 dict_byte; };
    std::vector<Blk> blks;
    size_t pos = n;
    while (pos >= 32) {
        while (pos >= 4 && in[pos - 1] == 0 && in[pos - 2] == 0 && in[pos - 3] == 0 && in[pos - 4] == 0) pos -= 4;   // stream padding
        if (pos < 32 || in[pos - 2] != 0x59 || in[pos - 1] != 0x5A) break;
        const size_t foot = pos - 12;
        const int ctype = in[foot + 9] & 0xF;
        const size_t csize = (size_t)check_size(ctype);
        const size_t index_size = ((size_t)le32(in + foot + 4) + 1) * 4;
        if (index_size + 12 > foot) break;
        const size_t istart = foot - index_size;
        if (in[istart] != 0) break;
        Rd ir{in, foot, istart + 1};
        int64_t count = 0;
        if (multibyte(ir, &count) || count < 0 || count > 1000000) break;
        std::vector<std::pair<int64_t, int64_t>> recs((size_t)count);
        bool bad = false; uint64_t blocks_total = 0;
        for (auto &rc : recs) {                                   // untrusted sizes: every sum is checked against the bytes before the index
            if (multibyte(ir, &rc.first) || multibyte(ir, &rc.second) || rc.first <= 0 || rc.second < 0) { bad = true; break; }
            if ((uint64_t)rc.first > (uint64_t)istart) { bad = true; break; }
            const uint64_t padded = ((uint64_t)rc.first + 3) & ~3ull;
            if (padded > (uint64_t)istart - blocks_total) { bad = true; break; }
            blocks_total += padded;
        }
        if (bad || blocks_total + 12 > istart) break;
        const size_t sstart = istart - (size_t)blocks_total - 12;
        static const uint8_t magic[6] = {0xFD, 0x37, 0x7A, 0x58, 0x5A, 0x00};
        if (memcmp(in + sstart, magic, 6) != 0) break;
        size_t boff = sstart + 12;
        for (auto &rc : recs) {
            if (boff + 2 > istart) { bad = true; break; }
            const size_t hsz = ((size_t)in[boff] + 1) * 4;
            if (hsz > istart - boff) { bad = true; break; }
            // single LZMA2 filter, optional size fields: flags, [comp], [uncomp], id 0x21, props size 1, dict byte
            Rd hr{in, boff + hsz, boff + 1};
            const unsigned flags = in[boff + 1]; hr.off = boff + 2;
            int64_t tmp; bool ok = (flags & 0x3F) == 0;
            if (ok && (flags & 0x40)) ok = multibyte(hr, &tmp) == 0;
            if (ok && (flags & 0x80)) ok = multibyte(hr, &tmp) == 0;
            if (ok && hr.off + 3 <= boff + hsz && in[hr.off] == 0x21 && in[hr.off + 1] == 1 && (size_t)rc.first > hsz + csize) {
                blks.push_back({boff + hsz, (size_t)rc.first - hsz - csize, (size_t)rc.second, in[hr.off + 2]});
            }
            boff += ((size_t)rc.first + 3) & ~(size_t)3;
        }
        if (bad) break;
        pos = sstart;
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
    lzma::Args a;
    a.mode = lzma::MODE_LZMA2; a.in_base = d_in; a.in_off = t.dev(c.in_off); a.in_len = t.dev(c.in_len); a.dict_bytes = t.dev(dict);
    a.props = nullptr; a.dict_size = nullptr; a.usize = nullptr;
    a.out_base = pf.out.as<u8>(); a.out_off = t.dev(c.out_off); a.out_cap = t.dev(c.out_cap); a.out_len = t.dev(c.out_len);
    a.consumed = t.dev(c.consumed); a.status = t.dev(c.status); a.n = nb; a.lit_scratch = nullptr;
    if ((st = lzma::launch(a, 0))) return st;
    std::vector<uint64_t> r_len, r_used;
    std::vector<int32_t> r_st;
    if ((st = t.fetch(c.out_len, r_len)) || (st = t.fetch(c.consumed, r_used)) || (st = t.fetch(c.status, r_st))) return st;
    for (size_t i = 0; i < nb; i++)
        if (r_st[i] == SWC_OK) pf.by_offset[blks[i].data_off] = PrefetchEntry{(size_t)o_off[i], (size_t)r_len[i], (size_t)r_used[i], blks[i].dict_byte};
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
        if ((st = xz_padding(r))) return st;
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
    if (!in_base || !in_off || !in_len || !props || !dict_size || !uncompressed_size || !out_base || !out_off || !out_cap || !out_len ||
        !consumed_bytes || !status)
        return SWC_ERR_INVALID_ARG;
    lzma::Args a;
    a.mode = lzma::MODE_RAW; a.in_base = in_base; a.in_off = in_off; a.in_len = in_len; a.dict_bytes = nullptr;
    a.props = props; a.dict_size = (const i64 *)dict_size; a.usize = (const i64 *)uncompressed_size;
    a.out_base = out_base; a.out_off = out_off; a.out_cap = out_cap; a.out_len = out_len; a.consumed = consumed_bytes;
    a.status = status; a.n = n; a.lit_scratch = nullptr;      // lc + lp > 4 would need 6 MB of literal coders per unit: refused here
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
    if (!in_base || !in_off || !in_len || !dict_bytes || !out_base || !out_off || !out_cap || !out_len || !consumed_bytes || !status)
        return SWC_ERR_INVALID_ARG;
    lzma::Args a;
    a.mode = lzma::MODE_LZMA2; a.in_base = in_base; a.in_off = in_off; a.in_len = in_len; a.dict_bytes = dict_bytes;
    a.props = nullptr; a.dict_size = nullptr; a.usize = nullptr;
    a.out_base = out_base; a.out_off = out_off; a.out_cap = out_cap; a.out_len = out_len; a.consumed = consumed_bytes;
    a.status = status; a.n = n; a.lit_scratch = nullptr;      // a chunk with lc + lp > 4 would need 6 MB of literal coders: refused here
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
