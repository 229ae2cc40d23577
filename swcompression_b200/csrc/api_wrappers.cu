// api_wrappers.cu — GzipArchive / ZlibArchive framing around the device Deflate decoder, and the checksum C ABI.
// Reference: Sources/GZip/GzipArchive.swift:38-100, GzipHeader.swift:68-199, Sources/Zlib/ZlibArchive.swift:25-42,
// ZlibHeader.swift:47-93.  Headers/trailers (tens of bytes) are parsed on the host with the grammar of archive_header.cuh;
// Deflate and CRC-32 / Adler-32 over the payload run on the device.  The batched form is unarchive_batch.cu.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "archive_header.cuh"
#include "checks.cuh"

using namespace swc;

namespace {

int gzip_header(const uint8_t *in, size_t n, size_t *off) {
    swc_gzip_header h;
    const int st = gzip_parse(in, n, *off, &h);
    if (st == SWC_OK) *off += h.header_len;
    return st;
}

// processMember GzipArchive.swift:79-100; d_in holds the whole archive on the device
int gzip_member(const uint8_t *in, size_t n, const u8 *d_in, size_t *off, HostOut &out, bool *crc_error) {
    if (n - *off < 20) return SWC_GZIP_WRONG_MAGIC;
    int st = gzip_header(in, n, off);
    if (st) return st;
    UnitResult r;
    if ((st = deflate_unit_device(d_in, n, (size_t)*off * 8, r))) return st;
    if (r.status != SWC_OK) return r.status;
    size_t p = *off + (r.consumed + 7) / 8;                          // align()
    if (n - p < 8) return SWC_GZIP_WRONG_MAGIC;
    const uint32_t crc = le32(in + p), isize = le32(in + p + 4);
    p += 8;
    if ((uint32_t)r.out_len != isize) return SWC_GZIP_WRONG_ISIZE;
    u64 got = 0;
    if ((st = checks::check_device(checks::CRC32, r.out.as<u8>(), r.out_len, &got))) return st;
    *crc_error = (uint32_t)got != crc;
    uint8_t *dst = out.grow(r.out_len);
    if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
    if (r.out_len) SWC_CUDA_TRY(cudaMemcpy(dst, r.out.p, r.out_len, cudaMemcpyDeviceToHost));
    *off = p;
    return SWC_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Batch path for multi-member archives (BGZF and friends).  Members are independent Deflate streams, so candidate member
// starts are found by signature, every candidate is decoded speculatively in ONE batched launch (its input ends 8 bytes
// before the next candidate; its capacity is the ISIZE found there), and the in-order walk of GzipArchive.multiUnarchive
// (GzipArchive.swift:52-77) then only *validates*: member k is accepted iff it decoded cleanly, stopped exactly at that
// trailer and produced ISIZE bytes — exactly what the sequential decoder would have computed from the same start.  A
// member that does not validate (a signature look-alike inside its payload, ISIZE wrap-around, damage) is decoded by the
// sequential path, and the walk resynchronises on the candidate list afterwards.
static size_t inflate_scratch_bytes(u64 n, u64 out_total) { return swc_deflate_batch_scratch_bytes(n, out_total); }

struct Cand { size_t at, dstart, next; uint32_t crc, isize; long unit; };

int gzip_multi_batch(const uint8_t *in, size_t n, const u8 *d_in, HostOut &o, std::vector<size_t> &ends, std::vector<size_t> &starts, size_t *off, int *result, bool *stop) {
    const bool trace = getenv("SWC_TRACE") != nullptr;
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t0 = now();
    std::vector<size_t> pos;
    {
        int st = checks::find_gzip_members(d_in, n, pos);              // device-side signature scan, sorted positions
        if (st) return st;
    }
    if (trace) fprintf(stderr, "[swc] gzip scan: %zu candidates, %.1f ms\n", pos.size(), now() - t0);
    if (pos.size() < 4 || pos[0] != 0) return SWC_OK;              // nothing to gain: the caller's loop handles it
    size_t free_b = 0, total_b = 0;
    SWC_CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    // a round needs its speculative outputs, the 4/3 x record scratch of the Deflate batch and the gather copy: ~3.3 x out_total
    const size_t budget = free_b / 5;
    cudaStream_t stream = 0;
    size_t idx = 0;
    while (idx < pos.size() && pos[idx] == *off && !*stop) {
        // ---- one round: candidates idx.. while the speculative outputs fit the budget
        std::vector<Cand> cs;
        size_t nu = 0, out_total = 0;
        for (size_t k = idx; k < pos.size() && cs.size() < (1u << 22); k++) {
            Cand c;
            c.at = pos[k]; c.next = k + 1 < pos.size() ? pos[k + 1] : n; c.unit = -1; c.crc = c.isize = 0;
            size_t d = c.at;
            const bool hdr_ok = gzip_header(in, c.next, &d) == SWC_OK;   // a real header never reaches the next member
            c.dstart = d;
            if (hdr_ok && c.next >= d + 8) {
                c.crc = le32(in + c.next - 8); c.isize = le32(in + c.next - 4);
                if ((u64)c.isize <= (u64)(c.next - 8 - d) * 1032 + 64) {    // Deflate cannot expand further than ~1032:1
                    const size_t cap16 = round16((size_t)c.isize);
                    if (out_total + cap16 > budget && !cs.empty()) break;
                    c.unit = (long)nu++;
                    out_total += cap16;
                }
            }
            cs.push_back(c);
        }
        UnitTable t;
        UnitCols uc(t, nu);
        const Col<uint32_t> crc = t.out<uint32_t>(nu);
        u64 *h_outoff = t.host(uc.out_off);
        for (size_t k = 0, run = 0; k < cs.size(); k++) {
            const Cand &c = cs[k];
            if (c.unit < 0) continue;
            t.host(uc.in_off)[c.unit] = c.dstart; t.host(uc.in_len)[c.unit] = c.next - 8 - c.dstart;
            h_outoff[c.unit] = run; t.host(uc.out_cap)[c.unit] = c.isize;
            run += round16((size_t)c.isize);
        }
        UnitCols::Results res;
        std::vector<uint32_t> h_crc;
        DevBuf d_out;
        if (nu) {
            // an allocation failure is not an error of the archive: hand the rest to the caller's sequential walk
            if (t.alloc()) return SWC_OK;
            if (d_out.alloc(out_total + 64)) return SWC_OK;
            { void *scr = nullptr; if (scratch_get(inflate_scratch_bytes(nu, out_total), &scr, stream)) return SWC_OK; }
            int st = t.upload(stream);
            if (st) return st;
            if ((st = deflate_batch_impl(uc.bind(t, d_in, d_out.as<u8>(), 0, nu), nullptr, out_total, nullptr, 0, stream))) return st;
            if ((st = checks::crc32_units(d_out.as<u8>(), t.dev(uc.out_off), t.dev(uc.out_len), t.dev(uc.status), t.dev(crc), nu, stream))) return st;
            if ((st = uc.fetch(t, res, stream)) || (st = t.fetch(crc, h_crc, stream))) return st;
        }
        if (trace) fprintf(stderr, "[swc] gzip round: %zu units, %.1f MB out, decode+crc done at %.1f ms\n", nu, out_total / 1e6, now() - t0);
        // ---- the in-order walk: accept the longest validated prefix
        size_t accepted = 0;
        for (; accepted < cs.size(); accepted++) {
            const Cand &c = cs[accepted];
            if (c.unit < 0) break;
            const size_t u = (size_t)c.unit;
            if (res.status[u] != SWC_OK || c.dstart + (res.consumed[u] + 7) / 8 + 8 != c.next || res.out_len[u] != c.isize) break;
            if (h_crc[u] != c.crc) { *result = SWC_GZIP_WRONG_CRC; *stop = true; accepted++; break; }   // the member is still returned
        }
        if (accepted) {
            UnitTable g;
            const Col<u64> src = g.in<u64>(accepted), len = g.in<u64>(accepted), dst = g.in<u64>(accepted);
            size_t acc_bytes = 0;
            for (size_t i = 0; i < accepted; i++) {
                const size_t u = (size_t)cs[i].unit;
                g.host(src)[i] = h_outoff[u]; g.host(len)[i] = res.out_len[u]; g.host(dst)[i] = acc_bytes;
                acc_bytes += res.out_len[u];
            }
            DevBuf d_g;
            if (g.alloc()) return SWC_OK;
            if (d_g.alloc(acc_bytes + 16)) return SWC_OK;
            int st = g.upload(stream);
            if (st) return st;
            if ((st = checks::gather_units(d_out.as<u8>(), g.dev(src), g.dev(len), d_g.as<u8>(), g.dev(dst), accepted, stream))) return st;
            const size_t base = o.len;
            uint8_t *out = o.grow(acc_bytes);
            if (!out) return SWC_ERR_OUTPUT_OVERFLOW;
            SWC_CUDA_TRY(cudaStreamSynchronize(stream));
            if ((st = copy_pageable(out, d_g.p, acc_bytes, false))) return st;
            for (size_t i = 0; i < accepted; i++) { ends.push_back(base + g.host(dst)[i] + g.host(len)[i]); starts.push_back(cs[i].at); }
            *off = cs[accepted - 1].next;
            if (trace) fprintf(stderr, "[swc] gzip round: %zu accepted, gathered + copied back at %.1f ms\n", accepted, now() - t0);
        }
        if (*stop) return SWC_OK;
        idx += accepted;
        if (accepted == cs.size()) continue;                             // next round (or done)
        // ---- member idx did not validate: decode it the sequential way, then resynchronise on the candidate list
        bool crc_error = false;
        const size_t member_at = *off;
        int st = gzip_member(in, n, d_in, off, o, &crc_error);
        if (st) return st;
        ends.push_back(o.len); starts.push_back(member_at);
        if (crc_error) { *result = SWC_GZIP_WRONG_CRC; *stop = true; return SWC_OK; }
        idx = (size_t)(std::lower_bound(pos.begin(), pos.end(), *off) - pos.begin());
    }
    return SWC_OK;
}

template <typename F>
int host_check(const uint8_t *in, size_t n, F fn) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d;
    int st = upload_input(d, in, n);
    if (st) return st;
    return fn(d.as<u8>());
}

}  // namespace

extern "C" {

int32_t swc_gzip_unarchive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, size_t *consumed_bytes) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bytes) *consumed_bytes = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    int st = upload_input(d_in, in, in_len);
    if (st) return st;
    HostOut o;
    size_t off = 0; bool crc_error = false;
    if ((st = gzip_member(in, in_len, d_in.as<u8>(), &off, o, &crc_error))) return st;
    if (consumed_bytes) *consumed_bytes = off;
    if ((st = o.release_to(out, out_len))) return st;
    return crc_error ? SWC_GZIP_WRONG_CRC : SWC_OK;
}

// GzipArchive.multiUnarchive GzipArchive.swift:52-77
static int gzip_multi(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, size_t **member_ends, size_t **member_in_off,
                      size_t *n_members) {
    if (!out || !out_len || !member_ends || !n_members) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0; *member_ends = nullptr; *n_members = 0;
    if (member_in_off) *member_in_off = nullptr;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    int st = upload_input(d_in, in, in_len);
    if (st) return st;
    HostOut o;
    std::vector<size_t> ends, starts;
    size_t off = 0;
    int result = SWC_OK;
    bool stop = false;
    if ((st = gzip_multi_batch(in, in_len, d_in.as<u8>(), o, ends, starts, &off, &result, &stop))) return st;
    while (off < in_len && !stop) {
        bool crc_error = false;
        const size_t member_at = off;
        if ((st = gzip_member(in, in_len, d_in.as<u8>(), &off, o, &crc_error))) return st;
        ends.push_back(o.len); starts.push_back(member_at);
        if (crc_error) { result = SWC_GZIP_WRONG_CRC; break; }
    }
    if ((st = o.release_to(out, out_len)) || (st = give_sizes(ends, member_ends, out, out_len))) return st;
    if (member_in_off) {
        starts.push_back(off);                                           // one past the last member
        if ((st = give_sizes(starts, member_in_off, out, out_len))) { swc_free(*member_ends); *member_ends = nullptr; return st; }
    }
    *n_members = ends.size();
    return result;
}

int32_t swc_gzip_multi_unarchive(const uint8_t *in, size_t in_len,
                                 uint8_t **out, size_t *out_len, size_t **member_ends, size_t *n_members) {
    return gzip_multi(in, in_len, out, out_len, member_ends, nullptr, n_members);
}

int32_t swc_gzip_multi_unarchive_members(const uint8_t *in, size_t in_len,
                                         uint8_t **out, size_t *out_len, size_t **member_ends, size_t **member_in_off,
                                         size_t *n_members) {
    if (!member_in_off) return SWC_ERR_INVALID_ARG;
    return gzip_multi(in, in_len, out, out_len, member_ends, member_in_off, n_members);
}

int32_t swc_gzip_header_parse(const uint8_t *in, size_t in_len, size_t member_off, swc_gzip_header *hdr) {
    if (!in || !hdr) return SWC_ERR_INVALID_ARG;
    return gzip_parse(in, in_len, member_off, hdr);
}

int32_t swc_zlib_header_parse(const uint8_t *in, size_t in_len, swc_zlib_header *hdr) {
    if (!in || !hdr) return SWC_ERR_INVALID_ARG;
    return zlib_parse(in, in_len, hdr);
}

int32_t swc_zlib_unarchive(const uint8_t *in, size_t n, uint8_t **out, size_t *out_len) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    swc_zlib_header zh;
    { const int hst = zlib_parse(in, n, &zh); if (hst) return hst; }
    const size_t off = zh.header_len;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    int st = upload_input(d_in, in, n);
    if (st) return st;
    UnitResult r;
    if ((st = deflate_unit_device(d_in.as<u8>(), n, off * 8, r))) return st;
    if (r.status != SWC_OK) return r.status;
    const size_t p = off + (r.consumed + 7) / 8;
    int result = SWC_OK;
    if (n - p < 4) {
        result = SWC_ZLIB_WRONG_ADLER32;                             // ZlibArchive.swift:34-35 (payload still returned)
    } else {
        const uint32_t adler = (uint32_t)in[p] << 24 | (uint32_t)in[p + 1] << 16 | (uint32_t)in[p + 2] << 8 | in[p + 3];
        u64 got = 0;
        if ((st = checks::check_device(checks::ADLER32, r.out.as<u8>(), r.out_len, &got))) return st;
        if ((uint32_t)got != adler) result = SWC_ZLIB_WRONG_ADLER32;
    }
    if ((st = to_host_alloc(r.out.p, r.out_len, out, out_len))) return st;
    return result;
}

int32_t swc_crc32_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len, const int32_t *status,
                        uint32_t *result, uint64_t n, void *cuda_stream) {
    if (n == 0) return SWC_OK;
    if (!in_base || !off || !len || !result) return SWC_ERR_INVALID_ARG;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    return checks::crc32_units(in_base, off, len, status, result, n, (cudaStream_t)cuda_stream);
}
int32_t swc_adler32_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len, const int32_t *status,
                          uint32_t *result, uint64_t n, void *cuda_stream) {
    if (n == 0) return SWC_OK;
    if (!in_base || !off || !len || !result) return SWC_ERR_INVALID_ARG;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    return checks::adler32_units(in_base, off, len, status, result, n, (cudaStream_t)cuda_stream);
}
int32_t swc_crc64_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len, const int32_t *status,
                        uint64_t *result, uint64_t n, void *cuda_stream) {
    if (n == 0) return SWC_OK;
    if (!in_base || !off || !len || !result) return SWC_ERR_INVALID_ARG;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    return checks::crc64_units(in_base, off, len, status, result, n, (cudaStream_t)cuda_stream);
}
int32_t swc_xxh32_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len,
                        uint32_t *result, uint64_t n, void *cuda_stream) {
    if (n == 0) return SWC_OK;
    if (!in_base || !off || !len || !result) return SWC_ERR_INVALID_ARG;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    return checks::xxh32_batch(in_base, off, len, result, n, (cudaStream_t)cuda_stream);
}

int32_t swc_crc32(const uint8_t *in, size_t n, uint32_t *result) {
    return host_check(in, n, [&](const u8 *d) { u64 v = 0; int st = checks::check_device(checks::CRC32, d, n, &v); *result = (uint32_t)v; return st; });
}
int32_t swc_bzip2_crc32(const uint8_t *in, size_t n, uint32_t *result) {
    return host_check(in, n, [&](const u8 *d) { u64 v = 0; int st = checks::check_device(checks::BZIP2_CRC32, d, n, &v); *result = (uint32_t)v; return st; });
}
int32_t swc_crc64(const uint8_t *in, size_t n, uint64_t *result) {
    return host_check(in, n, [&](const u8 *d) { u64 v = 0; int st = checks::check_device(checks::CRC64, d, n, &v); *result = v; return st; });
}
int32_t swc_adler32(const uint8_t *in, size_t n, uint32_t *result) {
    return host_check(in, n, [&](const u8 *d) { u64 v = 0; int st = checks::check_device(checks::ADLER32, d, n, &v); *result = (uint32_t)v; return st; });
}
int32_t swc_xxh32(const uint8_t *in, size_t n, uint32_t *result) {
    return host_check(in, n, [&](const u8 *d) { u64 v = 0; int st = checks::check_device(checks::XXH32, d, n, &v); *result = (uint32_t)v; return st; });
}
int32_t swc_sha256(const uint8_t *in, size_t n, uint8_t digest[32]) {
    return host_check(in, n, [&](const u8 *d) {
        DevBuf dg;
        int st = dg.alloc(32);
        if (st) return st;
        if ((st = checks::sha256(d, n, dg.as<u8>(), 0))) return st;
        SWC_CUDA_TRY(cudaMemcpy(digest, dg.p, 32, cudaMemcpyDeviceToHost));
        return (int)SWC_OK;
    });
}

}  // extern "C"
