// api_wrappers.cu — GzipArchive / ZlibArchive single and multi-member calls, and the checksum C ABI.
// Reference: Sources/GZip/GzipArchive.swift:38-100, Sources/Zlib/ZlibArchive.swift:25-42.  An archive or member is one unit
// of the device unarchive batch (unarchive_batch.cu), which parses the header, decodes the Deflate stream, checks the
// trailer and reports the reference's statuses; only multiUnarchive's walk over members stays on the host.
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

// GzipArchive.unarchive / ZlibArchive.unarchive of d_in[start, in_len) as a one-unit unarchive batch, r.consumed counted from
// `start`: 4 x the input plus 64 KiB first; a unit that needs more reports its exact size, and the rerun at that size is final.
int archive_unit(bool gzip, const u8 *d_in, size_t in_len, size_t start, UnitResult &r) {
    UnitTable t;
    const UnitCols c(t, 1);
    return decode_unit(t, c, d_in, start, in_len, (in_len - start) * 4 + 65536, 3, [](size_t, size_t need) { return need; },
                       [&](const DecodeIO &io, size_t cap) { return unarchive_batch_impl(gzip, io, nullptr, cap, nullptr, 0, 0); }, r);
}

// processMember GzipArchive.swift:79-100 at *off, appended to `out` with its end and start; *off moves past the member.  A
// member with a wrong CRC is still returned and sets *crc_error; any other failure is the result.
int next_member(const u8 *d_in, size_t n, size_t *off, HostOut &out, std::vector<size_t> &ends, std::vector<size_t> &starts,
                bool *crc_error) {
    UnitResult r;
    int st = archive_unit(true, d_in, n, *off, r);
    if (st) return st;
    if (r.status != SWC_OK && r.status != SWC_GZIP_WRONG_CRC) return r.status;
    uint8_t *dst = out.grow(r.out_len);
    if (!dst) return SWC_ERR_OUTPUT_OVERFLOW;
    if (r.out_len) SWC_CUDA_TRY(cudaMemcpy(dst, r.out.p, r.out_len, cudaMemcpyDeviceToHost));
    ends.push_back(out.len); starts.push_back(*off);
    *crc_error = r.status == SWC_GZIP_WRONG_CRC;
    *off += r.consumed;
    return SWC_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Batch path for multi-member archives (BGZF and friends).  Members are independent Deflate streams, so candidate member
// starts are found by signature, and every candidate is one unit [at, next) of ONE unarchive batch, its capacity the ISIZE
// found at next - 4.  The in-order walk of GzipArchive.multiUnarchive (GzipArchive.swift:52-77) then only *validates*:
// member k is accepted iff its status is OK or a wrong CRC and it consumed exactly next - at bytes — its trailer then sits
// at next - 8, so it is what the sequential decoder would have computed from the same start.  A member that does not
// validate (a signature look-alike inside its payload, ISIZE wrap-around, damage) is decoded by the sequential path, and
// the walk resynchronises on the candidate list afterwards.
struct Cand { size_t at, next; uint32_t isize; long unit; };

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
            c.at = pos[k]; c.next = k + 1 < pos.size() ? pos[k + 1] : n; c.unit = -1; c.isize = 0;
            if (c.next - c.at >= 20) {                                   // a shorter member fails the 20-byte guard anyway
                c.isize = le32(in + c.next - 4);
                if ((u64)c.isize <= (u64)(c.next - c.at) * 1032 + 64) {     // Deflate cannot expand further than ~1032:1
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
        u64 *h_outoff = t.host(uc.out_off);
        for (size_t k = 0, run = 0; k < cs.size(); k++) {
            const Cand &c = cs[k];
            if (c.unit < 0) continue;
            t.host(uc.in_off)[c.unit] = c.at; t.host(uc.in_len)[c.unit] = c.next - c.at;
            h_outoff[c.unit] = run; t.host(uc.out_cap)[c.unit] = c.isize;
            run += round16((size_t)c.isize);
        }
        UnitCols::Results res;
        DevBuf d_out;
        if (nu) {
            // an allocation failure is not an error of the archive: hand the rest to the caller's sequential walk
            if (t.alloc()) return SWC_OK;
            if (d_out.alloc(out_total + 64)) return SWC_OK;
            { void *scr = nullptr; if (scratch_get(swc_unarchive_batch_scratch_bytes(nu, out_total), &scr, stream)) return SWC_OK; }
            int st = t.upload(stream);
            if (st) return st;
            if ((st = unarchive_batch_impl(true, uc.bind(t, d_in, d_out.as<u8>(), 0, nu), nullptr, out_total, nullptr, 0, stream))) return st;
            if ((st = uc.fetch(t, res, stream))) return st;
        }
        if (trace) fprintf(stderr, "[swc] gzip round: %zu units, %.1f MB out, decode done at %.1f ms\n", nu, out_total / 1e6, now() - t0);
        // ---- the in-order walk: accept the longest validated prefix
        size_t accepted = 0;
        for (; accepted < cs.size(); accepted++) {
            const Cand &c = cs[accepted];
            if (c.unit < 0) break;
            const size_t u = (size_t)c.unit;
            if ((res.status[u] != SWC_OK && res.status[u] != SWC_GZIP_WRONG_CRC) || res.consumed[u] != c.next - c.at) break;
            if (res.status[u] == SWC_GZIP_WRONG_CRC) { *result = SWC_GZIP_WRONG_CRC; *stop = true; accepted++; break; }   // the member is still returned
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
        int st = next_member(d_in, n, off, o, ends, starts, &crc_error);
        if (st) return st;
        if (crc_error) { *result = SWC_GZIP_WRONG_CRC; *stop = true; return SWC_OK; }
        idx = (size_t)(std::lower_bound(pos.begin(), pos.end(), *off) - pos.begin());
    }
    return SWC_OK;
}

// GzipArchive.unarchive / ZlibArchive.unarchive GzipArchive.swift:38-47, ZlibArchive.swift:25-42
int single_unarchive(bool gzip, const uint8_t *in, size_t n, uint8_t **out, size_t *out_len, size_t *consumed_bytes) {
    if (!out || !out_len) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (consumed_bytes) *consumed_bytes = 0;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    UnitResult r;
    int st = upload_input(d_in, in, n);
    if (st || (st = archive_unit(gzip, d_in.as<u8>(), n, 0, r))) return st;
    if (consumed_bytes) *consumed_bytes = r.consumed;
    if (r.status != SWC_OK && r.status != (gzip ? SWC_GZIP_WRONG_CRC : SWC_ZLIB_WRONG_ADLER32)) return r.status;
    return (st = to_host_alloc(r.out.p, r.out_len, out, out_len)) ? st : r.status;
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
    return single_unarchive(true, in, in_len, out, out_len, consumed_bytes);
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
        if ((st = next_member(d_in.as<u8>(), in_len, &off, o, ends, starts, &crc_error))) return st;
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
    return single_unarchive(false, in, n, out, out_len, nullptr);
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
