// compress_host.h — host side shared by the batched compressors (api_lz4.cu, api_deflate_compress.cu,
// api_bzip2_compress.cu): the slice planner of a batch and the single-call driver.  The kernels and each slice's plan
// stay with the codec.
#pragma once
#include <cstring>
#include <vector>
#include "../../include/swcgpu.h"
#include "host_util.h"
#include "checks.cuh"

namespace swc {

constexpr u64 kCompressPoolLimit = 16ull << 30;      // library-pool scratch per slice of a compress batch

// Runs units [0, n) of a compress batch in slices (DESIGN §2).  A slice of `count` units takes head(count) bytes of plan
// at the front of the scratch, then need(i) bytes per unit i.  Without a caller scratch the library pool supplies
// head(n) + the sum of need(i), capped at kCompressPoolLimit but never below head(1) + the largest need.  A slice takes
// units while head(count + 1) + its units' needs still fit; a scratch that cannot hold one unit is SWC_ERR_INVALID_ARG.
// slice(first, count, scr, cap) lays out its plan in scr[0, cap) and launches the slice on `s`.
template <typename Need, typename Head, typename Slice>
int run_in_slices(u64 n, Need need, Head head, void *scratch, size_t scratch_bytes, cudaStream_t s, Slice slice) {
    size_t cap = scratch_bytes;
    if (!scratch) {
        u64 total = head(n), biggest = 0;
        for (u64 i = 0; i < n; i++) {
            const u64 q = need(i);
            total += q;
            if (q > biggest) biggest = q;
        }
        cap = (size_t)(total < kCompressPoolLimit ? total : kCompressPoolLimit);
        if (cap < head(1) + biggest) cap = (size_t)(head(1) + biggest);
        int st = scratch_get(cap, &scratch, s);
        if (st) return st;
    }
    for (u64 first = 0; first < n;) {
        u64 count = 0, used = 0;
        while (first + count < n) {
            const u64 q = need(first + count);
            if (head(count + 1) + used + q > cap) break;
            used += q;
            count++;
        }
        if (count == 0) return SWC_ERR_INVALID_ARG;                       // caller scratch smaller than one unit needs
        int st = slice(first, count, (u8 *)scratch, cap);
        if (st) return st;
        first += count;
    }
    return SWC_OK;
}

// The single call of a batched compressor: in[0, in_len) goes through batch() as a 1-unit batch on the library pool, into
// an output of `cap` bytes (the largest result the codec writes for in_len bytes).  `a` carries the codec's own fields;
// the unit table is filled here.  The result is handed back as one swc_alloc'ed buffer.
template <typename Args>
int compress_one(Args a, int (*batch)(const Args &, const std::vector<u64> &, void *, size_t, cudaStream_t), u64 cap,
                 const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in, d_out;
    int st;
    if ((st = upload_input(d_in, in, in_len))) return st;
    UnitTable t;
    const Col<u64> in_off = t.in<u64>(1), c_len = t.in<u64>(1), out_off = t.in<u64>(1), out_cap = t.in<u64>(1);
    const Col<u64> r_len = t.out<u64>(1);
    const Col<int32_t> r_st = t.out<int32_t>(1);
    cap = round16(cap);
    if ((st = t.alloc()) || (st = d_out.alloc(cap))) return st;
    *t.host(c_len) = in_len; *t.host(out_cap) = cap;
    if ((st = t.upload())) return st;
    a.in_base = d_in.as<u8>(); a.in_off = t.dev(in_off); a.in_len = t.dev(c_len);
    a.out_base = d_out.as<u8>(); a.out_off = t.dev(out_off); a.out_cap = t.dev(out_cap);
    a.out_len = t.dev(r_len); a.status = t.dev(r_st); a.n = 1;
    if ((st = batch(a, std::vector<u64>(1, in_len), nullptr, 0, 0))) return st;
    std::vector<u64> len;
    std::vector<int32_t> status;
    if ((st = t.fetch(r_len, len)) || (st = t.fetch(r_st, status))) return st;
    if (status[0] != SWC_OK) return status[0];
    const size_t n = (size_t)len[0];
    uint8_t *host = (uint8_t *)swc_alloc(n);
    if (!host) return SWC_ERR_OUTPUT_OVERFLOW;
    if (n && (st = copy_pageable(host, d_out.p, n, false))) { swc_free(host); return st; }
    *out = host; *out_len = n;
    return SWC_OK;
}

}  // namespace swc
