// host_util.h — host-side helpers shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <vector>
#include "common.cuh"
#include "archive_header.cuh"   // crc32_framing

#include <mutex>

namespace swc {

int ensure_device();

// ---- per-device library context (runtime.cu) -----------------------------------------------------------------------------
// The reference is re-entrant; here the mutable state is one lazily created context per device: scratch arenas, the streams /
// pinned result buffer of the *_batch_host paths, one-time kernel configuration flags.  Every C-ABI entry point that touches it
// holds the device's API mutex for the duration of the call (ApiLock), so any number of host threads may call into the library
// concurrently on the same or on different devices; calls on one device are serialised, calls on different devices are not.
struct DeviceCtx {
    std::recursive_mutex api_mu;
    std::mutex cfg_mu;
    bool configured[16] = {};
    cudaStream_t streams[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t tables_ready = nullptr;
    uint8_t *h_res = nullptr;
    size_t h_res_bytes = 0;
    int num_sms = 0;
};
DeviceCtx &device_ctx();                 // context of the CURRENT device
struct ApiLock {
    std::unique_lock<std::recursive_mutex> lk;
    ApiLock() : lk(device_ctx().api_mu) {}
};
enum { CFG_INFLATE_K1W = 0, CFG_INFLATE_K1L = 1, CFG_LZMA = 2, CFG_BZIP2_CRC = 3, CFG_LZ4 = 4, CFG_XZ = 5 };
// runs `f` (returning an swc status) once per device, thread-safe; a failing `f` is retried by the next caller
template <typename F> int configure_once(int slot, F f) {
    DeviceCtx &c = device_ctx();
    std::lock_guard<std::mutex> g(c.cfg_mu);
    if (c.configured[slot]) return SWC_OK;
    if (!c.num_sms) {
        int dev = 0;
        SWC_CUDA_TRY(cudaGetDevice(&dev));
        SWC_CUDA_TRY(cudaDeviceGetAttribute(&c.num_sms, cudaDevAttrMultiProcessorCount, dev));
    }
    const int st = f(c);
    if (st == SWC_OK) c.configured[slot] = true;
    return st;
}

// RAII device allocation (single-unit paths; the batch paths use caller memory + the scratch pool)
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    bool owned = true;          // false: a view into memory owned elsewhere (never freed here)
    DevBuf() {}
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    void release() { if (p && owned) cudaFree(p); p = nullptr; bytes = 0; owned = true; }
    void borrow(void *ptr, size_t n) { release(); p = ptr; bytes = n; owned = false; }
    void take(DevBuf &o) { release(); p = o.p; bytes = o.bytes; owned = o.owned; o.p = nullptr; o.bytes = 0; o.owned = true; }
    int alloc(size_t n) {
        release();
        cudaError_t e = cudaMalloc(&p, n ? n : 16);
        if (e != cudaSuccess) { p = nullptr; return cuda_fail(e, "cudaMalloc"); }
        bytes = n;
        return SWC_OK;
    }
    template <typename T> T *as() const { return (T *)p; }
};

inline size_t round16(size_t v) { return (v + 15) & ~(size_t)15; }
inline size_t round256(size_t v) { return (v + 255) & ~(size_t)255; }

// Lays typed columns out from `base`, each on a 256-byte boundary so that no column overlaps its neighbour whatever its
// type and length; `at` counts the bytes taken.  A null base only sizes the layout.  The batches that split their units
// into sub-units take their unit columns first, at offsets that do not depend on the table size, so the counts taken on a
// layout of n units and no table are valid in the same scratch's layout of n units and any table.
struct Carver {
    u8 *base;
    size_t at = 0;
    explicit Carver(void *b) : base((u8 *)b) {}
    template <typename... T> void cols(u64 count, T *&...p) { ((p = (T *)(base + at), at += round256(count * sizeof(T))), ...); }
    u8 *end() const { return base + at; }
};

// a batch's n u64 lengths (device) into `v` on the host, for planning the batch (blocking: waits for `s`)
inline int read_lens(const u64 *d, u64 n, cudaStream_t s, std::vector<u64> &v) {
    v.resize(n);
    SWC_CUDA_TRY(cudaMemcpyAsync(v.data(), d, n * 8, cudaMemcpyDeviceToHost, s));
    SWC_CUDA_TRY(cudaStreamSynchronize(s));
    return SWC_OK;
}

// ---- unit tables: the per-unit metadata of one batch, as typed columns in one device allocation ----
// Declare every column first, then seat the table with alloc() (its own cudaMalloc, kept when alloc() is called again) or
// place() (memory the caller owns); host() pointers stay valid from the last declaration on.  in<T>() columns have a
// zero-filled host side that upload() sends in one copy; out<T>() columns exist on the device only (kernel results, or
// filled by the caller's own copies).
// Every column starts on a 256-byte boundary, so a column never overlaps its neighbour whatever its type and length.
template <typename T> struct Col { size_t off = 0, n = 0; bool dev_only = false; };
class UnitTable {
  public:
    template <typename T> Col<T> in(size_t n) { Col<T> c{host_.size(), n, false}; host_.resize(host_.size() + round256(n * sizeof(T))); return c; }
    template <typename T> Col<T> out(size_t n) { Col<T> c{out_bytes_, n, true}; out_bytes_ += round256(n * sizeof(T)); return c; }
    template <typename T> T *host(Col<T> c) { return (T *)(host_.data() + c.off); }
    template <typename T> T *dev(Col<T> c) const { return (T *)(dev_.as<u8>() + (c.dev_only ? host_.size() : 0) + c.off); }
    size_t bytes() const { return host_.size() + out_bytes_; }
    int alloc() { return dev_.p && dev_.owned && dev_.bytes == bytes() ? SWC_OK : dev_.alloc(bytes()); }
    void place(void *p) { dev_.borrow(p, bytes()); }
    int upload(cudaStream_t s = 0) {
        if (!host_.empty()) SWC_CUDA_TRY(cudaMemcpyAsync(dev_.p, host_.data(), host_.size(), cudaMemcpyHostToDevice, s));
        return SWC_OK;
    }
    // one column back into `v` (blocking: waits for `s`)
    template <typename T> int fetch(Col<T> c, std::vector<T> &v, cudaStream_t s = 0) const {
        v.resize(c.n);
        if (c.n) SWC_CUDA_TRY(cudaMemcpyAsync(v.data(), dev(c), c.n * sizeof(T), cudaMemcpyDeviceToHost, s));
        SWC_CUDA_TRY(cudaStreamSynchronize(s));
        return SWC_OK;
    }
  private:
    std::vector<u8> host_;
    size_t out_bytes_ = 0;
    DevBuf dev_;
};

// a null pointer among a caller's unit table: the call returns SWC_ERR_INVALID_ARG
inline bool missing(const UnitIO &a) {
    return !a.in_base || !a.in_off || !a.in_len || !a.out_base || !a.out_off || !a.out_cap || !a.out_len || !a.status;
}
inline bool missing(const DecodeIO &a) { return missing((const UnitIO &)a) || !a.consumed; }

// the columns every batched decoder takes: the unit's input and output regions in, its results out.  With
// in_on_host = false the input columns are device-only too, for a table the caller's own copies fill.
struct UnitCols {
    Col<u64> in_off, in_len, out_off, out_cap, out_len, consumed;
    Col<int32_t> status;
    UnitCols(UnitTable &t, size_t n, bool in_on_host = true)
        : in_off(in_col(t, n, in_on_host)), in_len(in_col(t, n, in_on_host)), out_off(in_col(t, n, in_on_host)),
          out_cap(in_col(t, n, in_on_host)), out_len(t.out<u64>(n)), consumed(t.out<u64>(n)), status(t.out<int32_t>(n)) {}
    // a decoder's unit columns for units [first, first + count) of the seated table `t`, reading in_base, writing out_base
    DecodeIO bind(const UnitTable &t, const u8 *in_base, u8 *out_base, u64 first, u64 count) const {
        return DecodeIO{{in_base, t.dev(in_off) + first, t.dev(in_len) + first, out_base, t.dev(out_off) + first,
                         t.dev(out_cap) + first, t.dev(out_len) + first, t.dev(status) + first, count},
                        t.dev(consumed) + first};
    }
    struct Results {
        std::vector<u64> out_len, consumed;
        std::vector<int32_t> status;
    };
    // the whole table's results (blocking: waits for `s`)
    int fetch(const UnitTable &t, Results &r, cudaStream_t s = 0) const {
        int st;
        if ((st = t.fetch(out_len, r.out_len, s)) || (st = t.fetch(consumed, r.consumed, s)) || (st = t.fetch(status, r.status, s)))
            return st;
        return SWC_OK;
    }
  private:
    static Col<u64> in_col(UnitTable &t, size_t n, bool on_host) { return on_host ? t.in<u64>(n) : t.out<u64>(n); }
};

// result of decoding ONE unit that is already resident on the device
struct UnitResult {
    DevBuf out;            // decoded bytes (device)
    size_t out_len = 0;
    size_t consumed = 0;   // bits (Deflate/BZip2) or bytes (LZ4/LZMA)
    int status = 0;
};

// Decodes the unit d_in[start, in_len) described by the 1-unit table `t` / `c` (the codec's own columns already declared
// and filled) into r.out, growing the output until it fits: `cap` bytes first, then, while the unit overflows and
// `attempts` last, grow(cap, reported out_len) bytes — 0 stops.  launch(io, cap) runs the codec on the table's columns io.
template <typename Grow, typename Launch>
int decode_unit(UnitTable &t, const UnitCols &c, const u8 *d_in, size_t start, size_t in_len, size_t cap, int attempts,
                Grow grow, Launch launch, UnitResult &r) {
    int st = t.alloc();
    if (st) return st;
    *t.host(c.in_off) = start;
    *t.host(c.in_len) = in_len - start;
    for (int attempt = 0; attempt < attempts; attempt++) {
        cap = round16(cap);
        if ((st = r.out.alloc(cap))) return st;
        *t.host(c.out_cap) = cap;
        if ((st = t.upload())) return st;
        if ((st = launch(c.bind(t, d_in, r.out.as<u8>(), 0, 1), cap))) return st;
        UnitCols::Results res;
        if ((st = c.fetch(t, res))) return st;
        r.out_len = (size_t)res.out_len[0];
        r.consumed = (size_t)res.consumed[0];
        r.status = res.status[0];
        if (r.status != SWC_ERR_OUTPUT_OVERFLOW || !(cap = grow(cap, r.out_len))) break;
    }
    return SWC_OK;
}

// The scratch of a batch that splits its units into sub-units (DESIGN §2), and its count-first step for a call that
// leaves the table size to the library.  count_first() seats unit_bytes of unit columns on the caller's scratch
// (SWC_ERR_INVALID_ARG when that is smaller) or on the pool; launch(base, &totals) lays the codec's unit columns out at
// base, launches its count and points `totals` at its k device totals, which come back into `out` with one
// synchronisation.  seat() then takes the whole layout from the pool when the caller gave no scratch.  `counted` tells
// whether the unit columns at `p` hold the counts: always on the caller's scratch, on the pool only if it kept its contents.
struct SplitScratch {
    void *p;                 // the caller's scratch, or the pool once seated
    const bool caller;
    cudaStream_t s;
    bool counted = false;
    SplitScratch(void *scratch, cudaStream_t stream) : p(scratch), caller(scratch != nullptr), s(stream) {}
    template <typename Launch> int count_first(size_t scratch_bytes, size_t unit_bytes, int k, u64 *out, Launch launch) {
        int st;
        if (caller ? scratch_bytes < unit_bytes : (st = scratch_get(unit_bytes, &p, s)) != SWC_OK)
            return caller ? SWC_ERR_INVALID_ARG : st;
        const u64 *totals = nullptr;
        if ((st = launch(p, &totals))) return st;
        SWC_CUDA_TRY(cudaMemcpyAsync(out, totals, k * sizeof(u64), cudaMemcpyDeviceToHost, s));
        SWC_CUDA_TRY(cudaStreamSynchronize(s));
        counted = true;
        return SWC_OK;
    }
    int seat(size_t bytes) {
        if (caller) return SWC_OK;
        bool kept = false;
        const int st = scratch_get(bytes, &p, s, &kept);
        counted = counted && kept;
        return st;
    }
};

// the largest table size m in [1, hi] whose layout, bytes_of(m) bytes, fits `cap`; 1 when none does
template <typename Bytes> u64 largest_table(u64 hi, size_t cap, Bytes bytes_of) {
    u64 lo = 1;
    while (lo < hi) {
        const u64 mid = lo + (hi - lo + 1) / 2;
        if (bytes_of(mid) <= cap) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// batched Deflate on device-resident tables (api_deflate.cu); start_bits may be null; scratch == nullptr -> library pool
int deflate_batch_impl(const DecodeIO &io, const uint8_t *start_bits, uint64_t out_total, void *scratch, size_t scratch_bytes,
                       cudaStream_t stream);
// the same for GzipArchive / ZlibArchive.unarchive (unarchive_batch.cu); headers may be null (always for zlib)
int unarchive_batch_impl(bool gzip, const DecodeIO &io, swc_gzip_header *headers, uint64_t out_total, void *scratch,
                         size_t scratch_bytes, cudaStream_t stream);
// the inverse of swc_unarchive_batch_scratch_bytes: an output arena `bytes` of scratch covers for n units (0: none)
uint64_t unarchive_batch_arena(uint64_t n, size_t bytes);

// large transfers between pageable host memory and the device: T threads x (stream + two pinned bounce buffers) (runtime.cu)
int copy_pageable(void *dst, const void *src, size_t bytes, bool to_device);

// the caller's input on the device, with 256 bytes of slack behind it for the decoders' wide loads
int upload_input(DevBuf &d, const uint8_t *in, size_t n);

// hand a device buffer back to a C caller as swc_alloc'ed host memory
int to_host_alloc(const void *d, size_t n, uint8_t **out, size_t *out_len);

// growable malloc'ed host buffer that is handed to the C caller without another copy (swc_free == free)
struct HostOut {
    uint8_t *p = nullptr;
    size_t len = 0, cap = 0;
    HostOut() {}
    HostOut(const HostOut &) = delete;
    HostOut &operator=(const HostOut &) = delete;
    ~HostOut() { free(p); }
    uint8_t *grow(size_t add) {                                     // nullptr when out of memory
        if (len + add > cap || !p) {
            size_t nc = cap * 2 > len + add ? cap * 2 : len + add;
            if (nc < 64) nc = 64;
            uint8_t *q = (uint8_t *)realloc(p, nc);
            if (!q) return nullptr;
            p = q; cap = nc;
        }
        uint8_t *r = p + len;
        len += add;
        return r;
    }
    int release_to(uint8_t **out, size_t *out_len) {
        if (!p && !grow(0)) return SWC_ERR_OUTPUT_OVERFLOW;
        *out = p; *out_len = len;
        p = nullptr; len = cap = 0;
        return SWC_OK;
    }
};

// Hands `v` to a C caller as an swc_alloc'ed array.  When that allocation fails, the bytes this call already handed out
// (*out) are freed again and the call returns SWC_ERR_OUTPUT_OVERFLOW.
int give_sizes(const std::vector<size_t> &v, size_t **dst, uint8_t **out, size_t *out_len);

// checks shared by the *_batch_host calls: every unit lies inside the two host arenas (overflow-safe) and every output
// region is 16-byte aligned; *monotone tells whether the units follow each other on both sides
int check_host_units(const uint64_t *in_off, const uint64_t *in_len, uint64_t in_total, const uint64_t *out_off,
                     const uint64_t *out_cap, uint64_t out_total, uint64_t n, bool *monotone);
// copies the output regions of units [b, e) from d_out back to out_base — only those: the caller's bytes between and
// around them are not ours to overwrite (regions that touch are merged, so densely packed units are one copy)
int copy_back_regions(uint8_t *out_base, const u8 *d_out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t b,
                      uint64_t e, cudaStream_t s);

// ---- container framing (a few bytes per header / block mark) read on the host ----
inline uint32_t le32(const uint8_t *p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
inline void put_le32(uint8_t *p, uint32_t v) { for (int k = 0; k < 4; k++) p[k] = (uint8_t)(v >> (8 * k)); }

}  // namespace swc
