// unarchive_batch.cu — batched GzipArchive.unarchive / ZlibArchive.unarchive on device-resident archives: one archive per
// unit, everything enqueued on the caller's stream (no host read, no allocation when the caller passes scratch).
// Reference: Sources/GZip/GzipArchive.swift:38-47, 79-100, Sources/Zlib/ZlibArchive.swift:25-42.
//
// Four stages (DESIGN.md §4.12):
//   header   unarchive_header_kernel, one thread per unit: the `bytesLeft >= 20` guard (gzip), then the header grammar of
//            archive_header.cuh bounded by in_len[i]; writes the Deflate input column (in_off + header length, in_len -
//            header length, or length 0 when the header failed, so that the Deflate stage rejects the unit at once), the
//            header status and, for gzip, the caller's swc_gzip_header array;
//   Deflate  deflate_batch_impl on those columns, unchanged (K1w below 20 000 units, K1L from there, slow kernel, replay),
//            writing the caller's out_len / status and, in the caller's consumed array, the Deflate bits;
//   checksum checks::crc32_units (gzip) or checks::adler32_units (zlib), one warp per unit the Deflate stage decoded; a
//            one-unit batch (the single calls) spreads its unit over the whole GPU instead (checks::unit_check);
//   trailer  unarchive_trailer_kernel, one thread per unit: the final status, out_len and consumed in the reference's order.
#include "../../include/swcgpu.h"
#include "archive_header.cuh"
#include "checks.cuh"
#include "host_util.h"
#include "inflate.cuh"

namespace swc {
namespace {

// scratch: four n-entry columns (Deflate input offset and length, header status, checksum), then the Deflate scratch
struct Scratch {
    u64 *d_off, *d_len;
    int32_t *hstat;
    u32 *check;
    void *inflate;
    size_t inflate_bytes;
};
size_t columns_bytes(u64 n) { return 2 * round256(n * 8) + 2 * round256(n * 4); }
Scratch seat(void *p, u64 n, size_t bytes) {
    Scratch r;
    Carver c(p);
    c.cols(n, r.d_off, r.d_len, r.hstat, r.check);
    r.inflate = c.end();
    r.inflate_bytes = bytes - c.at;
    return r;
}

template <bool GZIP>
__global__ void __launch_bounds__(256) unarchive_header_kernel(const u8 *in_base, const u64 *in_off, const u64 *in_len, Scratch s,
                                                               swc_gzip_header *headers, u64 n) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u64 o = in_off[i], L = in_len[i];
    const u8 *p = in_base + o;
    size_t hl = 0;
    int st;
    if (GZIP) {
        swc_gzip_header h = {};
        st = L < 20 ? SWC_GZIP_WRONG_MAGIC : gzip_parse(p, L, 0, &h);          // GzipArchive.swift:83, then GzipHeader
        if (st == SWC_OK) {
            hl = h.header_len;
            if (h.has_file_name) h.file_name_off += o;                          // offsets relative to in_base
            if (h.has_comment) h.comment_off += o;
            if (h.extra_len) h.extra_off += o;
        }
        if (headers) headers[i] = h;
    } else {
        swc_zlib_header h;
        st = zlib_parse(p, L, &h);
        if (st == SWC_OK) hl = h.header_len;
    }
    s.hstat[i] = st;
    s.d_off[i] = o + hl;
    s.d_len[i] = st == SWC_OK ? L - hl : 0;
}

__device__ __forceinline__ u32 rd_le32(const u8 *q) { return (u32)q[0] | (u32)q[1] << 8 | (u32)q[2] << 16 | (u32)q[3] << 24; }
__device__ __forceinline__ u32 rd_be32(const u8 *q) { return (u32)q[0] << 24 | (u32)q[1] << 16 | (u32)q[2] << 8 | (u32)q[3]; }

// processMember GzipArchive.swift:84-99 / ZlibArchive.swift:29-41 after the Deflate stage.  `consumed` holds the Deflate bits
// on entry and the archive bytes the reference read on exit (0 unless the status is OK or payload-carrying).
template <bool GZIP>
__global__ void __launch_bounds__(256) unarchive_trailer_kernel(const u8 *in_base, const u64 *in_off, const u64 *in_len, Scratch s,
                                                                u64 *out_len, u64 *consumed, int32_t *status, u64 n) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int hs = s.hstat[i];
    if (hs != SWC_OK) {                                                          // header (and gzip's 20-byte guard)
        status[i] = hs; out_len[i] = 0; consumed[i] = 0;
        return;
    }
    if (status[i] != SWC_OK) {                                                   // any Deflate status is final
        consumed[i] = 0;
        return;
    }
    const u64 o = in_off[i], L = in_len[i];
    const u64 p = (s.d_off[i] - o) + (consumed[i] + 7) / 8;                      // align()
    const u64 left = p <= L ? L - p : 0;
    const u8 *q = in_base + o + p;
    int st;
    u64 used = 0;
    if (GZIP) {
        if (left < 8) {
            st = SWC_GZIP_WRONG_MAGIC;                                           // :88-89
        } else if ((u32)out_len[i] != rd_le32(q + 4)) {
            st = SWC_GZIP_WRONG_ISIZE;                                           // :94-95
        } else {
            st = s.check[i] == rd_le32(q) ? SWC_OK : SWC_GZIP_WRONG_CRC;         // :97-98 (the data is kept)
            used = p + 8;
        }
    } else if (left < 4) {
        st = SWC_ZLIB_WRONG_ADLER32;                                             // :34-35 (the data is kept)
        used = p;
    } else {
        st = s.check[i] == rd_be32(q) ? SWC_OK : SWC_ZLIB_WRONG_ADLER32;         // :37-40
        used = p + 4;
    }
    status[i] = st;
    consumed[i] = used;
}

}  // namespace

int unarchive_batch_impl(bool gzip, const DecodeIO &io, swc_gzip_header *headers, uint64_t out_total, void *scratch,
                         size_t scratch_bytes, cudaStream_t stream) {
    const u64 n = io.n;
    if (n == 0) return SWC_OK;
    if (missing(io)) return SWC_ERR_INVALID_ARG;
    const size_t need = swc_unarchive_batch_scratch_bytes(n, out_total);
    if (!scratch) {
        scratch_bytes = need;
        int st = scratch_get(need, &scratch, stream);
        if (st) return st;
    } else if (scratch_bytes < need) {
        return SWC_ERR_INVALID_ARG;
    }
    const Scratch s = seat(scratch, n, scratch_bytes);
    const unsigned blocks = (unsigned)((n + 255) / 256);
    timing_mark(stream);
    if (gzip) unarchive_header_kernel<true><<<blocks, 256, 0, stream>>>(io.in_base, io.in_off, io.in_len, s, headers, n);
    else unarchive_header_kernel<false><<<blocks, 256, 0, stream>>>(io.in_base, io.in_off, io.in_len, s, nullptr, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(stream);
    const DecodeIO dio{{io.in_base, s.d_off, s.d_len, io.out_base, io.out_off, io.out_cap, io.out_len, io.status, n}, io.consumed};
    int st = deflate_batch_impl(dio, nullptr, out_total, s.inflate, s.inflate_bytes, stream);
    if (st) return st;
    // one warp would hold a lone large unit back; its out_total / 512 bytes of partials fit the ~1.33 x out_total Deflate scratch
    if (n == 1)
        st = checks::unit_check(gzip ? checks::CRC32 : checks::ADLER32, io.out_base, io.out_off, io.out_len, io.status, out_total,
                                s.check, (u64 *)s.inflate, stream);
    else
        st = gzip ? checks::crc32_units(io.out_base, io.out_off, io.out_len, io.status, s.check, n, stream)
                  : checks::adler32_units(io.out_base, io.out_off, io.out_len, io.status, s.check, n, stream);
    if (st) return st;
    timing_mark(stream);
    if (gzip) unarchive_trailer_kernel<true><<<blocks, 256, 0, stream>>>(io.in_base, io.in_off, io.in_len, s, io.out_len, io.consumed, io.status, n);
    else unarchive_trailer_kernel<false><<<blocks, 256, 0, stream>>>(io.in_base, io.in_off, io.in_len, s, io.out_len, io.consumed, io.status, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(stream);
    return SWC_OK;
}

uint64_t unarchive_batch_arena(uint64_t n, size_t bytes) {
    const size_t cols = columns_bytes(n);
    return bytes < cols ? 0 : inflate::arena_covered(n, bytes - cols);
}

}  // namespace swc

using namespace swc;

extern "C" {

size_t swc_unarchive_batch_scratch_bytes(uint64_t n, uint64_t out_capacity_total) {
    return columns_bytes(n) + inflate::scratch_bytes(n, out_capacity_total);
}

int32_t swc_gzip_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                 uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t out_capacity_total,
                                 uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status, swc_gzip_header *headers,
                                 uint64_t n, void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    const DecodeIO io{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bytes};
    return unarchive_batch_impl(true, io, headers, out_capacity_total, scratch, scratch_bytes, (cudaStream_t)cuda_stream);
}

int32_t swc_zlib_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                 uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t out_capacity_total,
                                 uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                 uint64_t n, void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    const DecodeIO io{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bytes};
    return unarchive_batch_impl(false, io, nullptr, out_capacity_total, scratch, scratch_bytes, (cudaStream_t)cuda_stream);
}

}  // extern "C"
