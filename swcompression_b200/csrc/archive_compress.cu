// archive_compress.cu — batched GzipArchive.archive (reference Sources/GZip/GzipArchive.swift:126-241) and
// ZlibArchive.archive (Sources/Zlib/ZlibArchive.swift:54-70) on device-resident units: the framing runs on the device
// around the Deflate compressor of deflate_compress.cu.  With a caller scratch and max_in_bytes > 0 the call is a fixed
// sequence of launches: no host read, no allocation (DESIGN.md §4.16).
//
//   place      one CTA           fit rule, each unit's scratch and staging offsets, link-tile, emit-chunk and finish-CTA
//                                prefix sums (deflatec::Plan), status OK / UNSUPPORTED
//   checksum   warp per unit     CRC-32 (gzip) or Adler-32 (zlib) of the input, placed units only
//   link, parse, emit, seam      deflatec::run: each stream into staging in the scratch, which it never overflows
//   finish     CTA per 64 KiB    out_len and status; header, stream and trailer into the caller's region of a unit that
//                                fits, every byte once, 16-byte stores wherever the region allows
#include <vector>
#include "../../include/swcgpu.h"
#include "compress_host.h"
#include "deflate_compress.cuh"

namespace swc {
namespace {

using deflatec::MAX_UNIT;

constexpr u64 FIN_BYTES = 64u << 10;     // output bytes per finish CTA
constexpr u64 ZLIB_HDR = 2;              // 78 DA (ZlibArchive.swift:56-60)

// one archive batch: the caller's unit table and, for gzip, the header columns (hdr_base null: zlib)
struct ArcArgs : UnitIO {
    const u8 *hdr_base;
    const u64 *hdr_off, *hdr_len;
};

__host__ __device__ __forceinline__ u64 stream_max(u64 l) { return (9 * l + 17) / 8; }    // Deflate.compress's largest
// a unit's staging: its largest stream and 16 bytes for the finish kernel's aligned over-read, in whole 256-byte lines
__host__ __device__ __forceinline__ u64 stage_bytes(u64 l) { return deflatec::a256(stream_max(l) + 16); }
__host__ __device__ __forceinline__ u64 unit_need(u64 l) { return l >= MAX_UNIT ? 0 : deflatec::unit_scratch(l) + stage_bytes(l); }

// the per-unit columns of one slice (index j = unit - first), at the front of the scratch
struct Cols {
    u64 *scr_off, *tile_start, *chunk_start, *fin_start;       // the starts have count + 1 entries
    u64 *eff_len;              // the unit's length, or MAX_UNIT for a unit that is not placed (the parse rejects it)
    u64 *stage_off, *stage_cap, *s_len;
    int32_t *st, *s_st;        // place status; the Deflate stage's status
    u32 *ck;                   // CRC-32 or Adler-32 of the input
};

struct Layout {
    Cols c;
    size_t bytes;
    Layout(void *base, u64 count) {
        Carver k(base);
        k.cols(count, c.scr_off);
        k.cols(count + 1, c.tile_start, c.chunk_start, c.fin_start);
        k.cols(count, c.eff_len, c.stage_off, c.stage_cap, c.s_len, c.st, c.s_st, c.ck);
        bytes = k.at;
    }
};

__device__ __forceinline__ u64 header_len(const ArcArgs &a, u64 u) { return a.hdr_base ? a.hdr_len[u] : ZLIB_HDR; }
__device__ __forceinline__ u64 trailer_len(const ArcArgs &a) { return a.hdr_base ? 8 : 4; }

// Units [first, first + count), a contiguous run of them per thread.  Unit i is placed while the exclusive prefix sum of
// in_len plus its own length is at most `fit` (and it is under 4 GiB); placed units get their scratch and staging behind
// the `head` bytes of columns, in order.
__global__ void __launch_bounds__(1024) arc_place_kernel(ArcArgs a, Cols c, u64 first, u64 count, u64 fit, u64 head) {
    __shared__ u64 part[4][1024];
    u64 b, e;
    cta_unit_run(count, b, e);
    const u64 *len = a.in_len + first;
    u64 sum = 0;
    for (u64 j = b; j < e; j++) sum += len[j];
    part[0][threadIdx.x] = sum;
    cta_scan<1>(part);
    const u64 at0 = part[0][threadIdx.x] - sum;
    auto fits = [&](u64 at, u64 l) { return l < MAX_UNIT && at <= fit && l <= fit - at; };
    u64 s[4] = {0, 0, 0, 0};                             // need, tiles, chunks, finish CTAs
    for (u64 j = b, at = at0; j < e; at += len[j], j++) {
        const u64 l = len[j], el = fits(at, l) ? l : MAX_UNIT;
        s[0] += unit_need(el); s[1] += deflatec::unit_tiles(el); s[2] += deflatec::unit_chunks(el);
        s[3] += el == MAX_UNIT ? 1 : (header_len(a, first + j) + stream_max(l) + trailer_len(a) + 32 + FIN_BYTES - 1) / FIN_BYTES;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; k++) part[k][threadIdx.x] = s[k];
    cta_scan<4>(part);
    u64 o[4];
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = part[k][threadIdx.x] - s[k];
    for (u64 j = b, at = at0; j < e; at += len[j], j++) {
        const u64 l = len[j];
        const bool ok = fits(at, l);
        const u64 el = ok ? l : MAX_UNIT;
        c.scr_off[j] = head + o[0];
        c.stage_off[j] = head + o[0] + deflatec::unit_scratch(el);
        c.stage_cap[j] = ok ? stage_bytes(l) - 16 : 0;
        c.tile_start[j] = o[1]; c.chunk_start[j] = o[2]; c.fin_start[j] = o[3];
        c.eff_len[j] = el;
        c.st[j] = ok ? SWC_OK : SWC_ERR_UNSUPPORTED;
        o[0] += unit_need(el); o[1] += deflatec::unit_tiles(el); o[2] += deflatec::unit_chunks(el);
        o[3] += ok ? (header_len(a, first + j) + stream_max(l) + trailer_len(a) + 32 + FIN_BYTES - 1) / FIN_BYTES : 1;
    }
    if (threadIdx.x == 1023) { c.tile_start[count] = o[1]; c.chunk_start[count] = o[2]; c.fin_start[count] = o[3]; }
}

// the unit j of a slice whose range of `start` (count + 1 prefix sums) holds g
__device__ __forceinline__ u64 locate(const u64 *start, u64 count, u64 g) {
    u64 lo = 0, hi = count;
    while (hi - lo > 1) {
        const u64 mid = (lo + hi) >> 1;
        if (start[mid] <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// 16 stream bytes from stg[q, q + 16) with q = q0 + sh, q0 a multiple of 16: two aligned loads and funnel shifts
__device__ __forceinline__ uint4 shifted16(const u8 *stg, u64 q0, u32 sh) {
    const uint4 x = *(const uint4 *)(stg + q0), y = *(const uint4 *)(stg + q0 + 16);
    const u32 w[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
    const u32 ws = sh >> 2, bs = (sh & 3) * 8;
    u32 r[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const u32 lo = ws == 0 ? w[i] : ws == 1 ? w[i + 1] : ws == 2 ? w[i + 2] : w[i + 3];
        const u32 hi = ws == 0 ? w[i + 1] : ws == 1 ? w[i + 2] : ws == 2 ? w[i + 3] : w[i + 4];
        r[i] = __funnelshift_r(lo, hi, bs);
    }
    return make_uint4(r[0], r[1], r[2], r[3]);
}

// CTA g of the slice's finish range: FIN_BYTES / 16 aligned 16-byte vectors of its unit's region.  The first CTA of a
// unit writes out_len and status; a unit that is not OK or whose archive passes out_cap writes no byte.  The grid may be
// smaller than the range: CTAs stride over it.
__global__ void __launch_bounds__(256) arc_finish_kernel(ArcArgs a, Cols c, const u8 *scr, u64 first, u64 count) {
    const u64 nfin = c.fin_start[count];
    for (u64 g = blockIdx.x; g < nfin; g += gridDim.x) {
        const u64 j = locate(c.fin_start, count, g), k = g - c.fin_start[j], u = first + j;
        int st = c.st[j];
        if (st == SWC_OK) st = c.s_st[j];
        const bool gz = a.hdr_base != nullptr;
        const u64 hl = header_len(a, u), sl = st == SWC_OK ? c.s_len[j] : 0, total = hl + sl + trailer_len(a);
        if (st == SWC_OK && total > a.out_cap[u]) st = SWC_ERR_OUTPUT_OVERFLOW;
        if (k == 0 && threadIdx.x == 0) {
            a.status[u] = st;
            a.out_len[u] = st == SWC_OK || st == SWC_ERR_OUTPUT_OVERFLOW ? total : 0;
        }
        if (st != SWC_OK) continue;
        const u8 *hdr = gz ? a.hdr_base + a.hdr_off[u] : nullptr;
        const u8 *stg = scr + c.stage_off[j];
        const u32 ck = c.ck[j], isize = (u32)a.in_len[u];
        auto byte_at = [&](u64 q) -> u8 {                  // byte q of the archive
            if (q < hl) return gz ? hdr[q] : q ? 0xDA : 0x78;
            q -= hl;
            if (q < sl) return stg[q];
            q -= sl;
            if (gz) return (u8)((q < 4 ? ck : isize) >> (8 * (q & 3)));              // GzipArchive.swift:237-241, LE
            return (u8)(ck >> (8 * (3 - q)));                                         // ZlibArchive.swift:64-68, BE
        };
        u8 *dst = a.out_base + a.out_off[u];
        const u64 a0 = (u64)(uintptr_t)dst;
        const u64 v0 = a0 >> 4, vend = (a0 + total + 15) >> 4;
        const u64 vb = v0 + k * (FIN_BYTES / 16), ve = vend < vb + FIN_BYTES / 16 ? vend : vb + FIN_BYTES / 16;
        const u32 sh = (u32)(0 - (a0 + hl)) & 15;       // stream byte offset of every vector start, mod 16
        for (u64 v = vb + threadIdx.x; v < ve; v += blockDim.x) {
            const int64_t p = (int64_t)(v * 16 - a0);     // archive position of the vector's first byte
            if (p >= 0 && (u64)p + 16 <= total) {
                uint4 r;
                if ((u64)p >= hl && (u64)p + 16 <= hl + sl) {
                    r = shifted16(stg, (u64)p - hl - sh, sh);
                } else {
                    u32 w[4] = {0, 0, 0, 0};
#pragma unroll
                    for (int i = 0; i < 16; i++) w[i >> 2] |= (u32)byte_at((u64)p + i) << (8 * (i & 3));
                    r = make_uint4(w[0], w[1], w[2], w[3]);
                }
                *(uint4 *)(dst + p) = r;
            } else {
                for (int i = 0; i < 16; i++) {
                    const int64_t q = p + i;
                    if (q >= 0 && (u64)q < total) dst[q] = byte_at((u64)q);
                }
            }
        }
    }
}

// the grid of a slice whose placed units hold at most `in_bytes` input bytes: the bounds of DESIGN §4.16
struct Grids { u64 tiles, chunks, fin; };
Grids grids(u64 count, u64 in_bytes) {
    const u64 fin = stream_max(in_bytes) / FIN_BYTES + count;
    return Grids{in_bytes / deflatec::TILE + count, in_bytes / deflatec::CHUNK + count, fin < (1u << 20) ? fin : (1u << 20)};
}

// one slice: units [first, first + count) placed by `fit`, their input at most `in_bytes`, columns at the front of scr
int archive_slice(const ArcArgs &a, u64 first, u64 count, u8 *scr, u64 fit, u64 in_bytes, cudaStream_t s) {
    const u64 head = Layout(nullptr, count).bytes;
    const Cols c = Layout(scr, count).c;
    const Grids g = grids(count, in_bytes);
    timing_mark(s);
    arc_place_kernel<<<1, 1024, 0, s>>>(a, c, first, count, fit, head);
    count_launch();
    timing_mark(s);
    int st = a.hdr_base ? checks::crc32_units(a.in_base, a.in_off + first, a.in_len + first, c.st, c.ck, count, s)
                        : checks::adler32_units(a.in_base, a.in_off + first, a.in_len + first, c.st, c.ck, count, s);
    if (st) return st;
    // the streams go to staging: out_base is the scratch, and a unit that is not placed has a length the parse rejects
    const deflatec::Args d{{a.in_base, a.in_off + first, c.eff_len, scr, c.stage_off, c.stage_cap, c.s_len, c.s_st, count}};
    if ((st = deflatec::run(d, 0, count, scr, deflatec::Plan{c.scr_off, c.tile_start, c.chunk_start, g.tiles, g.chunks}, s)))
        return st;
    arc_finish_kernel<<<(unsigned)g.fin, 256, 0, s>>>(a, c, scr, first, count);
    count_launch();
    timing_mark(s);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

u64 capture_scratch(u64 n, u64 max_in) {
    // unit_scratch(l) <= 9 l + 2048 and stage_bytes(l) <= 9 l / 8 + 290, summed over the placed units
    return Layout(nullptr, n).bytes + 9 * max_in + (9 * max_in + 7) / 8 + n * (2048 + 512) + 256;
}

// the batch in slices of the scratch; `lens` is the host copy of in_len
int archive_slices(const ArcArgs &a, const std::vector<u64> &lens, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    return run_in_slices(a.n, [&](u64 i) { return unit_need(lens[i]); }, [](u64 count) { return (u64)Layout(nullptr, count).bytes; },
                         scratch, scratch_bytes, s, [&](u64 first, u64 count, u8 *scr, size_t) -> int {
        u64 in_bytes = 0;
        for (u64 j = first; j < first + count; j++) in_bytes += lens[j] < MAX_UNIT ? lens[j] : 0;
        return archive_slice(a, first, count, scr, ~0ull, in_bytes, s);
    });
}

int archive_batch(const ArcArgs &a, u64 max_in, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    if (max_in == 0) {                  // the library plans the slices: the lengths come back (one synchronisation)
        std::vector<u64> lens;
        int st = read_lens(a.in_len, a.n, s, lens);
        if (st) return st;
        return archive_slices(a, lens, scratch, scratch_bytes, s);
    }
    const u64 need = capture_scratch(a.n, max_in);
    if (scratch && scratch_bytes < need) return SWC_ERR_INVALID_ARG;
    if (!scratch) {
        int st = scratch_get((size_t)need, &scratch, s);
        if (st) return st;
    }
    return archive_slice(a, 0, a.n, (u8 *)scratch, max_in, max_in, s);
}

// GzipArchive.archive's header (GzipArchive.swift:126-235)
int gzip_header(const swc_gzip_options *o, std::vector<uint8_t> &h) {
    if (o->n_extra && (!o->extra_ids || !o->extra_lens || !o->extra_bytes)) return SWC_ERR_INVALID_ARG;
    uint64_t xlen = 0;
    for (size_t i = 0; i < o->n_extra; i++) xlen += 4 + o->extra_lens[i];
    if (xlen > 65535) return SWC_GZIP_CANNOT_ENCODE_ISO_LATIN1;                             // :205-207
    h = {0x1f, 0x8b, 8,
         (uint8_t)((o->comment ? 1 << 4 : 0) | (o->file_name ? 1 << 3 : 0) | (o->n_extra ? 1 << 2 : 0) |
                   (o->write_header_crc ? 1 << 1 : 0) | (o->is_text_file ? 1 : 0))};   // :130-176
    for (int k = 0; k < 4; k++) h.push_back(o->has_mtime ? (uint8_t)((uint64_t)o->mtime >> (8 * k)) : 0);   // :180-186
    h.push_back(2);
    h.push_back(o->os_type);
    if (o->n_extra) {                                                                       // :204-223
        h.push_back((uint8_t)xlen); h.push_back((uint8_t)(xlen >> 8));
        size_t at = 0;
        for (size_t i = 0; i < o->n_extra; i++) {
            const size_t l = (size_t)o->extra_lens[i];
            h.push_back(o->extra_ids[2 * i]); h.push_back(o->extra_ids[2 * i + 1]);
            h.push_back((uint8_t)l); h.push_back((uint8_t)(l >> 8));
            h.insert(h.end(), o->extra_bytes + at, o->extra_bytes + at + l);
            at += l;
        }
    }
    // ISO-Latin-1 text, NUL-terminated unless it already ends with NUL (:132-161)
    auto text = [&](const uint8_t *t, size_t n) {
        if (!t) return;
        h.insert(h.end(), t, t + n);
        if (n == 0 || t[n - 1] != 0) h.push_back(0);
    };
    text(o->file_name, o->file_name_len);
    text(o->comment, o->comment_len);
    if (o->write_header_crc) {                                                              // :230-235
        const uint32_t c = crc32_framing(h.data(), h.size());
        h.push_back((uint8_t)c); h.push_back((uint8_t)(c >> 8));
    }
    return SWC_OK;
}

// the single calls' batch: one unit whose length the host knows
int one_archive(const ArcArgs &a, const std::vector<u64> &lens, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    return archive_slices(a, lens, scratch, scratch_bytes, s);
}

bool missing_archive(const ArcArgs &a, bool gz) { return missing((const UnitIO &)a) || (gz && (!a.hdr_base || !a.hdr_off || !a.hdr_len)); }

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

int32_t swc_gzip_archive_header(const swc_gzip_options *options, uint8_t *buf, size_t cap, size_t *len) {
    if (!options || !len || (!buf && cap)) return SWC_ERR_INVALID_ARG;
    std::vector<uint8_t> h;
    int st = gzip_header(options, h);
    if (st) return st;
    *len = h.size();
    if (cap < h.size()) return SWC_ERR_OUTPUT_OVERFLOW;
    memcpy(buf, h.data(), h.size());
    return SWC_OK;
}

size_t swc_gzip_archive_max_bytes(uint64_t in_len, uint64_t header_len) { return (size_t)(header_len + stream_max(in_len) + 8); }
size_t swc_zlib_archive_max_bytes(uint64_t in_len) { return (size_t)(ZLIB_HDR + stream_max(in_len) + 4); }
size_t swc_archive_compress_batch_scratch_bytes(uint64_t n, uint64_t max_in_bytes) { return (size_t)capture_scratch(n, max_in_bytes); }

int32_t swc_gzip_archive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                               const uint8_t *hdr_base, const uint64_t *hdr_off, const uint64_t *hdr_len,
                               uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                               uint64_t *out_len, int32_t *status, uint64_t n, uint64_t max_in_bytes,
                               void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    ArcArgs a{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, hdr_base, hdr_off, hdr_len};
    if (missing_archive(a, true)) return SWC_ERR_INVALID_ARG;
    return archive_batch(a, max_in_bytes, scratch, scratch_bytes, (cudaStream_t)cuda_stream);
}

int32_t swc_zlib_archive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                               uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                               uint64_t *out_len, int32_t *status, uint64_t n, uint64_t max_in_bytes,
                               void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    ArcArgs a{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, nullptr, nullptr, nullptr};
    if (missing_archive(a, false)) return SWC_ERR_INVALID_ARG;
    return archive_batch(a, max_in_bytes, scratch, scratch_bytes, (cudaStream_t)cuda_stream);
}

// ZlibArchive.archive(data:) ZlibArchive.swift:54-70: the one-unit batch on the library pool
int32_t swc_zlib_archive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (in_len >= MAX_UNIT) return SWC_ERR_UNSUPPORTED;
    return compress_one(ArcArgs{}, one_archive, swc_zlib_archive_max_bytes(in_len), in, in_len, out, out_len);
}

// GzipArchive.archive(data:comment:fileName:writeHeaderCRC:isTextFile:osType:modificationTime:extraFields:)
// GzipArchive.swift:126-241: the header on the host, then the one-unit batch on the library pool
int32_t swc_gzip_archive(const uint8_t *in, size_t in_len, const swc_gzip_options *o, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || !o || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    std::vector<uint8_t> h;
    int st = gzip_header(o, h);
    if (st) return st;
    if (in_len >= MAX_UNIT) return SWC_ERR_UNSUPPORTED;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    // one upload: the header's offset and length columns (16 and its size), then its bytes
    std::vector<uint8_t> blob(16 + h.size());
    const u64 cols[2] = {16, h.size()};
    memcpy(blob.data(), cols, 16);
    memcpy(blob.data() + 16, h.data(), h.size());
    DevBuf d_hdr;
    if ((st = d_hdr.alloc(blob.size()))) return st;
    SWC_CUDA_TRY(cudaMemcpy(d_hdr.p, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    ArcArgs a{};
    a.hdr_base = d_hdr.as<u8>(); a.hdr_off = d_hdr.as<u64>(); a.hdr_len = d_hdr.as<u64>() + 1;
    return compress_one(a, one_archive, swc_gzip_archive_max_bytes(in_len, h.size()), in, in_len, out, out_len);
}

}  // extern "C"
