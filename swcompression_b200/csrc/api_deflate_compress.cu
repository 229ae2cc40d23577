// api_deflate_compress.cu — C ABI for Deflate compression: raw Deflate batches in device memory, and the single calls
// Deflate.compress (Deflate+Compress.swift:22-42), ZlibArchive.archive (ZlibArchive.swift:54-70) and GzipArchive.archive
// (GzipArchive.swift:126-241).  The stream and the CRC-32 / Adler-32 of the input are computed on the device; the host
// writes the few framing bytes around them.
#include <vector>
#include "../../include/swcgpu.h"
#include "compress_host.h"
#include "deflate_compress.cuh"

using namespace swc;

namespace {

inline u64 meta_bytes(u64 count) { return (3 * count + 2) * 8 + 3 * 256; }

// the batch on device-resident tables; `lens` is the host copy of in_len
int batch_impl(const deflatec::Args &a, const std::vector<u64> &lens, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    std::vector<u64> plan;
    return run_in_slices(a.n, [&](u64 i) { return deflatec::unit_scratch(lens[i]); }, meta_bytes, scratch, scratch_bytes, s,
                         [&](u64 first, u64 count, u8 *scr, size_t) -> int {
        // the slice's plan first (scratch offsets, tile and chunk prefix sums), then each unit's region
        plan.assign(3 * count + 2, 0);
        u64 *off = plan.data(), *tiles = off + count, *chunks = tiles + count + 1;
        u64 at = meta_bytes(count);
        for (u64 j = 0; j < count; j++) {
            const u64 l = lens[first + j];
            off[j] = at; at += deflatec::unit_scratch(l);
            tiles[j + 1] = tiles[j] + deflatec::unit_tiles(l);
            chunks[j + 1] = chunks[j] + deflatec::unit_chunks(l);
        }
        // a copy from pageable memory has read `plan` when it returns, so the next slice may refill it
        SWC_CUDA_TRY(cudaMemcpyAsync(scr, plan.data(), plan.size() * 8, cudaMemcpyHostToDevice, s));
        deflatec::Plan p;
        p.scr_off = (const u64 *)scr; p.tile_start = p.scr_off + count; p.chunk_start = p.tile_start + count + 1;
        p.tiles = tiles[count]; p.chunks = chunks[count];
        return deflatec::run(a, first, count, scr, p, s);
    });
}

// one framed result: `head`, the Deflate stream of `in`, then `tail_len` bytes of trailer written by `tail`
template <typename Tail>
int framed(const uint8_t *in, size_t in_len, const std::vector<uint8_t> &head, checks::Kind kind, size_t tail_len, Tail tail,
           uint8_t **out, size_t *out_len) {
    if (in_len >= deflatec::MAX_UNIT) return SWC_ERR_UNSUPPORTED;
    // (9 n + 17) / 8: the largest stream Deflate.compress writes for n bytes
    return compress_one(deflatec::Args{}, batch_impl, (9 * (u64)in_len + 17) / 8, in, in_len, out, out_len, head, kind, tail_len,
                        tail);
}

}  // namespace

extern "C" {

size_t swc_deflate_compress_batch_scratch_bytes(uint64_t n, uint64_t in_bytes_total) {
    // unit_scratch(l) <= 9 l + 2048 (link 2 l, chains 6 l, visited, checkpoints and alignment), plus the slice's plan
    return (size_t)(in_bytes_total * 9 + n * (2048 + 24) + 4096);
}

int32_t swc_deflate_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                   uint64_t *out_len, int32_t *status, uint64_t n,
                                   void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    if (!in_base || !in_off || !in_len || !out_base || !out_off || !out_cap || !out_len || !status) return SWC_ERR_INVALID_ARG;
    const cudaStream_t s = (cudaStream_t)cuda_stream;
    // the scratch layout is planned on the host from the unit sizes (n x 8 bytes)
    std::vector<u64> lens;
    int st = read_lens(in_len, n, s, lens);
    if (st) return st;
    const deflatec::Args a{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}};
    return batch_impl(a, lens, scratch, scratch_bytes, s);
}

// Deflate.compress(data:) Deflate+Compress.swift:22-42
int32_t swc_deflate_compress(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    return framed(in, in_len, {}, checks::CRC32, 0, [](uint8_t *, uint32_t) {}, out, out_len);
}

// ZlibArchive.archive(data:) ZlibArchive.swift:54-70
int32_t swc_zlib_archive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    return framed(in, in_len, {0x78, 0xDA}, checks::ADLER32, 4, [](uint8_t *p, uint32_t v) {
        for (int k = 0; k < 4; k++) p[k] = (uint8_t)(v >> (8 * (3 - k)));
    }, out, out_len);
}

// GzipArchive.archive(data:comment:fileName:writeHeaderCRC:isTextFile:osType:modificationTime:extraFields:)
// GzipArchive.swift:126-241
int32_t swc_gzip_archive(const uint8_t *in, size_t in_len, const swc_gzip_options *o, uint8_t **out, size_t *out_len) {
    if (!out || !out_len || !o || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (o->n_extra && (!o->extra_ids || !o->extra_lens || !o->extra_bytes)) return SWC_ERR_INVALID_ARG;
    uint64_t xlen = 0;
    for (size_t i = 0; i < o->n_extra; i++) xlen += 4 + o->extra_lens[i];
    if (xlen > 65535) return SWC_GZIP_CANNOT_ENCODE_ISO_LATIN1;                             // :205-207
    std::vector<uint8_t> h = {0x1f, 0x8b, 8,
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
    const uint32_t isize = (uint32_t)in_len;
    return framed(in, in_len, h, checks::CRC32, 8, [isize](uint8_t *p, uint32_t crc) {   // :237-260
        put_le32(p, crc); put_le32(p + 4, isize);
    }, out, out_len);
}

}  // extern "C"
