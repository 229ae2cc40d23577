// lz4_frame_batch.cu — batched LZ4.decompress(data:dictionary:dictionaryID:) on device-resident frames: the frame layer
// (reference Sources/LZ4/LZ4.swift:73-91, :148-330) walked on the device, feeding the block kernels of lz4.cu.  With a caller
// scratch and max_blocks > 0 the call is a fixed sequence of launches: no host read, no allocation (DESIGN.md §4.14).
//
//   walk<COUNT>   thread per unit   skippable frames, magic, descriptor and its checksum, then the chain of block marks:
//                                   kind, block count, record slots, the framing error and the block it stands behind
//   place         one CTA           first_blk / rec_first = exclusive sums over the units; units past the table are marked
//   walk<FILL>    thread per unit   the block columns (offset, length, stored bit, checksum word, "no dictionary")
//   parse         thread per block  lz4_parse_kernel with no capacity fence: every block's size and final status
//   xxh32         warp per block    block checksums over the compressed bytes (frames with the flag only)
//   chain         warp per unit     lz4_block_body over first_blk / n_blk for frames with dependent blocks
//   resolve       warp per unit     the first failure in the reference's order, output offsets of an independent frame's
//                                   blocks, content size, capacity; blocks of failed or overflowing units are switched off
//   exec          warp per block    lz4_exec_kernel / lz4_fallback_kernel, unchanged replay
//   xxh32, check  warp per unit     content checksum over the decoded bytes; turns OK into checksumMismatch
#include <climits>
#include "../../include/swcgpu.h"
#include "checks.cuh"
#include "host_util.h"
#include "lz4.cuh"
#include "lz4_frame.cuh"

namespace swc {
namespace {

typedef swc_lz4_frame_info Info;
enum : u32 { KIND_NONE = 0, KIND_INDEPENDENT = 1, KIND_DEPENDENT = 2, KIND_LEGACY = 3 };
using namespace lz4f;
constexpr u32 UNPLACED = 0x10000;          // internal: the unit's blocks do not fit the block table or the record area
constexpr u64 STORED = 1ull << 63;

__device__ __forceinline__ u32 rd32(const u8 *p) { return (u32)p[0] | (u32)p[1] << 8 | (u32)p[2] << 16 | (u32)p[3] << 24; }
__device__ __forceinline__ bool is_magic(u32 v) { return v == 0x184D2204u || v == 0x184C2102u || (v >= 0x184D2A50u && v <= 0x184D2A5Fu); }

// the block columns of the batch, indexed by block; walk<FILL> writes them
struct BlockCols {
    u64 *off, *len;        // compressed bytes (offset from in_base; bit 63 of len = stored)
    u64 *par_len;          // len for the blocks the parse decodes, 0 for blocks of dependent frames
    u64 *ck_len;           // len for blocks that carry a checksum, else 0
    u32 *stored_ck, *ck;   // the checksum word behind the block / the one computed
    u8 *no_dict;
    u64 *out_off, *cap, *out_len, *rec_base;
    int32_t *status;
    u32 *rec_count;
};

struct WalkArgs {
    const u8 *in_base;
    const u64 *in_off, *in_len;
    u64 n;
    int32_t has_dict, has_dict_id;
    u32 dict_id;
    Info *info;
    u64 *rec_need;                  // COUNT: record slots of the unit's parsed blocks (may be null)
    const u32 *first_blk;           // FILL
    const u64 *rec_first;
    BlockCols b;
};

// One unit's framing.  COUNT fills info[unit]; FILL writes the unit's blocks into the table from first_blk[unit] on.
template <bool FILL>
__global__ void __launch_bounds__(128) lz4f_walk_kernel(WalkArgs a) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= a.n) return;
    if (FILL && (a.info[unit].kind == KIND_NONE || (a.info[unit].flags & UNPLACED))) return;
    const u64 base = a.in_off[unit];
    const u8 *p = a.in_base + base;
    const u64 L = a.in_len[unit];
    Info r;
    r.status = SWC_OK; r.kind = KIND_NONE; r.n_blocks = 0; r.flags = 0; r.max_block_size = 0;
    r.content_size = ~0ull; r.frame_start = 0; r.frame_end = 0;
    u64 rec_need = 0, blk = FILL ? a.first_blk[unit] : 0, rec_at = FILL ? a.rec_first[unit] : 0;
    bool no_dict = !a.has_dict, has_id = a.has_dict_id != 0;
    u64 pos = 0;
    u32 magic = 0;
    for (;;) {                                                          // LZ4.swift:73-91
        if (L - pos < 4) { r.status = SWC_DATA_TRUNCATED; break; }
        magic = rd32(p + pos);
        if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) {             // :148-155, then decompress(data:) without dictionary (:85)
            if (L - pos - 4 < 4) { r.status = SWC_DATA_TRUNCATED; break; }
            const u64 size = rd32(p + pos + 4);
            if (L - pos - 4 < size + 4) { r.status = SWC_DATA_TRUNCATED; break; }
            pos += 8 + size;
            no_dict = true; has_id = false;
            r.flags |= SWC_LZ4F_DICTIONARY_DROPPED;
            continue;
        }
        if (magic != 0x184D2204u && magic != 0x184C2102u) r.status = SWC_DATA_CORRUPTED;
        break;
    }
    r.frame_start = pos;
    auto block = [&](u64 at, u64 size, bool stored, bool parsed, bool has_ck) {
        if (FILL) {
            a.b.off[blk] = base + at;
            a.b.len[blk] = size | (stored ? STORED : 0);
            a.b.par_len[blk] = parsed ? size | (stored ? STORED : 0) : 0;
            a.b.ck_len[blk] = has_ck ? size : 0;
            a.b.stored_ck[blk] = has_ck ? rd32(p + at + size) : 0;
            a.b.no_dict[blk] = no_dict;
            a.b.cap[blk] = ~0ull;
            a.b.rec_base[blk] = rec_at;
        }
        const u64 slots = parsed && !stored ? size / 3 + 2 : 0;
        blk++; rec_at += slots; rec_need += slots;
        r.n_blocks++;
    };
    if (r.status == SWC_OK && magic == 0x184C2102u) {                   // process(legacyFrame:) :160-186
        r.kind = KIND_LEGACY;
        no_dict = true;
        u64 off = pos + 4;
        while (off < L) {
            if (L - off < 4) { r.status = SWC_DATA_TRUNCATED; break; }
            const u32 raw = rd32(p + off);
            if (is_magic(raw)) break;
            off += 4;
            if (L - off < raw) { r.status = SWC_DATA_TRUNCATED; break; }
            block(off, raw, false, true, false);
            off += raw;
        }
        if (r.status == SWC_OK) r.frame_end = off;
    } else if (r.status == SWC_OK) do {                                 // process(frame:) :188-330
        const u8 *in = p + pos + 4;
        const u64 n = L - pos - 4;
        if (n < 7) { r.status = SWC_DATA_TRUNCATED; break; }
        const u32 flg = in[0];
        if (!(((flg & 0xC0) >> 6) == 1 && (flg & 0x2) == 0)) { r.status = SWC_DATA_CORRUPTED; break; }
        const u32 bd = in[1];
        if (bd != 0x40 && bd != 0x50 && bd != 0x60 && bd != 0x70) { r.status = SWC_DATA_CORRUPTED; break; }
        const u64 max_block = 64u << (10 + 2 * ((bd >> 4) - 4));
        u64 off = 2;
        u64 content_size = ~0ull;
        if (flg & FLG_CONTENT_SIZE) {
            if (n - off < 13) { r.status = SWC_DATA_TRUNCATED; break; }
            content_size = (u64)rd32(in + off) | (u64)rd32(in + off + 4) << 32;
            off += 8;
            if (content_size > (u64)INT64_MAX) { r.status = SWC_DATA_UNSUPPORTED_FEATURE; break; }
        }
        if (flg & FLG_DICT_ID) {
            if (no_dict) { r.status = SWC_DATA_CORRUPTED; break; }
            if (n - off < 9) { r.status = SWC_DATA_TRUNCATED; break; }
            const u32 id = rd32(in + off);
            off += 4;
            if (has_id && id != a.dict_id) { r.status = SWC_DATA_CORRUPTED; break; }
        }
        if (((xxh32_descriptor(in, (u32)off) >> 8) & 0xFF) != in[off]) { r.status = SWC_DATA_CORRUPTED; break; }
        off++;
        // from here on the frame has blocks to decode: an error below stands behind the blocks before it
        const bool independent = (flg & FLG_INDEPENDENT) != 0, block_ck = (flg & FLG_BLOCK_CK) != 0;
        r.kind = independent ? KIND_INDEPENDENT : KIND_DEPENDENT;
        r.flags |= flg;
        r.max_block_size = (u32)max_block;
        r.content_size = content_size;
        for (;;) {                                                      // :278-318, framing only
            if (n - off < 4) { r.status = SWC_DATA_TRUNCATED; break; }
            const u32 mark = rd32(in + off);
            off += 4;
            if (mark == 0) {
                if (flg & FLG_CONTENT_CK) {                             // :323-328; reported behind the content size check
                    if (n - off < 4) { r.status = SWC_DATA_TRUNCATED; r.flags |= SWC_LZ4F_CHECKSUM_CUT; break; }
                    off += 4;
                }
                r.frame_end = pos + 4 + off;
                break;
            }
            const u64 size = mark & 0x7FFFFFFFu;
            if (size > max_block) { r.status = SWC_DATA_CORRUPTED; break; }
            if (n - off < size + (block_ck ? 4 : 0) + 4) { r.status = SWC_DATA_TRUNCATED; break; }
            block(pos + 4 + off, size, (mark >> 31) != 0, independent, block_ck);
            off += size + (block_ck ? 4 : 0);
        }
    } while (0);
    if (!FILL) {
        a.info[unit] = r;
        if (a.rec_need) a.rec_need[unit] = rec_need;
    }
}

// the per-unit columns the stages hand to each other
struct UnitCols {
    Info *info;
    u64 *rec_need, *rec_first;
    u32 *first_blk, *n_chain;      // n_chain: the unit's blocks if it is a placed dependent frame, else 0
    u8 *no_dict;
    u64 *chain_len;                // the chain decoder's out_len / status
    int32_t *chain_status;
    u64 *cc_len;                   // decoded bytes to hash for the content checksum (0: none)
    u32 *cc;
    u64 *totals;                   // [0] blocks, [1] record slots of the whole batch
};

// exclusive sums of the units' block counts and record slots, one CTA; marks the units that do not fit
__global__ void __launch_bounds__(1024) lz4f_place_kernel(UnitCols c, u64 n, u64 max_blocks, u64 rec_cap) {
    __shared__ u64 part[2][1024];
    u64 b, e;
    cta_unit_run(n, b, e);
    u64 sb = 0, sr = 0;
    for (u64 i = b; i < e; i++) { sb += c.info[i].n_blocks; sr += c.rec_need[i]; }
    part[0][threadIdx.x] = sb; part[1][threadIdx.x] = sr;
    cta_scan<2>(part);
    if (threadIdx.x == 1023) { c.totals[0] = part[0][1023]; c.totals[1] = part[1][1023]; }
    u64 rb = part[0][threadIdx.x] - sb, rr = part[1][threadIdx.x] - sr;
    for (u64 i = b; i < e; i++) {
        Info &f = c.info[i];
        const u64 nb = f.n_blocks, need = c.rec_need[i];
        const bool fits = nb == 0 || (rb + nb <= max_blocks && rr + need <= rec_cap);
        f.flags = fits ? f.flags & ~UNPLACED : f.flags | UNPLACED;
        c.first_blk[i] = fits ? (u32)rb : 0;
        c.rec_first[i] = rr;
        c.n_chain[i] = fits && f.kind == KIND_DEPENDENT ? (u32)nb : 0;
        c.no_dict[i] = (f.flags & SWC_LZ4F_DICTIONARY_DROPPED) != 0;
        rb += nb; rr += need;
    }
}

// One warp per unit: the first failure the reference's sequential loop would meet, and the unit's results.
__global__ void __launch_bounds__(256) lz4f_resolve_kernel(UnitIO io, u64 *consumed, UnitCols c, BlockCols b) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= io.n) return;
    const u32 lane = lane_id();
    const Info f = c.info[unit];
    const u64 nb = f.n_blocks, b0 = c.first_blk[unit], cap = io.out_cap[unit];
    const bool block_ck = f.kind != KIND_LEGACY && (f.flags & FLG_BLOCK_CK);
    int status = SWC_OK;
    u64 total = 0;
    if (f.kind == KIND_NONE) status = f.status;
    else if (f.flags & UNPLACED) status = SWC_ERR_UNSUPPORTED;
    else {
        // block k: its checksum (:300), then its decode (:305-313); the chain decoder reports the one block it failed at
        const int cs = f.kind == KIND_DEPENDENT ? c.chain_status[unit] : SWC_OK;
        const bool chain_failed = cs != SWC_OK && cs != SWC_ERR_OUTPUT_OVERFLOW;
        const u64 chain_fail = chain_failed ? c.chain_len[unit] : nb;
        const u64 out0 = io.out_off[unit];
        for (u64 g = 0; g < nb && status == SWC_OK; g += 32) {
            const u64 k = g + lane;
            int fail = SWC_OK;
            u64 size = 0;
            if (k < nb) {
                if (block_ck && b.ck[b0 + k] != b.stored_ck[b0 + k]) fail = SWC_DATA_CORRUPTED;
                else if (f.kind == KIND_DEPENDENT) fail = k == chain_fail ? cs : SWC_OK;
                else {
                    const int s = b.status[b0 + k];
                    if (s != SWC_OK && s != lz4::LZ4_INTERNAL_FALLBACK) fail = s;
                    size = b.out_len[b0 + k];
                }
                if (f.kind == KIND_DEPENDENT && k > chain_fail) fail = SWC_OK;      // the reference never got there
            }
            const u32 m = __ballot_sync(SWC_FULL, fail != SWC_OK);
            if (m) { status = __shfl_sync(SWC_FULL, fail, __ffs(m) - 1); break; }
            if (f.kind != KIND_DEPENDENT) {                                          // where each block of the frame goes
                u64 incl = size;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const u64 v = __shfl_up_sync(SWC_FULL, incl, d);
                    if (lane >= (u32)d) incl += v;
                }
                if (k < nb) { b.out_off[b0 + k] = out0 + total + incl - size; b.cap[b0 + k] = size; }
                total += __shfl_sync(SWC_FULL, incl, 31);
            }
        }
        if (f.kind == KIND_DEPENDENT) total = chain_failed ? 0 : c.chain_len[unit];
        const bool cut_checksum = (f.flags & SWC_LZ4F_CHECKSUM_CUT) != 0;
        if (status == SWC_OK && f.status != SWC_OK && !cut_checksum) status = f.status;               // the framing error behind the blocks
        if (status == SWC_OK && (f.flags & FLG_CONTENT_SIZE) && f.kind != KIND_LEGACY && total != f.content_size) status = SWC_DATA_CORRUPTED;
        if (status == SWC_OK && cut_checksum) status = SWC_DATA_TRUNCATED;
        if (status == SWC_OK && total > cap) status = SWC_ERR_OUTPUT_OVERFLOW;
        if (status != SWC_OK && f.kind != KIND_DEPENDENT)                                              // nothing of this unit is stored
            for (u64 k = lane; k < nb; k += 32) b.status[b0 + k] = SWC_ERR_UNSUPPORTED;
    }
    if (lane == 0) {
        const bool has_cc = status == SWC_OK && f.kind != KIND_LEGACY && (f.flags & FLG_CONTENT_CK);
        io.status[unit] = status;
        io.out_len[unit] = status == SWC_OK || status == SWC_ERR_OUTPUT_OVERFLOW ? total : 0;
        consumed[unit] = status == SWC_OK ? f.frame_end : 0;
        c.cc_len[unit] = has_cc ? total : 0;
    }
}

// content checksum (:323-328): the word behind the EndMark against the hash of the unit's decoded bytes
__global__ void __launch_bounds__(128) lz4f_content_check_kernel(UnitIO io, UnitCols c) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= io.n) return;
    const Info f = c.info[unit];
    if (io.status[unit] != SWC_OK || f.kind == KIND_NONE || f.kind == KIND_LEGACY || !(f.flags & FLG_CONTENT_CK)) return;
    if (rd32(io.in_base + io.in_off[unit] + f.frame_end - 4) != c.cc[unit]) io.status[unit] = SWC_DATA_CHECKSUM_MISMATCH;
}

// ---- scratch layout: the unit columns, then the block columns, then the records ---------------------------------------
struct Layout {
    UnitCols u;
    BlockCols b;
    u64 *recs;
    size_t unit_bytes, fixed_bytes;      // up to the block columns / up to the records
    u8 *block_part;

    Layout(void *base, u64 n, u64 nblk) {
        Carver c(base);
        c.cols(n, u.info, u.rec_need, u.rec_first, u.first_blk, u.n_chain, u.no_dict, u.chain_len, u.chain_status, u.cc_len, u.cc);
        c.cols(2, u.totals);
        unit_bytes = c.at;
        block_part = c.end();
        c.cols(nblk, b.off, b.len, b.par_len, b.ck_len, b.stored_ck, b.ck, b.no_dict, b.out_off, b.cap, b.out_len, b.rec_base,
               b.status, b.rec_count);
        fixed_bytes = c.at;
        recs = (u64 *)c.end();
    }
};

size_t scratch_bytes_for(u64 n, u64 nblk, u64 rec_slots) { return Layout(nullptr, n, nblk).fixed_bytes + rec_slots * 8; }
// record slots of blocks that hold in_bytes_total bytes between them
u64 rec_slots_for(u64 in_bytes_total, u64 nblk) { return in_bytes_total / 3 + 2 * nblk; }

struct Call {
    UnitIO io;
    u64 *consumed;
    const u8 *dict;
    u64 dict_len;
    int32_t has_dict_id;
    u32 dict_id;
    cudaStream_t s;
};

int count_and_place(const Call &q, const Layout &l, u64 max_blocks, u64 rec_cap) {
    WalkArgs w{q.io.in_base, q.io.in_off, q.io.in_len, q.io.n, q.dict != nullptr, q.has_dict_id, q.dict_id, l.u.info, l.u.rec_need,
               nullptr, nullptr, BlockCols{}};
    lz4f_walk_kernel<false><<<(unsigned)((q.io.n + 127) / 128), 128, 0, q.s>>>(w);
    lz4f_place_kernel<<<1, 1024, 0, q.s>>>(l.u, q.io.n, max_blocks, rec_cap);
    count_launch(2);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// `counted`: the unit columns of `l` already hold this batch's count and placement
int decode(const Call &q, const Layout &l, u64 nblk, u64 rec_cap, bool counted) {
    const u64 n = q.io.n;
    const unsigned unit_warps = (unsigned)((n * 32 + 255) / 256);
    int st;
    timing_mark(q.s);
    if (!counted && (st = count_and_place(q, l, nblk, rec_cap))) return st;
    // idle table entries are empty blocks that every stage passes over
    SWC_CUDA_TRY(cudaMemsetAsync(l.block_part, 0, l.fixed_bytes - l.unit_bytes, q.s));
    WalkArgs w{q.io.in_base, q.io.in_off, q.io.in_len, n, q.dict != nullptr, q.has_dict_id, q.dict_id, l.u.info, nullptr,
               l.u.first_blk, l.u.rec_first, l.b};
    lz4f_walk_kernel<true><<<(unsigned)((n + 127) / 128), 128, 0, q.s>>>(w);
    count_launch();
    timing_mark(q.s);
    // independent and legacy blocks: one unit per block, no capacity fence
    lz4::Args blocks{{q.io.in_base, l.b.off, l.b.par_len, q.io.out_base, l.b.out_off, l.b.cap, l.b.out_len, l.b.status, nblk},
                     nullptr, nullptr, q.dict, q.dict ? q.dict_len : 0, nullptr, l.b.no_dict};
    if ((st = lz4::launch_parse(blocks, l.b.rec_base, l.recs, l.b.rec_count, q.s))) return st;
    timing_mark(q.s);
    if ((st = checks::xxh32_batch(q.io.in_base, l.b.off, l.b.ck_len, l.b.ck, nblk, q.s))) return st;
    timing_mark(q.s);
    // dependent frames: one warp per unit over its chain, the dictionary cut to its last 64 KiB (:309)
    lz4::Args chain{{q.io.in_base, l.b.off, l.b.len, q.io.out_base, q.io.out_off, q.io.out_cap, l.u.chain_len, l.u.chain_status, n},
                    l.u.first_blk, l.u.n_chain, q.dict, q.dict ? q.dict_len : 0, nullptr, l.u.no_dict};
    if (chain.dict_len > 65536) { chain.dict += chain.dict_len - 65536; chain.dict_len = 65536; }
    if ((st = lz4::launch(chain, q.s))) return st;
    timing_mark(q.s);
    lz4f_resolve_kernel<<<unit_warps, 256, 0, q.s>>>(q.io, q.consumed, l.u, l.b);
    count_launch();
    timing_mark(q.s);
    if ((st = lz4::launch_exec(blocks, l.b.rec_base, l.recs, l.b.rec_count, q.s))) return st;
    timing_mark(q.s);
    if ((st = checks::xxh32_batch(q.io.out_base, q.io.out_off, l.u.cc_len, l.u.cc, n, q.s))) return st;
    lz4f_content_check_kernel<<<(unsigned)((n + 127) / 128), 128, 0, q.s>>>(q.io, l.u);
    count_launch();
    timing_mark(q.s);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

size_t swc_lz4_frame_batch_scratch_bytes(uint64_t n, uint64_t in_bytes_total, uint64_t max_blocks) {
    return scratch_bytes_for(n, max_blocks, rec_slots_for(in_bytes_total, max_blocks));
}

int32_t swc_lz4_frame_info_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                 int32_t has_dict, int32_t has_dict_id, uint32_t dict_id,
                                 swc_lz4_frame_info *info, uint64_t n, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    if (!in_base || !in_off || !in_len || !info) return SWC_ERR_INVALID_ARG;
    WalkArgs w{in_base, in_off, in_len, n, has_dict, has_dict_id, dict_id, info, nullptr, nullptr, nullptr, BlockCols{}};
    lz4f_walk_kernel<false><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)cuda_stream>>>(w);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

int32_t swc_lz4_frame_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                       const uint8_t *dict, uint64_t dict_len, int32_t has_dict_id, uint32_t dict_id,
                                       uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                       uint64_t n, uint64_t max_blocks,
                                       void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    const Call q{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bytes, dict, dict_len,
                 has_dict_id, dict_id, (cudaStream_t)cuda_stream};
    if (missing(q.io) || !consumed_bytes || max_blocks > 0xFFFFFFFFull) return SWC_ERR_INVALID_ARG;
    int st;
    u64 nblk = max_blocks, rec_cap = 0;
    SplitScratch sc(scratch, q.s);
    if (max_blocks == 0) {
        // the library counts first: the walk on the unit columns alone, then the totals back
        auto launch = [&](void *base, const u64 **t) {
            const Layout l(base, n, 0);
            *t = l.u.totals;
            return count_and_place(q, l, ~0ull, ~0ull);
        };
        u64 totals[2];
        if ((st = sc.count_first(scratch_bytes, Layout(nullptr, n, 0).unit_bytes, 2, totals, launch))) return st;
        if (totals[0] > 0xFFFFFFFFull) return SWC_ERR_UNSUPPORTED;
        nblk = totals[0] ? totals[0] : 1;
        rec_cap = totals[1];
        if (scratch && scratch_bytes < scratch_bytes_for(n, nblk, rec_cap)) return SWC_ERR_INVALID_ARG;
    } else if (scratch) {
        const size_t fixed = scratch_bytes_for(n, nblk, 0);
        if (scratch_bytes < fixed) return SWC_ERR_INVALID_ARG;
        rec_cap = (scratch_bytes - fixed) / 8;
    } else {
        // no caller scratch to size the record area from: the units' lengths are read back (one synchronisation)
        std::vector<u64> lens;
        if ((st = read_lens(in_len, n, q.s, lens))) return st;
        u64 total = 0;
        for (u64 i = 0; i < n; i++) total += lens[i];
        rec_cap = rec_slots_for(total, nblk);
    }
    if ((st = sc.seat(scratch_bytes_for(n, nblk, rec_cap)))) return st;
    return decode(q, Layout(sc.p, n, nblk), nblk, rec_cap, sc.counted);
}

}  // extern "C"
