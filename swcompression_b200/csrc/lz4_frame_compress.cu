// lz4_frame_compress.cu — batched LZ4.compress(data:independentBlocks:blockChecksums:contentChecksum:contentSize:blockSize:
// dictionary:dictionaryID:) (reference Sources/LZ4/LZ4+Compress.swift:47-154) on device-resident units: the frame layer runs
// on the device around the block compressor of lz4_compress.cu.  A dependent block's dictionary is the previous block's
// input (:106-110), so every block of every frame is parsed at once.  With a caller scratch and max_blocks > 0 the call is
// a fixed sequence of launches: no host read, no allocation (DESIGN.md §4.15).
//
//   place        one CTA          first_blk = exclusive sum of the units' block counts; units past the table are unsupported
//   fill         thread per entry the block table: input, dictionary window; idle entries get a window the parse rejects
//   per slice of whole blocks:
//     chain, parse                lz4c: every block's exact compressed size and trap status, no capacity fence
//     layout     warp per unit    stored rule, block marks, payload offsets, the unit's running frame position, capacity
//     emit                        lz4c: payloads at their frame offsets, stored blocks raw
//   xxh32        warp per block   block checksums over the stored bytes in the output
//   xxh32        warp per unit    content checksum over the input
//   finish       warp per unit    header, checksum words, EndMark, content checksum; out_len and status
#include <vector>
#include "../../include/swcgpu.h"
#include "compress_host.h"
#include "lz4_compress.cuh"
#include "lz4_frame.cuh"

namespace swc {
namespace {

using namespace lz4f;

// one frame batch: the caller's unit table and the options, dictionary and dictionary ID the whole batch shares
struct FrameArgs : UnitIO {
    u64 bs;                        // block size
    u32 flg, bd, hdr;              // FLG and BD bytes; header length, magic to HC
    u32 dict_id;
    const u8 *dict;                // device, null: no dictionary
    u64 dict_len;
};

struct UnitCols {
    u64 *first_blk, *nb;           // the unit's entries in the block table (nb = 0: none, or not placed)
    u64 *pos;                      // frame bytes laid out so far: the header, then each block's mark, payload, checksum
    int32_t *st;                   // SWC_OK, SWC_ERR_UNSUPPORTED (not placed) or the first failing block's trap
    u64 *cc_len;                   // bytes to hash for the content checksum (0: none)
    u32 *cc;
};

struct BlockCols {
    u64 *in_off, *in_len, *dict_off, *dict_len;    // the block and its dictionary window (lz4c::Args)
    u64 *cap, *res_len, *out_off, *ck_len, *scr_off;
    int32_t *status;               // parse: trap or OK; layout: anything but OK switches the block's emit off
    u8 *stored;
    u32 *ck;
};

__device__ __forceinline__ void put32(u8 *p, u32 v) { p[0] = (u8)v; p[1] = (u8)(v >> 8); p[2] = (u8)(v >> 16); p[3] = (u8)(v >> 24); }
__host__ __device__ __forceinline__ u64 blocks_of(u64 len, u64 bs) { return len / bs + (len % bs != 0); }

__global__ void __launch_bounds__(1024) lz4fc_place_kernel(FrameArgs f, UnitCols c, u64 max_blocks) {
    __shared__ u64 part[1][1024];
    u64 b, e;
    cta_unit_run(f.n, b, e);
    u64 sum = 0;
    for (u64 i = b; i < e; i++) sum += blocks_of(f.in_len[i], f.bs);
    part[0][threadIdx.x] = sum;
    cta_scan<1>(part);
    u64 at = part[0][threadIdx.x] - sum;
    for (u64 i = b; i < e; i++) {
        const u64 len = f.in_len[i], nb = blocks_of(len, f.bs);
        const bool fits = nb <= (at < max_blocks ? max_blocks - at : 0);
        c.first_blk[i] = at;
        c.nb[i] = fits ? nb : 0;
        c.st[i] = fits ? SWC_OK : SWC_ERR_UNSUPPORTED;
        c.pos[i] = f.hdr;
        c.cc_len[i] = fits && (f.flg & FLG_CONTENT_CK) ? len : 0;
        at += nb;
    }
}

// Entry j of the table is block j - first_blk[u] of the last unit u with first_blk[u] <= j, or idle.  `scr_head` and
// `scr_need` place each slice's blocks in the scratch behind the columns.
__global__ void __launch_bounds__(256) lz4fc_fill_kernel(FrameArgs f, UnitCols c, BlockCols b, u64 nblk, u64 scr_head, u64 scr_need) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nblk) return;
    b.scr_off[j] = scr_head + j * scr_need;
    b.cap[j] = ~0ull;
    b.out_off[j] = 0; b.ck_len[j] = 0; b.stored[j] = 0;
    u64 lo = 0, hi = f.n;
    while (lo < hi) {
        const u64 mid = (lo + hi) / 2;
        if (c.first_blk[mid] <= j) lo = mid + 1; else hi = mid;
    }
    if (lo == 0 || j - c.first_blk[lo - 1] >= c.nb[lo - 1]) {
        // idle: a 1-byte window is the parse's trap (:283), so chain, parse and emit pass over the entry
        b.in_off[j] = 0; b.in_len[j] = 0; b.dict_off[j] = lz4c::USER_DICT; b.dict_len[j] = 1;
        return;
    }
    const u64 u = lo - 1, k = j - c.first_blk[u], start = k * f.bs, len = f.in_len[u];
    const u64 at = f.in_off[u] + start;
    b.in_off[j] = at;
    b.in_len[j] = len - start < f.bs ? len - start : f.bs;
    if ((f.flg & FLG_INDEPENDENT) || k == 0) {                                     // :105
        b.dict_off[j] = lz4c::USER_DICT; b.dict_len[j] = f.dict_len;
    } else {                                                                       // :106-110
        const u64 w = f.bs < lz4c::MAX_DICT ? f.bs : lz4c::MAX_DICT;
        b.dict_off[j] = at - w; b.dict_len[j] = w;
    }
}

// One warp per unit over its blocks in the slice [first, first + count), 32 at a time: the stored rule, each block's mark
// and payload offset, and the unit's running frame position, which carries over to the next slice.  A block whose end
// passes out_cap is not written; a failing block switches the rest of its unit off.
__global__ void __launch_bounds__(256) lz4fc_layout_kernel(FrameArgs f, UnitCols c, BlockCols b, u64 first, u64 count) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= f.n) return;
    const u32 lane = lane_id();
    const u64 b0 = c.first_blk[unit], e0 = b0 + c.nb[unit];
    const u64 lo = b0 > first ? b0 : first, hi = e0 < first + count ? e0 : first + count;
    if (lo >= hi) return;
    int st = c.st[unit];
    u64 pos = c.pos[unit];
    const u64 cap = f.out_cap[unit], out0 = f.out_off[unit];
    const u32 ck = f.flg & FLG_BLOCK_CK ? 4u : 0u;
    for (u64 g = lo; g < hi; g += 32) {
        const u64 j = g + lane;
        const bool have = j < hi;
        const int bst = have ? b.status[j] : SWC_OK;
        const u32 m = __ballot_sync(SWC_FULL, bst != SWC_OK);
        if (st == SWC_OK && m) st = __shfl_sync(SWC_FULL, bst, __ffs(m) - 1);
        if (st != SWC_OK) {                                                        // nothing more of this unit is written
            if (have) b.status[j] = SWC_ERR_UNSUPPORTED;
            continue;
        }
        const u64 len = have ? b.in_len[j] : 0, res = have ? b.res_len[j] : 0;
        const bool stored = res > len;                                             // :112
        const u64 pay = stored ? len : res, enc = have ? 4 + pay + ck : 0;
        u64 incl = enc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u64 v = __shfl_up_sync(SWC_FULL, incl, d);
            if (lane >= (u32)d) incl += v;
        }
        if (have) {
            const u64 at = pos + incl - enc;                                       // the block's mark in the frame
            const bool fits = at + enc <= cap;
            b.stored[j] = stored;
            b.out_off[j] = out0 + at + 4;
            b.ck_len[j] = fits ? (ck ? pay : 0) : 0;
            if (fits) put32(f.out_base + out0 + at, (stored ? 0x80000000u : 0u) | (u32)pay);    // :113-118
            else b.status[j] = SWC_ERR_OUTPUT_OVERFLOW;
        }
        pos += __shfl_sync(SWC_FULL, incl, 31);
    }
    if (lane == 0) { c.pos[unit] = pos; c.st[unit] = st; }
}

// One warp per unit: the header (:54-93), the block checksum words (:120-125, :133-138), the EndMark and the content
// checksum (:143-151) of every unit whose whole frame fits; out_len and status of every unit.
__global__ void __launch_bounds__(256) lz4fc_finish_kernel(FrameArgs f, UnitCols c, BlockCols b) {
    const u64 unit = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (unit >= f.n) return;
    const u32 lane = lane_id();
    int st = c.st[unit];
    const u64 end = c.pos[unit], total = end + 4 + (f.flg & FLG_CONTENT_CK ? 4 : 0);
    if (st == SWC_OK && total > f.out_cap[unit]) st = SWC_ERR_OUTPUT_OVERFLOW;
    if (st == SWC_OK) {
        u8 *out = f.out_base + f.out_off[unit];
        if (f.flg & FLG_BLOCK_CK)
            for (u64 j = c.first_blk[unit] + lane; j < c.first_blk[unit] + c.nb[unit]; j += 32) put32(f.out_base + b.out_off[j] + b.ck_len[j], b.ck[j]);
        if (lane == 0) {
            put32(out, 0x184D2204u);
            out[4] = (u8)f.flg; out[5] = (u8)f.bd;
            u32 h = 6;
            if (f.flg & FLG_CONTENT_SIZE) { const u64 v = f.in_len[unit]; put32(out + h, (u32)v); put32(out + h + 4, (u32)(v >> 32)); h += 8; }
            if (f.flg & FLG_DICT_ID) { put32(out + h, f.dict_id); h += 4; }
            out[h] = (u8)(xxh32_descriptor(out + 4, h - 4) >> 8);
            put32(out + end, 0);
            if (f.flg & FLG_CONTENT_CK) put32(out + end + 4, c.cc[unit]);
        }
    }
    if (lane == 0) {
        f.status[unit] = st;
        f.out_len[unit] = st == SWC_OK || st == SWC_ERR_OUTPUT_OVERFLOW ? total : 0;
    }
}

// ---- scratch: the unit columns, the block columns, then each slice's blocks ------------------------------------------
struct Layout {
    UnitCols u;
    BlockCols b;
    size_t bytes = 0;              // the columns

    Layout(void *base, u64 n, u64 nblk) {
        Carver c(base);
        c.cols(n, u.first_blk, u.nb, u.pos, u.st, u.cc_len, u.cc);
        c.cols(nblk, b.in_off, b.in_len, b.dict_off, b.dict_len, b.cap, b.res_len, b.out_off, b.ck_len, b.scr_off, b.status,
               b.stored, b.ck);
        bytes = c.at;
    }
};

bool valid_block_size(int64_t bs) { return bs >= 1 && bs <= (int64_t)lz4c::MAX_BLOCK; }

// the scratch of one block: its window is the block and the largest dictionary window a block of the batch can have
u64 block_need(u64 bs, bool independent, u64 dict_len) {
    u64 w = dict_len < lz4c::MAX_DICT ? dict_len : lz4c::MAX_DICT;
    if (!independent && w < (bs < lz4c::MAX_DICT ? bs : lz4c::MAX_DICT)) w = bs < lz4c::MAX_DICT ? bs : lz4c::MAX_DICT;
    return lz4c::unit_scratch(bs + w, bs);
}

FrameArgs frame_args(int32_t independent, int32_t block_ck, int32_t content_ck, int32_t content_size, int64_t block_size,
                     const u8 *dict, u64 dict_len, int32_t has_dict_id, u32 dict_id) {
    FrameArgs f{};
    f.bs = (u64)block_size;
    f.flg = 0x40 | (independent ? FLG_INDEPENDENT : 0) | (block_ck ? FLG_BLOCK_CK : 0) | (content_size ? FLG_CONTENT_SIZE : 0) |
            (content_ck ? FLG_CONTENT_CK : 0) | (has_dict_id ? FLG_DICT_ID : 0);                      // :57-81
    f.bd = f.bs <= (64u << 10) ? 0x40 : f.bs <= (256u << 10) ? 0x50 : f.bs <= (1u << 20) ? 0x60 : 0x70;   // :83-90
    f.hdr = 7 + (content_size ? 8 : 0) + (has_dict_id ? 4 : 0);
    f.dict_id = dict_id;
    f.dict = dict;
    f.dict_len = dict ? dict_len : 0;
    return f;
}

// the batch with a block table of `nblk` entries
int frame_batch(const FrameArgs &f, u64 nblk, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    const u64 n = f.n, head = Layout(nullptr, n, nblk).bytes;
    const u64 need = block_need(f.bs, (f.flg & FLG_INDEPENDENT) != 0, f.dict_len);
    const unsigned unit_warps = (unsigned)((n * 32 + 255) / 256);
    Layout l(nullptr, 0, 0);
    int st = run_in_slices(nblk, [&](u64) { return need; }, [&](u64) { return head; }, scratch, scratch_bytes, s,
                           [&](u64 first, u64 count, u8 *scr, size_t) -> int {
        if (first == 0) {                                           // the columns sit at the front of every slice's scratch
            timing_mark(s);
            l = Layout(scr, n, nblk);
            lz4fc_place_kernel<<<1, 1024, 0, s>>>(f, l.u, nblk);
            lz4fc_fill_kernel<<<(unsigned)((nblk + 255) / 256), 256, 0, s>>>(f, l.u, l.b, nblk, head, need);
            count_launch(2);
        }
        const lz4c::Args a{{f.in_base, l.b.in_off, l.b.in_len, f.out_base, l.b.out_off, l.b.cap, l.b.res_len, l.b.status, nblk},
                           l.b.dict_off, l.b.dict_len, l.b.stored, f.dict};
        int st = lz4c::parse(a, first, count, scr, l.b.scr_off, s);
        if (st) return st;
        lz4fc_layout_kernel<<<unit_warps, 256, 0, s>>>(f, l.u, l.b, first, count);
        count_launch();
        timing_mark(s);
        return lz4c::emit(a, first, count, scr, l.b.scr_off, s);
    });
    if (st) return st;
    if ((st = checks::xxh32_batch(f.out_base, l.b.out_off, l.b.ck_len, l.b.ck, nblk, s))) return st;
    timing_mark(s);
    if ((st = checks::xxh32_batch(f.in_base, f.in_off, l.u.cc_len, l.u.cc, n, s))) return st;
    timing_mark(s);
    lz4fc_finish_kernel<<<unit_warps, 256, 0, s>>>(f, l.u, l.b);
    count_launch();
    timing_mark(s);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// the single call's batch: one unit whose length the host knows
int one_frame(const FrameArgs &f, const std::vector<u64> &lens, void *scratch, size_t scratch_bytes, cudaStream_t s) {
    const u64 nb = blocks_of(lens[0], f.bs);
    return frame_batch(f, nb ? nb : 1, scratch, scratch_bytes, s);
}

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

size_t swc_lz4_frame_compress_max_bytes(uint64_t in_len, int64_t block_size, int32_t block_checksums, int32_t content_checksum,
                                        int32_t content_size, int32_t has_dict_id) {
    if (!valid_block_size(block_size)) return 0;
    const u64 nb = blocks_of(in_len, (u64)block_size);
    return (size_t)(7 + (content_size ? 8 : 0) + (has_dict_id ? 4 : 0) + in_len + nb * (block_checksums ? 8 : 4) + 4 +
                    (content_checksum ? 4 : 0));
}

size_t swc_lz4_frame_compress_batch_scratch_bytes(uint64_t n, uint64_t max_blocks, int64_t block_size,
                                                  int32_t independent_blocks, uint64_t dict_len) {
    if (!valid_block_size(block_size)) return 0;
    return (size_t)(Layout(nullptr, n, max_blocks).bytes + max_blocks * block_need((u64)block_size, independent_blocks != 0, dict_len));
}

int32_t swc_lz4_frame_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     int32_t independent_blocks, int32_t block_checksums, int32_t content_checksum,
                                     int32_t content_size, int64_t block_size, const uint8_t *dict, uint64_t dict_len,
                                     int32_t has_dict_id, uint32_t dict_id,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t *out_len, int32_t *status, uint64_t n, uint64_t max_blocks,
                                     void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (!valid_block_size(block_size)) return SWC_ERR_REFERENCE_TRAP;                                    // :51
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    FrameArgs f = frame_args(independent_blocks, block_checksums, content_checksum, content_size, block_size, dict, dict_len,
                             has_dict_id, dict_id);
    static_cast<UnitIO &>(f) = UnitIO{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n};
    if (missing(f) || max_blocks > 0xFFFFFFFFull) return SWC_ERR_INVALID_ARG;
    const cudaStream_t s = (cudaStream_t)cuda_stream;
    u64 nblk = max_blocks;
    if (nblk == 0) {                    // the library counts the blocks: the lengths come back (one synchronisation)
        std::vector<u64> lens;
        int st = read_lens(in_len, n, s, lens);
        if (st) return st;
        for (u64 i = 0; i < n; i++) nblk += blocks_of(lens[i], f.bs);
        if (nblk > 0xFFFFFFFFull) return SWC_ERR_UNSUPPORTED;
        if (nblk == 0) nblk = 1;
    }
    return frame_batch(f, nblk, scratch, scratch_bytes, s);
}

// LZ4.compress(data:independentBlocks:blockChecksums:contentChecksum:contentSize:blockSize:dictionary:dictionaryID:)
// LZ4+Compress.swift:47-154: the one-unit batch on the library pool
int32_t swc_lz4_compress(const uint8_t *in, size_t in_len, int32_t independent_blocks, int32_t block_checksums,
                         int32_t content_checksum, int32_t content_size, int64_t block_size,
                         const uint8_t *dict, size_t dict_len, int32_t has_dict_id, uint32_t dict_id,
                         uint8_t **out, size_t *out_len) {
    if (!out || !out_len || (!in && in_len)) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0;
    if (!valid_block_size(block_size)) return SWC_ERR_REFERENCE_TRAP;                                    // :51
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    // only the dictionary's last 64 KiB reaches a window (:95-101); an empty one still needs a non-null pointer
    const size_t d = !dict ? 0 : dict_len > lz4c::MAX_DICT ? lz4c::MAX_DICT : dict_len;
    DevBuf d_dict;
    int st;
    if (dict) {
        if ((st = d_dict.alloc(d + 16))) return st;
        if (d) SWC_CUDA_TRY(cudaMemcpy(d_dict.p, dict + (dict_len - d), d, cudaMemcpyHostToDevice));
    }
    const FrameArgs f = frame_args(independent_blocks, block_checksums, content_checksum, content_size, block_size,
                                   d_dict.as<u8>(), d, has_dict_id, dict_id);
    return compress_one(f, one_frame, swc_lz4_frame_compress_max_bytes(in_len, block_size, block_checksums, content_checksum,
                                                                       content_size, has_dict_id),
                        in, in_len, out, out_len);
}

}  // extern "C"
