// xz_batch.cu — batched XZArchive.unarchive on device-resident archives: one whole .xz file per unit, one warp per unit,
// everything enqueued on the caller's stream in one launch (no host read, no allocation, no scratch).
// Reference: Sources/XZ/XZArchive.swift:27-218, XZBlock.swift:18-97, Sources/LZMA2/LZMA2Decoder.swift:17-99,
// Sources/Common/DeltaFilter.swift:11-32, Sources/Common/CheckSums.swift, Sources/XZ/Sha256.swift.
//
// xz_kernel walks the container with the grammar of xz_framing.cuh, every lane in lock-step (uniform control flow).  Blocks
// are found only by decoding their predecessors, so an archive is serial, as in the reference; the parallelism is across
// archives, as in lzma_kernel, with the same 2 warps and 2 x 28 304 B of model per CTA (DESIGN.md §4.13).  Per block:
//   LZMA2    lzma::lzma2_decode with a fresh Dec straight into the unit's output region (a block never sees earlier blocks'
//            bytes: the reference builds a new LZMA2Decoder per block);
//   Delta    in place over the block's output, the listed Deltas last to first;
//   check    CRC-32 / CRC-64 by the warp (warp_crc) with slicing tables built in the warp's model area, which is dead once
//            the block's LZMA2 decode has finished, or SHA-256 on lane 0.
// The index is compared with the blocks by walking the stream's block headers and LZMA2 chunk headers again (no per-block
// state is kept: the sizes of a block that decoded cleanly can be read back from its headers).
#include "../../include/swcgpu.h"
#include "checks_device.cuh"
#include "host_util.h"
#include "lzma.cuh"
#include "lzma_dec.cuh"
#include "xz_framing.cuh"

namespace swc {
namespace {

using lzma::Dec;
constexpr int WARPS = lzma::WARPS;

// an LZMA2 stream at p that lzma2_decode took cleanly: its chunk headers give the bytes it read and the bytes it produced
__device__ void lzma2_skim(const u8 *p, u64 *used, u64 *produced) {
    u64 o = 0, out = 0;
    for (;;) {
        const u32 c = p[o++];
        if (c == 0) break;
        if (c == 1 || c == 2) {
            const u64 size = ((u64)p[o] << 8 | p[o + 1]) + 1;
            o += 2 + size; out += size;
            continue;
        }
        out += ((u64)(c & 0x1F) << 16 | (u64)p[o] << 8 | p[o + 1]) + 1;
        const u64 comp = ((u64)p[o + 2] << 8 | p[o + 3]) + 1;
        o += 4 + (((c & 0x60) >> 5) >= 2 ? 1 : 0) + comp;
    }
    *used = o; *produced = out;
}

// the blocks' index records, read back from the stream's blocks in order (each one parsed and decoded cleanly before)
struct BlockRecords {
    const u8 *p; size_t n, pos; int csize;
    __device__ void operator()(int64_t, int64_t *unpadded, int64_t *uncompressed) {
        xz::Rd q{p, n, pos + 1};
        xz::BlockHeader h;
        xz::block_header(q, p[pos], h);
        u64 used, produced;
        lzma2_skim(p + q.off, &used, &produced);
        const int64_t unp = (int64_t)(q.off + used - h.hstart);
        *unpadded = unp + csize;
        *uncompressed = (int64_t)produced;
        pos = h.hstart + (size_t)((unp + 3) & ~(int64_t)3) + csize;
    }
};

// DeltaFilter.swift:11-32 in place: out[j] += out[j - dist] for j >= dist.  The warp takes rows of `dist` bytes, lanes on
// columns; a column is one lane's all the way down, so rows need no barrier.
__device__ void delta_in_place(u8 *b, u64 n, u32 dist) {
    for (u64 row = dist; row < n; row += dist)
        for (u64 j = row + lane_id(); j < row + dist && j < n; j += 32) b[j] = (u8)(b[j] + b[j - dist]);
    __syncwarp();
}

// the block's check against the `stored` field; `P` is the warp's model area (free once the block has decoded)
__device__ bool check_matches(u16 *P, const u8 *blk, u64 n, int ctype, const u8 *stored) {
    __syncwarp();
    if (ctype == 1) {
        u32 (*tab)[256] = (u32 (*)[256])P;
        checks::crc_tables<checks::Crc32R>(tab, lane_id(), 32);
        __syncwarp();
        const u32 c = checks::warp_crc<checks::Crc32R>(tab, blk, n);
        __syncwarp();
        return c == xz::rd32(stored);
    }
    if (ctype == 4) {
        u64 (*tab)[256] = (u64 (*)[256])P;
        checks::crc_tables<checks::Crc64R>(tab, lane_id(), 32);
        __syncwarp();
        const u64 c = checks::warp_crc<checks::Crc64R>(tab, blk, n);
        __syncwarp();
        return c == ((u64)xz::rd32(stored) | (u64)xz::rd32(stored + 4) << 32);
    }
    int bad = 0;
    if (lane_id() == 0) {
        u8 dg[32];
        checks::sha256_buffer(blk, n, dg);
        for (int k = 0; k < 32; k++) bad |= dg[k] != stored[k];
    }
    return __shfl_sync(SWC_FULL, bad, 0) == 0;
}

// processStream XZArchive.swift:90-130 (+ processIndex, processFooter); the stream's data is appended at out + *written
__device__ int xz_stream(xz::Rd &r, u16 *P, u8 *out, u64 cap, u64 *written, bool *check_error) {
    int ctype = 0;
    int st = xz::stream_header(r, &ctype);
    if (st) return st;
    const int csize = xz::check_size(ctype);
    const size_t first_block = r.off;
    int64_t nblocks = 0, index_size = -1;
    for (;;) {
        if (!r.need(1)) return SWC_ERR_REFERENCE_TRAP;
        const unsigned hs = r.p[r.off++];
        if (hs == 0) {
            if ((st = xz::index(r, nblocks, BlockRecords{r.p, r.n, first_block, csize}, &index_size))) return st;
            break;
        }
        xz::BlockHeader h;
        if ((st = xz::block_header(r, hs, h))) return st;
        // the filter chains this kernel runs: zero to three Deltas, then LZMA2 (DESIGN.md §6)
        const int last = h.nfilters - 1;
        bool supported = h.kind[last] == xz::FILTER_LZMA2;
        for (int f = 0; f < last; f++) supported = supported && h.kind[f] == xz::FILTER_DELTA;
        if (!supported) return SWC_ERR_UNSUPPORTED;
        const size_t data_start = r.off;
        u8 *blk = out + *written;
        Dec d;
        d.start(P, blk, cap - *written);
        d.in_init(r.p + r.off, r.n - r.off);
        const u64 addr0 = d.addr;
        if ((st = lzma::lzma2_decode(d, (u32)h.param[last], nullptr))) return st;
        r.off += d.addr - addr0;
        const u64 n = (u64)d.dict_end;
        __syncwarp();
        for (int f = last - 1; f >= 0; f--) delta_in_place(blk, n, (u32)h.param[f]);
        int64_t unp = 0;
        if ((st = xz::block_tail(r, h, data_start, (int64_t)n, csize, &unp))) return st;
        const u8 *stored = nullptr;
        if ((st = xz::check_field(r, ctype, &stored))) return st;
        *written += n;
        if (ctype != 0 && !check_matches(P, blk, n, ctype, stored)) { *check_error = true; return SWC_OK; }
        nblocks++;
    }
    return xz::footer(r, ctype, index_size);
}

__global__ void __launch_bounds__(WARPS * 32) xz_kernel(UnitIO a) {
    extern __shared__ u16 smem16[];
    const u32 warp = threadIdx.x >> 5;
    const u64 unit = (u64)blockIdx.x * WARPS + warp;
    if (unit >= a.n) return;
    u16 *P = smem16 + warp * lzma::SMEM_U16;
    const u8 *in = a.in_base + a.in_off[unit];
    const u64 L = a.in_len[unit];
    u8 *out = a.out_base + a.out_off[unit];
    const u64 cap = a.out_cap[unit];
    u64 written = 0;
    bool check_error = false;
    int st = SWC_OK;
    xz::Rd r{in, L, 0};
    while (r.off < r.n) {                                                     // XZArchive.unarchive :27-50
        if (r.n - r.off < 32) { st = SWC_XZ_WRONG_MAGIC; break; }
        if ((st = xz_stream(r, P, out, cap, &written, &check_error)) || check_error) break;
        if ((st = xz::padding(r))) break;
    }
    if (check_error) st = SWC_XZ_WRONG_CHECK;
    if (lane_id() == 0) {
        a.out_len[unit] = st == SWC_OK || st == SWC_XZ_WRONG_CHECK ? written
                          : st == SWC_ERR_OUTPUT_OVERFLOW ? xz::declared_size(in, L) : 0;
        a.status[unit] = st;
    }
}

int configure() {
    return configure_once(CFG_XZ, [](DeviceCtx &) {
        SWC_CUDA_TRY(cudaFuncSetAttribute(xz_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lzma::SMEM_BYTES));
        return (int)SWC_OK;
    });
}

int xz_batch(const UnitIO &a, cudaStream_t stream) {
    if (a.n == 0) return SWC_OK;
    if (missing(a)) return SWC_ERR_INVALID_ARG;
    if (int st = configure()) return st;
    xz_kernel<<<(unsigned)((a.n + WARPS - 1) / WARPS), WARPS * 32, lzma::SMEM_BYTES, stream>>>(a);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

int32_t swc_xz_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                               uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                               uint64_t *out_len, int32_t *status, uint64_t n, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    return xz_batch(UnitIO{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, (cudaStream_t)cuda_stream);
}

int32_t swc_xz_occupancy(int32_t *lzma_warps_per_sm, int32_t *xz_warps_per_sm) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    int lb = 0, xb = 0;
    if (lzma_warps_per_sm) {
        if (int st = lzma::occupancy_blocks(&lb)) return st;
        *lzma_warps_per_sm = lb * WARPS;
    }
    if (xz_warps_per_sm) {
        if (int st = configure()) return st;
        SWC_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&xb, xz_kernel, WARPS * 32, lzma::SMEM_BYTES));
        *xz_warps_per_sm = xb * WARPS;
    }
    return SWC_OK;
}

}  // extern "C"
