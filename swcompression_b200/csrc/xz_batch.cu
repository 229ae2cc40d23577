// xz_batch.cu — batched XZArchive.unarchive on device-resident archives, one whole .xz file per unit.
// swc_xz_unarchive_batch: one warp per unit, everything enqueued on the caller's stream in one launch (no host read, no
// allocation, no scratch).  swc_xz_block_unarchive_batch: every block of every unit side by side, validated by the
// reference's walk, with xz_kernel as the fallback (the stages are listed above xzb_walk_kernel).
// Reference: Sources/XZ/XZArchive.swift:27-218, XZBlock.swift:18-97, Sources/LZMA2/LZMA2Decoder.swift:17-99,
// Sources/Common/DeltaFilter.swift:11-32, Sources/Common/CheckSums.swift, Sources/XZ/Sha256.swift.
//
// xz_kernel walks the container with the grammar of xz_framing.cuh, every lane in lock-step (uniform control flow).  Walking
// forward, blocks are found only by decoding their predecessors, so in xz_kernel an archive is serial, as in the reference
// (the block-parallel batch finds them from the indexes instead); the parallelism is across archives, as in lzma_kernel,
// with the same 2 warps and 2 x 28 304 B of model per CTA (DESIGN.md §4.13).  Per block:
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

// One block (XZBlock.swift:18-97, XZArchive.swift:105-118) of a stream with check type `ctype`, from its header-size byte
// `hs` (non-zero, read already) to the end of its check field, decoded with a fresh Dec into blk[0, cap).  xz_kernel and
// xzb_block_kernel both run this one copy, so the fresh-decoder rule, the filter rule and the order of checks are shared.
// On SWC_OK: *n is the decoded size, *unpadded the index's Unpadded Size and *check_ok whether the stored check matched.
__device__ __forceinline__ int xz_block(xz::Rd &r, unsigned hs, int ctype, u16 *P, u8 *blk, u64 cap, u64 *n,
                                        int64_t *unpadded, bool *check_ok) {
    int st;
    xz::BlockHeader h;
    if ((st = xz::block_header(r, hs, h))) return st;
    // the filter chains this kernel runs: zero to three Deltas, then LZMA2 (DESIGN.md §6)
    const int last = h.nfilters - 1;
    bool supported = h.kind[last] == xz::FILTER_LZMA2;
    for (int f = 0; f < last; f++) supported = supported && h.kind[f] == xz::FILTER_DELTA;
    if (!supported) return SWC_ERR_UNSUPPORTED;
    const size_t data_start = r.off;
    Dec d;
    d.start(P, blk, cap);
    d.in_init(r.p + r.off, r.n - r.off);
    const u64 addr0 = d.addr;
    if ((st = lzma::lzma2_decode(d, (u32)h.param[last], nullptr))) return st;
    r.off += d.addr - addr0;
    *n = (u64)d.dict_end;
    __syncwarp();
    for (int f = last - 1; f >= 0; f--) delta_in_place(blk, *n, (u32)h.param[f]);
    if ((st = xz::block_tail(r, h, data_start, (int64_t)*n, xz::check_size(ctype), unpadded))) return st;
    const u8 *stored = nullptr;
    if ((st = xz::check_field(r, ctype, &stored))) return st;
    *check_ok = ctype == 0 || check_matches(P, blk, *n, ctype, stored);
    return SWC_OK;
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
        u64 n = 0;
        int64_t unp = 0;
        bool check_ok = false;
        if ((st = xz_block(r, hs, ctype, P, out + *written, cap - *written, &n, &unp, &check_ok))) return st;
        *written += n;
        if (!check_ok) { *check_error = true; return SWC_OK; }
        nblocks++;
    }
    return xz::footer(r, ctype, index_size);
}

// `run` (per unit, or nullptr: every unit runs): 0 skips the unit, which writes nothing, not even its results.
// `parallel_blocks` (or nullptr): 0 for every unit this kernel decodes.
__global__ void __launch_bounds__(WARPS * 32) xz_kernel(UnitIO a, const u8 *run, u32 *parallel_blocks) {
    extern __shared__ u16 smem16[];
    const u32 warp = threadIdx.x >> 5;
    const u64 unit = (u64)blockIdx.x * WARPS + warp;
    if (unit >= a.n || (run && !run[unit])) return;
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
        if (parallel_blocks) parallel_blocks[unit] = 0;
    }
}

// ---- block-parallel batch (swc_xz_block_unarchive_batch, DESIGN.md §4.19) ------------------------------------------------
// The stream indexes, read backwards, give every block's start (header-size byte) and its place in the unit's output, so all
// blocks of all units decode side by side straight into their regions; the reference's forward walk then validates them.
//   walk<false>  thread per unit    backward walk to byte 0: records and declared total; the unit qualifies when the walk
//                                   covers it and the total fits out_cap
//   place        one CTA            first entry = exclusive sum of the record counts of qualifying units; placed iff its
//                                   records end inside max_blocks.  Every unit starts marked for the fallback
//   walk<true>   thread per unit    the placed units' block table from the same walk
//   order        one CTA            launch order, largest expected decoded size first
//   block        warp per entry     xz_block at the entry's start into out + its offset, capacity = its expected size
//   resolve      thread per unit    the forward walk with each block taken from the table; a unit that comes out SWC_OK is
//                                   final and unmarked
//   fallback     warp per unit      xz_kernel over the marked units
// The walks and the resolve are one thread's work: the index records are a chain of variable-length integers and the
// container grammar reads byte by byte.
constexpr u64 MAX63 = (1ull << 63) - 1;
enum : u8 { F_OK = 1, F_PLACED = 2 };

struct Units {
    u64 *count;      // index records of a qualifying unit
    u64 *total;      // its declared decoded size
    u64 *first;      // its first entry in the block table
    u8 *flags, *run; // run: 1 = xz_kernel decodes the unit
    u64 *sums;       // [0] entries of the placed units, [1] records of every qualifying unit
};

struct Table {
    u32 *unit;
    u8 *ctype;                 // check type from the stream footer
    u64 *start;                // offset of the block's header-size byte in the unit
    u64 *out_at;               // output offset in the unit's region: the sum of the Uncompressed Sizes in front of it
    u64 *size;                 // its index record's Uncompressed Size
    u32 *order;                // launch position -> entry
    int32_t *status;           // block stage results, per entry
    u64 *end, *got;            // offset behind the check field, bytes decoded
    int64_t *unpadded;
};

template <bool FILL>
__global__ void __launch_bounds__(256) xzb_walk_kernel(UnitIO io, Units u, Table t) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= io.n || (FILL && !(u.flags[unit] & F_PLACED))) return;
    const u8 *in = io.in_base + io.in_off[unit];
    size_t pos = io.in_len[unit];
    u64 recs = FILL ? u.count[unit] : 0, out = FILL ? u.total[unit] : 0;
    bool ok = true;
    while (pos > 0) {
        xz::BackStream s;
        if (!xz::back_stream(in, pos, s) || !s.uncomp_ok || (!FILL && s.uncomp > MAX63 - out)) { ok = false; break; }
        if (FILL) {
            // this stream's records are the `count` entries in front of the later streams' (the walk goes backwards)
            recs -= (u64)s.count; out -= s.uncomp;
            xz::Rd ir{in, s.foot, s.rec_off};
            u64 e = u.first[unit] + recs, at = s.start + 12, o = out;
            for (int64_t k = 0; k < s.count; k++, e++) {
                int64_t unp = 0, unc = 0;
                xz::multibyte(ir, &unp);          // the first walk read the same bytes cleanly
                xz::multibyte(ir, &unc);
                t.unit[e] = (u32)unit; t.ctype[e] = (u8)s.ctype; t.start[e] = at; t.out_at[e] = o; t.size[e] = (u64)unc;
                at += ((u64)unp + 3) & ~3ull;
                o += (u64)unc;
            }
        } else {
            recs += (u64)s.count; out += s.uncomp;
        }
        pos = s.start;
    }
    if (!FILL) {
        const bool q = ok && out <= io.out_cap[unit];
        u.count[unit] = q ? recs : 0;
        u.total[unit] = q ? out : 0;
        u.flags[unit] = q ? F_OK : 0;
    }
}

// exclusive sum of the qualifying units' record counts in unit order; a unit is placed iff its records end inside the
// table (a prefix rule).  Marks every unit for the fallback.
__global__ void __launch_bounds__(1024) xzb_place_kernel(Units u, u64 n, u64 max_blocks) {
    __shared__ u64 part[1][1024];
    u64 b, e;
    cta_unit_run(n, b, e);
    u64 s = 0;
    for (u64 i = b; i < e; i++) s += (u.flags[i] & F_OK) ? u.count[i] : 0;
    part[0][threadIdx.x] = s;
    if (threadIdx.x == 0) u.sums[0] = 0;
    cta_scan<1>(part);
    if (threadIdx.x == 1023) u.sums[1] = part[0][1023];
    u64 at = part[0][threadIdx.x] - s, used = 0;
    for (u64 i = b; i < e; i++) {
        const bool ok = (u.flags[i] & F_OK) != 0;
        const u64 nb = ok ? u.count[i] : 0;
        const bool fits = ok && at + nb <= max_blocks;
        u.flags[i] = (ok ? F_OK : 0) | (fits ? F_PLACED : 0);
        u.first[i] = at;
        u.run[i] = 1;
        if (fits && at + nb > used) used = at + nb;
        at += nb;
    }
    // the placed units' entries are a prefix of the table: past the first unit that does not fit, only empty ones fit
    atomicMax((unsigned long long *)&u.sums[0], (unsigned long long)used);
}

// One CTA: the entries in launch order, largest expected decoded size first (a counting sort on its leading zeros).  A CTA
// of the block kernel holds its 2 x 28 304 B of model until its slower warp ends, so the long blocks go first, 2 to a CTA,
// and a file's short last block fills in behind them instead of idling its partner's slot.
__global__ void __launch_bounds__(1024) xzb_order_kernel(Units u, Table t) {
    clz_order(u.sums[0], [&](u64 e) -> u32 { return __clzll((long long)t.size[e]); }, [&](u64 e, u32 at) { t.order[at] = (u32)e; });
}

// Warp per launch position: the block at the entry's start, as xz_kernel would decode it there (the input bounded by the
// unit's end), into its own part of the unit's region and no further.  Positions past the placed entries exit at once.
// __maxnreg__ rather than __launch_bounds__: under the 64-thread bound ptxas keeps this kernel to 96 registers and spills.
__global__ void __maxnreg__(128) xzb_block_kernel(UnitIO io, Units u, Table t) {
    extern __shared__ u16 smem16[];
    const u32 warp = threadIdx.x >> 5;
    const u64 k = (u64)blockIdx.x * WARPS + warp;
    if (k >= u.sums[0]) return;
    const u32 e = t.order[k], unit = t.unit[e];
    const u8 *in = io.in_base + io.in_off[unit];
    const u64 at = t.start[e];
    xz::Rd r{in, io.in_len[unit], at + 1};
    const unsigned hs = in[at];
    // the walk keeps out_at + size within the declared total, which fits out_cap; the clamp keeps the write bound local
    const u64 cap = io.out_cap[unit], o = t.out_at[e], room = o < cap ? cap - o : 0;
    u64 n = 0;
    int64_t unp = 0;
    bool check_ok = false;
    int st = hs == 0 ? SWC_XZ_WRONG_FIELD        // an index indicator: the forward walk never takes this entry
                     : xz_block(r, hs, t.ctype[e], smem16 + warp * lzma::SMEM_U16, io.out_base + io.out_off[unit] + o,
                                t.size[e] < room ? t.size[e] : room, &n, &unp, &check_ok);
    if (st == SWC_OK && !check_ok) st = SWC_XZ_WRONG_CHECK;
    if (lane_id() == 0) { t.status[e] = st; t.end[e] = r.off; t.got[e] = n; t.unpadded[e] = unp; }
}

// the index records of a stream's blocks as the block stage found them
struct TableRecords {
    const Table &t;
    u64 first;
    __device__ void operator()(int64_t k, int64_t *unpadded, int64_t *uncompressed) const {
        *unpadded = t.unpadded[first + k];
        *uncompressed = (int64_t)t.got[first + k];
    }
};

// Thread per placed unit: XZArchive.unarchive's walk (:27-50, processStream :90-130, processIndex :132-167, processFooter
// :169-192, processPadding :194-218) with each block taken from the unit's next entry: it must start at r.off, with the
// stream's check type, at the output offset the earlier blocks produced, and be SWC_OK.  A walk that ends SWC_OK over all of
// the unit's entries is xz_kernel's answer; any other outcome, a wrong check included, is left to xz_kernel.
__global__ void __launch_bounds__(256) xzb_resolve_kernel(UnitIO io, Units u, Table t, u32 *parallel_blocks) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= io.n || !(u.flags[unit] & F_PLACED)) return;
    const u64 f = u.first[unit], last = f + u.count[unit];
    xz::Rd r{io.in_base + io.in_off[unit], io.in_len[unit], 0};
    u64 e = f, written = 0;
    while (r.off < r.n) {
        int ctype = 0;
        if (r.n - r.off < 32 || xz::stream_header(r, &ctype)) return;
        const u64 first = e;
        int64_t index_size = -1;
        for (;;) {
            if (!r.need(1)) return;
            const unsigned hs = r.p[r.off++];
            if (hs == 0) {
                if (xz::index(r, (int64_t)(e - first), TableRecords{t, first}, &index_size)) return;
                break;
            }
            if (e == last || t.start[e] != r.off - 1 || t.ctype[e] != ctype || t.out_at[e] != written || t.status[e] != SWC_OK) return;
            r.off = t.end[e];
            written += t.got[e];
            e++;
        }
        if (xz::footer(r, ctype, index_size) || xz::padding(r)) return;
    }
    if (e != last) return;
    io.status[unit] = SWC_OK;
    io.out_len[unit] = written;
    if (parallel_blocks) parallel_blocks[unit] = (u32)(last - f);
    u.run[unit] = 0;
}

int configure() {
    return configure_once(CFG_XZ, [](DeviceCtx &) {
        SWC_CUDA_TRY(cudaFuncSetAttribute(xz_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lzma::SMEM_BYTES));
        SWC_CUDA_TRY(cudaFuncSetAttribute(xzb_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lzma::SMEM_BYTES));
        return (int)SWC_OK;
    });
}

int xz_batch(const UnitIO &a, cudaStream_t stream) {
    if (a.n == 0) return SWC_OK;
    if (missing(a)) return SWC_ERR_INVALID_ARG;
    if (int st = configure()) return st;
    xz_kernel<<<(unsigned)((a.n + WARPS - 1) / WARPS), WARPS * 32, lzma::SMEM_BYTES, stream>>>(a, nullptr, nullptr);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// scratch layout: the unit columns, then the block table of nblk entries
struct Layout {
    Units u;
    Table t;
    size_t unit_bytes, bytes;

    Layout(void *base, u64 n, u64 nblk) {
        Carver c(base);
        c.cols(n, u.count, u.total, u.first, u.flags, u.run);
        c.cols(2, u.sums);
        unit_bytes = c.at;
        c.cols(nblk, t.unit, t.ctype, t.start, t.out_at, t.size, t.order, t.status, t.end, t.got, t.unpadded);
        bytes = c.at;
    }
};

size_t block_scratch_bytes(u64 n, u64 nblk) { return Layout(nullptr, n, nblk).bytes; }

// the walk, unless the unit columns of `l` already hold it (`counted`), and the placement in a table of max_blocks entries
int count_and_place(const UnitIO &io, const Layout &l, u64 max_blocks, bool counted, cudaStream_t s) {
    if (!counted) xzb_walk_kernel<false><<<(unsigned)((io.n + 255) / 256), 256, 0, s>>>(io, l.u, l.t);
    xzb_place_kernel<<<1, 1024, 0, s>>>(l.u, io.n, max_blocks);
    count_launch(counted ? 1 : 2);
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// `counted`: the unit columns of `l` already hold this batch's walk
int block_batch(const UnitIO &io, u32 *parallel_blocks, const Layout &l, u64 nblk, bool counted, cudaStream_t s) {
    const unsigned unit_threads = (unsigned)((io.n + 255) / 256);
    int st;
    timing_mark(s);
    if ((st = count_and_place(io, l, nblk, counted, s))) return st;
    xzb_walk_kernel<true><<<unit_threads, 256, 0, s>>>(io, l.u, l.t);
    xzb_order_kernel<<<1, 1024, 0, s>>>(l.u, l.t);
    count_launch(2);
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(s);
    xzb_block_kernel<<<(unsigned)((nblk + WARPS - 1) / WARPS), WARPS * 32, lzma::SMEM_BYTES, s>>>(io, l.u, l.t);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(s);
    xzb_resolve_kernel<<<unit_threads, 256, 0, s>>>(io, l.u, l.t, parallel_blocks);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(s);
    xz_kernel<<<(unsigned)((io.n + WARPS - 1) / WARPS), WARPS * 32, lzma::SMEM_BYTES, s>>>(io, l.u.run, parallel_blocks);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(s);
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

size_t swc_xz_block_batch_scratch_bytes(uint64_t n, uint64_t max_blocks) {
    return block_scratch_bytes(n, max_blocks ? max_blocks : 1);
}

int32_t swc_xz_block_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t *out_len, int32_t *status, uint32_t *parallel_blocks,
                                     uint64_t n, uint64_t max_blocks,
                                     void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    const UnitIO io{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n};
    const cudaStream_t s = (cudaStream_t)cuda_stream;
    if (missing(io) || max_blocks > 0xFFFFFFFFull || n > 0xFFFFFFFFull) return SWC_ERR_INVALID_ARG;
    if (scratch && scratch_bytes < swc_xz_block_batch_scratch_bytes(n, max_blocks)) return SWC_ERR_INVALID_ARG;
    int st;
    if ((st = configure())) return st;
    u64 nblk = max_blocks;
    SplitScratch sc(scratch, s);
    if (max_blocks == 0) {
        // the library counts first: the walk on the unit columns alone, then the record total back
        auto launch = [&](void *base, const u64 **t) {
            const Layout l(base, n, 0);
            *t = l.u.sums + 1;
            return count_and_place(io, l, ~0ull, false, s);
        };
        u64 records = 0;
        if ((st = sc.count_first(scratch_bytes, Layout(nullptr, n, 0).unit_bytes, 1, &records, launch))) return st;
        nblk = records < 1 ? 1 : records > 0xFFFFFFFFull ? 0xFFFFFFFFull : records;
        // the largest table the caller's scratch holds; the units past it fall back
        if (scratch) nblk = largest_table(nblk, scratch_bytes, [&](u64 m) { return block_scratch_bytes(n, m); });
    }
    if ((st = sc.seat(block_scratch_bytes(n, nblk)))) return st;
    return block_batch(io, parallel_blocks, Layout(sc.p, n, nblk), nblk, sc.counted, s);
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
