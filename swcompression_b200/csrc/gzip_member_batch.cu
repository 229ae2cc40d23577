// gzip_member_batch.cu — batched GzipArchive.multiUnarchive (reference Sources/GZip/GzipArchive.swift:52-100) on
// device-resident files, every member of every file decoded side by side.  With a caller scratch and max_members > 0 the
// call is a fixed sequence of launches: no host read, no allocation (DESIGN.md §4.20).
//
//   scan<count>  checks::gzip_scan   candidate member starts per unit: the signature with 20 bytes left, and position 0
//   place        one CTA             first entry = exclusive sum of the candidate counts; placed iff they fit max_members
//   scan<fill>   checks::gzip_scan   the placed units' candidates into the table (any order)
//   sort         CTA per unit        the unit's candidates into position order
//   span         thread per unit     cuts the unit into member spans: from a candidate with
//                                    a BGZF BSIZE hint to c + BSIZE + 1 when that is a candidate or the unit end, else to
//                                    the next candidate; capacity = the ISIZE in the span's last 4 bytes, output offset = the
//                                    exclusive sum of those ISIZEs, clamped to the unit's region
//   decode       unarchive_batch_impl(gzip) over every table entry: header, Deflate, CRC-32 and trailer, straight into place
//   validate     thread per unit     the reference's in-order walk over the results: member k is accepted iff it is OK or
//                                    wrongCRC, consumed exactly its span and starts where member k - 1 ended
//   fallback     thread per unit     from the first member that was not accepted, the sequential walk: gzip_parse,
//                                    inflate_serial, serial CRC-32 and trailer, member after member
#include <vector>
#include "../../include/swcgpu.h"
#include "archive_header.cuh"
#include "checks.cuh"
#include "host_util.h"
#include "inflate_serial.cuh"

namespace swc {
namespace {

constexpr u64 NONE = ~0ull;

struct Units {
    unsigned long long *count, *fill;   // candidates (scan<count>) / placed so far (scan<fill>)
    u64 *first;                         // first table entry, NONE: not placed
    u64 *spans;                         // member spans at first ..
    u64 *resume, *written, *members;    // fallback: where the walk resumes, with the output and members accepted so far
    u8 *run;                            // 1: the fallback finishes the unit
    u64 *sums;                          // [0] candidates of every unit
};

// the member table: candidates, then the decode stage's columns per span
struct Table {
    u64 *cand;
    u64 *in_off, *in_len, *out_off, *out_cap;   // contiguous: zeroed together, so idle entries are zero-length units
    u64 *out_len, *consumed;
    int32_t *status;
};

// the caller's member table and counters (any pointer may be null)
struct Members {
    u64 *count;
    const u64 *off, *cap;
    u64 *end, *in_off;
    u32 *parallel;
    __device__ void put(u64 unit, u64 k, u64 end_at, u64 start) const {
        if (off && k < cap[unit]) { end[off[unit] + k] = end_at; in_off[off[unit] + k] = start; }
    }
};

__device__ __forceinline__ u32 le16(const u8 *q) { return (u32)q[0] | (u32)q[1] << 8; }
__device__ __forceinline__ u32 le32d(const u8 *q) { return le16(q) | le16(q + 2) << 16; }

// BSIZE + 1 from a BGZF "BC" subfield of the FEXTRA field of the header at `at`, or 0.  A hint only: the reference never
// reads it, and a hint that does not lead to a candidate or to the unit end is ignored.
__device__ u64 bsize_hint(const u8 *p, u64 L, u64 at) {
    if (at + 12 > L || !(p[at + 3] & 0x04)) return 0;
    const u64 end = at + 12 + le16(p + at + 10);
    if (end > L) return 0;
    for (u64 x = at + 12; x + 4 <= end; x += 4 + le16(p + x + 2))
        if (p[x] == 'B' && p[x + 1] == 'C' && le16(p + x + 2) == 2 && x + 6 <= end) return (u64)le16(p + x + 4) + 1;
    return 0;
}

// the fill scan appends in any order (its CTAs race for the slots): a heap sort by one thread, for the units too large for
// gzm_sort_kernel's shared memory
__device__ void sort_positions(u64 *a, u64 m) {
    bool sorted = true;
    for (u64 i = 1; i < m && sorted; i++) sorted = a[i - 1] <= a[i];
    if (sorted) return;
    auto sift = [&](u64 i, u64 end) {
        const u64 v = a[i];
        for (;;) {
            u64 c = 2 * i + 1;
            if (c >= end) break;
            if (c + 1 < end && a[c + 1] > a[c]) c++;
            if (a[c] <= v) break;
            a[i] = a[c];
            i = c;
        }
        a[i] = v;
    };
    for (u64 i = m / 2; i-- > 0;) sift(i, m);
    for (u64 e = m; e-- > 1;) {
        const u64 t = a[0];
        a[0] = a[e]; a[e] = t;
        sift(0, e);
    }
}

// CTA per placed unit (strided): the unit's candidates into position order, a bitonic sort in shared memory for up to
// SORT_SMEM of them, else one thread's heap sort
constexpr u32 SORT_SMEM = 4096;
__global__ void __launch_bounds__(1024) gzm_sort_kernel(Units u, u64 *cand, u64 n) {
    __shared__ u64 s[SORT_SMEM];
    for (u64 unit = blockIdx.x; unit < n; unit += gridDim.x) {
        const u64 f = u.first[unit], m = u.count[unit];
        if (f == NONE || m < 2) continue;
        u64 *a = cand + f;
        if (m > SORT_SMEM) {
            if (threadIdx.x == 0) sort_positions(a, m);
            continue;
        }
        u32 p2 = 2;
        while (p2 < m) p2 <<= 1;
        for (u32 i = threadIdx.x; i < p2; i += blockDim.x) s[i] = i < m ? a[i] : NONE;
        __syncthreads();
        for (u32 k = 2; k <= p2; k <<= 1)
            for (u32 j = k >> 1; j > 0; j >>= 1) {
                for (u32 i = threadIdx.x; i < p2; i += blockDim.x) {
                    const u32 l = i ^ j;
                    if (l > i) {
                        const u64 x = s[i], y = s[l];
                        if ((x > y) == ((i & k) == 0)) { s[i] = y; s[l] = x; }
                    }
                }
                __syncthreads();
            }
        for (u32 i = threadIdx.x; i < m; i += blockDim.x) a[i] = s[i];
        __syncthreads();
    }
}

// exclusive sum of the candidate counts in unit order; a unit is placed iff its candidates end inside the table
__global__ void __launch_bounds__(1024) gzm_place_kernel(Units u, u64 n, u64 max_members) {
    __shared__ u64 part[1][1024];
    u64 b, e;
    cta_unit_run(n, b, e);
    u64 s = 0;
    for (u64 i = b; i < e; i++) s += u.count[i];
    part[0][threadIdx.x] = s;
    cta_scan<1>(part);
    if (threadIdx.x == 1023) u.sums[0] = part[0][1023];
    u64 at = part[0][threadIdx.x] - s;
    for (u64 i = b; i < e; i++) {
        const u64 nb = u.count[i];
        u.first[i] = at + nb <= max_members ? at : NONE;
        u.fill[i] = 0;
        at += nb;
    }
}

// Thread per unit: the member spans of a placed unit (rule above), written as decode-stage units.  Every unit starts
// marked for the fallback from byte 0.  `arena`: the output arena the decode stage's scratch covers.
//
// A span's region is either empty or at least MIN_REGION bytes, and lies inside the arena; any other span gets capacity 0,
// so a member with output fails the decode stage and the fallback decodes it (with every member behind it).  The Huffman
// stages store literal bytes only below out_cap (K1w byte by byte, K1L in 8-byte words that end at or below out_cap) but do
// not check them against the unit's scratch region (inflate.cuh), which holds 4 floor(cap / 3) bytes or more.  For a cap of
// 1, 2 or 5 that is less than cap, and the literals would land in the scratch of whatever region follows: the next span, or
// another unit's region packed right behind this one.  From 6 bytes on the region holds every literal; 16 keeps a margin.
// A region past the arena would have its records indexed past the scratch.
constexpr u64 MIN_REGION = 16;
__global__ void __launch_bounds__(256) gzm_span_kernel(UnitIO io, Units u, Table t, u64 arena) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= io.n) return;
    u.run[unit] = 1; u.resume[unit] = 0; u.written[unit] = 0; u.members[unit] = 0; u.spans[unit] = 0;
    const u64 f = u.first[unit];
    if (f == NONE) return;
    const u64 m = u.count[unit];
    const u64 *c = t.cand + f;                                       // in position order (gzm_sort_kernel)
    const u8 *p = io.in_base + io.in_off[unit];
    const u64 L = io.in_len[unit], cap = io.out_cap[unit];
    u64 k = 0, o = 0, e = f;
    while (k < m) {
        const u64 at = c[k];
        u64 next = k + 1 < m ? c[k + 1] : L, nk = k + 1;
        const u64 hint = bsize_hint(p, L, at);
        if (hint && at + hint == L) {
            next = L; nk = m;
        } else if (hint && at + hint < L) {
            u64 lo = k + 1, hi = m;                                  // the first candidate >= at + hint
            while (lo < hi) { const u64 mid = (lo + hi) / 2; if (c[mid] < at + hint) lo = mid + 1; else hi = mid; }
            if (lo < m && c[lo] == at + hint) { next = at + hint; nk = lo; }
        }
        u64 isize = 0;
        if (next - at >= 20) {
            isize = le32d(p + next - 4);
            if (isize > (next - at) * 1032 + 64) isize = 0;            // Deflate cannot expand further than ~1032:1
        }
        const u64 room = o < cap ? cap - o : 0, out_at = io.out_off[unit] + (o < cap ? o : cap);
        u64 region = isize < room ? isize : room;
        if (region < MIN_REGION || out_at + region > arena) region = 0;
        t.in_off[e] = io.in_off[unit] + at;
        t.in_len[e] = next - at;
        t.out_off[e] = out_at;
        t.out_cap[e] = region;
        o += isize;
        e++;
        k = nk;
    }
    u.spans[unit] = e - f;
}

// Thread per unit: GzipArchive.multiUnarchive's walk (:57-76) over the decoded spans.  A unit whose spans are all
// accepted, or whose walk ends at an accepted wrongCRC member, is final; any other placed unit resumes in the fallback at
// its first span that was not accepted, with the accepted members kept in place.
__global__ void __launch_bounds__(256) gzm_validate_kernel(DecodeIO io, Units u, Table t, Members mb) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= io.n) return;
    if (mb.parallel) mb.parallel[unit] = 0;
    const u64 f = u.first[unit];
    if (f == NONE) return;
    const u64 ns = u.spans[unit], in0 = io.in_off[unit], out0 = io.out_off[unit];
    u64 w = 0, k = 0;
    for (; k < ns; k++) {
        const u64 e = f + k;
        const int st = t.status[e];
        if ((st != SWC_OK && st != SWC_GZIP_WRONG_CRC) || t.consumed[e] != t.in_len[e] || t.out_off[e] - out0 != w) break;
        mb.put(unit, k, w + t.out_len[e], t.in_off[e] - in0);
        w += t.out_len[e];
        if (st == SWC_GZIP_WRONG_CRC) {                                 // the member is returned, the walk ends
            io.status[unit] = st; io.out_len[unit] = w; io.consumed[unit] = t.in_off[e] - in0 + t.in_len[e];
            if (mb.count) mb.count[unit] = k + 1;
            if (mb.parallel) mb.parallel[unit] = (u32)(k + 1);
            u.run[unit] = 0;
            return;
        }
    }
    if (mb.parallel) mb.parallel[unit] = (u32)k;
    if (k == ns) {                                                      // the spans end at the unit end
        io.status[unit] = SWC_OK; io.out_len[unit] = w; io.consumed[unit] = io.in_len[unit];
        if (mb.count) mb.count[unit] = ns;
        u.run[unit] = 0;
        return;
    }
    u.resume[unit] = t.in_off[f + k] - in0;
    u.written[unit] = w;
    u.members[unit] = k;
}

// Thread per marked unit: the sequential walk (GzipArchive.swift:57-76, processMember :79-100) from the resume point, one
// member after another into the unit's region.  Once a member does not fit, the walk goes on counting: members decode
// without keeping their bytes and their CRC-32 is not checked, and the unit reports SWC_ERR_OUTPUT_OVERFLOW with the bytes
// counted up to where the walk stops.
__global__ void __launch_bounds__(64) gzm_fallback_kernel(DecodeIO io, Units u, Members mb) {
    __shared__ u32 tab[256];
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) {
        u32 c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
        tab[i] = c;
    }
    __syncthreads();
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= io.n || !u.run[unit]) return;
    const u8 *p = io.in_base + io.in_off[unit];
    const u64 L = io.in_len[unit], cap = io.out_cap[unit];
    u8 *out = io.out_base + io.out_off[unit];
    u64 off = u.resume[unit], w = u.written[unit], k = u.members[unit];
    bool over = false;
    int st = SWC_OK;
    while (off < L) {
        if (L - off < 20) { st = SWC_GZIP_WRONG_MAGIC; break; }                  // :83
        swc_gzip_header h;
        if ((st = gzip_parse(p, L, off, &h))) break;
        const u64 d = off + h.header_len;
        const u64 room = !over && w < cap ? cap - w : 0;
        u64 got = 0, used = 0;
        st = inflate::inflate_serial(p + d, (L - d) * 8, 0, out + (w < cap ? w : cap), room, &got, &used);
        if (st == SWC_ERR_OUTPUT_OVERFLOW) { over = true; st = SWC_OK; }
        if (st == SWC_OK) {
            const u64 q = d + (used + 7) / 8;                                     // align()
            if (L - q < 8) st = SWC_GZIP_WRONG_MAGIC;                             // :88-89
            else if ((u32)got != le32d(p + q + 4)) st = SWC_GZIP_WRONG_ISIZE;     // :94-95
            else {
                bool crc_ok = true;
                if (!over) {
                    u32 c = 0xFFFFFFFFu;
                    for (u64 i = 0; i < got; i++) c = tab[(c ^ out[w + i]) & 0xFF] ^ (c >> 8);
                    crc_ok = ~c == le32d(p + q);                                   // :97-98
                    mb.put(unit, k, w + got, off);
                    k++;
                }
                off = q + 8;
                if (!crc_ok) st = SWC_GZIP_WRONG_CRC;
            }
        }
        w += got;
        if (st != SWC_OK) break;
    }
    const bool kept = !over && (st == SWC_OK || st == SWC_GZIP_WRONG_CRC);
    io.status[unit] = over ? SWC_ERR_OUTPUT_OVERFLOW : st;
    io.out_len[unit] = kept || over ? w : 0;
    io.consumed[unit] = kept ? off : 0;
    if (mb.count) mb.count[unit] = kept ? k : 0;
}

// ---- scratch layout: the unit columns, the member table, then the decode stage's scratch ----------------------------
struct Layout {
    Units u;
    Table t;
    size_t unit_bytes, cols_bytes, table_bytes;
    void *inner;

    Layout(void *base, u64 n, u64 nblk) {
        Carver c(base);
        c.cols(n, u.count, u.fill, u.first, u.spans, u.resume, u.written, u.members, u.run);
        c.cols(1, u.sums);
        unit_bytes = c.at;
        c.cols(nblk, t.cand);
        const size_t cols = c.at;
        c.cols(nblk, t.in_off, t.in_len, t.out_off, t.out_cap);
        cols_bytes = c.at - cols;
        c.cols(nblk, t.out_len, t.consumed, t.status);
        table_bytes = c.at;
        inner = c.end();
    }
};

size_t batch_scratch_bytes(u64 n, u64 nblk, u64 out_total) {
    return Layout(nullptr, n, nblk).table_bytes + swc_unarchive_batch_scratch_bytes(nblk, out_total);
}

struct Call {
    DecodeIO io;
    Members mb;
    cudaStream_t s;
};

// the candidate counts, unless the unit columns of `l` already hold them (`counted`), and the placement in a table of
// max_members entries
int count(const Call &q, const Layout &l, u64 max_members, bool counted) {
    if (!counted) {
        SWC_CUDA_TRY(cudaMemsetAsync(l.u.count, 0, q.io.n * 8, q.s));
        int st = checks::gzip_scan(checks::GzipScan{q.io.in_base, q.io.in_off, q.io.in_len, q.io.n, l.u.count, nullptr, nullptr, 0, true}, q.s);
        if (st) return st;
    }
    gzm_place_kernel<<<1, 1024, 0, q.s>>>(l.u, q.io.n, max_members);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// `counted`: the unit columns of `l` already hold this batch's candidate counts; the decode stage has `inner` bytes,
// enough for an output arena of out_total bytes
int decode(const Call &q, const Layout &l, u64 nblk, bool counted, u64 out_total, size_t inner) {
    const u64 n = q.io.n;
    const unsigned unit_threads = (unsigned)((n + 255) / 256);
    int st;
    timing_mark(q.s);
    if ((st = count(q, l, nblk, counted))) return st;
    if ((st = checks::gzip_scan(checks::GzipScan{q.io.in_base, q.io.in_off, q.io.in_len, n, l.u.fill, l.u.first, l.t.cand, 0, true}, q.s)))
        return st;
    timing_mark(q.s);
    gzm_sort_kernel<<<(unsigned)(n < 65535 ? n : 65535), 1024, 0, q.s>>>(l.u, l.t.cand, n);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(q.s);
    SWC_CUDA_TRY(cudaMemsetAsync(l.t.in_off, 0, l.cols_bytes, q.s));
    gzm_span_kernel<<<unit_threads, 256, 0, q.s>>>(q.io, l.u, l.t, out_total);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(q.s);
    const DecodeIO members{{q.io.in_base, l.t.in_off, l.t.in_len, q.io.out_base, l.t.out_off, l.t.out_cap, l.t.out_len, l.t.status, nblk},
                           l.t.consumed};
    if ((st = unarchive_batch_impl(true, members, nullptr, out_total, l.inner, inner, q.s))) return st;
    timing_mark(q.s);
    gzm_validate_kernel<<<unit_threads, 256, 0, q.s>>>(q.io, l.u, l.t, q.mb);
    gzm_fallback_kernel<<<(unsigned)((n + 63) / 64), 64, 0, q.s>>>(q.io, l.u, q.mb);
    count_launch(2);
    SWC_CUDA_TRY(cudaGetLastError());
    timing_mark(q.s);
    return SWC_OK;
}

// the output arena the units span: max(out_off[i] + out_cap[i]) (blocking: waits for `s`)
int arena_bytes(const UnitIO &io, cudaStream_t s, u64 *total) {
    std::vector<u64> off, cap;
    int st;
    if ((st = read_lens(io.out_off, io.n, s, off)) || (st = read_lens(io.out_cap, io.n, s, cap))) return st;
    *total = 0;
    for (u64 i = 0; i < io.n; i++) *total = off[i] + cap[i] > *total ? off[i] + cap[i] : *total;
    return SWC_OK;
}

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

size_t swc_gzip_member_batch_scratch_bytes(uint64_t n, uint64_t max_members, uint64_t out_capacity_total) {
    return batch_scratch_bytes(n, max_members ? max_members : 1, out_capacity_total);
}

int32_t swc_gzip_multi_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                       uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                       uint64_t *n_members, const uint64_t *member_off, const uint64_t *member_cap,
                                       uint64_t *member_end, uint64_t *member_in_off, uint32_t *parallel_members,
                                       uint64_t n, uint64_t max_members, void *scratch, size_t scratch_bytes, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    if (n == 0) return SWC_OK;
    const bool table = member_off || member_cap || member_end || member_in_off;
    const Call q{{{in_base, in_off, in_len, out_base, out_off, out_cap, out_len, status, n}, consumed_bytes},
                 {n_members, member_off, member_cap, member_end, member_in_off, parallel_members},
                 (cudaStream_t)cuda_stream};
    if (missing(q.io) || max_members > 0xFFFFFFFFull || n > 0xFFFFFFFFull) return SWC_ERR_INVALID_ARG;
    if (table && !(member_off && member_cap && member_end && member_in_off)) return SWC_ERR_INVALID_ARG;
    int st;
    u64 nblk = max_members, arena = 0;
    SplitScratch sc(scratch, q.s);
    if (max_members == 0) {
        // the library counts first: the scan on the unit columns alone, then the candidate total back
        auto launch = [&](void *base, const u64 **t) {
            const Layout l(base, n, 0);
            *t = l.u.sums;
            return count(q, l, ~0ull, false);
        };
        u64 total = 0;
        if ((st = sc.count_first(scratch_bytes, Layout(nullptr, n, 0).unit_bytes, 1, &total, launch))) return st;
        // the table is capped at in_len / 20 + 1 entries per unit, as many members as a unit can hold: a file of
        // look-alikes (one candidate every 4 bytes) must not size the scratch, its units past the cap fall back
        std::vector<u64> lens;
        if ((st = read_lens(in_len, n, q.s, lens))) return st;
        u64 bound = 0;
        for (u64 x : lens) bound += x / 20 + 1;
        total = total < bound ? total : bound;
        nblk = total < 1 ? 1 : total > 0xFFFFFFFFull ? 0xFFFFFFFFull : total;
    }
    if (!scratch || max_members == 0) {
        if ((st = arena_bytes(q.io, q.s, &arena))) return st;
    }
    if (scratch) {
        if (max_members == 0) {
            // the largest table the caller's scratch holds beside the decode stage's scratch; the units past it fall back
            if (batch_scratch_bytes(n, 1, arena) > scratch_bytes) return SWC_ERR_INVALID_ARG;
            nblk = largest_table(nblk, scratch_bytes, [&](u64 m) { return batch_scratch_bytes(n, m, arena); });
        } else if (scratch_bytes < batch_scratch_bytes(n, nblk, 0)) {
            return SWC_ERR_INVALID_ARG;
        }
    } else {
        scratch_bytes = batch_scratch_bytes(n, nblk, arena);
        if ((st = sc.seat(scratch_bytes))) return st;
    }
    const Layout l(sc.p, n, nblk);
    // the decode stage takes the rest of the scratch and the arena it covers; spans outside that arena take the fallback
    const size_t inner = scratch_bytes - l.table_bytes;
    const u64 out_total = unarchive_batch_arena(nblk, inner);
    return decode(q, l, nblk, sc.counted, out_total, inner);
}

}  // extern "C"
