// tar.cu — TarContainer.open / info / formatOf walked on the device: one warp per archive (DESIGN §4.18).
//
// The walk is TarParser.next() (Sources/TAR/TarParser.swift:35-79) hop by hop.  Each hop is one dependent 512-byte
// header read, so an archive is inherently sequential; a warp per archive keeps every hop to a handful of instructions:
// the 32 lanes load the header (16 B each) into shared memory, vote on the 1 024-byte EOF marker, reduce both checksum
// sums, parse the ten numeric fields in ten lanes at once, and find string ends with ballots over the header's NUL mask.
// PAX payloads are walked by the warp too: record boundaries by ballot, UTF-8 validation lane-parallel.
#include <cuda_runtime.h>
#include "common.cuh"
#include "host_util.h"
#include "../../include/swcgpu.h"

namespace swc {
namespace {

constexpr int WARPS = 4;                              // warps (archives) per block
constexpr int REC_WORDS = sizeof(swc_tar_entry) / 8;
static_assert(sizeof(swc_tar_entry) % 8 == 0, "swc_tar_entry is copied as 8-byte words");

// TarExtendedHeader (TarExtendedHeader.swift:9-101): Int fields as values, text fields as ranges of their last record
struct Pax {
    u32 present;                                      // SWC_TAR_UID / SWC_TAR_GID
    u32 has;                                          // bit r: range r set (0 mtime 1 atime 2 ctime 3 uname 4 gname
    int has_size;                                     //   5 path 6 linkpath 7 charset 8 comment)
    i64 uid, gid, size;
    u64 off[9], len[9];
    u64 poff, plen;
};

struct alignas(16) WarpSmem {
    u8 hdr[512];
    u32 nul[16];                                      // bit b of word j: hdr[32 j + b] == 0
    i64 val[10];                                      // tarInt of the ten numeric fields
    u32 ok;                                           // bit k: val[k] parsed
    Pax pax[2];                                       // 0 global, 1 local
    swc_tar_entry rec;
};

struct Args {
    const u8 *in_base;
    const u64 *in_off, *in_len;
    const u64 *in_cap;                                // optional: a unit is at most in_cap[i] bytes
    const int32_t *in_status;                         // optional: a unit whose in_status[i] != 0 is not walked
    swc_tar_entry *entries;
    const u64 *entry_off, *entry_cap;
    u64 *n_entries;
    int32_t *info_status, *open_status, *format, *format_status;
    u64 n;
};

// the ten numeric header fields (TarHeader.swift:58-128): mode uid gid size mtime chksum devmajor devminor atime ctime
__constant__ u16 c_field_pos[10] = {100, 108, 116, 124, 136, 148, 329, 337, 345, 357};
__constant__ u8 c_field_len[10] = {8, 8, 8, 12, 12, 8, 8, 8, 12, 12};
// the keys TarExtendedHeader.init keeps as text (TarExtendedHeader.swift:67-91), in Pax range order
__constant__ char c_pax_keys[9][9] = {"mtime", "atime", "ctime", "uname", "gname", "path", "linkpath", "charset", "comment"};

__device__ __forceinline__ bool add_ovf(i64 a, i64 b, i64 *r) {
    const i64 s = (i64)((u64)a + (u64)b);
    *r = s;
    return ((a ^ s) & (b ^ s)) < 0;
}
__device__ __forceinline__ i64 round512(i64 v) { return v >= INT64_MAX - 510 ? INT64_MAX : (v + 511) & ~(i64)511; }
__device__ __forceinline__ i64 shfl64(i64 v, int src) { return (i64)__shfl_sync(SWC_FULL, (long long)v, src); }

// Swift Int(String): decimal, optional sign, nil on overflow or any other byte
__device__ bool swift_int(const u8 *p, u64 n, i64 *v) {
    if (n == 0) return false;
    bool neg = false;
    u64 i = 0;
    if (p[0] == '+' || p[0] == '-') { neg = p[0] == '-'; i = 1; if (n == 1) return false; }
    const u64 lim = neg ? (u64)INT64_MAX + 1 : (u64)INT64_MAX;
    u64 acc = 0;
    for (; i < n; i++) {
        const u64 d = (u64)p[i] - '0';
        if (d > 9 || acc > (lim - d) / 10) return false;
        acc = acc * 10 + d;
    }
    *v = neg ? (i64)(0 - acc) : (i64)acc;
    return true;
}

// tarInt(maxLength:) (LittleEndianByteReader+Tar.swift:38-91) on the field f[0, m) of the shared header
__device__ bool tar_int(const u8 *f, int m, i64 *v) {
    if (f[0] & 0x80) {                                                  // base-256
        const u64 inv = (f[0] & 0x40) ? 0xFF : 0;
        u64 r = 0;
        for (int i = 0; i < m; i++) {
            u64 b = (f[i] ^ inv) & 0xFF;
            if (i == 0) b &= 0x7F;
            if ((i64)r >> 56 > 0) return false;
            r = (r << 8) | b;
        }
        *v = inv ? (i64)~r : (i64)r;
        return true;
    }
    // octal: the skip loop leaves the reader one byte early, so the last byte of the field is never read
    int s = 0;
    u8 b;
    do { b = f[s]; s++; } while ((b == 0 || b == 0x20) && s < m);
    const int first = s - 1, count = m - s;
    int n = 0;
    while (n < count && f[first + n] != 0 && f[first + n] != 0x20) n++;
    if (n == 0) return false;
    const u8 *p = f + first;
    bool neg = false;
    int i = 0;
    if (p[0] == '+' || p[0] == '-') { neg = p[0] == '-'; i = 1; if (n == 1) return false; }
    const u64 lim = neg ? (u64)INT64_MAX + 1 : (u64)INT64_MAX;
    u64 acc = 0;
    for (; i < n; i++) {
        const u64 d = (u64)p[i] - '0';
        if (d > 7 || acc > (lim - d) / 8) return false;
        acc = acc * 8 + d;
    }
    *v = neg ? (i64)(0 - acc) : (i64)acc;
    return true;
}

// first index in [i, e) whose byte is c, else e (a ballot per 32 bytes)
__device__ i64 warp_find(const u8 *in, i64 i, i64 e, u8 c) {
    for (i64 base = i; base < e; base += 32) {
        const i64 p = base + lane_id();
        const u32 m = __ballot_sync(SWC_FULL, p < e && in[p] == c);
        if (m) return base + __ffs(m) - 1;
    }
    return e;
}

// String(data:encoding: .utf8) succeeds on in[s, s + n): strict UTF-8, every lane checks the sequences starting at its
// positions, and the byte after each sequence must not be a continuation byte (so none is left unclaimed)
__device__ bool warp_utf8(const u8 *in, i64 s, i64 n) {
    bool bad = false;
    for (i64 p = lane_id(); p < n && !bad; p += 32) {
        const u8 b = in[s + p];
        if ((b & 0xC0) == 0x80) { bad = p == 0; continue; }
        int k = 0;
        u8 lo = 0x80, hi = 0xBF;
        if (b < 0x80) k = 0;
        else if (b >= 0xC2 && b <= 0xDF) k = 1;
        else if (b >= 0xE0 && b <= 0xEF) { k = 2; if (b == 0xE0) lo = 0xA0; if (b == 0xED) hi = 0x9F; }
        else if (b >= 0xF0 && b <= 0xF4) { k = 3; if (b == 0xF0) lo = 0x90; if (b == 0xF4) hi = 0x8F; }
        else { bad = true; break; }
        if (n - p - 1 < k) { bad = true; break; }
        if (k) {
            if (in[s + p + 1] < lo || in[s + p + 1] > hi) { bad = true; break; }
            for (int j = 2; j <= k; j++) if ((in[s + p + j] & 0xC0) != 0x80) bad = true;
        }
        if (p + k + 1 < n && (in[s + p + k + 1] & 0xC0) == 0x80) bad = true;
    }
    return __all_sync(SWC_FULL, !bad);
}

__device__ __forceinline__ bool key_is(const u8 *k, i64 n, const char *s) {
    int i = 0;
    for (; s[i]; i++) if (i >= n || k[i] != (u8)s[i]) return false;
    return i == n;
}

// TarExtendedHeader.init(_:) over the slice in[s, e): an index outside the slice is a trap
__device__ int parse_pax(const u8 *in, i64 s, i64 e, Pax *h) {
    if (lane_id() == 0) {
        *h = Pax{};
        h->poff = (u64)s; h->plen = (u64)(e - s);
    }
    __syncwarp();
    i64 i = s;
    while (i < e) {
        const i64 ls = i;
        const i64 sp = warp_find(in, i, e, 0x20);
        if (sp >= e) return SWC_ERR_REFERENCE_TRAP;
        i64 length = 0;
        int ok = 0;
        if (lane_id() == 0) ok = swift_int(in + ls, (u64)(sp - ls), &length);
        ok = __shfl_sync(SWC_FULL, ok, 0);
        length = shfl64(length, 0);
        if (!ok) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
        const i64 ks = sp + 1;
        const i64 eq = warp_find(in, ks, e, 0x3D);
        if (eq >= e) return SWC_ERR_REFERENCE_TRAP;
        if (!warp_utf8(in, ks, eq - ks)) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
        const i64 vs = eq + 1;
        i = vs;
        if (i - ls + 1 < length) {                                      // the value runs to ls + length - 1
            i64 need;
            if (add_ovf(ls, length - 1, &need) || need >= e) return SWC_ERR_REFERENCE_TRAP;
            i = need;
        }
        if (i >= e) return SWC_ERR_REFERENCE_TRAP;
        if (in[i] != 0x0A) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
        const i64 ve = i++;
        if (!warp_utf8(in, vs, ve - vs)) continue;                      // a value that is not UTF-8 skips the record
        if (lane_id() == 0) {
            const u8 *k = in + ks, *v = in + vs;
            const i64 kn = eq - ks;
            const u64 vl = (u64)(ve - vs);
            i64 x = 0;
            if (key_is(k, kn, "uid")) {
                if (swift_int(v, vl, &x)) { h->uid = x; h->present |= SWC_TAR_UID; } else h->present &= ~SWC_TAR_UID;
            } else if (key_is(k, kn, "gid")) {
                if (swift_int(v, vl, &x)) { h->gid = x; h->present |= SWC_TAR_GID; } else h->present &= ~SWC_TAR_GID;
            } else if (key_is(k, kn, "size")) {
                h->has_size = swift_int(v, vl, &x);
                h->size = x;
            } else {
                for (int r = 0; r < 9; r++)
                    if (key_is(k, kn, c_pax_keys[r])) { h->off[r] = (u64)vs; h->len[r] = vl; h->has |= 1u << r; break; }
            }
        }
        __syncwarp();
    }
    if (e > s && in[e - 1] != 0x0A) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
    return SWC_OK;
}

// length of the C string at hdr[s, s + m), from the NUL mask
__device__ u64 hdr_cstr(const WarpSmem &w, int s, int m) {
    for (int p = s; p < s + m;) {
        const int j = p >> 5, b = p & 31;
        const u32 bits = w.nul[j] >> b;
        if (bits) return (u64)min(p + __ffs(bits) - 1, s + m) - s;
        p = (j + 1) << 5;
    }
    return (u64)m;
}

// 16 bytes at p, one vector load when p is aligned
__device__ __forceinline__ uint4 load16(const u8 *p) {
    if (((uintptr_t)p & 15) == 0) return __ldg((const uint4 *)p);
    u32 v[4];
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = (u32)p[4 * k] | (u32)p[4 * k + 1] << 8 | (u32)p[4 * k + 2] << 16 | (u32)p[4 * k + 3] << 24;
    return make_uint4(v[0], v[1], v[2], v[3]);
}

__global__ void __launch_bounds__(WARPS * 32, 1) tar_walk_kernel(const Args a) {
    __shared__ WarpSmem smem[WARPS];
    const u64 unit = (u64)blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (unit >= a.n) return;
    WarpSmem &w = smem[threadIdx.x >> 5];
    const int lane = lane_id();
    if (a.in_status && a.in_status[unit] != SWC_OK) {                  // the decode that produced the unit failed
        if (lane_id() == 0) {
            const int32_t up = a.in_status[unit];
            a.n_entries[unit] = 0;
            a.info_status[unit] = a.open_status[unit] = a.format_status[unit] = up;
            a.format[unit] = SWC_TAR_PRE_POSIX;
        }
        return;
    }
    const u8 *in = a.in_base + a.in_off[unit];
    const i64 L = (i64)(a.in_cap ? min(a.in_len[unit], a.in_cap[unit]) : a.in_len[unit]);
    swc_tar_entry *out = a.entries + a.entry_off[unit];
    const u64 cap = a.entry_cap[unit];
    const u64 max_hops = 2 * (((u64)L + 511) / 512) + 2;

    i64 off = 0;
    u64 hops = 0, count = 0;
    int st = SWC_OK, ost = -1, fst = -1, fmt = SWC_TAR_PRE_POSIX;
    bool ustar_seen = false, has_g = false, has_l = false, has_ln = false, has_ll = false;
    u64 ln_off = 0, ln_len = 0, ll_off = 0, ll_len = 0;

    while (true) {
        if (off >= L) break;                                            // .finished
        if (off < 0) { st = SWC_ERR_REFERENCE_TRAP; break; }            // a negative size took the reader before 0
        if (L - off < 512) { st = SWC_TAR_TOO_SMALL_FILE_IS_PASSED; break; }   // .truncated (no EOF marker fits)
        __syncwarp();                                                   // every lane is done with the last header
        const uint4 x = load16(in + off + 16 * lane);
        *(uint4 *)(w.hdr + 16 * lane) = x;
        if (L - off >= 1024) {                                          // .eofMarker: 1 024 zero bytes
            const uint4 y = load16(in + off + 512 + 16 * lane);
            if (__all_sync(SWC_FULL, !(x.x | x.y | x.z | x.w | y.x | y.y | y.z | y.w))) break;
        }
        if (++hops > max_hops) { st = SWC_ERR_REFERENCE_TRAP; break; } // some block parsed a third time: a cycle
        __syncwarp();
        // checksum sums with bytes 148..155 as spaces, NUL mask, numeric fields
        u32 us = 0;
        int ss = 0;
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int p = 16 * lane + k;
            const u8 b = (p >= 148 && p < 156) ? 0x20 : w.hdr[p];
            us += b; ss += (int8_t)b;
        }
        us = __reduce_add_sync(SWC_FULL, us);
        ss = __reduce_add_sync(SWC_FULL, ss);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const u32 m = __ballot_sync(SWC_FULL, w.hdr[32 * j + lane] == 0);
            if (lane == 0) w.nul[j] = m;
        }
        u64 magic = 0;                                                  // reader.uint64() at offset 257
#pragma unroll
        for (int k = 7; k >= 0; k--) magic = magic << 8 | w.hdr[257 + k];
        const bool gnu = magic == 0x0020207261747375ull;
        const bool ustar = magic == 0x3030007261747375ull || magic == 0x3030207261747375ull;
        // fields: 0 mode 1 uid 2 gid 3 size 4 mtime 5 chksum 6 devmajor 7 devminor 8 atime 9 ctime
        {
            bool ok = false;
            i64 v = 0;
            if (lane < 10 && (lane < 6 || ((gnu || ustar) && (lane < 8 || gnu))))
                ok = tar_int(w.hdr + c_field_pos[lane], c_field_len[lane], &v);
            if (lane < 10) w.val[lane] = v;
            const u32 okm = __ballot_sync(SWC_FULL, ok);
            if (lane == 0) w.ok = okm;
        }
        __syncwarp();
        const u32 okm = w.ok;
        if (!(okm >> 3 & 1)) { st = SWC_TAR_WRONG_FIELD; break; }      // size, before the checksum (TarHeader.swift:72-73)
        if (!(okm >> 5 & 1)) { st = SWC_TAR_WRONG_HEADER_CHECKSUM; break; }
        const i64 chk = w.val[5], size = w.val[3];
        if (!((u64)us == (u64)chk || (i64)ss == chk)) { st = SWC_TAR_WRONG_HEADER_CHECKSUM; break; }
        const int hf = gnu ? SWC_TAR_GNU : ustar ? SWC_TAR_USTAR : SWC_TAR_PRE_POSIX;
        const u8 tf = w.hdr[156];
        const i64 ds = off + 512;
        if (tf == 'L' || tf == 'K' || tf == 'g' || tf == 'x' || tf == 'X') {   // special entries (TarParser.swift:51-69)
            i64 de;
            if (size < 0 || add_ovf(ds, size, &de) || de > L) { st = SWC_ERR_REFERENCE_TRAP; break; }
            if (tf == 'L' || tf == 'K') {
                const u64 cut = (u64)(warp_find(in, ds, de, 0) - ds);     // tarCString(maxLength: size)
                if (tf == 'L') { has_ln = true; ln_off = (u64)ds; ln_len = cut; }
                else { has_ll = true; ll_off = (u64)ds; ll_len = cut; }
            } else {
                const int r = parse_pax(in, ds, de, &w.pax[tf == 'g' ? 0 : 1]);
                if (r) { st = r; break; }
                if (tf == 'g') has_g = true; else has_l = true;
            }
            if (add_ovf(ds, round512(size), &off)) { st = SWC_ERR_REFERENCE_TRAP; break; }
            if (fst < 0 && (tf == 'g' || tf == 'x')) { fst = SWC_OK; fmt = SWC_TAR_PAX; }
            if (fst < 0 && (tf == 'L' || tf == 'K')) { fst = SWC_OK; fmt = SWC_TAR_GNU; }
            continue;
        }
        i64 noff;                                                       // TarParser.swift:73, before next() returns
        if (add_ovf(ds, round512(size), &noff)) { st = SWC_ERR_REFERENCE_TRAP; break; }
        // TarEntryInfo.init (TarEntryInfo.swift:184-242), resolved by lane 0 into the shared record
        i64 info_size = size;
        if (lane == 0) {
            swc_tar_entry &e = w.rec;
            e = swc_tar_entry{};
            const Pax *lp = has_l ? &w.pax[1] : nullptr, *gp = has_g ? &w.pax[0] : nullptr;
            e.header_off = (u64)off; e.data_off = (u64)ds; e.typeflag = tf;
            if (okm & 1) { e.mode = w.val[0] & 0xFFF; e.present |= SWC_TAR_MODE; }
            if (lp && (lp->present & SWC_TAR_UID)) { e.uid = lp->uid; e.present |= SWC_TAR_UID; }
            else if (gp && (gp->present & SWC_TAR_UID)) { e.uid = gp->uid; e.present |= SWC_TAR_UID; }
            else if (okm >> 1 & 1) { e.uid = w.val[1]; e.present |= SWC_TAR_UID; }
            if (lp && (lp->present & SWC_TAR_GID)) { e.gid = lp->gid; e.present |= SWC_TAR_GID; }
            else if (gp && (gp->present & SWC_TAR_GID)) { e.gid = gp->gid; e.present |= SWC_TAR_GID; }
            else if (okm >> 2 & 1) { e.gid = w.val[2]; e.present |= SWC_TAR_GID; }
            e.size = lp && lp->has_size ? lp->size : gp && gp->has_size ? gp->size : size;
            if (okm >> 4 & 1) { e.mtime = w.val[4]; e.present |= SWC_TAR_MTIME; }
            if (okm >> 6 & 1) { e.dev_major = w.val[6]; e.present |= SWC_TAR_DEV_MAJOR; }
            if (okm >> 7 & 1) { e.dev_minor = w.val[7]; e.present |= SWC_TAR_DEV_MINOR; }
            if (okm >> 8 & 1) { e.atime = w.val[8]; e.present |= SWC_TAR_ATIME; }
            if (okm >> 9 & 1) { e.ctime = w.val[9]; e.present |= SWC_TAR_CTIME; }
            for (int k = 0; k < 3; k++) {
                if (lp && (lp->has >> k & 1)) { e.pax_time_off[k] = lp->off[k]; e.pax_time_len[k] = lp->len[k]; e.present |= SWC_TAR_PAX_TIME0 << k; }
                if (gp && (gp->has >> k & 1)) { e.pax_time_off[3 + k] = gp->off[k]; e.pax_time_len[3 + k] = gp->len[k]; e.present |= SWC_TAR_PAX_TIME0 << (3 + k); }
            }
            auto pick = [&](int r, u64 &o, u64 &n) -> bool {
                const Pax *h = lp && (lp->has >> r & 1) ? lp : gp && (gp->has >> r & 1) ? gp : nullptr;
                if (h) { o = h->off[r]; n = h->len[r]; }
                return h != nullptr;
            };
            if (pick(3, e.uname_off, e.uname_len)) e.present |= SWC_TAR_UNAME;
            else if (hf != SWC_TAR_PRE_POSIX) { e.uname_off = (u64)off + 265; e.uname_len = hdr_cstr(w, 265, 32); e.present |= SWC_TAR_UNAME; }
            if (pick(4, e.gname_off, e.gname_len)) e.present |= SWC_TAR_GNAME;
            else if (hf != SWC_TAR_PRE_POSIX) { e.gname_off = (u64)off + 297; e.gname_len = hdr_cstr(w, 297, 32); e.present |= SWC_TAR_GNAME; }
            if (!pick(5, e.name_off, e.name_len)) {
                if (has_ln) { e.name_off = ln_off; e.name_len = ln_len; }
                else {
                    e.name_off = (u64)off; e.name_len = hdr_cstr(w, 0, 100);
                    if (hf == SWC_TAR_USTAR && w.hdr[345]) {
                        e.prefix_off = (u64)off + 345; e.prefix_len = hdr_cstr(w, 345, 155); e.present |= SWC_TAR_PREFIX;
                    }
                }
            }
            if (!pick(6, e.link_off, e.link_len)) {
                if (has_ll) { e.link_off = ll_off; e.link_len = ll_len; }
                else { e.link_off = (u64)off + 157; e.link_len = hdr_cstr(w, 157, 100); }
            }
            if (pick(7, e.charset_off, e.charset_len)) e.present |= SWC_TAR_CHARSET;
            if (pick(8, e.comment_off, e.comment_len)) e.present |= SWC_TAR_COMMENT;
            if (lp) { e.local_off = lp->poff; e.local_len = lp->plen; e.present |= SWC_TAR_LOCAL; }
            if (gp) { e.global_off = gp->poff; e.global_len = gp->plen; e.present |= SWC_TAR_GLOBAL; }
            e.open_size = tf == '5' ? 0 : e.size;
            info_size = e.size;
        }
        info_size = shfl64(info_size, 0);
        __syncwarp();
        if (count < cap) {
            const u64 *src = (const u64 *)&w.rec;
            u64 *dst = (u64 *)(out + count);
            for (int k = lane; k < REC_WORDS; k += 32) dst[k] = src[k];
        }
        __syncwarp();
        count++;
        off = noff;
        has_l = has_ln = has_ll = false;
        if (ost < 0 && tf != '5') {                                     // open's data bound (TarContainer.swift:197-211)
            i64 de;
            if (add_ovf(ds, info_size, &de)) ost = SWC_ERR_REFERENCE_TRAP;
            else if (!(de < L)) ost = SWC_TAR_TOO_SMALL_FILE_IS_PASSED;
            else if (de < ds) ost = SWC_ERR_REFERENCE_TRAP;
        }
        if (fst < 0 && hf == SWC_TAR_GNU) { fst = SWC_OK; fmt = SWC_TAR_GNU; }   // formatOf (TarContainer.swift:49-59)
        if (hf == SWC_TAR_USTAR) ustar_seen = true;
    }
    if (fst < 0) { fst = st; fmt = st == SWC_OK && ustar_seen ? SWC_TAR_USTAR : SWC_TAR_PRE_POSIX; }
    if (ost < 0) ost = st;
    if (count > cap) {
        if (st == SWC_OK) st = SWC_ERR_OUTPUT_OVERFLOW;
        if (ost == SWC_OK) ost = SWC_ERR_OUTPUT_OVERFLOW;
    }
    if (lane == 0) {
        a.n_entries[unit] = count;
        a.info_status[unit] = st;
        a.open_status[unit] = ost;
        a.format[unit] = fmt;
        a.format_status[unit] = fst;
    }
}

int tar_walk(const Args &a, cudaStream_t stream) {
    if (a.n == 0) return SWC_OK;
    if (!a.in_base || !a.in_off || !a.in_len || !a.entries || !a.entry_off || !a.entry_cap || !a.n_entries ||
        !a.info_status || !a.open_status || !a.format || !a.format_status)
        return SWC_ERR_INVALID_ARG;
    tar_walk_kernel<<<(unsigned)((a.n + WARPS - 1) / WARPS), WARPS * 32, 0, stream>>>(a);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

// one host container as a one-unit batch; the table starts at in_len / 512 + 1 records and is rerun once at the
// reported count (only a walk with negative sizes can need more)
int tar_single(const uint8_t *in, size_t in_len, swc_tar_entry **entries, size_t *n_entries, int32_t *st_out,
               int which) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    DevBuf d_in;
    if (int st = upload_input(d_in, in, in_len)) return st;
    DevBuf d_cols;
    // columns: in_off, in_len, entry_off, entry_cap, n_entries (u64) + 4 int32 statuses
    if (int st = d_cols.alloc(5 * 8 + 4 * 4)) return st;
    u64 *c = d_cols.as<u64>();
    int32_t *s32 = (int32_t *)(c + 5);
    u64 cap = in_len / 512 + 1;
    for (int attempt = 0; attempt < 2; attempt++) {
        DevBuf d_tab;
        if (int st = d_tab.alloc(cap * sizeof(swc_tar_entry))) return st;
        const u64 cols[4] = {0, (u64)in_len, 0, cap};
        SWC_CUDA_TRY(cudaMemcpy(c, cols, sizeof cols, cudaMemcpyHostToDevice));
        Args a{d_in.as<u8>(), c, c + 1, nullptr, nullptr, d_tab.as<swc_tar_entry>(), c + 2, c + 3, c + 4, s32, s32 + 1, s32 + 2, s32 + 3, 1};
        if (int st = tar_walk(a, 0)) return st;
        u64 res[5];
        SWC_CUDA_TRY(cudaMemcpy(res, c, sizeof res, cudaMemcpyDeviceToHost));
        int32_t sts[4];
        SWC_CUDA_TRY(cudaMemcpy(sts, s32, sizeof sts, cudaMemcpyDeviceToHost));
        const u64 n = res[4];
        if (which == 2) { st_out[0] = sts[3]; st_out[1] = sts[2]; return SWC_OK; }
        const int32_t st = sts[which];
        if (st == SWC_ERR_OUTPUT_OVERFLOW && attempt == 0) { cap = n; continue; }
        st_out[0] = st;
        if (st != SWC_OK) return SWC_OK;
        *entries = (swc_tar_entry *)swc_alloc(sizeof(swc_tar_entry) * (n + 1));
        if (!*entries) { st_out[0] = SWC_ERR_OUTPUT_OVERFLOW; return SWC_OK; }
        SWC_CUDA_TRY(cudaMemcpy(*entries, d_tab.p, n * sizeof(swc_tar_entry), cudaMemcpyDeviceToHost));
        *n_entries = n;
        return SWC_OK;
    }
    return SWC_ERR_OUTPUT_OVERFLOW;
}

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

int32_t swc_tar_walk_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                           const uint64_t *in_cap, const int32_t *in_status, swc_tar_entry *entries, const uint64_t *entry_off, const uint64_t *entry_cap,
                           uint64_t *n_entries, int32_t *info_status, int32_t *open_status, int32_t *format,
                           int32_t *format_status, uint64_t n, void *cuda_stream) {
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    return tar_walk(Args{in_base, in_off, in_len, in_cap, in_status, entries, entry_off, entry_cap, n_entries, info_status, open_status,
                         format, format_status, n}, (cudaStream_t)cuda_stream);
}

int32_t swc_tar_info(const uint8_t *in, size_t in_len, swc_tar_entry **entries, size_t *n_entries) {
    if ((!in && in_len) || !entries || !n_entries) return SWC_ERR_INVALID_ARG;
    *entries = nullptr; *n_entries = 0;
    int32_t st = SWC_OK;
    if (int r = tar_single(in, in_len, entries, n_entries, &st, 0)) return r;
    return st;
}

int32_t swc_tar_open(const uint8_t *in, size_t in_len, swc_tar_entry **entries, size_t *n_entries) {
    if ((!in && in_len) || !entries || !n_entries) return SWC_ERR_INVALID_ARG;
    *entries = nullptr; *n_entries = 0;
    int32_t st = SWC_OK;
    if (int r = tar_single(in, in_len, entries, n_entries, &st, 1)) return r;
    return st;
}

int32_t swc_tar_format(const uint8_t *in, size_t in_len, int32_t *format) {
    if ((!in && in_len) || !format) return SWC_ERR_INVALID_ARG;
    int32_t st[2] = {SWC_OK, 0};
    swc_tar_entry *unused = nullptr;
    size_t n = 0;
    if (int r = tar_single(in, in_len, &unused, &n, st, 2)) return r;
    if (st[0] == SWC_OK) *format = st[1];
    return st[0];
}

}  // extern "C"
