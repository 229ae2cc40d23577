/* tar.c — CPU restatement of TarContainer.open / info / formatOf.  TEST INFRASTRUCTURE ONLY (see swco.h).
 *
 *   TarParser.next()                  Sources/TAR/TarParser.swift:35-79
 *   TarHeader.init(_:)                Sources/TAR/TarHeader.swift:54-135
 *   tarInt / tarCString               Sources/TAR/LittleEndianByteReader+Tar.swift:23-91
 *   TarExtendedHeader.init(_:)        Sources/TAR/TarExtendedHeader.swift:31-101
 *   TarEntryInfo.init(...)            Sources/TAR/TarEntryInfo.swift:184-242
 *   TarContainer.open/info/formatOf   Sources/TAR/TarContainer.swift:36-71, 187-261
 *
 * swco_tar_walk runs the three calls over one archive at once and fills swc_tar_entry records (include/swcgpu.h), the
 * same contract as one unit of swc_tar_walk_batch.  Where Swift traps (index / range / overflow) or never returns, the
 * status is SWC_ERR_REFERENCE_TRAP. */
#include <stdint.h>
#include <string.h>
#include "../include/swcgpu.h"

typedef struct {
    uint32_t present;                    /* SWC_TAR_UID / GID bits for Int fields; bit 16 + k for ranges below */
    int64_t uid, gid, size;
    int has_size;
    /* ranges: 0 mtime 1 atime 2 ctime 3 uname 4 gname 5 path 6 linkpath 7 charset 8 comment */
    uint64_t off[9], len[9];
    uint32_t has;                        /* bit k: range k set */
    uint64_t poff, plen;
} pax;

static int is_cont(uint8_t b) { return (b & 0xC0) == 0x80; }

/* String(data:encoding: .utf8) succeeds (strict UTF-8: no overlongs, surrogates or code points past U+10FFFF) */
static int utf8_ok(const uint8_t *p, uint64_t n) {
    uint64_t i = 0;
    while (i < n) {
        uint8_t b = p[i];
        if (b < 0x80) { i++; continue; }
        int k; uint8_t lo = 0x80, hi = 0xBF;
        if (b >= 0xC2 && b <= 0xDF) k = 1;
        else if (b >= 0xE0 && b <= 0xEF) { k = 2; if (b == 0xE0) lo = 0xA0; if (b == 0xED) hi = 0x9F; }
        else if (b >= 0xF0 && b <= 0xF4) { k = 3; if (b == 0xF0) lo = 0x90; if (b == 0xF4) hi = 0x8F; }
        else return 0;
        if (n - i - 1 < (uint64_t)k) return 0;
        if (p[i + 1] < lo || p[i + 1] > hi) return 0;
        for (int j = 2; j <= k; j++) if (!is_cont(p[i + j])) return 0;
        i += k + 1;
    }
    return 1;
}

/* Swift Int(String) (decimal, optional + / -, no whitespace, nil on overflow) */
static int swift_int(const uint8_t *p, uint64_t n, int64_t *v) {
    if (n == 0) return 0;
    int neg = 0; uint64_t i = 0;
    if (p[0] == '+' || p[0] == '-') { neg = p[0] == '-'; i = 1; if (n == 1) return 0; }
    uint64_t acc = 0, lim = neg ? (uint64_t)INT64_MAX + 1 : (uint64_t)INT64_MAX;
    for (; i < n; i++) {
        if (p[i] < '0' || p[i] > '9') return 0;
        uint64_t d = p[i] - '0';
        if (acc > (lim - d) / 10) return 0;
        acc = acc * 10 + d;
    }
    *v = neg ? (int64_t)(0 - acc) : (int64_t)acc;
    return 1;
}

/* tarInt(maxLength:) on field f[0, m) */
static int tar_int(const uint8_t *f, int m, int64_t *v) {
    if (f[0] & 0x80) {                                            /* base-256 :47-66 */
        uint64_t inv = (f[0] & 0x40) ? 0xFF : 0, r = 0;
        for (int i = 0; i < m; i++) {
            uint64_t b = (f[i] ^ inv) & 0xFF;
            if (i == 0) b &= 0x7F;
            if ((int64_t)r >> 56 > 0) return 0;
            r = (r << 8) | b;
        }
        if ((int64_t)r >> 63 > 0) return 0;                      /* never: arithmetic shift of a negative is -1 */
        *v = inv ? (int64_t)~r : (int64_t)r;
        return 1;
    }
    /* octal :68-89: the skip loop stops one byte early when it runs to the end, and the last byte is never read */
    int s = 0;
    uint8_t b;
    do { b = f[s]; s++; } while ((b == 0 || b == 0x20) && s < m);
    s--;                                                          /* offset -= 1 */
    uint8_t buf[16]; int n = 0;
    /* for _ in actualStartIndex..<maxLength: reads bytes f[s], f[s+1], ... (maxLength - actualStartIndex) of them */
    int count = m - (s + 1);
    for (int k = 0; k < count; k++) {
        uint8_t c = f[s + k];
        if (c == 0 || c == 0x20) break;
        buf[n++] = c;
    }
    /* String(bytes:encoding:.utf8) then Int(_, radix: 8) */
    if (n == 0) return 0;
    int i = 0, neg = 0;
    if (buf[0] == '+' || buf[0] == '-') { neg = buf[0] == '-'; i = 1; if (n == 1) return 0; }
    uint64_t acc = 0, lim = neg ? (uint64_t)INT64_MAX + 1 : (uint64_t)INT64_MAX;
    for (; i < n; i++) {
        if (buf[i] < '0' || buf[i] > '7') return 0;
        uint64_t d = buf[i] - '0';
        if (acc > (lim - d) / 8) return 0;
        acc = acc * 8 + d;
    }
    *v = neg ? (int64_t)(0 - acc) : (int64_t)acc;
    return 1;
}

static uint64_t cstr_len(const uint8_t *p, uint64_t m) {
    uint64_t i = 0;
    while (i < m && p[i]) i++;
    return i;
}

static int add_ovf(int64_t a, int64_t b, int64_t *r) { return __builtin_add_overflow(a, b, r); }

static int64_t round512(int64_t v) { return v >= INT64_MAX - 510 ? INT64_MAX : (v + 511) & ~(int64_t)511; }

/* TarExtendedHeader.init over in[s, e) (a slice: indices outside it trap) */
static int parse_pax(const uint8_t *in, int64_t s, int64_t e, pax *h) {
    memset(h, 0, sizeof *h);
    h->poff = (uint64_t)s; h->plen = (uint64_t)(e - s);
    int64_t i = s;
    while (i < e) {
        int64_t ls = i;
        while (1) { if (i >= e) return SWC_ERR_REFERENCE_TRAP; if (in[i] == 0x20) break; i++; }
        int64_t length;
        if (!swift_int(in + ls, (uint64_t)(i - ls), &length)) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
        i++;
        int64_t ks = i;
        while (1) { if (i >= e) return SWC_ERR_REFERENCE_TRAP; if (in[i] == 0x3D) break; i++; }
        if (!utf8_ok(in + ks, (uint64_t)(i - ks))) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
        int64_t klen = i - ks;
        i++;
        int64_t vs = i;
        /* while i - lengthStartIndex + 1 < length: value bytes up to ls + length - 1 */
        int64_t need;
        if (i - ls + 1 < length) {
            if (__builtin_add_overflow(ls, length - 1, &need) || need >= e) return SWC_ERR_REFERENCE_TRAP;
            i = need;
        }
        if (i >= e) return SWC_ERR_REFERENCE_TRAP;
        if (in[i] != 0x0A) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
        int64_t ve = i;
        i++;
        if (!utf8_ok(in + vs, (uint64_t)(ve - vs))) continue;
        const char *k = (const char *)in + ks;
        const uint8_t *v = in + vs;
        uint64_t vl = (uint64_t)(ve - vs);
#define KEY(str) (klen == (int64_t)strlen(str) && !memcmp(k, str, klen))
        int64_t x;
        if (KEY("uid")) { if (swift_int(v, vl, &x)) { h->uid = x; h->present |= SWC_TAR_UID; } else h->present &= ~SWC_TAR_UID; }
        else if (KEY("gid")) { if (swift_int(v, vl, &x)) { h->gid = x; h->present |= SWC_TAR_GID; } else h->present &= ~SWC_TAR_GID; }
        else if (KEY("size")) { h->has_size = swift_int(v, vl, &x); h->size = x; }
        else {
            static const char *names[9] = {"mtime", "atime", "ctime", "uname", "gname", "path", "linkpath", "charset", "comment"};
            for (int r = 0; r < 9; r++)
                if (KEY(names[r])) { h->off[r] = (uint64_t)vs; h->len[r] = vl; h->has |= 1u << r; break; }
        }
#undef KEY
    }
    if (e > s && in[e - 1] != 0x0A) return SWC_TAR_WRONG_PAX_HEADER_ENTRY;
    return SWC_OK;
}

int swco_tar_walk(const uint8_t *in, uint64_t len, swc_tar_entry *entries, uint64_t cap, uint64_t *n_entries,
                  int32_t *info_st, int32_t *open_st, int32_t *format, int32_t *format_st) {
    const int64_t L = (int64_t)len;
    int64_t off = 0;
    pax g, l;
    int has_g = 0, has_l = 0, has_ln = 0, has_ll = 0;
    uint64_t ln_off = 0, ln_len = 0, ll_off = 0, ll_len = 0;
    uint64_t count = 0;
    int st = SWC_OK, ost = -1, fst = -1, fmt = SWC_TAR_PRE_POSIX, ustar_seen = 0;
    const uint64_t max_hops = 2 * ((len + 511) / 512) + 2;
    uint64_t hops = 0;
    while (1) {
        if (off >= L) break;                                              /* finished */
        if (off < 0) { st = SWC_ERR_REFERENCE_TRAP; break; }
        if (L - off >= 1024) {                                            /* EOF marker */
            int z = 1;
            for (int k = 0; k < 1024 && z; k++) z = in[off + k] == 0;
            if (z) break;
        }
        if (L - off < 512) { st = SWC_TAR_TOO_SMALL_FILE_IS_PASSED; break; }
        if (++hops > max_hops) { st = SWC_ERR_REFERENCE_TRAP; break; }  /* a block parsed a third time: a cycle */
        const uint8_t *h = in + off;
        int64_t mode, uid, gid, size, mtime, chk, dmaj = 0, dmin = 0, at = 0, ct = 0;
        int hm = tar_int(h + 100, 8, &mode), hu = tar_int(h + 108, 8, &uid), hg = tar_int(h + 116, 8, &gid);
        if (!tar_int(h + 124, 12, &size)) { st = SWC_TAR_WRONG_FIELD; break; }
        int ht = tar_int(h + 136, 12, &mtime);
        if (!tar_int(h + 148, 8, &chk)) { st = SWC_TAR_WRONG_HEADER_CHECKSUM; break; }
        uint64_t us = 0; int64_t ss = 0;
        for (int k = 0; k < 512; k++) {
            uint8_t b = (k >= 148 && k < 156) ? 0x20 : h[k];
            us += b; ss += (int8_t)b;
        }
        if (!(us == (uint64_t)chk || ss == chk)) { st = SWC_TAR_WRONG_HEADER_CHECKSUM; break; }
        const uint8_t tf = h[156];
        uint64_t magic = 0;
        for (int k = 7; k >= 0; k--) magic = magic << 8 | h[257 + k];
        int hf = SWC_TAR_PRE_POSIX, hdj = 0, hdn = 0, ha = 0, hc = 0;
        if (magic == 0x0020207261747375ull || magic == 0x3030007261747375ull || magic == 0x3030207261747375ull) {
            hdj = tar_int(h + 329, 8, &dmaj); hdn = tar_int(h + 337, 8, &dmin);
            if (magic == 0x0020207261747375ull) { ha = tar_int(h + 345, 12, &at); hc = tar_int(h + 357, 12, &ct); hf = SWC_TAR_GNU; }
            else hf = SWC_TAR_USTAR;
        }
        const int64_t ds = off + 512;
        if (tf == 'L' || tf == 'K' || tf == 'g' || tf == 'x' || tf == 'X') {
            int64_t de;
            if (size < 0 || add_ovf(ds, size, &de) || de > L) { st = SWC_ERR_REFERENCE_TRAP; break; }
            if (tf == 'g' || tf == 'x' || tf == 'X') {
                pax *t = tf == 'g' ? &g : &l;
                int r = parse_pax(in, ds, de, t);
                if (r) { st = r; break; }
                if (tf == 'g') has_g = 1; else has_l = 1;
            } else if (tf == 'L') { has_ln = 1; ln_off = (uint64_t)ds; ln_len = cstr_len(in + ds, (uint64_t)size); }
            else { has_ll = 1; ll_off = (uint64_t)ds; ll_len = cstr_len(in + ds, (uint64_t)size); }
            if (add_ovf(ds, round512(size), &off)) { st = SWC_ERR_REFERENCE_TRAP; break; }
            if (fst < 0 && (tf == 'g' || tf == 'x')) { fst = SWC_OK; fmt = SWC_TAR_PAX; }
            if (fst < 0 && (tf == 'L' || tf == 'K')) { fst = SWC_OK; fmt = SWC_TAR_GNU; }
            continue;
        }
        /* TarEntryInfo.init */
        swc_tar_entry e;
        memset(&e, 0, sizeof e);
        e.header_off = (uint64_t)off; e.data_off = (uint64_t)ds; e.typeflag = tf;
        const pax *lp = has_l ? &l : NULL, *gp = has_g ? &g : NULL;
        if (hm) { e.mode = mode & 0xFFF; e.present |= SWC_TAR_MODE; }
        if (lp && (lp->present & SWC_TAR_UID)) { e.uid = lp->uid; e.present |= SWC_TAR_UID; }
        else if (gp && (gp->present & SWC_TAR_UID)) { e.uid = gp->uid; e.present |= SWC_TAR_UID; }
        else if (hu) { e.uid = uid; e.present |= SWC_TAR_UID; }
        if (lp && (lp->present & SWC_TAR_GID)) { e.gid = lp->gid; e.present |= SWC_TAR_GID; }
        else if (gp && (gp->present & SWC_TAR_GID)) { e.gid = gp->gid; e.present |= SWC_TAR_GID; }
        else if (hg) { e.gid = gid; e.present |= SWC_TAR_GID; }
        e.size = lp && lp->has_size ? lp->size : gp && gp->has_size ? gp->size : size;
        if (ht) { e.mtime = mtime; e.present |= SWC_TAR_MTIME; }
        if (ha) { e.atime = at; e.present |= SWC_TAR_ATIME; }
        if (hc) { e.ctime = ct; e.present |= SWC_TAR_CTIME; }
        if (hdj) { e.dev_major = dmaj; e.present |= SWC_TAR_DEV_MAJOR; }
        if (hdn) { e.dev_minor = dmin; e.present |= SWC_TAR_DEV_MINOR; }
        for (int k = 0; k < 3; k++) {
            if (lp && (lp->has >> k & 1)) { e.pax_time_off[k] = lp->off[k]; e.pax_time_len[k] = lp->len[k]; e.present |= SWC_TAR_PAX_TIME0 << k; }
            if (gp && (gp->has >> k & 1)) { e.pax_time_off[3 + k] = gp->off[k]; e.pax_time_len[3 + k] = gp->len[k]; e.present |= SWC_TAR_PAX_TIME0 << (3 + k); }
        }
#define PICK(r, O, N, BIT)                                                                  \
        if (lp && (lp->has >> r & 1)) { e.O = lp->off[r]; e.N = lp->len[r]; e.present |= BIT; } \
        else if (gp && (gp->has >> r & 1)) { e.O = gp->off[r]; e.N = gp->len[r]; e.present |= BIT; }
        PICK(3, uname_off, uname_len, SWC_TAR_UNAME)
        else if (hf != SWC_TAR_PRE_POSIX) { e.uname_off = (uint64_t)off + 265; e.uname_len = cstr_len(h + 265, 32); e.present |= SWC_TAR_UNAME; }
        PICK(4, gname_off, gname_len, SWC_TAR_GNAME)
        else if (hf != SWC_TAR_PRE_POSIX) { e.gname_off = (uint64_t)off + 297; e.gname_len = cstr_len(h + 297, 32); e.present |= SWC_TAR_GNAME; }
        PICK(5, name_off, name_len, 0)
        else if (has_ln) { e.name_off = ln_off; e.name_len = ln_len; }
        else {
            e.name_off = (uint64_t)off; e.name_len = cstr_len(h, 100);
            if (hf == SWC_TAR_USTAR && h[345]) { e.prefix_off = (uint64_t)off + 345; e.prefix_len = cstr_len(h + 345, 155); e.present |= SWC_TAR_PREFIX; }
        }
        PICK(6, link_off, link_len, 0)
        else if (has_ll) { e.link_off = ll_off; e.link_len = ll_len; }
        else { e.link_off = (uint64_t)off + 157; e.link_len = cstr_len(h + 157, 100); }
        PICK(7, charset_off, charset_len, SWC_TAR_CHARSET)
        PICK(8, comment_off, comment_len, SWC_TAR_COMMENT)
#undef PICK
        if (lp) { e.local_off = lp->poff; e.local_len = lp->plen; e.present |= SWC_TAR_LOCAL; }
        if (gp) { e.global_off = gp->poff; e.global_len = gp->plen; e.present |= SWC_TAR_GLOBAL; }
        const int is_dir = tf == '5';
        e.open_size = is_dir ? 0 : e.size;
        int64_t noff;                                                     /* TarParser.swift:73, before next() returns */
        if (add_ovf(ds, round512(size), &noff)) { st = SWC_ERR_REFERENCE_TRAP; break; }
        off = noff;
        if (count < cap) entries[count] = e;
        count++;
        has_l = has_ln = has_ll = 0;
        /* open's data bound (TarContainer.swift:197-211) */
        if (ost < 0 && !is_dir) {
            int64_t de;
            if (add_ovf(ds, e.size, &de)) ost = SWC_ERR_REFERENCE_TRAP;
            else if (!(de < L)) ost = SWC_TAR_TOO_SMALL_FILE_IS_PASSED;
            else if (de < ds) ost = SWC_ERR_REFERENCE_TRAP;
        }
        /* formatOf (TarContainer.swift:49-59) */
        if (fst < 0 && hf == SWC_TAR_GNU) { fst = SWC_OK; fmt = SWC_TAR_GNU; }
        if (hf == SWC_TAR_USTAR) ustar_seen = 1;
    }
    if (fst < 0) { fst = st; fmt = st == SWC_OK ? (ustar_seen ? SWC_TAR_USTAR : SWC_TAR_PRE_POSIX) : SWC_TAR_PRE_POSIX; }
    if (ost < 0) ost = st;
    if (count > cap) {
        if (st == SWC_OK) st = SWC_ERR_OUTPUT_OVERFLOW;
        if (ost == SWC_OK) ost = SWC_ERR_OUTPUT_OVERFLOW;
    }
    *n_entries = count; *info_st = st; *open_st = ost; *format = fmt; *format_st = fst;
    return SWC_OK;
}
