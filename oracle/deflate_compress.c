/* deflate_compress.c — ORACLE (test infrastructure): restatement of Sources/Deflate/Deflate+Compress.swift (Deflate
 * compression), GzipArchive.archive (Sources/GZip/GzipArchive.swift:126-241) and ZlibArchive.archive
 * (Sources/Zlib/ZlibArchive.swift:54-70).  Line references are to Deflate+Compress.swift unless a file is named.
 * Built on its own with checksums.c into libswco_deflatec.so (swco_deflatec.py); never linked into the product. */
#define _POSIX_C_SOURCE 200809L
#include <pthread.h>
#include <stdatomic.h>
#include <time.h>
#include "swco.h"

int swco_deflate_compress(const uint8_t *data, size_t n, swco_buf *out);
int swco_zlib_archive(const uint8_t *data, size_t n, swco_buf *out);
int swco_gzip_archive(const uint8_t *data, size_t n, const uint8_t *comment, size_t comment_len, int has_comment,
                      const uint8_t *name, size_t name_len, int has_name, int header_crc, int is_text, uint8_t os,
                      int has_mtime, int64_t mtime, size_t n_extra, const uint8_t *extra_ids, const uint64_t *extra_lens,
                      const uint8_t *extra_bytes, swco_buf *out);
int swco_deflatec_batch_mt(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint64_t n, uint64_t total,
                           int nthreads, double *seconds, uint64_t *out_bytes, uint64_t *failures);

/* matchStorage: [UInt32: Int] keyed by the exact three bytes (:139).  Open addressing over exact keys: a lookup finds
 * the last position stored under that very key. */
typedef struct { uint32_t *key; int64_t *pos; size_t mask; } storage_t;

static int storage_init(storage_t *s, size_t n_positions) {
    size_t cap = 16;
    while (cap < 2 * n_positions + 16) cap *= 2;
    s->key = (uint32_t *)malloc(cap * sizeof(uint32_t));
    s->pos = (int64_t *)malloc(cap * sizeof(int64_t));
    s->mask = cap - 1;
    if (!s->key || !s->pos) { free(s->key); free(s->pos); return -1; }
    for (size_t i = 0; i < cap; i++) s->pos[i] = -1;
    return 0;
}
static void storage_free(storage_t *s) { free(s->key); free(s->pos); }
static size_t storage_slot(const storage_t *s, uint32_t k) {
    size_t h = (size_t)((k * 2654435761u) >> 5) & s->mask;
    while (s->pos[h] >= 0 && s->key[h] != k) h = (h + 1) & s->mask;
    return h;
}

/* Constants.lengthBase / distanceBase (Deflate+Constants.swift), RFC 1951 3.2.5 */
static const int length_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99,
                                    115, 131, 163, 195, 227, 258};
static const int distance_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025,
                                      1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};

/* Constants.lengthCode[length - 3]: the length symbol */
static int length_symbol(int length) {
    int s = 28;
    while (length_base[s] > length) s--;
    return 257 + s;
}
/* (distanceBase.firstIndex { $0 > distance } ?? 30) - 1 */
static int distance_symbol(int distance) {
    int i = 0;
    while (i < 30 && distance_base[i] <= distance) i++;
    return i - 1;
}

/* the LsbBitWriter: bits go in from the least significant end of each byte */
typedef struct { swco_buf *out; uint32_t acc; int nbits; int fail; } bitw_t;
static void bw_bit(bitw_t *w, int bit) {
    w->acc |= (uint32_t)(bit & 1) << w->nbits;
    if (++w->nbits == 8) { if (swco_buf_push(w->out, (uint8_t)w->acc)) w->fail = 1; w->acc = 0; w->nbits = 0; }
}
static void bw_number(bitw_t *w, int number, int count) { for (int k = 0; k < count; k++) bw_bit(w, (number >> k) & 1); }
static void bw_align(bitw_t *w) { if (w->nbits) { if (swco_buf_push(w->out, (uint8_t)w->acc)) w->fail = 1; w->acc = 0; w->nbits = 0; } }
/* EncodingTree.code(symbol:) with reverseCodes: the code's bits, most significant first */
static void bw_code(bitw_t *w, int code, int len) { for (int k = len - 1; k >= 0; k--) bw_bit(w, (code >> k) & 1); }
static void bw_literal(bitw_t *w, int sym) {           /* Constants.staticHuffmanLiteralCodes */
    if (sym <= 143) bw_code(w, 0x30 + sym, 8);
    else if (sym <= 255) bw_code(w, 0x190 + sym - 144, 9);
    else if (sym <= 279) bw_code(w, sym - 256, 7);
    else bw_code(w, 0xC0 + sym - 280, 8);
}

/* lengthEncode(_:) :134-197 as codes (length << 32 | distance, or the byte with length 0) and stats (:140) */
typedef struct { uint64_t *code; size_t count; int64_t stats[316]; } bld_t;

static int length_encode(const uint8_t *data, size_t n, bld_t *b) {
    memset(b->stats, 0, sizeof(b->stats));
    b->count = 0;
    b->code = (uint64_t *)malloc((n + 1) * sizeof(uint64_t));
    storage_t st;
    if (!b->code || storage_init(&st, n)) { free(b->code); b->code = NULL; return -1; }
    uint64_t *codes = b->code;
    size_t i = 0;                                                                   /* :141 */
    while ((long long)i < (long long)n - 2) {                                       /* :143 */
        const uint8_t byte = data[i];
        const uint32_t match_id = (uint32_t)data[i] << 16 | (uint32_t)data[i + 1] << 8 | data[i + 2];   /* :145-147 */
        const size_t h = storage_slot(&st, match_id);
        if (st.pos[h] < 0) {                                                        /* :148-155 */
            st.key[h] = match_id; st.pos[h] = (int64_t)i;
            codes[b->count++] = byte;
            b->stats[byte]++;
            i++;
            continue;
        }
        const size_t match_start = (size_t)st.pos[h];
        st.pos[h] = (int64_t)i;                                                     /* :158 */
        size_t match_length = 3;                                                    /* :161 */
        size_t match_index = match_start + match_length;                            /* :163 */
        const size_t distance = i - match_start;                                    /* :165 */
        if (distance > 32768) {                                                     /* :166-171 */
            codes[b->count++] = byte;
            b->stats[byte]++;
            i++;
            continue;
        }
        while (i + match_length < n && data[i + match_length] == data[match_index] && match_length < 258) {   /* :173 */
            match_length++; match_index++;
        }
        codes[b->count++] = (uint64_t)match_length << 32 | distance;                /* :177-178 */
        b->stats[length_symbol((int)match_length)]++;                               /* :179 */
        b->stats[286 + distance_symbol((int)distance)]++;                           /* :180 */
        i += match_length;                                                          /* :181 */
    }
    while (i < n) {                                                                 /* :186-191 */
        codes[b->count++] = data[i];
        b->stats[data[i]]++;
        i++;
    }
    b->stats[256]++;                                                                /* :194 */
    storage_free(&st);
    return 0;
}

/* staticHuffmanBitSize(_:) :44-72, in bytes */
static uint64_t static_huffman_size(const int64_t *stats) {
    uint64_t bits = 3;
    for (int symbol = 0; symbol < 316; symbol++) {
        int code_size, extra;
        if (symbol <= 143) { code_size = 8; extra = 0; }
        else if (symbol <= 255) { code_size = 9; extra = 0; }
        else if (symbol <= 279) { code_size = 7; extra = symbol <= 260 ? 0 : ((symbol - 257) >> 2) - 1; }
        else if (symbol <= 285) { code_size = 8; extra = symbol == 285 ? 0 : ((symbol - 257) >> 2) - 1; }
        else { code_size = 5; extra = symbol == 286 || symbol == 287 ? 0 : ((symbol - 286) >> 1) - 1; }
        bits += (uint64_t)stats[symbol] * (uint64_t)(code_size + extra);
    }
    return bits % 8 == 0 ? bits / 8 : bits / 8 + 1;
}

/* compress(data:) :22-42 — appends the Deflate stream to `out` */
int swco_deflate_compress(const uint8_t *data, size_t n, swco_buf *out) {
    bld_t b;
    if (length_encode(data, n, &b)) return SWC_ERR_OUTPUT_OVERFLOW;
    const uint64_t uncomp = 1 + 2 + 2 + (uint64_t)n;                                /* :27 */
    const uint64_t stat = static_huffman_size(b.stats);                             /* :30 */
    int status = SWC_OK;
    if (uncomp <= stat && uncomp <= 65535) {                                        /* :35 createUncompressedBlock :74-83 */
        const unsigned nl = (unsigned)n ^ 0xFFFFu;
        const uint8_t hdr[5] = {1, (uint8_t)(n & 0xFF), (uint8_t)((n >> 8) & 0xFF), (uint8_t)(nl & 0xFF), (uint8_t)((nl >> 8) & 0xFF)};
        if (swco_buf_append(out, hdr, 5) || swco_buf_append(out, data, n)) status = SWC_ERR_OUTPUT_OVERFLOW;
    } else {                                                                        /* encodeHuffmanBlock :85-125 */
        bitw_t w = {out, 0, 0, 0};
        bw_bit(&w, 1);
        bw_bit(&w, 1); bw_bit(&w, 0);
        const uint64_t *codes = b.code;
        for (size_t k = 0; k < b.count; k++) {
            const uint64_t c = codes[k];
            if (c >> 32 == 0) { bw_literal(&w, (int)c); continue; }
            const int length = (int)(c >> 32), distance = (int)(c & 0xFFFFFFFFu);
            const int ls = length_symbol(length);
            const int lx = (ls >= 257 && ls <= 260) || ls == 285 ? 0 : ((ls - 257) >> 2) - 1;
            bw_literal(&w, ls);
            bw_number(&w, length - length_base[ls - 257], lx);
            const int ds = distance_symbol(distance);
            const int dx = ds == 0 || ds == 1 ? 0 : (ds >> 1) - 1;
            bw_code(&w, ds, 5);
            bw_number(&w, distance - distance_base[ds], dx);
        }
        bw_literal(&w, 256);                                                        /* :121 */
        bw_align(&w);
        if (w.fail) status = SWC_ERR_OUTPUT_OVERFLOW;
    }
    free(b.code);
    return status;
}

/* ZlibArchive.archive(data:) ZlibArchive.swift:54-70 */
int swco_zlib_archive(const uint8_t *data, size_t n, swco_buf *out) {
    const uint8_t hdr[2] = {120, 218};
    if (swco_buf_append(out, hdr, 2)) return SWC_ERR_OUTPUT_OVERFLOW;
    int st = swco_deflate_compress(data, n, out);
    if (st) return st;
    const uint32_t a = swco_adler32(data, n);
    const uint8_t t[4] = {(uint8_t)(a >> 24), (uint8_t)(a >> 16), (uint8_t)(a >> 8), (uint8_t)a};
    return swco_buf_append(out, t, 4) ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
}

/* GzipArchive.archive(data:comment:fileName:writeHeaderCRC:isTextFile:osType:modificationTime:extraFields:)
 * GzipArchive.swift:126-241.  comment / name are ISO-Latin-1 bytes (the caller encodes them and reports
 * cannotEncodeISOLatin1 itself); os is osTypeByte (255 for nil); mtime is Int(timeIntervalSince1970). */
int swco_gzip_archive(const uint8_t *data, size_t n, const uint8_t *comment, size_t comment_len, int has_comment,
                      const uint8_t *name, size_t name_len, int has_name, int header_crc, int is_text, uint8_t os,
                      int has_mtime, int64_t mtime, size_t n_extra, const uint8_t *extra_ids, const uint64_t *extra_lens,
                      const uint8_t *extra_bytes, swco_buf *out) {
    uint8_t flags = 0;
    if (has_comment) flags |= 1 << 4;                                               /* :133 */
    if (has_name) flags |= 1 << 3;                                                  /* :147 */
    if (n_extra) flags |= 1 << 2;                                                   /* :161 */
    if (header_crc) flags |= 1 << 1;                                                /* :165 */
    if (is_text) flags |= 1 << 0;                                                   /* :169 */
    uint8_t mt[4] = {0, 0, 0, 0};                                                   /* :175-181 */
    if (has_mtime) for (int i = 0; i < 4; i++) mt[i] = (uint8_t)(((uint64_t)mtime >> (8 * i)) & 0xFF);
    const size_t start = out->len;
    const uint8_t h[10] = {0x1f, 0x8b, 8, flags, mt[0], mt[1], mt[2], mt[3], 2, os};  /* :183-193 */
    int st = SWC_OK;
    if (swco_buf_append(out, h, 10)) return SWC_ERR_OUTPUT_OVERFLOW;
    if (n_extra) {                                                                  /* :195-214 */
        uint64_t xlen = 0;
        for (size_t i = 0; i < n_extra; i++) xlen += 4 + extra_lens[i];
        if (xlen > 65535) { out->len = start; return SWC_GZIP_CANNOT_ENCODE_ISO_LATIN1; }
        if (swco_buf_push(out, (uint8_t)(xlen & 0xFF)) || swco_buf_push(out, (uint8_t)((xlen >> 8) & 0xFF))) return SWC_ERR_OUTPUT_OVERFLOW;
        size_t at = 0;
        for (size_t i = 0; i < n_extra; i++) {
            const uint64_t len = extra_lens[i];
            const uint8_t f[4] = {extra_ids[2 * i], extra_ids[2 * i + 1], (uint8_t)(len & 0xFF), (uint8_t)((len >> 8) & 0xFF)};
            if (swco_buf_append(out, f, 4) || swco_buf_append(out, extra_bytes + at, (size_t)len)) return SWC_ERR_OUTPUT_OVERFLOW;
            at += (size_t)len;
        }
    }
    /* :216-219: the file name, then the comment; each gets a NUL unless its last character is one (:134-136, :148-150) */
    if (has_name && (swco_buf_append(out, name, name_len) || ((name_len == 0 || name[name_len - 1] != 0) && swco_buf_push(out, 0))))
        return SWC_ERR_OUTPUT_OVERFLOW;
    if (has_comment && (swco_buf_append(out, comment, comment_len) ||
                        ((comment_len == 0 || comment[comment_len - 1] != 0) && swco_buf_push(out, 0))))
        return SWC_ERR_OUTPUT_OVERFLOW;
    if (header_crc) {                                                               /* :221-226 */
        const uint32_t c = swco_crc32(out->data + start, out->len - start, 0);
        if (swco_buf_push(out, (uint8_t)(c & 0xFF)) || swco_buf_push(out, (uint8_t)((c >> 8) & 0xFF))) return SWC_ERR_OUTPUT_OVERFLOW;
    }
    if ((st = swco_deflate_compress(data, n, out))) return st;                      /* :228 */
    const uint32_t crc = swco_crc32(data, n, 0);                                     /* :230-235 */
    const uint32_t isize = (uint32_t)((uint64_t)n % ((uint64_t)1 << 32));           /* :237-242 */
    const uint8_t t[8] = {(uint8_t)crc, (uint8_t)(crc >> 8), (uint8_t)(crc >> 16), (uint8_t)(crc >> 24),
                          (uint8_t)isize, (uint8_t)(isize >> 8), (uint8_t)(isize >> 16), (uint8_t)(isize >> 24)};
    return swco_buf_append(out, t, 8) ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
}

/* The CPU arm of the compression benchmark: `total` units (wrapping over the n given ones) through swco_deflate_compress
 * on `nthreads` pthreads, handed out through one atomic counter.  `out_bytes` counts compressed bytes. */
typedef struct {
    const uint8_t *base;
    const uint64_t *off, *len;
    uint64_t n, total;
    atomic_ullong next, bytes, failures;
} deflatec_job_t;

static void *deflatec_worker(void *arg) {
    deflatec_job_t *j = (deflatec_job_t *)arg;
    unsigned long long bytes = 0, fails = 0;
    for (;;) {
        const unsigned long long k = atomic_fetch_add_explicit(&j->next, 1, memory_order_relaxed);
        if (k >= j->total) break;
        const uint64_t i = k % j->n;
        swco_buf out = {0, 0, 0};
        if (swco_deflate_compress(j->base + j->off[i], (size_t)j->len[i], &out) != 0) fails++;
        bytes += out.len;
        free(out.data);
    }
    atomic_fetch_add(&j->bytes, bytes);
    atomic_fetch_add(&j->failures, fails);
    return NULL;
}

int swco_deflatec_batch_mt(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint64_t n, uint64_t total,
                           int nthreads, double *seconds, uint64_t *out_bytes, uint64_t *failures) {
    if (n == 0 || nthreads < 1) return -1;
    deflatec_job_t j;
    j.base = base; j.off = off; j.len = len; j.n = n; j.total = total;
    atomic_init(&j.next, 0); atomic_init(&j.bytes, 0); atomic_init(&j.failures, 0);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    if (!th) return -1;
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    int started = 0;
    for (; started < nthreads; started++)
        if (pthread_create(&th[started], NULL, deflatec_worker, &j) != 0) break;
    for (int i = 0; i < started; i++) pthread_join(th[i], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    free(th);
    if (started == 0) return -1;
    *seconds = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
    *out_bytes = atomic_load(&j.bytes);
    *failures = atomic_load(&j.failures);
    return 0;
}
