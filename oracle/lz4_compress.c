/* lz4_compress.c — ORACLE (test infrastructure): restatement of Sources/LZ4/LZ4+Compress.swift:16-298, the LZ4 frame
 * compressor.  Line references are to that file.  The reference cannot fail; the inputs on which it traps (a failed
 * precondition or an invalid range) return SWC_ERR_REFERENCE_TRAP here.
 * Built on its own with checksums.c into libswco_lz4c.so (swco_lz4c.py); never linked into the product. */
#define _POSIX_C_SOURCE 200809L
#include <pthread.h>
#include <stdatomic.h>
#include <time.h>
#include "swco.h"

int swco_lz4_block_compress(const uint8_t *block, size_t block_len, const uint8_t *dict, size_t dict_len, swco_buf *out);
int swco_lz4_compress(const uint8_t *data, size_t n, int independent, int block_checksums, int content_checksum,
                      int content_size, int64_t block_size, const uint8_t *dict /* NULL = nil */, size_t dict_len,
                      int has_dict_id, uint32_t dict_id, swco_buf *out);
int swco_lz4c_batch_mt(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint64_t n, uint64_t total,
                       int nthreads, double *seconds, uint64_t *out_bytes, uint64_t *failures);

/* matchStorage: [UInt32: Int] keyed by the exact four bytes (:160, :177-178, :279-288).  Open addressing over exact keys:
 * no buckets are shared between keys, so a lookup finds the last position stored under that very key. */
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
    size_t h = (size_t)((k * 2654435761u) >> 7) & s->mask;
    while (s->pos[h] >= 0 && s->key[h] != k) h = (h + 1) & s->mask;
    return h;
}

/* combine(_:from:) :290-298 */
static inline uint32_t combine(const uint8_t *b, size_t i) {
    return (uint32_t)b[i] << 24 | (uint32_t)b[i + 1] << 16 | (uint32_t)b[i + 2] << 8 | (uint32_t)b[i + 3];
}

/* the "count - 15, emit min(255, rest), subtract 255 while >= 0" length bytes of :222-230 and :240-248 */
static int put_len(swco_buf *out, long long rest) {
    while (rest >= 0) {
        if (swco_buf_push(out, rest > 255 ? 255 : (uint8_t)rest)) return -1;
        rest -= 255;
    }
    return 0;
}

/* compress(block:_:) :156-277 — appends the raw compressed block to `out`.  `dict` is used as given (the frame layer
 * passes at most its last 64 KiB). */
int swco_lz4_block_compress(const uint8_t *block, size_t block_len, const uint8_t *dict, size_t dict_len, swco_buf *out) {
    if (dict_len >= 1 && dict_len <= 3) return SWC_ERR_REFERENCE_TRAP;        /* :283 `0 ..< dict.endIndex - 4` is invalid */
    const size_t end = dict_len + block_len;                                  /* blockBytes.endIndex */
    uint8_t *bytes = (uint8_t *)malloc(end ? end : 1);
    if (!bytes) return SWC_ERR_OUTPUT_OVERFLOW;
    if (dict_len) memcpy(bytes, dict, dict_len);                              /* :159 */
    if (block_len) memcpy(bytes + dict_len, block, block_len);                /* :162 */
    storage_t st;
    if (storage_init(&st, end)) { free(bytes); return SWC_ERR_OUTPUT_OVERFLOW; }
    int status = SWC_OK;
#define PUT(v) do { if (swco_buf_push(out, (uint8_t)(v))) { status = SWC_ERR_OUTPUT_OVERFLOW; goto done; } } while (0)
    for (size_t i = 0; dict_len && i < dict_len - 4; i++) {                   /* populateMatchStorage :279-288 */
        const size_t h = storage_slot(&st, combine(bytes, i));
        st.key[h] = combine(bytes, i); st.pos[h] = (int64_t)i;
    }
    size_t i = dict_len;                                                      /* :161 */
    size_t lit_start = i, lit_count = 0;                                      /* currentLiterals: always bytes[lit_start ..< i] */
    while ((long long)i < (long long)end - 9) {                               /* :176 */
        const uint32_t id = combine(bytes, i);
        const size_t h = storage_slot(&st, id);
        if (st.pos[h] < 0) {                                                  /* :178-185 */
            st.key[h] = id; st.pos[h] = (int64_t)i;
            lit_count++; i++;
            continue;
        }
        const size_t match_start = (size_t)st.pos[h];
        st.pos[h] = (int64_t)i;                                               /* :187 */
        size_t match_length = 4;                                              /* :190 */
        size_t match_index = match_start + match_length;
        const size_t distance = i - match_start;
        if (distance > 65535) { lit_count++; i++; continue; }                 /* :195-199 */
        while ((long long)(i + match_length) < (long long)end - 5 && bytes[i + match_length] == bytes[match_index]) {  /* :205 */
            match_length++; match_index++;
        }
        if (end - i < 12) break;                                              /* :210-214 */
        PUT((lit_count < 15 ? lit_count : 15) << 4 | (match_length - 4 < 15 ? match_length - 4 : 15));   /* :218-220 */
        if (put_len(out, (long long)lit_count - 15)) { status = SWC_ERR_OUTPUT_OVERFLOW; goto done; }   /* :222-230 */
        if (swco_buf_append(out, bytes + lit_start, lit_count)) { status = SWC_ERR_OUTPUT_OVERFLOW; goto done; }  /* :231-233 */
        PUT(distance & 0xFF); PUT((distance >> 8) & 0xFF);                    /* :235-236 */
        i += match_length;                                                    /* :239 */
        if (put_len(out, (long long)match_length - 19)) { status = SWC_ERR_OUTPUT_OVERFLOW; goto done; }  /* :240-248 */
        lit_start = i; lit_count = 0;                                         /* :249 */
    }
    lit_count += end - i;                                                     /* :254-257 */
    /* :261 `assert(currentLiterals.count > 0)` only fails for an empty block; asserts are compiled out of the reference's
     * release builds, which write the single token 0x00 below, and so does this restatement */
    PUT((lit_count < 15 ? lit_count : 15) << 4);                              /* :262 */
    if (put_len(out, (long long)lit_count - 15)) { status = SWC_ERR_OUTPUT_OVERFLOW; goto done; }   /* :263-271 */
    if (swco_buf_append(out, bytes + lit_start, lit_count)) status = SWC_ERR_OUTPUT_OVERFLOW;     /* :272-274 */
done:
#undef PUT
    storage_free(&st);
    free(bytes);
    return status;
}

static int put32(swco_buf *out, uint32_t v) {
    const uint8_t b[4] = {(uint8_t)v, (uint8_t)(v >> 8), (uint8_t)(v >> 16), (uint8_t)(v >> 24)};
    return swco_buf_append(out, b, 4);
}

/* compress(data:independentBlocks:blockChecksums:contentChecksum:contentSize:blockSize:dictionary:dictionaryID:) :47-154.
 * dict == NULL is `dictionary: nil`; has_dict_id == 0 is `dictionaryID: nil`.  The frame is appended to `out`. */
int swco_lz4_compress(const uint8_t *data, size_t n, int independent, int block_checksums, int content_checksum,
                      int content_size, int64_t block_size, const uint8_t *dict, size_t dict_len, int has_dict_id,
                      uint32_t dict_id, swco_buf *out) {
    if (!(block_size <= 4 * 1024 * 1024 && block_size > 0)) return SWC_ERR_REFERENCE_TRAP;    /* :51 */
    const size_t bs = (size_t)block_size;
    const size_t start = out->len;
    uint8_t hdr[19];
    size_t h = 0;
    hdr[h++] = 0x04; hdr[h++] = 0x22; hdr[h++] = 0x4D; hdr[h++] = 0x18;                     /* :55 */
    hdr[h++] = (uint8_t)(0x40 | (independent ? 0x20 : 0) | (block_checksums ? 0x10 : 0) | (content_size ? 0x8 : 0) |
                         (content_checksum ? 0x4 : 0) | (has_dict_id ? 0x1 : 0));               /* :58-63 */
    hdr[h++] = bs <= 64 * 1024 ? 0x40 : bs <= 256 * 1024 ? 0x50 : bs <= 1024 * 1024 ? 0x60 : 0x70;   /* :66-76 */
    if (content_size) for (int k = 0; k < 8; k++) hdr[h++] = (uint8_t)((uint64_t)n >> (8 * k));  /* :78-83 */
    if (has_dict_id) for (int k = 0; k < 4; k++) hdr[h++] = (uint8_t)(dict_id >> (8 * k));        /* :85-89 */
    const uint32_t hc = swco_xxh32(hdr + 4, h - 4);                                              /* :92-93 */
    hdr[h++] = (uint8_t)((hc >> 8) & 0xFF);
    if (swco_buf_append(out, hdr, h)) return SWC_ERR_OUTPUT_OVERFLOW;

    const uint8_t *d = NULL;                                                                     /* :95-101 */
    size_t dl = 0;
    if (dict) { dl = dict_len > 64 * 1024 ? 64 * 1024 : dict_len; d = dict + (dict_len - dl); }
    swco_buf blk; swco_buf_init(&blk);
    int status = SWC_OK;
    for (size_t i = 0; i < n; i += bs) {                                                         /* :103 */
        const size_t len = n - i < bs ? n - i : bs;
        const uint8_t *block = data + i;
        blk.len = 0;
        if ((status = swco_lz4_block_compress(block, len, d, dl, &blk))) goto done;              /* :105 */
        if (!independent) { dl = len > 64 * 1024 ? 64 * 1024 : len; d = block + (len - dl); }   /* :106-110 */
        const int stored = blk.len > len;                                                        /* :112 */
        const uint8_t *payload = stored ? block : blk.data;
        const size_t plen = stored ? len : blk.len;
        if (put32(out, (stored ? 0x80000000u : 0u) | (uint32_t)plen) || swco_buf_append(out, payload, plen) ||
            (block_checksums && put32(out, swco_xxh32(payload, plen)))) { status = SWC_ERR_OUTPUT_OVERFLOW; goto done; }  /* :113-139 */
    }
    if (put32(out, 0) || (content_checksum && put32(out, swco_xxh32(data, n)))) status = SWC_ERR_OUTPUT_OVERFLOW;  /* :143-151 */
done:
    swco_buf_free(&blk);
    if (status) out->len = start;
    return status;
}

/* The CPU arm of the compression benchmark: `total` raw blocks (wrapping over the n given ones) through
 * swco_lz4_block_compress on `nthreads` pthreads, handed out through one atomic counter, as batch_mt.c does for the
 * decoders.  `out_bytes` counts compressed bytes.  Returns 0, or -1 if no thread could start. */
typedef struct {
    const uint8_t *base;
    const uint64_t *off, *len;
    uint64_t n, total;
    atomic_ullong next, bytes, failures;
} lz4c_job_t;

static void *lz4c_worker(void *arg) {
    lz4c_job_t *j = (lz4c_job_t *)arg;
    unsigned long long bytes = 0, fails = 0;
    for (;;) {
        const unsigned long long k = atomic_fetch_add_explicit(&j->next, 1, memory_order_relaxed);
        if (k >= j->total) break;
        const uint64_t i = k % j->n;
        swco_buf out = {0, 0, 0};
        if (swco_lz4_block_compress(j->base + j->off[i], (size_t)j->len[i], NULL, 0, &out) != 0) fails++;
        bytes += out.len;
        free(out.data);
    }
    atomic_fetch_add(&j->bytes, bytes);
    atomic_fetch_add(&j->failures, fails);
    return NULL;
}

int swco_lz4c_batch_mt(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint64_t n, uint64_t total,
                       int nthreads, double *seconds, uint64_t *out_bytes, uint64_t *failures) {
    if (n == 0 || nthreads < 1) return -1;
    lz4c_job_t j;
    j.base = base; j.off = off; j.len = len; j.n = n; j.total = total;
    atomic_init(&j.next, 0); atomic_init(&j.bytes, 0); atomic_init(&j.failures, 0);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    if (!th) return -1;
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    int started = 0;
    for (; started < nthreads; started++)
        if (pthread_create(&th[started], NULL, lz4c_worker, &j) != 0) break;
    for (int i = 0; i < started; i++) pthread_join(th[i], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    free(th);
    if (started == 0) return -1;
    *seconds = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
    *out_bytes = atomic_load(&j.bytes);
    *failures = atomic_load(&j.failures);
    return 0;
}
