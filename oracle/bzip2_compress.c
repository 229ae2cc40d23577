/* bzip2_compress.c — ORACLE (test infrastructure): restatement of Sources/BZip2/BZip2+Compress.swift (BZip2
 * compression) with the helpers it calls: BurrowsWheeler.transform (BurrowsWheeler.swift:8-27), SuffixArray.make
 * (SuffixArray.swift, SA-IS as written), BZip2.lengths(from:) (BZip2+Lengths.swift), Code.huffmanCodes (Code.swift) and
 * EncodingTree (EncodingTree.swift).  Line references are to BZip2+Compress.swift unless a file is named.
 * Built on its own with checksums.c into libswco_bzip2c.so (swco_bzip2c.py); never linked into the product. */
#define _POSIX_C_SOURCE 200809L
#include <pthread.h>
#include <stdatomic.h>
#include <time.h>
#include "swco.h"

int swco_bzip2c_batch_mt(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint64_t n, uint64_t total,
                         int block_size, int nthreads, double *seconds, uint64_t *out_bytes, uint64_t *failures);
int swco_bzip2_compress(const uint8_t *data, size_t n, int block_size, swco_buf *out);
int swco_bzip2c_suffix_array(const int32_t *bytes, int64_t n, int32_t alphabet, int64_t *sa);
int swco_bzip2c_lengths(const int64_t *stats, int64_t n, int32_t *lengths);

/* ---- MsbBitWriter ---- */
typedef struct { swco_buf *b; uint32_t acc; int fill; int err; } msbw;

static void w_bit(msbw *w, int bit) {
    w->acc = (w->acc << 1) | (uint32_t)(bit & 1);
    if (++w->fill == 8) { if (swco_buf_push(w->b, (uint8_t)w->acc)) w->err = 1; w->acc = 0; w->fill = 0; }
}
static void w_num(msbw *w, uint64_t v, int bits) { for (int k = bits - 1; k >= 0; k--) w_bit(w, (int)((v >> k) & 1)); }
static void w_bits(msbw *w, const uint8_t *bits, int n) { for (int k = 0; k < n; k++) w_bit(w, bits[k]); }
static void w_align(msbw *w) { while (w->fill) w_bit(w, 0); }

/* ---- SuffixArray.swift: SA-IS, statement for statement ---- */
typedef struct {
    const int64_t *input; int64_t n;
    uint8_t *stype;                   /* typemap: 1 = sType, 0 = lType (n + 1 entries) */
    int64_t *heads, *tails; int64_t alpha;
} sa_state;

static int sa_make(const int64_t *bytes, int64_t n, int64_t alpha, int64_t *result /* n + 1 */);

static int is_lms(int64_t off, const sa_state *s) {
    if (off == 0) return 0;
    return s->stype[off] && !s->stype[off - 1];
}

static int lms_equal(int64_t a, int64_t b, const sa_state *s) {
    if (a == s->n || b == s->n) return 0;
    for (int64_t i = 0;; i++) {
        const int al = is_lms(a + i, s), bl = is_lms(b + i, s);
        if (i > 0 && al && bl) return 1;
        if (al != bl) return 0;
        if (s->input[i + a] != s->input[i + b]) return 0;
    }
}

static void induce(int64_t *sa, const sa_state *s, int64_t *heads, int64_t *tails) {
    memcpy(heads, s->heads, (size_t)s->alpha * 8);
    memcpy(tails, s->tails, (size_t)s->alpha * 8);
    for (int64_t i = 0; i < s->n + 1; i++) {
        const int64_t j = sa[i] - 1;
        if (!(j >= 0 && !s->stype[j])) continue;
        sa[heads[s->input[j]]++] = j;
    }
    for (int64_t i = s->n; i >= 0; i--) {
        const int64_t j = sa[i] - 1;
        if (!(j >= 0 && s->stype[j])) continue;
        sa[tails[s->input[j]]--] = j;
    }
}

static int sa_make(const int64_t *bytes, int64_t n, int64_t alpha, int64_t *result) {
    int rc = -1;
    sa_state s = {bytes, n, NULL, NULL, NULL, alpha};
    int64_t *sizes = calloc((size_t)alpha + 1, 8), *h = malloc(((size_t)alpha + 1) * 8), *t = malloc(((size_t)alpha + 1) * 8);
    int64_t *names = NULL, *sum_off = NULL, *sum_bytes = NULL, *sum_sa = NULL;
    s.stype = calloc((size_t)n + 1, 1);
    s.heads = calloc((size_t)alpha + 1, 8); s.tails = calloc((size_t)alpha + 1, 8);
    if (!sizes || !h || !t || !s.stype || !s.heads || !s.tails) goto done;
    /* State.init */
    s.stype[n] = 1;
    if (n != 0) { sizes[bytes[n - 1]]++; s.stype[n - 1] = 0; }
    for (int64_t i = n - 2; i >= 0; i--) {
        if (bytes[i] > bytes[i + 1]) s.stype[i] = 0;
        else if (bytes[i] == bytes[i + 1] && !s.stype[i + 1]) s.stype[i] = 0;
        else s.stype[i] = 1;
        sizes[bytes[i]]++;
    }
    int64_t offset = 1;
    for (int64_t c = 0; c < alpha; c++) { s.heads[c] = offset; offset += sizes[c]; s.tails[c] = offset - 1; }
    /* guessLMSSort */
    for (int64_t i = 0; i < n + 1; i++) result[i] = -1;
    memcpy(t, s.tails, (size_t)alpha * 8);
    for (int64_t i = 0; i < n; i++) {
        if (!is_lms(i, &s)) continue;
        result[t[bytes[i]]--] = i;
    }
    result[0] = n;
    induce(result, &s, h, t);
    /* Summary.init */
    names = malloc(((size_t)n + 1) * 8);
    sum_off = malloc(((size_t)n + 1) * 8);
    sum_bytes = malloc(((size_t)n + 1) * 8);
    if (!names || !sum_off || !sum_bytes) goto done;
    for (int64_t i = 0; i < n + 1; i++) names[i] = -1;
    int64_t name = 0, last = result[0];
    names[result[0]] = name;
    for (int64_t i = 1; i < n + 1; i++) {
        const int64_t off = result[i];
        if (!is_lms(off, &s)) continue;
        if (!lms_equal(last, off, &s)) name++;
        last = off;
        names[off] = name;
    }
    int64_t m = 0;
    for (int64_t i = 0; i < n + 1; i++) {
        if (names[i] == -1) continue;
        sum_off[m] = i; sum_bytes[m] = names[i]; m++;
    }
    const int64_t sum_alpha = name + 1;
    /* Summary.makeSuffixArray */
    sum_sa = malloc(((size_t)m + 1) * 8);
    if (!sum_sa) goto done;
    if (sum_alpha == m) {
        for (int64_t i = 0; i < m + 1; i++) sum_sa[i] = -1;
        sum_sa[0] = m;
        for (int64_t i = 0; i < m; i++) sum_sa[sum_bytes[i] + 1] = i;
    } else if (sa_make(sum_bytes, m, sum_alpha, sum_sa)) {
        goto done;
    }
    /* accurateLMSSort */
    for (int64_t i = 0; i < n + 1; i++) result[i] = -1;
    memcpy(t, s.tails, (size_t)alpha * 8);
    for (int64_t i = m; i > 1; i--) {
        const int64_t at = sum_off[sum_sa[i]];
        result[t[bytes[at]]--] = at;
    }
    result[0] = n;
    induce(result, &s, h, t);
    rc = 0;
done:
    free(sizes); free(h); free(t); free(s.stype); free(s.heads); free(s.tails);
    free(names); free(sum_off); free(sum_bytes); free(sum_sa);
    return rc;
}

int swco_bzip2c_suffix_array(const int32_t *bytes, int64_t n, int32_t alphabet, int64_t *sa) {
    int64_t *b = malloc(((size_t)n + 1) * 8);
    if (!b) return SWC_ERR_OUTPUT_OVERFLOW;
    for (int64_t i = 0; i < n; i++) b[i] = bytes[i];
    const int rc = sa_make(b, n, alphabet, sa);
    free(b);
    return rc ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
}

/* ---- BZip2+Lengths.swift ---- */
int swco_bzip2c_lengths(const int64_t *stats_in, int64_t n, int32_t *lengths) {
    if (n == 0) return SWC_OK;
    if (n == 1) { lengths[0] = 1; return SWC_OK; }
    int64_t *stats = malloc((size_t)n * 8), *cl = calloc((size_t)n, 8), *others = malloc((size_t)n * 8), *bits = calloc((size_t)n, 8);
    if (!stats || !cl || !others || !bits) { free(stats); free(cl); free(others); free(bits); return SWC_ERR_OUTPUT_OVERFLOW; }
    memcpy(stats, stats_in, (size_t)n * 8);
    for (int64_t i = 0; i < n; i++) others[i] = -1;
    for (;;) {                                                  /* calculateCodeLengths */
        int64_t c1 = -1, minf = INT64_MAX;
        for (int64_t i = 0; i < n; i++)
            if (stats[i] > 0 && stats[i] <= minf) { minf = stats[i]; c1 = i; }
        int64_t c2 = -1;
        minf = INT64_MAX;
        for (int64_t i = 0; i < n; i++)
            if (stats[i] > 0 && stats[i] <= minf && i != c1) { minf = stats[i]; c2 = i; }
        if (c2 < 0) break;
        stats[c1] += stats[c2];
        stats[c2] = 0;
        cl[c1]++;
        while (others[c1] >= 0) { c1 = others[c1]; cl[c1]++; }
        others[c1] = c2;
        cl[c2]++;
        while (others[c2] >= 0) { c2 = others[c2]; cl[c2]++; }
    }
    for (int64_t i = 0; i < n; i++) bits[cl[i]]++;                /* count */
    for (int64_t i = n - 1; i > 20; i--) {                         /* adjust */
        while (bits[i] > 0) {
            int64_t j = i - 2;
            while (bits[j] == 0) j--;
            bits[i] -= 2; bits[i - 1] += 1; bits[j + 1] += 2; bits[j] -= 1;
        }
    }
    int64_t sym = 0;                                               /* generateSizeTable */
    const int64_t top = n - 1 < 20 ? n - 1 : 20;
    for (int64_t i = 1; i <= top; i++)
        for (int64_t j = 1; j <= bits[i]; j++) lengths[sym++] = (int32_t)i;
    for (; sym < n; sym++) lengths[sym] = 0;                       /* never reached: every symbol has a length */
    free(stats); free(cl); free(others); free(bits);
    return SWC_OK;
}

/* ---- process(_:_:) :76-262 ---- */
static const uint8_t block_marker[48] = {0, 0, 1, 1, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0, 1, 0, 1, 0, 1, 1, 0, 0, 1,
                                         0, 0, 1, 0, 0, 1, 1, 0, 0, 1, 0, 1, 0, 0, 1, 1, 0, 1, 0, 1, 1, 0, 0, 1};
static const uint8_t eos_marker[48] = {0, 0, 0, 1, 0, 1, 1, 1, 0, 1, 1, 1, 0, 0, 1, 0, 0, 1, 0, 0, 0, 1, 0, 1,
                                       0, 0, 1, 1, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 1, 0, 0, 1, 0, 0, 0, 0};

typedef struct { int32_t len[258]; uint32_t code[258]; int count; } table_t;

/* Code.huffmanCodes + EncodingTree: the canonical code in (length, symbol) order, reversed and reversed back */
static void make_table(const int32_t *lengths, int count, table_t *t) {
    t->count = count;
    int order[258];
    for (int i = 0; i < count; i++) order[i] = i;
    for (int i = 1; i < count; i++) {                              /* lengths.sorted(): by length, then symbol */
        const int v = order[i];
        int j = i - 1;
        while (j >= 0 && (lengths[order[j]] > lengths[v] || (lengths[order[j]] == lengths[v] && order[j] > v))) { order[j + 1] = order[j]; j--; }
        order[j + 1] = v;
    }
    int64_t symbol = -1, loop_bits = -1;
    for (int k = 0; k < count; k++) {
        const int s = order[k];
        if (lengths[s] <= 0) continue;
        symbol++;
        if (lengths[s] != loop_bits) { symbol <<= (lengths[s] - loop_bits); loop_bits = lengths[s]; }
        t->len[s] = lengths[s];
        t->code[s] = (uint32_t)symbol;
    }
}

static int64_t bit_size(const table_t *t, const int64_t *stats, int count) {
    int64_t total = 0;
    for (int s = 0; s < count; s++) if (stats[s] > 0) total += stats[s] * t->len[s];
    return total;
}

static int process(const uint8_t *block, size_t bn, msbw *w) {
    int rc = SWC_ERR_OUTPUT_OVERFLOW;
    /* initialRle :265-283 */
    int64_t *rle = malloc((bn + bn / 4 + 8) * 8), *dbl = NULL, *sa = NULL;
    int32_t *bwt = NULL, *out = NULL;
    uint8_t *sel = NULL;
    table_t *tables = NULL;
    if (!rle) return rc;
    size_t rn = 0;
    for (size_t i = 0; i < bn; i++) {
        int run = 1;
        while (i + 1 < bn && block[i] == block[i + 1] && run < 255) { run++; i++; }
        for (int k = 0; k < (run < 4 ? run : 4); k++) rle[rn++] = block[i];
        if (run >= 4) rle[rn++] = run - 4;
    }
    /* BurrowsWheeler.transform */
    dbl = malloc((2 * rn + 1) * 8); sa = malloc((2 * rn + 1) * 8); bwt = malloc((rn + 1) * 4);
    if (!dbl || !sa || !bwt) goto done;
    memcpy(dbl, rle, rn * 8); memcpy(dbl + rn, rle, rn * 8);
    if (sa_make(dbl, (int64_t)(2 * rn), 256, sa)) goto done;
    size_t bw = 0, pointer = 0;
    for (size_t i = 1; i < 2 * rn + 1; i++) {
        const int64_t x = sa[i];
        if (x < (int64_t)rn) bwt[bw++] = (int32_t)(x > 0 ? rle[x - 1] : rle[rn - 1]);
        else if (x == (int64_t)rn) pointer = bw;
    }
    /* Set(out).sorted(), mtfRle :299-349 */
    int used[256] = {0}, nused = 0, dict[256];
    for (size_t i = 0; i < rn; i++) used[bwt[i]] = 1;
    for (int c = 0; c < 256; c++) if (used[c]) dict[nused++] = c;
    out = malloc((rn + 2) * 4);
    if (!out) goto done;
    size_t on = 0;
    int64_t zrun = 0;
    int max_symbol = 1;
    for (size_t i = 0; i < rn; i++) {
        int idx = 0;
        while (dict[idx] != bwt[i]) idx++;
        if (idx == 0) zrun++;
        if ((idx == 0 && i == rn - 1) || idx != 0) {
            if (zrun > 0) {
                int digits = 0;
                for (int64_t v = zrun + 1; v > 1; v >>= 1) digits++;   /* floor(log2(zrun + 1)) */
                int64_t rem = zrun;
                for (int d = 0; d < digits; d++) {
                    const int64_t q = (rem + 1) / 2 - 1;               /* ceil(rem / 2) - 1 */
                    out[on++] = rem - 2 * q == 1 ? 0 : 1;
                    rem = q;
                }
                zrun = 0;
            }
        }
        if (idx != 0) {
            out[on++] = idx + 1;
            if (idx + 1 > max_symbol) max_symbol = idx + 1;
        }
        const int old = dict[idx];
        memmove(dict + 1, dict, (size_t)idx * sizeof(int));
        dict[0] = old;
    }
    out[on++] = max_symbol + 1;
    /* table choice :93-148 */
    const int A = max_symbol + 2;
    int64_t stats[258];
    int32_t lens[258];
    tables = malloc(7 * sizeof(table_t));
    sel = malloc(on / 50 + 2);
    if (!tables || !sel) goto done;
    int ntab = 0;
    size_t nsel = 0;
    int processed = 50;
    for (int s = 0; s < A; s++) stats[s] = 1;
    for (size_t i = 0; i < on; i++) {
        stats[out[i]]++;
        processed--;
        if (processed <= 0 || i == on - 1) {
            processed = 50;
            int64_t min_size = INT64_MAX;
            int min_sel = -1;
            for (int t = 0; t < ntab; t++) {
                const int64_t b = bit_size(&tables[t], stats, A);
                if (b < min_size) { min_size = b; min_sel = t; }
            }
            if (ntab == 6) {
                sel[nsel++] = (uint8_t)min_sel;
            } else {
                swco_bzip2c_lengths(stats, A, lens);
                make_table(lens, A, &tables[ntab]);
                if (bit_size(&tables[ntab], stats, A) < min_size) { sel[nsel++] = (uint8_t)ntab; ntab++; }
                else sel[nsel++] = (uint8_t)min_sel;
            }
            for (int s = 0; s < A; s++) stats[s] = 1;
        }
    }
    if (ntab == 1) { tables[1] = tables[0]; ntab = 2; }
    /* block header :150-221 */
    w_bit(w, 0);
    w_num(w, pointer, 24);
    uint8_t map[16] = {0};
    for (int k = 0; k < nused; k++) map[dict[k] / 16] = 1;     /* dict still holds the used bytes */
    w_bits(w, map, 16);
    for (int i = 0; i < 16; i++) {
        if (!map[i]) continue;
        for (int j = 0; j < 16; j++) w_bit(w, used[i * 16 + j]);
    }
    w_num(w, (uint64_t)ntab, 3);
    w_num(w, nsel, 15);
    int mtf[6] = {0, 1, 2, 3, 4, 5};
    for (size_t i = 0; i < nsel; i++) {                          /* mtf(_:maxValue:) :286-297 */
        int idx = 0;
        while (mtf[idx] != sel[i]) idx++;
        for (int k = 0; k < idx; k++) w_bit(w, 1);
        w_bit(w, 0);
        memmove(mtf + 1, mtf, (size_t)idx * sizeof(int));
        mtf[0] = sel[i];
    }
    for (int t = 0; t < ntab; t++) {
        int prev = tables[t].len[0];
        w_num(w, (uint64_t)prev, 5);
        for (int s = 0; s < A; s++) {
            const int l = tables[t].len[s];
            if (prev > l) w_num(w, (1ull << (2 * (prev - l))) - 1, 2 * (prev - l));
            else if (prev < l) w_num(w, ((1ull << (2 * (l - prev))) - 1) * 2 / 3, 2 * (l - prev));
            prev = l;
            w_bit(w, 0);
        }
    }
    /* contents :223-240 */
    size_t si = 0;
    int encoded = 0;
    const table_t *tab = &tables[sel[si++]];
    for (size_t i = 0; i < on; i++) {
        if (encoded >= 50) { tab = &tables[sel[si++]]; encoded = 0; }
        w_num(w, tab->code[out[i]], tab->len[out[i]]);
        encoded++;
    }
    rc = w->err ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
done:
    free(rle); free(dbl); free(sa); free(bwt); free(out); free(sel); free(tables);
    return rc;
}

/* compress(data:blockSize:) :44-74 */
int swco_bzip2_compress(const uint8_t *data, size_t n, int block_size, swco_buf *out) {
    if (block_size < 1 || block_size > 9) return SWC_ERR_INVALID_ARG;
    msbw w = {out, 0, 0, 0};
    const size_t raw = (size_t)block_size * 100 * 800;
    w_num(&w, 0x425a, 16);
    w_num(&w, 0x68, 8);
    w_num(&w, (uint64_t)(block_size + 0x30), 8);
    uint32_t total = 0;
    for (size_t i = 0; i < n; i += raw) {
        const size_t bn = n - i < raw ? n - i : raw;
        const uint32_t crc = swco_bzip2_crc32(data + i, bn);
        total = (total << 1) | (total >> 31);
        total ^= crc;
        w_bits(&w, block_marker, 48);
        w_num(&w, crc, 32);
        const int st = process(data + i, bn, &w);
        if (st) return st;
    }
    w_bits(&w, eos_marker, 48);
    w_num(&w, total, 32);
    w_align(&w);
    return w.err ? SWC_ERR_OUTPUT_OVERFLOW : SWC_OK;
}

/* The CPU arm of the compression benchmark: `total` units (wrapping over the n given ones) through swco_bzip2_compress
 * on `nthreads` pthreads, handed out through one atomic counter.  `out_bytes` counts compressed bytes. */
typedef struct {
    const uint8_t *base;
    const uint64_t *off, *len;
    uint64_t n, total;
    int block_size;
    atomic_ullong next, bytes, failures;
} bzip2c_job_t;

static void *bzip2c_worker(void *arg) {
    bzip2c_job_t *j = (bzip2c_job_t *)arg;
    unsigned long long bytes = 0, fails = 0;
    for (;;) {
        const unsigned long long k = atomic_fetch_add_explicit(&j->next, 1, memory_order_relaxed);
        if (k >= j->total) break;
        const uint64_t i = k % j->n;
        swco_buf out = {0, 0, 0};
        if (swco_bzip2_compress(j->base + j->off[i], (size_t)j->len[i], j->block_size, &out) != 0) fails++;
        bytes += out.len;
        free(out.data);
    }
    atomic_fetch_add(&j->bytes, bytes);
    atomic_fetch_add(&j->failures, fails);
    return NULL;
}

int swco_bzip2c_batch_mt(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint64_t n, uint64_t total,
                         int block_size, int nthreads, double *seconds, uint64_t *out_bytes, uint64_t *failures) {
    if (n == 0 || nthreads < 1) return -1;
    bzip2c_job_t j;
    j.base = base; j.off = off; j.len = len; j.n = n; j.total = total; j.block_size = block_size;
    atomic_init(&j.next, 0); atomic_init(&j.bytes, 0); atomic_init(&j.failures, 0);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    if (!th) return -1;
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    int started = 0;
    for (; started < nthreads; started++)
        if (pthread_create(&th[started], NULL, bzip2c_worker, &j) != 0) break;
    for (int i = 0; i < started; i++) pthread_join(th[i], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    free(th);
    if (started == 0) return -1;
    *seconds = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
    *out_bytes = atomic_load(&j.bytes);
    *failures = atomic_load(&j.failures);
    return 0;
}
