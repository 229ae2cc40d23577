/* lzma.c — ORACLE (test infrastructure): restatement of
 *   Sources/LZMA/LZMA.swift:25-73, LZMAProperties.swift:49-64, LZMADecoder.swift:79-298, LZMARangeDecoder.swift:20-80,
 *   LZMABitTreeDecoder.swift:18-43, LZMALenDecoder.swift:14-38, LZMAConstants.swift,
 *   Sources/LZMA2/LZMA2.swift:25-36, LZMA2Decoder.swift:17-99.
 * Probabilities are u16 here (64-bit Int in the reference; values never exceed 2^11). The reference's flat
 * `probabilities` array has 432 entries but is indexed up to 432 (state=11,posState=15) — a trap; sized 448 here and
 * the access reported as SWC_ERR_REFERENCE_TRAP. */
#include "swco.h"

#define TOP_VALUE (1u << 24)
#define PROB_INIT 1024
#define NUM_POS_BITS_MAX 4

typedef struct {
    const uint8_t *in; size_t n, ip;   /* byte reader */
    int trap;                          /* read past the end (BitByteData precondition) */
    uint32_t range, code;
} rc_t;

typedef struct { uint16_t choice, choice2, low[16][8], mid[16][8], high[256]; } len_dec;

typedef struct {
    rc_t rc;
    int lc, lp, pb;
    int64_t dict_size;
    int64_t uncompressed_size;
    swco_buf *out;
    size_t out_base;                   /* out->len at decoder creation: the reference's `out` starts empty */
    int64_t dict_start, dict_end;
    int64_t rep0, rep1, rep2, rep3;
    int state;
    int tables_ready;                  /* resetStateAndDecoders() has run at least once */
    uint16_t probs[448];
    uint16_t *lit;                     /* (1 << (lc+lp)) * 0x300 */
    size_t lit_count;
    uint16_t pos_slot[4][64];
    uint16_t align[16];
    uint16_t pos_dec[1 + 128 - 14];    /* 1 + numFullDistances - endPosModelIndex = 115 */
    len_dec len, rep_len;
} lzma_dec;

static inline uint8_t rc_byte(rc_t *r) {
    if (r->ip >= r->n) { r->trap = 1; return 0; }
    return r->in[r->ip++];
}
static inline void rc_normalize(rc_t *r) {                               /* LZMARangeDecoder.swift:38-43 */
    if (r->range < TOP_VALUE) { r->range <<= 8; r->code = (r->code << 8) | rc_byte(r); }
}
static int rc_init(rc_t *r) {                                            /* LZMARangeDecoder.swift:20-31 */
    if (r->n - r->ip < 5) return SWC_LZMA_RANGE_DECODER_INIT_ERROR;
    uint8_t b = r->in[r->ip++];
    r->code = (uint32_t)r->in[r->ip] << 24 | (uint32_t)r->in[r->ip + 1] << 16 | (uint32_t)r->in[r->ip + 2] << 8 | r->in[r->ip + 3];
    r->ip += 4;
    r->range = 0xFFFFFFFFu;
    if (b != 0) return SWC_LZMA_RANGE_DECODER_INIT_ERROR;
    return SWC_OK;
}
static inline int rc_bit(rc_t *r, uint16_t *prob) {                      /* LZMARangeDecoder.swift:65-80 */
    uint32_t bound = (r->range >> 11) * (uint32_t)*prob;
    int sym;
    if (r->code < bound) { *prob += ((1 << 11) - *prob) >> 5; r->range = bound; sym = 0; }
    else { *prob -= *prob >> 5; r->code -= bound; r->range -= bound; sym = 1; }
    rc_normalize(r);
    return sym;
}
static inline int rc_direct(rc_t *r, int count) {                        /* LZMARangeDecoder.swift:46-62 (repeat-while: >= 1 pass) */
    uint32_t res = 0;
    do {
        r->range >>= 1;
        r->code -= r->range;
        uint32_t t = 0u - (r->code >> 31);
        r->code += r->range & t;
        rc_normalize(r);
        res = (res << 1) + (t + 1);
        count--;
    } while (count > 0);
    return (int)res;
}
static inline int bittree(rc_t *r, uint16_t *probs, int nbits) {         /* LZMABitTreeDecoder.swift:18-24 */
    int m = 1;
    for (int i = 0; i < nbits; i++) m = (m << 1) + rc_bit(r, &probs[m]);
    return m - (1 << nbits);
}
static inline int bittree_rev(rc_t *r, uint16_t *probs, int nbits) {     /* LZMABitTreeDecoder.swift:32-43 (probs already offset) */
    int m = 1, sym = 0;
    for (int i = 0; i < nbits; i++) { int b = rc_bit(r, &probs[m]); m = (m << 1) + b; sym |= b << i; }
    return sym;
}
static void len_init(len_dec *l) {
    l->choice = l->choice2 = PROB_INIT;
    for (int i = 0; i < 16; i++) for (int j = 0; j < 8; j++) l->low[i][j] = l->mid[i][j] = PROB_INIT;
    for (int i = 0; i < 256; i++) l->high[i] = PROB_INIT;
}
static inline int len_decode(rc_t *r, len_dec *l, int pos_state) {       /* LZMALenDecoder.swift:28-38 */
    if (rc_bit(r, &l->choice) == 0) return bittree(r, l->low[pos_state], 3);
    if (rc_bit(r, &l->choice2) == 0) return 8 + bittree(r, l->mid[pos_state], 3);
    return 16 + bittree(r, l->high, 8);
}

static int reset_state(lzma_dec *d) {                                    /* LZMADecoder.swift:79-100 */
    d->state = 0; d->rep0 = d->rep1 = d->rep2 = d->rep3 = 0;
    for (int i = 0; i < 448; i++) d->probs[i] = PROB_INIT;
    size_t cnt = ((size_t)1 << (d->lc + d->lp)) * 0x300;
    if (cnt != d->lit_count) {
        free(d->lit);
        d->lit = (uint16_t *)malloc(sizeof(uint16_t) * cnt);
        if (!d->lit) { d->lit_count = 0; return -1; }
        d->lit_count = cnt;
    }
    for (size_t i = 0; i < cnt; i++) d->lit[i] = PROB_INIT;
    for (int i = 0; i < 4; i++) for (int j = 0; j < 64; j++) d->pos_slot[i][j] = PROB_INIT;
    for (int i = 0; i < 16; i++) d->align[i] = PROB_INIT;
    for (int i = 0; i < 115; i++) d->pos_dec[i] = PROB_INIT;
    len_init(&d->len); len_init(&d->rep_len);
    d->tables_ready = 1;
    return 0;
}

static inline int put(lzma_dec *d, uint8_t b) {                          /* LZMADecoder.swift:288-294 */
    if (swco_buf_push(d->out, b)) return -1;
    d->dict_end += 1;
    if (d->dict_end - d->dict_start == d->dict_size) d->dict_start += 1;
    return 0;
}
/* byte(at:) LZMADecoder.swift:296-298; *trap set when the array index is out of range */
static inline uint8_t byte_at(lzma_dec *d, int64_t distance, int *trap) {
    int64_t idx = distance <= d->dict_end ? d->dict_end - distance : d->dict_size - distance + d->dict_end;
    if (idx < 0 || idx >= d->dict_end) { *trap = 1; return 0; }          /* out.count == dictEnd */
    return d->out->data[d->out_base + (size_t)idx];
}

/* LZMADecoder.decode() LZMADecoder.swift:107-284 */
static int lzma_decode(lzma_dec *d) {
    rc_t *r = &d->rc;
    int st = rc_init(r);
    if (st) return st;
    if (!d->tables_ready) {
        /* LZMA2 chunk with reset kind 0/1 before any props: `probabilities`/`literalProbs` are empty arrays -> trap.
           (reset kind 1 calls resetStateAndDecoders, so only kind 0 gets here.) An immediately finished chunk
           (uncompressedSize == 0 && code == 0) cannot occur: LZMA2 sizes are >= 1. */
        return SWC_ERR_REFERENCE_TRAP;
    }
    int trap = 0;
    const int pb_mask = (1 << d->pb) - 1, lp_mask = (1 << d->lp) - 1;
    for (;;) {
        if (r->trap || trap) return SWC_ERR_REFERENCE_TRAP;
        if (d->uncompressed_size == 0 && r->code == 0) break;                                     /* :112-114 */
        int pos_state = (int)(d->dict_end & pb_mask);
        if (rc_bit(r, &d->probs[(d->state << NUM_POS_BITS_MAX) + pos_state]) == 0) {             /* :119-172 literal */
            if (r->trap) return SWC_ERR_REFERENCE_TRAP;
            if (d->uncompressed_size == 0) return SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE;
            int prev = d->dict_end == d->dict_start ? 0 : byte_at(d, 1, &trap);
            int symbol = 1;
            size_t lit_state = (size_t)((d->dict_end & lp_mask) << d->lc) + (size_t)(prev >> (8 - d->lc));
            uint16_t *lp = d->lit + lit_state * 0x300;
            if (d->state >= 7) {
                unsigned match_byte = byte_at(d, d->rep0 + 1, &trap);
                if (trap) return SWC_ERR_REFERENCE_TRAP;
                do {
                    int match_bit = (match_byte >> 7) & 1;
                    match_byte = (match_byte << 1) & 0xFF;
                    int bit = rc_bit(r, &lp[((1 + match_bit) << 8) + symbol]);
                    symbol = (symbol << 1) | bit;
                    if (match_bit != bit) break;
                } while (symbol < 0x100);
            }
            while (symbol < 0x100) symbol = (symbol << 1) | rc_bit(r, &lp[symbol]);
            if (r->trap) return SWC_ERR_REFERENCE_TRAP;
            d->uncompressed_size -= 1;
            if (put(d, (uint8_t)(symbol - 0x100))) return SWC_ERR_OUTPUT_OVERFLOW;
            d->state = d->state < 4 ? 0 : (d->state < 10 ? d->state - 3 : d->state - 6);
            continue;
        }
        int64_t len;
        if (rc_bit(r, &d->probs[193 + d->state]) != 0) {                                          /* :176-215 rep */
            if (r->trap) return SWC_ERR_REFERENCE_TRAP;
            if (d->uncompressed_size == 0) return SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE;
            if (d->dict_end == d->dict_start) return SWC_LZMA_WINDOW_IS_EMPTY;
            if (rc_bit(r, &d->probs[205 + d->state]) == 0) {
                int idx = 241 + (d->state << NUM_POS_BITS_MAX) + pos_state;
                if (idx >= 432) return SWC_ERR_REFERENCE_TRAP;                                    /* 432-entry array */
                if (rc_bit(r, &d->probs[idx]) == 0) {
                    if (r->trap) return SWC_ERR_REFERENCE_TRAP;
                    d->state = d->state < 7 ? 9 : 11;
                    uint8_t b = byte_at(d, d->rep0 + 1, &trap);
                    if (trap) return SWC_ERR_REFERENCE_TRAP;
                    if (put(d, b)) return SWC_ERR_OUTPUT_OVERFLOW;
                    d->uncompressed_size -= 1;
                    continue;
                }
            } else {
                int64_t dist;
                if (rc_bit(r, &d->probs[217 + d->state]) == 0) {
                    dist = d->rep1;
                } else {
                    if (rc_bit(r, &d->probs[229 + d->state]) == 0) dist = d->rep2;
                    else { dist = d->rep3; d->rep3 = d->rep2; }
                    d->rep2 = d->rep1;
                }
                d->rep1 = d->rep0;
                d->rep0 = dist;
            }
            len = len_decode(r, &d->rep_len, pos_state);
            d->state = d->state < 7 ? 8 : 11;
        } else {                                                                                  /* :216-272 match */
            d->rep3 = d->rep2; d->rep2 = d->rep1; d->rep1 = d->rep0;
            len = len_decode(r, &d->len, pos_state);
            d->state = d->state < 7 ? 7 : 10;
            int len_state = len > 3 ? 3 : (int)len;
            int pos_slot = bittree(r, d->pos_slot[len_state], 6);
            if (pos_slot < 4) {
                d->rep0 = pos_slot;
            } else {
                int ndirect = (pos_slot >> 1) - 1;
                int64_t dist = (int64_t)(2 | (pos_slot & 1)) << ndirect;
                if (pos_slot < 14) {
                    dist += bittree_rev(r, d->pos_dec + (dist - pos_slot), ndirect);
                } else {
                    dist += (int64_t)rc_direct(r, ndirect - 4) << 4;
                    dist += bittree_rev(r, d->align, 4);
                }
                d->rep0 = dist;
            }
            if (r->trap) return SWC_ERR_REFERENCE_TRAP;
            if ((uint32_t)d->rep0 == 0xFFFFFFFFu) {                                               /* :260-264 */
                if (r->code != 0) return SWC_LZMA_RANGE_DECODER_FINISH_ERROR;
                break;
            }
            if (d->uncompressed_size == 0) return SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE;
            if (d->rep0 >= d->dict_size || (d->rep0 > d->dict_end && d->dict_end < d->dict_size))
                return SWC_LZMA_NOT_ENOUGH_TO_REPEAT;                                             /* :269 */
        }
        if (r->trap) return SWC_ERR_REFERENCE_TRAP;
        len += 2;
        if (d->uncompressed_size > -1 && d->uncompressed_size < len) return SWC_LZMA_REPEAT_WILL_EXCEED;
        for (int64_t i = 0; i < len; i++) {                                                       /* :278-282 */
            uint8_t b = byte_at(d, d->rep0 + 1, &trap);
            if (trap) return SWC_ERR_REFERENCE_TRAP;
            if (put(d, b)) return SWC_ERR_OUTPUT_OVERFLOW;
            d->uncompressed_size -= 1;
        }
    }
    return SWC_OK;
}

static void dec_init(lzma_dec *d, const uint8_t *in, size_t n, size_t ip, swco_buf *out) {
    memset(d, 0, sizeof(*d));
    d->rc.in = in; d->rc.n = n; d->rc.ip = ip;
    d->lc = 3; d->lp = 0; d->pb = 2; d->dict_size = 1 << 24;       /* LZMAProperties defaults */
    d->uncompressed_size = -1;
    d->out = out; d->out_base = out->len;
}

int swco_lzma_decompress_raw(const uint8_t *in, size_t in_len, int lc, int lp, int pb, int64_t dict_size,
                             int64_t uncompressed_size, swco_buf *out, size_t *consumed) {
    lzma_dec *d = (lzma_dec *)malloc(sizeof(lzma_dec));
    if (!d) return SWC_ERR_OUTPUT_OVERFLOW;
    dec_init(d, in, in_len, 0, out);
    d->lc = lc; d->lp = lp; d->pb = pb; d->dict_size = dict_size;
    d->uncompressed_size = uncompressed_size < 0 ? -1 : uncompressed_size;   /* LZMA.swift:69 nil -> -1 */
    int st;
    /* properties no properties byte can express: the reference ("no validation") decodes some such streams -- Swift's >> by
       a negative count shifts left -- and traps on others; refused as valid input the engine does not take (DESIGN §6) */
    if (lc < 0 || lp < 0 || pb < 0 || lc > 8 || lp > 4 || pb > 4) st = SWC_ERR_UNSUPPORTED;
    else if (reset_state(d)) st = SWC_ERR_OUTPUT_OVERFLOW;
    else st = lzma_decode(d);
    if (consumed) *consumed = d->rc.ip;
    free(d->lit); free(d);
    return st;
}

/* LZMA.decompress(data:) LZMA.swift:25-34 */
int swco_lzma_decompress(const uint8_t *in, size_t in_len, swco_buf *out, size_t *consumed) {
    if (in_len < 13) return SWC_LZMA_WRONG_PROPERTIES;
    unsigned b = in[0];
    if (b >= 9 * 5 * 5) return SWC_LZMA_WRONG_PROPERTIES;                    /* LZMAProperties.swift:50 */
    int lc = b % 9, pb = (b / 9) / 5, lp = (b / 9) % 5;
    int64_t dict = (int64_t)in[1] | (int64_t)in[2] << 8 | (int64_t)in[3] << 16 | (int64_t)in[4] << 24; /* no clamp in init */
    uint64_t us = 0;
    for (int i = 0; i < 8; i++) us |= (uint64_t)in[5 + i] << (8 * i);
    int64_t usize = (int64_t)us;          /* int(fromBytes: 8): all-ones -> -1; any negative value never reaches 0 */
    size_t used = 0;
    int st = swco_lzma_decompress_raw(in + 13, in_len - 13, lc, lp, pb, dict, usize, out, &used);
    if (consumed) *consumed = 13 + used;
    return st;
}

/* LZMA2Decoder LZMA2Decoder.swift:17-99 */
int swco_lzma2_decompress_raw(const uint8_t *in, size_t n, uint8_t dict_byte, swco_buf *out, size_t *consumed) {
    if (dict_byte & 0xC0) return SWC_LZMA2_WRONG_DICTIONARY_SIZE;             /* :21-22 */
    int bits = dict_byte & 0x3F;
    if (bits >= 40) return SWC_LZMA2_WRONG_DICTIONARY_SIZE;
    uint32_t ds = (uint32_t)(2 | (bits & 1)) << (bits / 2 + 11);
    lzma_dec *d = (lzma_dec *)malloc(sizeof(lzma_dec));
    if (!d) return SWC_ERR_OUTPUT_OVERFLOW;
    dec_init(d, in, n, 0, out);
    d->dict_size = ds < 4096 ? 4096 : ds;                                     /* didSet clamp, LZMAProperties.swift:26-32 */
    int st = SWC_OK;
    rc_t *r = &d->rc;
#define NEED(k) do { if (r->n - r->ip < (size_t)(k)) { st = SWC_ERR_REFERENCE_TRAP; goto done; } } while (0)
    for (;;) {                                                                /* :34-53 */
        NEED(1);
        unsigned control = r->in[r->ip++];
        if (control == 0) break;
        if (control == 1 || control == 2) {                                   /* :84-89 decodeUncompressed */
            if (control == 1) d->dict_start = d->dict_end;                    /* resetDictionary */
            NEED(2);
            size_t size = ((size_t)r->in[r->ip] << 8) + r->in[r->ip + 1] + 1; r->ip += 2;
            NEED(size);
            for (size_t i = 0; i < size; i++) if (put(d, r->in[r->ip++])) { st = SWC_ERR_OUTPUT_OVERFLOW; goto done; }
            continue;
        }
        if (control < 0x80) { st = SWC_LZMA2_WRONG_CONTROL_BYTE; goto done; }
        /* dispatch :56-82 */
        int reset = (control & 0x60) >> 5;
        NEED(4);
        int64_t unpack = ((int64_t)(control & 0x1F) << 16) + ((int64_t)r->in[r->ip] << 8) + r->in[r->ip + 1] + 1;
        int64_t comp = ((int64_t)r->in[r->ip + 2] << 8) + r->in[r->ip + 3] + 1;
        r->ip += 4;
        if (reset == 1) {
            if (reset_state(d)) { st = SWC_ERR_OUTPUT_OVERFLOW; goto done; }
        } else if (reset >= 2) {                                              /* updateProperties :95-99 */
            NEED(1);
            unsigned b = r->in[r->ip++];
            if (b >= 225) { st = SWC_LZMA_WRONG_PROPERTIES; goto done; }
            d->lc = b % 9; d->pb = (b / 9) / 5; d->lp = (b / 9) % 5;
            if (reset_state(d)) { st = SWC_ERR_OUTPUT_OVERFLOW; goto done; }
            if (reset == 3) d->dict_start = d->dict_end;
        }
        d->uncompressed_size = unpack;
        size_t out_start = out->len, in_start = r->ip;
        st = lzma_decode(d);
        if (st) goto done;
        if (!(unpack == (int64_t)(out->len - out_start) && (int64_t)(r->ip - in_start) == comp)) { st = SWC_LZMA2_WRONG_SIZES; goto done; }
    }
done:
    if (consumed) *consumed = r->ip;
    free(d->lit); free(d);
    return st;
#undef NEED
}

/* LZMA2.decompress(data:) LZMA2.swift:25-30 */
int swco_lzma2_decompress(const uint8_t *in, size_t n, swco_buf *out, size_t *consumed) {
    if (n < 1) return SWC_LZMA_RANGE_DECODER_INIT_ERROR;
    size_t used = 0;
    int st = swco_lzma2_decompress_raw(in + 1, n - 1, in[0], out, &used);
    if (consumed) *consumed = 1 + used;
    return st;
}
