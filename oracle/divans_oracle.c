/*
 * divans_oracle.c -- CPU restatement of the dropbox/divans entropy path (decode + encode).
 *
 * TEST INFRASTRUCTURE ONLY (see divans_oracle.h).  "parity unpinned" versus the real Rust
 * binary (no rustc in the container, no golden .divans vectors in the reference); pinned
 * against all reference known-answer tests for this path.
 *
 * Reference citations are file:line in dropbox/divans @ 23459c22.
 */
#include "divans_oracle.h"
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------
 * RFC 7932 static data (dictionary, transforms, context LUTs): tools/gen_brotli_tables.py
 * ------------------------------------------------------------------------------------------ */
#ifndef DVO_TABLES_PATH
#error "DVO_TABLES_PATH must point at brotli_tables.bin"
#endif
__asm__(".section .rodata\n"
        ".global dvo_tables_blob\n"
        ".balign 16\n"
        "dvo_tables_blob:\n"
        ".incbin \"" DVO_TABLES_PATH "\"\n"
        ".global dvo_tables_blob_end\n"
        "dvo_tables_blob_end:\n"
        ".previous\n");
extern const uint8_t dvo_tables_blob[];
#define TB_SIZE_BITS (dvo_tables_blob + 24)
#define TB_OFFSETS ((const uint32_t *)(dvo_tables_blob + 56))
#define TB_CTX (dvo_tables_blob + 184)
#define TB_TRANSFORMS (dvo_tables_blob + 2232)
#define TB_PSMAP ((const uint16_t *)(dvo_tables_blob + 2616))
#define TB_PS (dvo_tables_blob + 2744)
#define TB_DICT (dvo_tables_blob + 3000)
#define TB_DICT_SIZE 122784u

/* ------------------------------------------------------------------------------------------
 * small helpers
 * ------------------------------------------------------------------------------------------ */
typedef struct { uint8_t *p; size_t n, cap; } bytevec;
static void bv_reserve(bytevec *v, size_t extra) {
    if (v->n + extra > v->cap) {
        size_t nc = v->cap ? v->cap * 2 : 256;
        while (nc < v->n + extra) nc *= 2;
        v->p = (uint8_t *)realloc(v->p, nc);
        v->cap = nc;
    }
}
static void bv_push(bytevec *v, const uint8_t *d, size_t n) { bv_reserve(v, n); memcpy(v->p + v->n, d, n); v->n += n; }
static void bv_free(bytevec *v) { free(v->p); v->p = NULL; v->n = v->cap = 0; }
static inline uint32_t bitlen32(uint32_t v) { return v ? 32u - (uint32_t)__builtin_clz(v) : 0u; }
/* codec/interface.rs:180-182 (u8 arithmetic, wrapping) */
static inline uint8_t round_up_mod_4(uint8_t v) { return (uint8_t)((((uint8_t)(v - 1)) | 3) + 1); }

/* ------------------------------------------------------------------------------------------
 * CRC32C  (codec/crc32.rs:17-86: state is the finalised value; init 0)
 * ------------------------------------------------------------------------------------------ */
static uint32_t crc_table[256];
static int crc_table_ready = 0;
static void crc_init_table(void) {
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : (c >> 1);
        crc_table[i] = c;
    }
    crc_table_ready = 1;
}
uint32_t dvo_crc32c(uint32_t crc, const uint8_t *buf, size_t n) {
    if (!crc_table_ready) crc_init_table();
    crc = ~crc;
    for (size_t i = 0; i < n; i++) crc = crc_table[(crc ^ buf[i]) & 0xff] ^ (crc >> 8);
    return ~crc;
}

/* ------------------------------------------------------------------------------------------
 * exact division by cdf max: OptFrequentistCDF16 (the default build's DefaultCDF16,
 * src/interface.rs:152-153) caches numeric::lookup_divisor(max) = RECIPROCAL[max as u16]
 * whose entries are compute_divisor(d as u16) (probability/numeric.rs:14-17, make_div_lut.rs:29-41)
 * ------------------------------------------------------------------------------------------ */
static inline void compute_divisor(uint16_t d, int64_t *inv, uint8_t *shift) {
    if (d == 0) { *inv = 0; *shift = 0; return; } /* div_lut.rs RECIPROCAL[0] = (0,0) */
    uint8_t bit_len = (uint8_t)(16 - __builtin_clz((uint32_t)d) + 16); /* 16 - leading_zeros(u16) */
    *inv = ((((int64_t)1 << bit_len) - (int64_t)d) << 31) / (int64_t)d + 1;
    *shift = (uint8_t)(bit_len - 1);
}
static inline int32_t fast_divide_30bit_by_16bit(int32_t num, int64_t inv, uint8_t shift) {
    /* probability/numeric.rs:26-31 */
    int64_t m = inv * (int64_t)num;
    int32_t t = (int32_t)(m >> 31);
    return (t + (((int32_t)((int64_t)num - (m >> 31))) >> 1)) >> shift;
}
int32_t dvo_fast_divide(int32_t num, int16_t denom) {
    int64_t inv; uint8_t sh;
    compute_divisor((uint16_t)denom, &inv, &sh);
    return fast_divide_30bit_by_16bit(num, inv, sh);
}

#ifdef DVO_FEATURE_BLEND
/* ------------------------------------------------------------------------------------------
 * BlendCDF16  (probability/blend_cdf.rs:109-208; generic BaseCDF paths probability/interface.rs:97-108,136-198)
 * ------------------------------------------------------------------------------------------ */
#define BLEND_CDF_MAX 32767                 /* probability/interface.rs:429 */
#define BLEND_DEL (BLEND_CDF_MAX - 16)      /* blend_cdf.rs:80,90 */
int dvo_feature_blend(void) { return 1; }
void dvo_cdf_default(dvo_cdf16 *c) { memset(c->c, 0, sizeof c->c); c->mix_rate = (1 << 10) + (1 << 9); c->count = 0; }   /* blend_cdf.rs:128-136 */

/* mul_blend (:15-55) + the early-growth step (:116-124) */
static void blend_internal(dvo_cdf16 *c, const int16_t to_blend[16], int32_t mix_rate) {
    const int32_t bias = (c->count & 0xf) << (15 - 4);
    const int32_t scale_minus_blend = (1 << 15) - mix_rate;
    for (int i = 0; i < 16; i++) {
        int32_t e = (int32_t)((uint32_t)(int32_t)to_blend[i] * (uint32_t)mix_rate);
        e = (int32_t)((uint32_t)e + (uint32_t)(int32_t)c->c[i] * (uint32_t)scale_minus_blend + (uint32_t)bias);
        c->c[i] = (int16_t)(e >> 15);
    }
    if (c->c[15] < (int16_t)(BLEND_DEL - (c->c[15] >> 1)))
        for (int i = 0; i < 16; i++) c->c[i] = (int16_t)(c->c[i] + (c->c[i] >> 1));
}
int16_t dvo_cdf_value(const dvo_cdf16 *c, uint8_t sym) {   /* :160-171: the bias is the latent uniform distribution */
    if (sym == 15) return BLEND_CDF_MAX;
    int16_t bias = (int16_t)(BLEND_CDF_MAX - c->c[15]);
    return (int16_t)(c->c[sym] + (int16_t)(((int32_t)bias * (int32_t)(sym + 1)) >> 4));
}
void dvo_cdf_sym_start_freq(const dvo_cdf16 *c, uint8_t sym, int16_t *start, int16_t *freq) {
    /* probability/interface.rs:97-108 with div_by_max = >> log_max = >> 15 (blend_cdf.rs:154-159) */
    int32_t cdf_sym = ((int32_t)dvo_cdf_value(c, sym & 15) << 15) >> 15;
    int32_t cdf_prev = sym ? ((int32_t)dvo_cdf_value(c, (uint8_t)((sym - 1) & 15)) << 15) >> 15 : 0;
    int32_t f = cdf_sym - cdf_prev;
    *start = (int16_t)((int16_t)cdf_prev + 1);
    *freq = (int16_t)((int16_t)f - 1);
}
uint8_t dvo_cdf_lookup(const dvo_cdf16 *c, int16_t cdf_offset, int16_t *start, int16_t *freq) {
    /* probability/interface.rs:136-198 (max() = CDF_MAX) */
    int16_t r = (int16_t)(((int32_t)cdf_offset * (int32_t)BLEND_CDF_MAX) >> 15);
    uint8_t sym = 15;
    for (uint8_t i = 0; i < 15; i++) {
        if (r < dvo_cdf_value(c, i)) { sym = i; break; }
    }
    dvo_cdf_sym_start_freq(c, sym, start, freq);
    return sym;
}
void dvo_cdf_blend(dvo_cdf16 *c, uint8_t sym, dvo_speed s) {
    /* blend_cdf.rs:186-208: the speed is computed and NOT used (`_mix_rate`); the CDF's own decaying mix_rate is */
    (void)s;
    c->count = (int32_t)((uint32_t)c->count + 1u);
    int16_t to_blend[16];
    for (int i = 0; i < 16; i++) to_blend[i] = i >= sym ? BLEND_DEL : 0;   /* to_blend_lut :87-108 */
    blend_internal(c, to_blend, c->mix_rate);
    c->mix_rate -= c->mix_rate >> 7;
}
void dvo_cdf_average(const dvo_cdf16 *self, const dvo_cdf16 *other, int32_t mix_rate, dvo_cdf16 *out) {
    /* blend_cdf.rs:181-185 */
    *out = *self;
    blend_internal(out, other->c, mix_rate);
}
#else
int dvo_feature_blend(void) { return 0; }
/* ------------------------------------------------------------------------------------------
 * FrequentistCDF16  (probability/frequentist_cdf.rs:12-86, probability/interface.rs:97-198)
 * ------------------------------------------------------------------------------------------ */
void dvo_cdf_default(dvo_cdf16 *c) { for (int i = 0; i < 16; i++) c->c[i] = (int16_t)(4 * (i + 1)); }

void dvo_cdf_sym_start_freq(const dvo_cdf16 *c, uint8_t sym, int16_t *start, int16_t *freq) {
    /* probability/interface.rs:97-108 */
    int64_t inv; uint8_t sh;
    compute_divisor((uint16_t)c->c[15], &inv, &sh);
    int32_t cdf_sym = fast_divide_30bit_by_16bit((int32_t)c->c[sym & 15] << 15, inv, sh);
    int32_t cdf_prev = sym ? fast_divide_30bit_by_16bit((int32_t)c->c[(sym - 1) & 15] << 15, inv, sh) : 0;
    int32_t f = cdf_sym - cdf_prev;
    *start = (int16_t)((int16_t)cdf_prev + 1); /* "major hax" */
    *freq = (int16_t)((int16_t)f - 1);
}

uint8_t dvo_cdf_lookup(const dvo_cdf16 *c, int16_t cdf_offset, int16_t *start, int16_t *freq) {
    /* probability/interface.rs:136-198 */
    int16_t cdfmax = c->c[15];
    int16_t r = (int16_t)(((int32_t)cdf_offset * (int32_t)cdfmax) >> 15);
    uint8_t sym = 15;
    for (uint8_t i = 0; i < 15; i++) {
        if (r < c->c[i]) { sym = i; break; }
    }
    dvo_cdf_sym_start_freq(c, sym, start, freq);
    return sym;
}

void dvo_cdf_blend(dvo_cdf16 *c, uint8_t sym, dvo_speed s) {
    /* probability/frequentist_cdf.rs:74-85 (i16 wrapping arithmetic) */
    for (int i = sym; i < 16; i++) c->c[i] = (int16_t)((uint16_t)c->c[i] + (uint16_t)s.inc);
    if (c->c[15] >= s.lim) {
        for (int i = 0; i < 16; i++) {
            int16_t t = (int16_t)((uint16_t)c->c[i] + (uint16_t)(i + 1));
            c->c[i] = (int16_t)((uint16_t)t - (uint16_t)(t >> 2));
        }
    }
}

void dvo_cdf_average(const dvo_cdf16 *self, const dvo_cdf16 *other, int32_t mix_rate, dvo_cdf16 *out) {
    /* probability/frequentist_cdf.rs:58-72 (i32 wrapping arithmetic) */
    int32_t ourmax = self->c[15], othermax = other->c[15];
    int32_t prod = (int32_t)((uint32_t)ourmax * (uint32_t)othermax);
    uint32_t lz = prod == 0 ? 32u : (uint32_t)__builtin_clz((uint32_t)prod);
    if (lz > 17) lz = 17;
    uint32_t shift = 17 - lz;
    int32_t inv_mix = (1 << 15) - mix_rate;
    for (int i = 0; i < 16; i++) {
        int32_t rs = (int32_t)((uint32_t)(int32_t)self->c[i] * (uint32_t)othermax) >> shift;
        int32_t ro = (int32_t)((uint32_t)(int32_t)other->c[i] * (uint32_t)ourmax) >> shift;
        uint32_t acc = (uint32_t)rs * (uint32_t)mix_rate + (uint32_t)ro * (uint32_t)inv_mix + 1u;
        out->c[i] = (int16_t)((int32_t)acc >> 15);
    }
}

#endif /* DVO_FEATURE_BLEND */

/* probability/interface.rs:566-585 (i16 versions) */
uint8_t dvo_speed_to_u8(int16_t data) {
    uint8_t length = (uint8_t)(16 - (data == 0 ? 16 : (__builtin_clz((uint32_t)(uint16_t)data) - 16)));
    uint8_t mantissa = 0;
    if (data != 0) {
        int16_t rem = (int16_t)(data - (int16_t)(1 << (length - 1)));
        mantissa = (uint8_t)((int16_t)((int16_t)(rem << 3)) >> (length - 1));
    }
    return (uint8_t)((length << 3) | mantissa);
}
int16_t dvo_u8_to_speed(uint8_t data) {
    if (data < 8) return 0;
    uint8_t log_val = (uint8_t)((data >> 3) - 1);
    int16_t rem = (int16_t)(((int16_t)data & 0x7) << log_val);
    return (int16_t)((int16_t)(1 << log_val) | (rem >> 3));
}
/* the brotli crate's u16 flavour used when the decoded f8 nibbles are stored into the
 * PredictionModeContextMap (codec/context_map.rs:262-266 -> brotli::enc::interface::{u8_to_speed,speed_to_u8},
 * NOT-IN-TREE; restated from the published crate, same formula on u16) */
static uint16_t brotli_u8_to_speed(uint8_t data) {
    if (data < 8) return 0;
    uint8_t log_val = (uint8_t)((data >> 3) - 1);
    uint16_t rem = (uint16_t)(((uint16_t)data & 0x7) << log_val);
    return (uint16_t)((uint16_t)(1u << log_val) | (rem >> 3));
}
static uint8_t brotli_speed_to_u8(uint16_t data) {
    uint8_t length = (uint8_t)(data == 0 ? 0 : 32 - __builtin_clz((uint32_t)data));
    uint8_t mantissa = 0;
    if (data != 0) {
        uint16_t rem = (uint16_t)(data - (uint16_t)(1u << (length - 1)));
        mantissa = (uint8_t)((uint16_t)(rem << 3) >> (length - 1));
    }
    return (uint8_t)((length << 3) | mantissa);
}

static const dvo_speed SPEED_MUD = {0x10, 0x2000}, SPEED_SLOW = {0x20, 0x1000}, SPEED_MED = {0x30, 0x4000},
                       SPEED_FAST = {0x60, 0x4000}, SPEED_PLANE = {0x80, 0x4000}, SPEED_ROCKET = {0x180, 0x4000};
/* probability/interface.rs:321-328 */

/* ------------------------------------------------------------------------------------------
 * mixing weights  (codec/weights.rs)
 * ------------------------------------------------------------------------------------------ */
void dvo_weights_init(dvo_weights *w) { w->w[0] = w->w[1] = 1; w->mixing_param = 1; w->norm = 1 << 14; }
static int32_t compute_new_weight(const int16_t probs[2], int16_t weighted_prob, const int32_t weights[2], int index) {
    /* codec/weights.rs:110-133 (the integer version: the cfg(features=...) typo keeps the float one out) */
    int64_t full_model_sum_p1 = weighted_prob;
    int64_t full_model_total = 1 << 15;
    int64_t full_model_sum_p0 = full_model_total - (int64_t)weighted_prob;
    int64_t n1i = probs[index];
    int64_t ni = 1 << 15;
    int64_t error = full_model_total - full_model_sum_p1;
    int64_t wi = weights[index];
    int64_t efficacy = (int64_t)((uint64_t)full_model_total * (uint64_t)n1i) - (int64_t)((uint64_t)full_model_sum_p1 * (uint64_t)ni);
    uint64_t geo = (uint64_t)full_model_sum_p1 * (uint64_t)full_model_sum_p0;
    uint32_t log_geo = 64u - (geo == 0 ? 64u : (uint32_t)__builtin_clzll(geo));
    int64_t prod = (int64_t)((uint64_t)error * (uint64_t)efficacy);
    int64_t adj = log_geo >= 64 ? (prod < 0 ? -1 : 0) : (prod >> log_geo);
    int32_t nw = (int32_t)(uint32_t)(uint64_t)(wi + adj);
    return nw > 1 ? nw : 1;
}
static int16_t compute_normalized_weight(const int32_t mw[2]) {
    /* codec/weights.rs:54-62 ; numeric.rs:60-62 with RECIPROCAL8[d] = 1 + (1<<24)/d, [0]=0 */
    int64_t total = (int64_t)mw[0] + (int64_t)mw[1];
    int lz = total == 0 ? 64 : __builtin_clzll((uint64_t)total);
    int16_t shift = (int16_t)(56 - lz);
    if (shift < 0) shift = 0;
    int64_t total_8bit = total >> shift;
    uint8_t d = (uint8_t)total_8bit;
    int32_t recip = d ? 1 + (1 << 24) / (int32_t)d : 0;
    uint16_t num = (uint16_t)((uint16_t)(mw[0] >> shift) << 8);
    int16_t q = (int16_t)(((int64_t)recip * (int64_t)num) >> 24);
    return (int16_t)((uint16_t)q << 7);
}
void dvo_weights_update(dvo_weights *w, int16_t p0, int16_t p1, int16_t weighted) {
    /* codec/weights.rs:23-38, 64-79 */
    if (((w->w[0] | w->w[1]) & 0x7f000000) != 0) {
        uint32_t lz0 = w->w[0] == 0 ? 32 : (uint32_t)__builtin_clz((uint32_t)w->w[0]);
        uint32_t lz1 = w->w[1] == 0 ? 32 : (uint32_t)__builtin_clz((uint32_t)w->w[1]);
        uint32_t ilog = 32 - (lz0 < lz1 ? lz0 : lz1);
        if (ilog >= 24) { w->w[0] >>= ilog - 24; w->w[1] >>= ilog - 24; }
    }
    int16_t probs[2] = {p0, p1};
    int32_t w0 = compute_new_weight(probs, weighted, w->w, 0);
    int32_t w1 = compute_new_weight(probs, weighted, w->w, 1);
    w->w[0] = w0; w->w[1] = w1;
    w->norm = compute_normalized_weight(w->w);
}

/* batch helpers for the arithmetic tests (tests/test_gpu_arith.py, tests/test_arith_domains.py): many cases per call */
void dvo_weights_update_batch(size_t n, const int32_t *w0, const int32_t *w1, const int16_t *p0, const int16_t *p1,
                              const int16_t *weighted, int32_t *out_w0, int32_t *out_w1, int16_t *out_norm) {
    for (size_t i = 0; i < n; i++) {
        dvo_weights w; dvo_weights_init(&w);
        w.w[0] = w0[i]; w.w[1] = w1[i];
        dvo_weights_update(&w, p0[i], p1[i], weighted[i]);
        out_w0[i] = w.w[0]; out_w1[i] = w.w[1]; out_norm[i] = w.norm;
    }
}
void dvo_cdf_step_batch(size_t n, int mix, int enc, const int16_t *cdf, const int16_t *cdf2, const int32_t *wts,
                        const dvo_speed *speeds, const uint64_t *state, const uint8_t *sym_in, uint8_t *sym_out, int16_t *start_out,
                        int16_t *freq_out, uint64_t *state_out, int16_t *cdf_out, int16_t *cdf2_out, int32_t *wts_out) {
    /* one literal nibble as code_lit_nibble codes it (codec/literal.rs:154-259): cdf = the stride prior, cdf2 = the
     * context-map prior and wts = (w0, w1, norm) when mixing, speeds[2i] / [2i+1] = stride / context-map speed; decode
     * takes the symbol from the rANS state (ans.rs:230-244, before renormalisation), encode from sym_in */
    for (size_t i = 0; i < n; i++) {
        dvo_cdf16 nb, cm, prob;
        memcpy(nb.c, cdf + 16 * i, 32);
        const dvo_cdf16 *coded = &nb;
        dvo_weights w; dvo_weights_init(&w);
        if (mix) {
            memcpy(cm.c, cdf2 + 16 * i, 32);
            w.w[0] = wts[3 * i]; w.w[1] = wts[3 * i + 1]; w.norm = (int16_t)wts[3 * i + 2];
            dvo_cdf_average(&cm, &nb, (int32_t)(uint16_t)w.norm, &prob);
            coded = &prob;
        }
        const uint64_t a = enc ? 0 : state[i];
        int16_t start, freq;
        uint8_t sym;
        if (enc) { sym = sym_in[i] & 15; dvo_cdf_sym_start_freq(coded, sym, &start, &freq); }
        else sym = dvo_cdf_lookup(coded, (int16_t)(a & 0x7fff), &start, &freq);
        if (!enc) state_out[i] = (uint64_t)(int64_t)freq * (a >> 15) + (a & 0x7fff) - (uint64_t)(int64_t)start;
        if (mix) {
            int16_t st, f_cm, f_nb;
            dvo_cdf_sym_start_freq(&cm, sym, &st, &f_cm);
            dvo_cdf_sym_start_freq(&nb, sym, &st, &f_nb);
            dvo_weights_update(&w, f_cm, f_nb, freq);
            dvo_cdf_blend(&cm, sym, speeds[2 * i + 1]);
            memcpy(cdf2_out + 16 * i, cm.c, 32);
            wts_out[3 * i] = w.w[0]; wts_out[3 * i + 1] = w.w[1]; wts_out[3 * i + 2] = (uint16_t)w.norm;
        }
        dvo_cdf_blend(&nb, sym, speeds[2 * i]);
        memcpy(cdf_out + 16 * i, nb.c, 32);
        sym_out[i] = sym; start_out[i] = start; freq_out[i] = freq;
    }
}
void dvo_cdf_walk_batch(size_t n_walks, size_t n_steps, const dvo_speed *speeds, const uint8_t *syms, dvo_cdf16 *trace) {
    /* walk w starts at the default CDF and blends syms[w * n_steps + j] under speeds[w]; trace[w * (n_steps + 1) + j] is
     * the CDF before step j (the last entry: after the walk) */
    for (size_t w = 0; w < n_walks; w++) {
        dvo_cdf16 c; dvo_cdf_default(&c);
        for (size_t j = 0; j < n_steps; j++) {
            trace[w * (n_steps + 1) + j] = c;
            dvo_cdf_blend(&c, syms[w * n_steps + j], speeds[w]);
        }
        trace[w * (n_steps + 1) + n_steps] = c;
    }
}

/* ------------------------------------------------------------------------------------------
 * prior tables: flat arrays, index rule of src/priors.rs:211-237 incl. the fall-through quirk
 * (a type that is not listed resolves to the LAST listed entry's offset)
 * ------------------------------------------------------------------------------------------ */
typedef struct { int type; int ndim; int dim[3]; } prior_ent;
static size_t prior_index(const prior_ent *t, int n, int type, size_t i0, size_t i1, size_t i2) {
    size_t off = 0;
    for (int k = 0; k < n; k++) {
        const prior_ent *e = &t[k];
        if (e->type == type || k == n - 1) {
            /* linearize_index!: car + d0*(cadr + d1*(caddr)) -- only as many dims as listed */
            size_t idx = i0;
            if (e->ndim >= 2) idx += (size_t)e->dim[0] * (e->ndim >= 3 ? (i1 + (size_t)e->dim[1] * i2) : i1);
            return off + idx;
        }
        size_t prod = 1;
        for (int d = 0; d < e->ndim; d++) prod *= (size_t)e->dim[d];
        off += prod;
    }
    return 0;
}
static size_t prior_total(const prior_ent *t, int n) {
    size_t off = 0;
    for (int k = 0; k < n; k++) { size_t prod = 1; for (int d = 0; d < t[k].ndim; d++) prod *= (size_t)t[k].dim[d]; off += prod; }
    return off;
}
/* codec/priors.rs:12-133 */
enum { CC_FullSelection, CC_EndIndicator };
static const prior_ent T_CC[] = {{CC_FullSelection, 2, {16, 1}}, {CC_EndIndicator, 2, {1, 256}}};
enum { LL_CountSmall, LL_SizeBegNib, LL_SizeLastNib, LL_SizeMantissaNib };
static const prior_ent T_LL[] = {{LL_CountSmall, 2, {256, 16}}, {LL_SizeBegNib, 1, {256}}, {LL_SizeLastNib, 1, {256}}, {LL_SizeMantissaNib, 1, {256}}};
enum { CM_FirstNibble, CM_SecondNibble };
static const prior_ent T_CM[] = {{CM_FirstNibble, 2, {1, 256}}, {CM_SecondNibble, 3, {1, 16, 256}}};
enum { LN_CombinedNibble };
static const prior_ent T_LN[] = {{LN_CombinedNibble, 3, {3, 256, 256}}};
enum { CP_DistanceBegNib, CP_DistanceLastNib, CP_DistanceMnemonic, CP_DistanceMnemonicTwo, CP_DistanceMantissaNib,
       CP_CountSmall, CP_CountBegNib, CP_CountLastNib, CP_CountMantissaNib };
static const prior_ent T_CP[] = {{CP_DistanceBegNib, 2, {256, 64}}, {CP_DistanceMnemonic, 2, {256, 2}}, {CP_DistanceLastNib, 2, {256, 1}},
                                 {CP_DistanceMantissaNib, 2, {256, 5}}, {CP_CountSmall, 2, {256, 64}}, {CP_CountBegNib, 2, {256, 64}},
                                 {CP_CountLastNib, 2, {256, 64}}, {CP_CountMantissaNib, 2, {256, 64}}};
enum { DC_SizeBegNib, DC_SizeLastNib, DC_Index, DC_Transform };
static const prior_ent T_DC[] = {{DC_SizeBegNib, 1, {256}}, {DC_SizeLastNib, 1, {256}}, {DC_Index, 2, {256, 5}}, {DC_Transform, 2, {2, 25}}};
enum { BT_Mnemonic, BT_FirstNibble, BT_SecondNibble, BT_StrideNibble };
static const prior_ent T_BT[] = {{BT_Mnemonic, 1, {3}}, {BT_FirstNibble, 1, {3}}, {BT_SecondNibble, 1, {3}}, {BT_StrideNibble, 1, {1}}};
enum { PM_Only, PM_DynamicContextMixingSpeed, PM_PriorDepth, PM_PriorMixingValue, PM_LiteralSpeed, PM_Mnemonic, PM_FirstNibble,
       PM_SecondNibble, PM_ContextMapSpeedPalette };
static const prior_ent T_PM[] = {{PM_Only, 1, {1}}, {PM_LiteralSpeed, 1, {1}}, {PM_FirstNibble, 1, {2}}, {PM_SecondNibble, 1, {2}},
                                 {PM_Mnemonic, 1, {4}}, {PM_PriorMixingValue, 1, {17}}, {PM_ContextMapSpeedPalette, 1, {4}}};
#define NEL(a) ((int)(sizeof(a) / sizeof((a)[0])))

/* The two 3*256*256 literal tables (6 MB each) are recycled per thread: the reference allocates and default-initialises
 * them per decompressor object (codec/interface.rs:728-729); we keep the initialisation (it is part of the reference's
 * cost) but not the mmap/munmap churn, which would understate the CPU baseline on many-core hosts. */
static __thread dvo_cdf16 *tl_pool[2];
static dvo_cdf16 *alloc_priors(size_t n) {
    dvo_cdf16 *p = NULL;
    if (n == 3u * 256 * 256) { for (int i = 0; i < 2; i++) if (tl_pool[i]) { p = tl_pool[i]; tl_pool[i] = NULL; break; } }
    if (!p) p = (dvo_cdf16 *)malloc(n * sizeof(dvo_cdf16));
    dvo_cdf16 d; dvo_cdf_default(&d);
    for (size_t i = 0; i < n; i++) p[i] = d;
    return p;
}

/* ------------------------------------------------------------------------------------------
 * rANS coder  (src/ans.rs)
 * ------------------------------------------------------------------------------------------ */
#define NUM_SYMBOLS_BEFORE_FLUSH 65536u /* ans.rs:57,138 */
typedef struct {
    uint64_t a, b; uint16_t sym_count; uint8_t need_a, need_b; /* ans.rs:142-148 */
    const uint8_t *p; size_t n, pos;
    int underflow; uint64_t n_syms;
} ans_dec;
static void ans_dec_init(ans_dec *d, const uint8_t *p, size_t n) {
    memset(d, 0, sizeof(*d)); d->need_a = 8; d->p = p; d->n = n; /* ans.rs:150-162 */
}
static void ans_dec_fill(ans_dec *d) {
    /* ans.rs:428-442 push_data + :173-189 (whole-stream: the 1..3-byte partial paths never arise) */
    if (d->need_a == 0) return;
    if (d->need_a == 1) {
        if (d->pos + 4 > d->n) { d->underflow = 1; d->a <<= 32; d->need_a = 0; d->pos = d->n; return; }
        const uint8_t *q = d->p + d->pos;
        d->a = (d->a << 32) | ((uint64_t)q[0] | ((uint64_t)q[1] << 8) | ((uint64_t)q[2] << 16) | ((uint64_t)q[3] << 24));
        d->pos += 4; d->need_a = 0;
        return;
    }
    /* need_a in 5..15: (re)initialise both states from 16 bytes */
    d->sym_count = 0; d->a = 0; d->b = 0;
    if (d->pos + 16 > d->n) { d->underflow = 1; d->need_a = 0; d->pos = d->n; return; }
    const uint8_t *q = d->p + d->pos;
    for (int i = 0; i < 8; i++) { d->a |= (uint64_t)q[i] << (8 * i); d->b |= (uint64_t)q[8 + i] << (8 * i); }
    d->pos += 16; d->need_a = 0;
}
static inline void ans_dec_advance(ans_dec *d, int16_t start, int16_t freq) {
    /* ans.rs:230-244 */
    d->need_a = d->need_b;
    d->need_a |= (uint8_t)((d->sym_count == (uint16_t)(NUM_SYMBOLS_BEFORE_FLUSH - 1)) << 3);
    uint64_t x = (uint64_t)(int64_t)freq * (d->a >> 15) + (d->a & 0x7fff) - (uint64_t)(int64_t)start;
    d->sym_count = (uint16_t)(d->sym_count + 1);
    d->need_b = (uint8_t)(x < ((uint64_t)1 << 31));
    d->a = d->b; d->b = x; d->n_syms++;
}

typedef struct {
    uint32_t *sf; size_t n_sf; /* (start | freq<<16) recorded for the current chunk, ans.rs:289-301 */
    bytevec out; uint64_t n_syms;
    int bad; /* a symbol with frequency <= 0 was put: the reference's flush divides by it (ans.rs:362-366) and panics */
} ans_enc;
static void ans_enc_init(ans_enc *e) { memset(e, 0, sizeof(*e)); e->sf = (uint32_t *)malloc(NUM_SYMBOLS_BEFORE_FLUSH * 4); }
static void ans_enc_free(ans_enc *e) { free(e->sf); bv_free(&e->out); }
static void ans_enc_flush_chunk(ans_enc *e) {
    /* ans.rs:302-378: walk symbols last->first, bytes are stacked in FRONT of what was emitted before */
    size_t len = e->n_sf;
    if (len == 0) return;
    uint8_t *tmp = (uint8_t *)malloc(len * 4 + 16);
    size_t top = len * 4 + 16; /* stack grows down */
    uint64_t sa = (uint64_t)1 << 31, sb = (uint64_t)1 << 31;
    for (size_t k = len; k-- > 0;) {
        int16_t start = (int16_t)(e->sf[k] & 0xffff), freq = (int16_t)(e->sf[k] >> 16);
        uint64_t f = (uint64_t)(int64_t)freq;
        uint64_t lim = (((uint64_t)1 << 31 >> 15) << 32) * f;
        uint64_t st = sa;
        if (st >= lim) {
            top -= 4;
            tmp[top] = (uint8_t)st; tmp[top + 1] = (uint8_t)(st >> 8); tmp[top + 2] = (uint8_t)(st >> 16); tmp[top + 3] = (uint8_t)(st >> 24);
            st >>= 32;
        }
        uint64_t x = ((st / f) << 15) + (st % f) + (uint64_t)(int64_t)start;
        sa = sb; sb = x;
    }
    { uint64_t t = sa; sa = sb; sb = t; }
    top -= 16;
    for (int i = 0; i < 8; i++) { tmp[top + i] = (uint8_t)(sa >> (8 * i)); tmp[top + 8 + i] = (uint8_t)(sb >> (8 * i)); }
    bv_push(&e->out, tmp + top, len * 4 + 16 - top);
    free(tmp);
    e->n_sf = 0;
}
static inline void ans_enc_put(ans_enc *e, int16_t start, int16_t freq) {
    if (freq <= 0) { e->bad = 1; freq = 1; start = 0; } /* only reachable after a stream-supplied speed wrapped an i16 counter */
    e->sf[e->n_sf++] = (uint32_t)(uint16_t)start | ((uint32_t)(uint16_t)freq << 16);
    e->n_syms++;
    if (e->n_sf == NUM_SYMBOLS_BEFORE_FLUSH) ans_enc_flush_chunk(e);
}

/* one coder of the pair, in either direction (ArithmeticEncoderOrDecoder, arithmetic_coder.rs:179-256) */
typedef struct { int encoding; ans_dec d; ans_enc e; } coder;
static inline uint8_t code_nibble(coder *k, uint8_t nib, const dvo_cdf16 *cdf, int16_t *freq_out) {
    int16_t start, freq;
    if (k->encoding) {
        dvo_cdf_sym_start_freq(cdf, nib, &start, &freq); /* ans.rs:279-288 */
        ans_enc_put(&k->e, start, freq);
    } else {
        ans_dec_fill(&k->d);                              /* drain_or_fill_static_buffer, codec/interface.rs:868-917 */
        nib = dvo_cdf_lookup(cdf, (int16_t)(k->d.a & 0x7fff), &start, &freq); /* ans.rs:246-252 */
        ans_dec_advance(&k->d, start, freq);
    }
    if (freq_out) *freq_out = freq;
    return nib;
}
static inline uint8_t code_and_blend(coder *k, uint8_t nib, dvo_cdf16 *cdf, dvo_speed sp) {
    nib = code_nibble(k, nib, cdf, NULL);
    dvo_cdf_blend(cdf, nib, sp);
    return nib;
}

/* ------------------------------------------------------------------------------------------
 * ring buffer replay  (src/cmd_to_raw/mod.rs) -- whole-stream flavour: every byte that enters the
 * ring is also appended to `out` (flush only changes WHEN bytes reach the caller, :90-121)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    uint8_t *ring; uint32_t ring_len; uint32_t idx; /* ring_buffer_decode_index */
    uint8_t *out; size_t out_cap, out_len; int overflow;
} recoder;
static inline void rc_put(recoder *r, uint8_t b) {
    r->ring[r->idx] = b;
    r->idx++; if (r->idx == r->ring_len) r->idx = 0;
    if (r->out_len < r->out_cap) r->out[r->out_len] = b; else r->overflow = 1;
    r->out_len++;
}
static void rc_last_8(const recoder *r, uint8_t ret[8]) {
    /* cmd_to_raw/mod.rs:69-86: NOTE the byte order flips when ring_buffer_decode_index < 8 */
    if (r->idx < 8) {
        for (uint32_t i = 0; i < 8; i++) ret[i] = r->ring[(r->idx + r->ring_len - i - 1) & (r->ring_len - 1)];
    } else {
        memcpy(ret, r->ring + r->idx - 8, 8);
    }
}
static int rc_copy(recoder *r, uint32_t distance, uint32_t num_bytes) {
    /* cmd_to_raw/mod.rs:245-283 + :159-195.  Byte-wise equivalent of both the repeat-buffer fast path
     * and the chunked non-overlapping path.  distance > idx + ring_len is the reference's
     * DistanceGreaterRingBuffer error (:166-168); distance >= ring_len makes the reference loop
     * forever / alias, we report failure for it. */
    if (distance == 0 || distance >= r->ring_len) return DVO_FAILURE;
    for (uint32_t i = 0; i < num_bytes; i++) {
        uint32_t src = (r->idx + r->ring_len - distance) & (r->ring_len - 1);
        rc_put(r, r->ring[src]);
    }
    return DVO_SUCCESS;
}
int dvo_dict_word(uint32_t word_size, uint32_t word_id, uint32_t transform, uint8_t *out) {
    /* cmd_to_raw/mod.rs:284-309 ; transform = RFC 7932 section 8 / appendix B (brotli crate, NOT-IN-TREE) */
    if (word_size < 4 || word_size > 24 || transform >= 121) return -1;
    uint64_t word_index = (uint64_t)word_id * word_size + TB_OFFSETS[word_size];
    if (word_index + word_size > TB_DICT_SIZE) return -1;
    const uint8_t *word = TB_DICT + word_index;
    const uint8_t *tr = TB_TRANSFORMS + 3 * transform;
    const uint8_t *prefix = TB_PS + TB_PSMAP[tr[0]];
    const uint8_t *suffix = TB_PS + TB_PSMAP[tr[2]];
    int type = tr[1];
    int idx = 0;
    int len = (int)word_size;
    { int plen = *prefix++; while (plen--) out[idx++] = *prefix++; }
    {
        int t = type;
        int skip = t < 12 ? 0 : t - 11;          /* OMIT_FIRST_1..9 = 12..20 */
        if (skip > len) skip = len;
        word += skip; len -= skip;
        if (t <= 9) len -= t;                      /* OMIT_LAST_1..9 = 1..9 */
        for (int i = 0; i < len; i++) out[idx++] = word[i];
        uint8_t *up = out + idx - (len > 0 ? len : 0);
        if (len > 0 && (t == 10 || t == 11)) {     /* UPPERCASE_FIRST / UPPERCASE_ALL */
            int remaining = t == 10 ? 1 : len;
            while (remaining > 0) {
                int step;
                if (up[0] < 0xc0) { if (up[0] >= 'a' && up[0] <= 'z') up[0] ^= 32; step = 1; }
                else if (up[0] < 0xe0) { up[1] ^= 32; step = 2; }
                else { up[2] ^= 5; step = 3; }
                up += step; remaining -= step;
                if (t == 10) break;
            }
        }
    }
    { int slen = *suffix++; while (slen--) out[idx++] = *suffix++; }
    return idx;
}
static int rc_dict(recoder *r, uint32_t word_size, uint32_t word_id, uint32_t transform, uint32_t final_size) {
    uint8_t buf[64]; memset(buf, 0, sizeof buf);
    int n = dvo_dict_word(word_size, word_id, transform, buf);
    if (n < 0) return DVO_FAILURE;
    if (final_size != 0 && (uint32_t)n != final_size) return DVO_FAILURE; /* DictTransformDiffersFromExpectedSize */
    for (int i = 0; i < n; i++) rc_put(r, buf[i]);
    return DVO_SUCCESS;
}

/* ------------------------------------------------------------------------------------------
 * codec state  (codec/interface.rs:125-168, 246-264, 348-402, 713-775)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    /* CrossCommandBookKeeping */
    dvo_cdf16 *lit_len_priors, *cc_priors, *copy_priors, *dict_priors, *pred_priors, *btype_priors;
    uint8_t distance_context_map[1024];
    uint8_t cmap_lru[13];
    uint32_t distance_lru[4];
    uint8_t btype_lru[3][2];
    uint8_t btype_max_seen[3];
    uint8_t last_dlen, last_clen; uint32_t last_llen; uint8_t last_4_states;
    /* encoder wishes */
    uint8_t desired_prior_depth, desired_context_mixing; int desired_do_context_map; int desired_force_stride;
    int have_desired_adapt; dvo_speed desired_adapt[4];
    /* LiteralBookKeeping */
    uint64_t last_8_literals;
    uint8_t literal_context_map[16384];
    uint8_t btype_last, stride;
    uint8_t literal_prediction_mode;
    dvo_speed literal_adaptation[4];
    const uint8_t *lut0, *lut1;
    uint8_t mixing_mask[8192];
    dvo_weights model_weights[2];
    dvo_cdf16 *lit_cm_priors; /* allocated on first mixing>=2, codec/interface.rs:322-329 */
    dvo_cdf16 *lit_high_priors, *lit_low_priors;
    /* the single recycled PredictionMode scratch (codec/context_map.rs:69-94, threading.rs:494-526) */
    uint8_t pm_lit_map[16384]; uint8_t pm_dist_map[1024]; uint8_t pm_mixing[8192];
    uint32_t pm_map_len[2]; uint8_t pm_f8[4][2], pm_mode; /* what the last PredictionMode command carried (for dvo_decode_cmds) */
    /* coders + ring */
    coder cmd, lit;
    recoder rc;
    int mixing_trait; /* specializations.rs:26-36 */
    uint64_t n_cmds;
    int model_rev;    /* DVO_MODEL_CURRENT / DVO_MODEL_WASM_2018: see divans_oracle.h */
    dvo_cmdlist *rec; /* decoder: when non-NULL every decoded command is appended here */
} codec;

static void set_pred_mode_luts(codec *s, uint8_t mode) {
    /* codec/interface.rs:199-238 == brotli's context lookup table, modes LSB6=0 MSB6=1 UTF8=2 SIGN=3 */
    s->literal_prediction_mode = mode;
    s->lut0 = TB_CTX + 512 * (mode & 3);
    s->lut1 = TB_CTX + 512 * (mode & 3) + 256;
}
static void codec_init(codec *s, int window, int encoding) {
    memset(s, 0, sizeof(*s));
    s->lit_len_priors = alloc_priors(prior_total(T_LL, NEL(T_LL)));
    s->cc_priors = alloc_priors(prior_total(T_CC, NEL(T_CC)));
    s->copy_priors = alloc_priors(prior_total(T_CP, NEL(T_CP)));
    s->dict_priors = alloc_priors(prior_total(T_DC, NEL(T_DC)));
    s->pred_priors = alloc_priors(prior_total(T_PM, NEL(T_PM)));
    s->btype_priors = alloc_priors(prior_total(T_BT, NEL(T_BT)));
    s->lit_high_priors = alloc_priors(prior_total(T_LN, NEL(T_LN)));
    s->lit_low_priors = alloc_priors(prior_total(T_LN, NEL(T_LN)));
    s->last_dlen = 1; s->last_llen = 1; s->last_clen = 1;
    s->last_4_states = 3 << 4;
    s->distance_lru[0] = 4; s->distance_lru[1] = 11; s->distance_lru[2] = 15; s->distance_lru[3] = 16;
    for (int i = 0; i < 3; i++) { s->btype_lru[i][0] = 0; s->btype_lru[i][1] = 1; }
    for (int i = 0; i < 4; i++) s->literal_adaptation[i] = SPEED_MUD;
    /* LiteralPredictionModeNibble::default() lives in the brotli crate (NOT-IN-TREE): LSB6 assumed -- UNPINNED,
     * unobservable for streams that start with a PredictionMode command (all encoders emit one first) */
    set_pred_mode_luts(s, 0);
    dvo_weights_init(&s->model_weights[0]); dvo_weights_init(&s->model_weights[1]);
    s->rc.ring_len = 1u << window;
    s->rc.ring = (uint8_t *)calloc(1, s->rc.ring_len);
    s->cmd.encoding = s->lit.encoding = encoding;
    if (encoding) { ans_enc_init(&s->cmd.e); ans_enc_init(&s->lit.e); }
}
static void codec_free(codec *s) {
    free(s->lit_len_priors); free(s->cc_priors); free(s->copy_priors); free(s->dict_priors); free(s->pred_priors);
    free(s->btype_priors); free(s->lit_cm_priors); free(s->rc.ring);
    { dvo_cdf16 *big[2] = {s->lit_high_priors, s->lit_low_priors};
      for (int k = 0; k < 2; k++) { int put = 0; for (int i = 0; i < 2 && !put; i++) if (!tl_pool[i]) { tl_pool[i] = big[k]; put = 1; } if (!put) free(big[k]); } }
    if (s->cmd.encoding) { ans_enc_free(&s->cmd.e); ans_enc_free(&s->lit.e); }
}
#define P(tbl, T, type, i0, i1, i2) (&(tbl)[prior_index(T, NEL(T), type, i0, i1, i2)])

static inline void next_state(codec *s) { s->last_4_states >>= 2; }
static uint32_t get_distance_prior(codec *s, uint32_t copy_len) {
    /* codec/interface.rs:426-430 */
    uint32_t dtype = s->btype_lru[2][0];
    uint32_t m = copy_len < 2 ? 2 : copy_len;
    m -= 2; if (m > 3) m = 3;
    return s->distance_context_map[dtype * 4 + m];
}
static void get_distance_from_mnemonic_code(const uint32_t lru[4], uint8_t code, uint32_t *dist, int *ok) {
    /* codec/interface.rs:979-1009 */
    if (code < 4) { *dist = lru[code]; *ok = 1; return; }
    int32_t us = code >> 2;
    int32_t ss = us - (((-(int32_t)(code & 1)) & us) << 1);
    uint32_t index = (code & 2) >> 1;
    int32_t ret = (int32_t)lru[index] + ss;
    *dist = (uint32_t)ret; *ok = ret > 0;
}
static void obs_distance(codec *s, uint32_t distance) {
    /* codec/interface.rs:509-527 */
    uint32_t *l = s->distance_lru;
    if (distance == l[1]) { uint32_t n[4] = {distance, l[0], l[2], l[3]}; memcpy(l, n, sizeof n); }
    else if (distance == l[2]) { uint32_t n[4] = {distance, l[0], l[1], l[3]}; memcpy(l, n, sizeof n); }
    else if (distance != l[0]) { uint32_t n[4] = {distance, l[0], l[1], l[2]}; memcpy(l, n, sizeof n); }
}
static void obs_btype(codec *s, int which, uint8_t btype) {
    /* codec/interface.rs:528-532 */
    next_state(s);
    s->btype_lru[which][1] = s->btype_lru[which][0];
    s->btype_lru[which][0] = btype;
    if (btype > s->btype_max_seen[which]) s->btype_max_seen[which] = btype;
}

/* ---- literal length (codec/literal.rs:561-661) ---- */
static int code_literal_len(codec *s, uint32_t *len_io, int *high_entropy_io) {
    uint32_t literal_len = *len_io;
    uint32_t serialized_large = literal_len - 15u;
    uint8_t lllen = (uint8_t)bitlen32(serialized_large);
    uint32_t ctype = s->btype_lru[1][0];
    int he_flag = 0;
    for (;;) {
        uint32_t lm1 = literal_len - 1u;
        uint8_t nib = (uint8_t)(lm1 < 14 ? lm1 : 14);
        if (s->cmd.encoding && *high_entropy_io && !he_flag) nib = 15;
        nib = code_and_blend(&s->cmd, nib, P(s->lit_len_priors, T_LL, LL_CountSmall, ctype, 0, 0), SPEED_MED);
        if (nib == 14) break;
        if (nib == 15) { *high_entropy_io = 1; he_flag = 1; continue; }
        *len_io = (uint32_t)nib + 1; s->last_llen = *len_io;
        return DVO_SUCCESS;
    }
    uint8_t beg = (uint8_t)(lllen < 15 ? lllen : 15);
    beg = code_and_blend(&s->cmd, beg, P(s->lit_len_priors, T_LL, LL_SizeBegNib, ctype, 0, 0), SPEED_MUD);
    uint8_t len_remaining; uint32_t decoded;
    if (beg == 15) {
        uint8_t last = (uint8_t)(lllen - 15);
        last = code_and_blend(&s->cmd, last, P(s->lit_len_priors, T_LL, LL_SizeLastNib, ctype, 0, 0), SPEED_MUD);
        len_remaining = round_up_mod_4((uint8_t)(last + 14));
        decoded = (last + 14) < 32 ? (1u << (last + 14)) : 0;
    } else if (beg <= 1) {
        *len_io = 15u + beg; /* note: last_llen is NOT updated on this path (literal.rs:608-616) */
        return DVO_SUCCESS;
    } else {
        len_remaining = round_up_mod_4((uint8_t)(beg - 1));
        decoded = 1u << (beg - 1);
    }
    while (1) {
        uint8_t next_rem = (uint8_t)(len_remaining - 4);
        uint8_t nib = (uint8_t)((serialized_large ^ decoded) >> next_rem);
        nib = code_and_blend(&s->cmd, nib, P(s->lit_len_priors, T_LL, LL_SizeMantissaNib, ctype, 0, 0), SPEED_MUD);
        decoded |= (uint32_t)nib << next_rem;
        if (next_rem == 0) break;
        len_remaining = next_rem;
    }
    *len_io = decoded + 15u; s->last_llen = *len_io;
    return DVO_SUCCESS;
}

/* ---- one literal nibble (codec/literal.rs:154-259) ---- */
static inline uint8_t code_lit_nibble(codec *s, int is_high, uint8_t nib, uint8_t actual_context, uint8_t prev_byte,
                                      uint64_t stride_bytes, uint8_t cur_byte_prior, dvo_cdf16 **blendable) {
    uint32_t mmi = actual_context;
    if (!is_high) { mmi |= (uint32_t)(cur_byte_prior & 0xf) << 8; mmi |= 4096; }
    else mmi |= ((uint32_t)prev_byte >> 4) << 8;
    uint8_t mm_opts = s->mixing_mask[mmi];
    uint8_t fast_cm_prior_mask = (uint8_t)(-(int8_t)(mm_opts != 3));
    uint8_t mm = (uint8_t)(-(int)(mm_opts != 0 && mm_opts != 3));
    uint8_t opt_1_f_mask = (uint8_t)((-(int8_t)(mm_opts == 1)) & 0xf);
    uint32_t stride_offset = mm_opts < 4 ? 0 : (((uint32_t)(mm_opts ^ 4) < 7 ? (uint32_t)(mm_opts ^ 4) : 7u) << 3);
    uint8_t ssb = (uint8_t)(stride_bytes >> (0x38 - stride_offset));
    uint32_t index_b, index_c;
    if (is_high) {
        index_b = (uint8_t)(ssb & mm & (uint8_t)~opt_1_f_mask);
        index_c = actual_context;
    } else {
        index_b = (uint8_t)((mm & ssb) | ((uint8_t)~mm & actual_context));
        index_c = (uint8_t)((cur_byte_prior & fast_cm_prior_mask) | ((actual_context & opt_1_f_mask) << 4));
    }
    uint32_t which = (uint32_t)((mm >> 7) ^ (opt_1_f_mask >> 2));
    dvo_cdf16 *nibble_prob = P(is_high ? s->lit_high_priors : s->lit_low_priors, T_LN, LN_CombinedNibble, which, index_b, index_c);
    if (s->mixing_trait) {
        dvo_cdf16 *cm_prob = is_high ? P(s->lit_cm_priors, T_CM, CM_FirstNibble, 0, actual_context, 0)
                                     : P(s->lit_cm_priors, T_CM, CM_SecondNibble, 0, cur_byte_prior, actual_context);
        dvo_cdf16 prob;
        dvo_weights *mw = &s->model_weights[is_high ? 1 : 0];
        dvo_cdf_average(cm_prob, nibble_prob, (int32_t)(uint16_t)mw->norm, &prob);
        int16_t wfreq;
        nib = code_nibble(&s->lit, nib, &prob, &wfreq);
        int16_t st, f_cm, f_nb;
        dvo_cdf_sym_start_freq(cm_prob, nib, &st, &f_cm);
        dvo_cdf_sym_start_freq(nibble_prob, nib, &st, &f_nb);
        dvo_weights_update(mw, f_cm, f_nb, wfreq);
        dvo_cdf_blend(cm_prob, nib, s->literal_adaptation[2 | (is_high ? 1 : 0)]);
    } else {
        dvo_cdf16 dflt;
        const dvo_cdf16 *coder_prior = nibble_prob;
        if (mm_opts == 2) { dvo_cdf_default(&dflt); coder_prior = &dflt; }
        nib = code_nibble(&s->lit, nib, coder_prior, NULL);
    }
    *blendable = mm_opts == 2 ? NULL : nibble_prob;
    return nib;
}

/* ---- literal content bytes (codec/literal.rs:261-394, get_prev_word_context :87-117) ---- */
static void code_literal_bytes(codec *s, uint8_t *data, uint32_t len) {
    /* codec/decoder.rs:361-375 / codec/mod.rs:771-785: re-seed last_8_literals from the ring */
    uint8_t l8[8]; rc_last_8(&s->rc, l8);
    s->last_8_literals = 0;
    for (int i = 0; i < 8; i++) s->last_8_literals |= (uint64_t)l8[i] << (8 * i);
    for (uint32_t i = 0; i < len; i++) {
        uint8_t prev_byte = (uint8_t)(s->last_8_literals >> 0x38);
        uint8_t prev_prev = (uint8_t)(s->last_8_literals >> 0x30);
        uint8_t selected = s->lut0[prev_byte] | s->lut1[prev_prev];
        uint8_t actual_context = s->literal_context_map[(uint32_t)selected + ((uint32_t)s->btype_last << 6)];
        uint8_t byte = data[i];
        dvo_cdf16 *bl;
        uint8_t h = code_lit_nibble(s, 1, byte >> 4, actual_context, prev_byte, s->last_8_literals, 0, &bl);
        if (bl) dvo_cdf_blend(bl, h, s->literal_adaptation[0]);
        uint8_t l = code_lit_nibble(s, 0, byte & 0xf, actual_context, prev_byte, s->last_8_literals, h, &bl);
        uint8_t cur = (uint8_t)(l | (h << 4));
        s->last_8_literals = (s->last_8_literals >> 8) | ((uint64_t)cur << 0x38); /* push_literal_byte, interface.rs:280-284 */
        data[i] = cur;
        if (bl) dvo_cdf_blend(bl, l, s->literal_adaptation[0]);
    }
}

/* ---- copy (codec/copy.rs:50-286) ---- */
static int code_copy(codec *s, uint32_t *dist_io, uint32_t *num_io) {
    uint32_t in_dist = *dist_io, in_num = *num_io;
    uint8_t dlen = (uint8_t)bitlen32(in_dist), clen = (uint8_t)bitlen32(in_num);
    if (s->cmd.encoding && dlen == 0) return DVO_FAILURE;
    uint32_t ctype = s->btype_lru[1][0];
    uint32_t num_bytes, distance;
    {
        uint32_t ll = s->last_llen - 1u; if (ll > 3) ll = 3;
        uint32_t index = ((s->last_4_states >> 4) & 3u) + 4u * ll;
        uint8_t nib = (uint8_t)(in_num < 15 ? in_num : 15);
        nib = code_and_blend(&s->cmd, nib, P(s->copy_priors, T_CP, CP_CountSmall, ctype, index, 0), SPEED_MUD);
        if (nib != 15) {
            num_bytes = nib; s->last_clen = (uint8_t)bitlen32(num_bytes);
        } else {
            uint8_t beg = (uint8_t)(clen - 4); if (beg > 15) beg = 15;
            beg = code_and_blend(&s->cmd, beg, P(s->copy_priors, T_CP, CP_CountBegNib, ctype, 0, 0), SPEED_FAST);
            uint8_t len_remaining; uint32_t decoded;
            if (beg == 15) {
                uint8_t last = (uint8_t)(clen - 19);
                last = code_and_blend(&s->cmd, last, P(s->copy_priors, T_CP, CP_CountLastNib, ctype, 0, 0), SPEED_FAST);
                s->last_clen = (uint8_t)(last + 19);
                len_remaining = round_up_mod_4((uint8_t)(last + 18));
                /* last 14 / 15 (decoder only: no u32 count needs them) shift by 32 and 33 here and by 32 in the first mantissa
                 * step: every shift count is taken mod 32, as the reference's release build does (copy.rs:136,148) */
                decoded = 1u << ((last + 18) & 31);
            } else {
                s->last_clen = (uint8_t)(beg + 4);
                len_remaining = round_up_mod_4((uint8_t)(beg + 4 - 1));
                decoded = 1u << (beg + 4 - 1);
            }
            uint8_t len_decoded = 0;
            for (;;) {
                uint8_t next_rem = (uint8_t)(len_remaining - 4);
                uint8_t nb = (uint8_t)((in_num ^ decoded) >> (next_rem & 31));
                uint32_t index2 = len_decoded == 0 ? (uint32_t)((s->last_clen % 4) + 1) : 0u;
                nb = code_and_blend(&s->cmd, nb, P(s->copy_priors, T_CP, CP_CountMantissaNib, ctype, index2, 0), SPEED_SLOW);
                decoded |= (uint32_t)nb << (next_rem & 31);
                if (next_rem == 0) break;
                len_decoded = (uint8_t)(len_decoded + 4); len_remaining = next_rem;
            }
            num_bytes = decoded;
        }
    }
    {
        uint8_t beg = 15;
        if (s->cmd.encoding) { /* distance_mnemonic_code, codec/interface.rs:469-477 */
            for (uint8_t i = 0; i < 15; i++) {
                uint32_t d; int ok; get_distance_from_mnemonic_code(s->distance_lru, i, &d, &ok);
                if (d == in_dist && ok) { beg = i; break; }
            }
        }
        uint32_t ap = get_distance_prior(s, num_bytes);
        beg = code_and_blend(&s->cmd, beg, P(s->copy_priors, T_CP, CP_DistanceMnemonic, ap, (s->last_llen < 8), 0), SPEED_SLOW);
        if (beg != 15) {
            int ok; get_distance_from_mnemonic_code(s->distance_lru, beg, &distance, &ok);
            s->last_dlen = (uint8_t)bitlen32(distance);
            if (!ok) return DVO_FAILURE; /* CopyDistanceMnemonicCodeBad */
        } else {
            uint8_t bn = (uint8_t)(dlen - 1); if (bn > 14) bn = 14;
            /* copy.rs:199-201; the DVO_MODEL_WASM_2018 encoder did not take this shortcut (the decoder accepts both) */
            if ((uint32_t)(s->distance_lru[1] - 3u) == in_dist && !(s->cmd.encoding && s->model_rev == DVO_MODEL_WASM_2018)) bn = 15;
            uint32_t index = bitlen32(num_bytes) >> 2;
            bn = code_and_blend(&s->cmd, bn, P(s->copy_priors, T_CP, CP_DistanceBegNib, ap, index, 0), SPEED_SLOW);
            if (bn == 15) {
                distance = s->distance_lru[1] - 3u;
                s->last_dlen = (uint8_t)bitlen32(distance);
            } else if (bn == 0) {
                s->last_dlen = 1; distance = 1;
            } else {
                uint8_t start_rem; uint32_t decoded;
                if (bn == 14) {
                    uint8_t last = (uint8_t)(dlen - 15);
                    last = code_and_blend(&s->cmd, last, P(s->copy_priors, T_CP, CP_DistanceLastNib, ap, 0, 0), SPEED_ROCKET);
                    s->last_dlen = (uint8_t)(last + 14 + 1);
                    start_rem = round_up_mod_4((uint8_t)(last + 14));
                    decoded = (last + 14) < 32 ? (1u << (last + 14)) : 0;
                } else {
                    s->last_dlen = (uint8_t)(bn + 1);
                    start_rem = round_up_mod_4(bn);
                    decoded = 1u << bn;
                }
                uint8_t len_decoded = 0;
                for (int sr2 = (int)((start_rem + 3) >> 2) - 1; sr2 >= 0; sr2--) {
                    uint8_t next_rem = (uint8_t)(sr2 << 2);
                    uint8_t nb = (uint8_t)((in_dist ^ decoded) >> next_rem);
                    uint32_t index2 = len_decoded == 0 ? (uint32_t)((s->last_dlen & 3) + 1) : 0u;
                    dvo_speed sp; sp.inc = (int16_t)(0x4 << ((index2 & 6) << ((index2 & 2) >> 1))); sp.lim = 0x4000;
                    nb = code_and_blend(&s->cmd, nb, P(s->copy_priors, T_CP, CP_DistanceMantissaNib, ap, index2, 0), sp);
                    decoded |= (uint32_t)nb << next_rem;
                    len_decoded = (uint8_t)(len_decoded + 4);
                }
                distance = decoded;
            }
        }
    }
    *dist_io = distance; *num_io = num_bytes;
    return DVO_SUCCESS;
}

/* ---- dict (codec/dict.rs:49-176) ---- */
static int code_dict(codec *s, uint32_t *word_id_io, uint32_t *word_size_io, uint32_t *transform_io, uint32_t *final_size_out) {
    uint32_t in_id = *word_id_io; uint8_t in_size = (uint8_t)*word_size_io, in_tr = (uint8_t)*transform_io;
    uint32_t ctype = s->btype_lru[1][0];
    uint8_t beg = (uint8_t)(in_size - 4); if (beg > 15) beg = 15;
    beg = code_and_blend(&s->cmd, beg, P(s->dict_priors, T_DC, DC_SizeBegNib, ctype, 0, 0), SPEED_MUD);
    uint8_t word_size;
    if (beg == 15) {
        uint8_t b2 = (uint8_t)(in_size - 19);
        b2 = code_and_blend(&s->cmd, b2, P(s->dict_priors, T_DC, DC_SizeLastNib, ctype, 0, 0), SPEED_MUD);
        word_size = (uint8_t)(b2 + 19);
        if (word_size > 24) return DVO_FAILURE; /* DictWordSizeTooLarge */
    } else word_size = (uint8_t)(beg + 4);
    uint8_t bits = TB_SIZE_BITS[word_size];
    uint8_t len_remaining = round_up_mod_4(bits);
    uint32_t decoded = 0; uint8_t len_decoded = 0;
    for (;;) {
        uint8_t next_rem = (uint8_t)(len_remaining - 4);
        uint8_t nb = (uint8_t)((in_id ^ decoded) >> next_rem);
        uint32_t index = len_decoded == 0 ? (uint32_t)((bits % 4) + 1) : 0u;
        uint32_t ap = get_distance_prior(s, word_size);
        nb = code_and_blend(&s->cmd, nb, P(s->dict_priors, T_DC, DC_Index, ap, index, 0), SPEED_MUD);
        decoded |= (uint32_t)nb << next_rem;
        if (next_rem == 0) break;
        len_decoded = (uint8_t)(len_decoded + 4); len_remaining = next_rem;
    }
    uint8_t hi = (uint8_t)(in_tr >> 4);
    hi = code_and_blend(&s->cmd, hi, P(s->dict_priors, T_DC, DC_Transform, 0, (uint32_t)word_size >> 1, 0), SPEED_FAST);
    uint8_t tr = (uint8_t)(hi << 4);
    uint8_t lo = (uint8_t)(in_tr & 0xf);
    lo = code_and_blend(&s->cmd, lo, P(s->dict_priors, T_DC, DC_Transform, 1, (uint32_t)tr >> 4, 0), SPEED_FAST);
    tr |= lo;
    if (tr >= 121) return DVO_FAILURE; /* DictTransformIndexUndefined */
    /* final_size = length of the transformed word (content independent) */
    uint8_t tmp[64]; memset(tmp, 0, sizeof tmp);
    uint64_t wi = (uint64_t)decoded * word_size + TB_OFFSETS[word_size];
    int fl = (wi + word_size <= TB_DICT_SIZE) ? dvo_dict_word(word_size, decoded, tr, tmp) : -1;
    *word_id_io = decoded; *word_size_io = word_size; *transform_io = tr; *final_size_out = fl < 0 ? 0 : (uint32_t)fl;
    return DVO_SUCCESS;
}

/* ---- block switch (codec/block_type.rs:27-110,121-194) ---- */
static uint8_t code_btype(codec *s, int which, uint8_t in_bt) {
    uint8_t varint;
    if (in_bt == s->btype_lru[which][1]) varint = 0;
    else if (in_bt == (uint8_t)(s->btype_max_seen[which] + 1)) varint = 1;
    else if (in_bt <= 12) varint = (uint8_t)(in_bt + 2);
    else varint = 15;
    varint = code_and_blend(&s->cmd, varint, P(s->btype_priors, T_BT, BT_Mnemonic, which, 0, 0), SPEED_SLOW);
    if (varint == 0) return s->btype_lru[which][1];
    if (varint == 1) return (uint8_t)(s->btype_max_seen[which] + 1);
    if (varint != 15) return (uint8_t)(varint - 2);
    uint8_t first = (uint8_t)(in_bt & 0xf), second = (uint8_t)(in_bt >> 4);
    first = code_and_blend(&s->cmd, first, P(s->btype_priors, T_BT, BT_FirstNibble, which, 0, 0), SPEED_SLOW);
    second = code_and_blend(&s->cmd, second, P(s->btype_priors, T_BT, BT_SecondNibble, which, 0, 0), SPEED_SLOW);
    return (uint8_t)((second << 4) | first);
}

/* ---- prediction mode / context maps (codec/context_map.rs:105-428) ---- */
static void obs_context_map_for_lru(codec *s, uint8_t val) {
    /* codec/interface.rs:439-453 */
    int found = -1;
    for (int i = 0; i < 13; i++) if (s->cmap_lru[i] == val) { found = i; break; }
    if (found < 0) found = 12; /* shift everything, drop the last */
    for (int i = found; i > 0; i--) s->cmap_lru[i] = s->cmap_lru[i - 1];
    s->cmap_lru[0] = val;
}
static int code_context_map(codec *s, int is_distance, const uint8_t *in_map, uint32_t in_len, uint8_t *out_map, uint32_t out_cap) {
    const dvo_speed sp = SPEED_MED;
    for (uint32_t index = 0;; index++) {
        uint8_t mn;
        if (index >= in_len) mn = 14;
        else {
            uint8_t target = in_map[index];
            mn = 15;
            uint8_t mx = 0;
            for (int i = 0; i < 13; i++) { if (s->cmap_lru[i] == target) mn = (uint8_t)i; if (s->cmap_lru[i] > mx) mx = s->cmap_lru[i]; }
            if (target == (uint8_t)(mx + 1)) mn = 13;
        }
        /* context_map.rs:273 + codec/priors.rs:130: Mnemonic has its own four slots.  DVO_MODEL_WASM_2018 (the build
         * that produced wasm/wasm.html:98-107): both mnemonic priors are the CDF that ContextMapSpeedPalette[0],
         * DynamicContextMixingSpeed and PriorDepth share (the priors.rs:226-236 fall-through slot). */
        dvo_cdf16 *mn_prior = s->model_rev == DVO_MODEL_WASM_2018 ? P(s->pred_priors, T_PM, PM_ContextMapSpeedPalette, 0, 0, 0)
                                                                  : P(s->pred_priors, T_PM, PM_Mnemonic, is_distance, 0, 0);
        mn = code_and_blend(&s->cmd, mn, mn_prior, sp);
        if (mn == 14) { s->pm_map_len[is_distance] = index; return DVO_SUCCESS; }
        uint8_t val;
        if (mn == 15) {
            uint8_t msn = index >= in_len ? 0 : (uint8_t)(in_map[index] >> 4);
            msn = code_and_blend(&s->cmd, msn, P(s->pred_priors, T_PM, PM_FirstNibble, is_distance, 0, 0), sp);
            uint8_t lsn = index >= in_len ? 0 : (uint8_t)(in_map[index] & 0xf);
            lsn = code_and_blend(&s->cmd, lsn, P(s->pred_priors, T_PM, PM_SecondNibble, is_distance, 0, 0), sp);
            val = (uint8_t)((msn << 4) | lsn);
            if (index >= out_cap) return DVO_FAILURE; /* IndexBeyondContextMapSize */
            out_map[index] = val;
            obs_context_map_for_lru(s, val);
            if (is_distance) s->distance_context_map[index] = val;
        } else {
            if (mn == 13) { uint8_t mx = 0; for (int i = 0; i < 13; i++) if (s->cmap_lru[i] > mx) mx = s->cmap_lru[i]; val = (uint8_t)(mx + 1); }
            else val = s->cmap_lru[mn];
            if (is_distance && index >= 1024) return DVO_FAILURE;
            obs_context_map_for_lru(s, val);
            if (is_distance) s->distance_context_map[index] = val;
            if (index >= out_cap) return DVO_FAILURE;
            out_map[index] = val;
        }
    }
}
static int code_predmode(codec *s, const dvo_predmode *in) {
    /* encoder speed wishes: codec/context_map.rs:123-146 */
    dvo_speed desired[4] = {SPEED_MUD, SPEED_MUD, SPEED_MUD, SPEED_MUD};
    if (s->cmd.encoding && in) {
        if (in->has_speeds) {
            const uint16_t(*st)[2] = s->desired_context_mixing != 0 ? in->combined_speed : in->stride_speed;
            /* the encoder input stores f8 bytes; speeds given as u16 go through speed_to_u8 first (brotli setters) */
            for (int k = 0; k < 2; k++) {
                uint8_t a = brotli_speed_to_u8(in->cm_speed[k][0]), b = brotli_speed_to_u8(in->cm_speed[k][1]);
                if (a != 0 || b != 0) { desired[2 + k].inc = dvo_u8_to_speed(a); desired[2 + k].lim = dvo_u8_to_speed(b); }
                a = brotli_speed_to_u8(st[k][0]); b = brotli_speed_to_u8(st[k][1]);
                if (a != 0 || b != 0) { desired[k].inc = dvo_u8_to_speed(a); desired[k].lim = dvo_u8_to_speed(b); }
            }
        }
        if (s->have_desired_adapt) memcpy(desired, s->desired_adapt, sizeof desired);
    }
    /* Begin */
    for (int i = 0; i < 13; i++) s->cmap_lru[i] = (uint8_t)i;
    for (int i = 0; i < 1024; i++) s->distance_context_map[i] = (uint8_t)(i & 3);
    uint8_t pm = in ? in->pred_mode : 0;
    pm = code_and_blend(&s->cmd, pm, P(s->pred_priors, T_PM, PM_Only, 0, 0, 0), SPEED_MED);
    /* LiteralPredictionModeNibble::new(): < 16 ok (brotli crate); obs_pred_mode rejects > 3 (codec/interface.rs:268-279) */
    uint8_t mixnib = (uint8_t)(s->desired_context_mixing | ((in ? in->is_adv : 0) << 3));
    mixnib = code_and_blend(&s->cmd, mixnib, P(s->pred_priors, T_PM, PM_DynamicContextMixingSpeed, 0, 0, 0), SPEED_MED);
    uint8_t mixing_math = mixnib & 3;
    int combine = mixnib != 0;
    uint8_t pd = s->desired_prior_depth;
    pd = code_and_blend(&s->cmd, pd, P(s->pred_priors, T_PM, PM_PriorDepth, 0, 0, 0), SPEED_FAST);
    uint8_t f8[4][2]; memset(f8, 0, sizeof f8);
    for (uint32_t index = 0; index < 16; index++) {
        uint32_t si = index >> 2, pt = index & 3;
        uint8_t c0 = dvo_speed_to_u8(desired[si].inc), c1 = dvo_speed_to_u8(desired[si].lim);
        uint8_t nib;
        if (pt == 0) nib = (uint8_t)((c0 & 0x7f) >> 3);
        else if (pt == 1) nib = (uint8_t)((c0 & 0x7f) & 7);
        else if (pt == 2) nib = (uint8_t)((c1 & 0x7f) >> 3);
        else nib = (uint8_t)((c1 & 0x7f) & 7);
        nib = code_and_blend(&s->cmd, nib, P(s->pred_priors, T_PM, PM_ContextMapSpeedPalette, pt, 0, 0), SPEED_FAST);
        if (pt == 0) f8[si][0] |= (uint8_t)(nib << 3);
        if (pt == 1) f8[si][0] |= nib;
        if (pt == 2) f8[si][1] |= (uint8_t)(nib << 3);
        if (pt == 3) f8[si][1] |= nib;
    }
    /* literal then distance context map */
    int do_cm = s->cmd.encoding ? s->desired_do_context_map : 1;
    int rc = code_context_map(s, 0, in ? in->lit_map : NULL, (in && do_cm) ? in->lit_map_len : 0, s->pm_lit_map, 16384);
    if (rc != DVO_SUCCESS) return rc;
    for (int i = 0; i < 13; i++) s->cmap_lru[i] = (uint8_t)i;
    rc = code_context_map(s, 1, in ? in->dist_map : NULL, (in && do_cm) ? in->dist_map_len : 0, s->pm_dist_map, 1024);
    if (rc != DVO_SUCCESS) return rc;
    for (uint32_t index = 0; index < 8192; index++) {
        uint8_t mv;
        if (!s->cmd.encoding) mv = 0;
        else if (!s->desired_do_context_map) mv = 4;
        else if (!combine) mv = 0;
        else mv = in ? in->mixing[index] : 0;
        if (mv > 15) return DVO_FAILURE; /* no nibble: the record is refused (record_representable) */
        /* context_map.rs:395-399; DVO_MODEL_WASM_2018: one prior (slot 16) for every mixing value */
        uint32_t prior = (index >= 256 && s->model_rev != DVO_MODEL_WASM_2018) ? (uint32_t)(s->pm_mixing[index - 256] & 0xf) : 16u;
        mv = code_and_blend(&s->cmd, mv, P(s->pred_priors, T_PM, PM_PriorMixingValue, prior, 0, 0), SPEED_PLANE);
        s->pm_mixing[index] = mv;
    }
    /* obs_prediction_mode_context_map, codec/interface.rs:293-321 */
    s->model_weights[0].mixing_param = mixing_math; s->model_weights[1].mixing_param = mixing_math;
    if (mixing_math >= 2 && !s->lit_cm_priors) s->lit_cm_priors = alloc_priors(prior_total(T_CM, NEL(T_CM)));
    if (pm > 3) return DVO_FAILURE; /* PredictionModeOutOfBounds */
    set_pred_mode_luts(s, pm);
    for (int k = 0; k < 4; k++) {
        /* f8 nibbles -> u16 speed (brotli u8_to_speed) -> stored as f8 (brotli speed_to_u8) -> Speed::from_f8_tuple */
        uint8_t a = brotli_speed_to_u8(brotli_u8_to_speed(f8[k][0])), b = brotli_speed_to_u8(brotli_u8_to_speed(f8[k][1]));
        s->literal_adaptation[k].inc = dvo_u8_to_speed(a);
        s->literal_adaptation[k].lim = dvo_u8_to_speed(b);
    }
    memcpy(s->pm_f8, f8, sizeof f8); s->pm_mode = pm;
    memcpy(s->literal_context_map, s->pm_lit_map, 16384);
    memcpy(s->mixing_mask, s->pm_mixing, 8192);
    s->mixing_trait = (s->model_weights[0].mixing_param > 1) || (s->model_weights[1].mixing_param > 1);
    return DVO_SUCCESS;
}

/* ------------------------------------------------------------------------------------------
 * framing  (src/mux.rs)
 * ------------------------------------------------------------------------------------------ */
int dvo_demux(const uint8_t *in, size_t n, uint8_t *cmd, size_t *cmd_len, uint8_t *lit, size_t *lit_len, size_t *consumed) {
    /* header already skipped by the caller? no: `in` starts at the first record. mux.rs:384-444 */
    size_t pos = 0; size_t ln[2] = {0, 0}; uint8_t *dst[2] = {cmd, lit};
    for (;;) {
        if (pos >= n) return DVO_NEEDS_MORE_INPUT;
        uint8_t b = in[pos];
        if (b == 0xff) { /* EOF marker ff fe ff, only recognised at a record boundary (mux.rs:54,410-419) */
            if (pos + 3 > n) return DVO_NEEDS_MORE_INPUT;
            if (in[pos + 1] != 0xfe || in[pos + 2] != 0xff) return DVO_FAILURE;
            pos += 3; break;
        }
        uint32_t sid = b & 1, count;
        if (b < 16) {
            if (pos + 3 > n) return DVO_NEEDS_MORE_INPUT;
            count = ((uint32_t)in[pos + 1] | ((uint32_t)in[pos + 2] << 8)) + 1; pos += 3;
        } else {
            uint32_t k = b >> 4;
            if (k > 3) return DVO_FAILURE; /* the reference would mis-size these; never produced */
            count = 1024u << (k << 1); pos += 1;
        }
        if (pos + count > n) return DVO_NEEDS_MORE_INPUT;
        if (dst[sid]) memcpy(dst[sid] + ln[sid], in + pos, count);
        ln[sid] += count; pos += count;
    }
    *cmd_len = ln[0]; *lit_len = ln[1]; *consumed = pos;
    return DVO_SUCCESS;
}
static void mux_record(bytevec *out, int sid, const uint8_t *p, size_t n, size_t *taken) {
    /* get_code(stream, n, is_lagging=true), mux.rs:55-78 */
    if (n == 4096 || n == 16384 || n >= 65536) {
        uint8_t h; size_t w;
        if (n < 16384) { h = (uint8_t)(sid | (1 << 4)); w = 4096; }
        else if (n < 65536) { h = (uint8_t)(sid | (2 << 4)); w = 16384; }
        else { h = (uint8_t)(sid | (3 << 4)); w = 65536; }
        bv_push(out, &h, 1); bv_push(out, p, w); *taken = w;
    } else {
        uint8_t h[3] = {(uint8_t)sid, (uint8_t)((n - 1) & 0xff), (uint8_t)(((n - 1) >> 8) & 0xff)};
        bv_push(out, h, 3); bv_push(out, p, n); *taken = n;
    }
}
static void mux_close(bytevec *out, const uint8_t *p0, size_t n0, const uint8_t *p1, size_t n1) {
    /* serialize_close -> flush_internal with everything still buffered (mux.rs:478-561): the record
     * boundaries the reference produces depend on the caller's buffer sizes (SURVEY 8c note); this is the
     * boundary set for "nothing was linearized before close". */
    const uint8_t *p[2] = {p0, p1}; size_t rem[2] = {n0, n1}; size_t last_flush[2] = {0, 0}; size_t bytes_flushed = 0;
    for (;;) {
        int flushed_any = 0; int have = 0; size_t lf = 0;
        for (int i = 0; i < 2; i++) if (rem[i]) { if (!have || last_flush[i] < lf) { lf = last_flush[i]; have = 1; } }
        for (int i = 0; i < 2; i++) {
            if (!have || last_flush[i] <= lf + 131073) {
                if (rem[i]) {
                    size_t taken; mux_record(out, i, p[i], rem[i], &taken);
                    p[i] += taken; rem[i] -= taken; bytes_flushed += taken; last_flush[i] = bytes_flushed; flushed_any = 1;
                }
            }
        }
        if (!flushed_any) break;
    }
    static const uint8_t eof[3] = {0xff, 0xfe, 0xff};
    bv_push(out, eof, 3);
}
size_t dvo_mux_single(int stream_id, const uint8_t *data, size_t n, uint8_t *out, size_t cap) {
    bytevec v = {0};
    if (stream_id == 0) mux_close(&v, data, n, NULL, 0); else mux_close(&v, NULL, 0, data, n);
    size_t r = v.n; if (r <= cap) memcpy(out, v.p, r);
    bv_free(&v); return r;
}

/* ------------------------------------------------------------------------------------------
 * whole-stream decode  (divans_decompressor.rs:38-52,111-161 ; codec/decoder.rs:230-419 ; codec/mod.rs:652-1024)
 * ------------------------------------------------------------------------------------------ */
static dvo_cmd *cl_add(dvo_cmdlist *l);
static size_t cl_add_lit(dvo_cmdlist *l, const uint8_t *p, size_t n);
static dvo_predmode *cl_add_pm(dvo_cmdlist *l);
static void record_predmode(codec *s) {
    dvo_cmd *c = cl_add(s->rec); c->type = DVO_CMD_PREDMODE; c->a = (uint32_t)s->rec->n_pms;
    dvo_predmode *pm = cl_add_pm(s->rec);
    pm->pred_mode = s->pm_mode; pm->has_speeds = 1;
    for (int k = 0; k < 2; k++) for (int j = 0; j < 2; j++) {
        pm->stride_speed[k][j] = pm->combined_speed[k][j] = brotli_u8_to_speed(s->pm_f8[k][j]);
        pm->cm_speed[k][j] = brotli_u8_to_speed(s->pm_f8[2 + k][j]);
    }
    pm->lit_map_len = s->pm_map_len[0]; memcpy(pm->lit_map, s->pm_lit_map, pm->lit_map_len);
    pm->dist_map_len = s->pm_map_len[1]; memcpy(pm->dist_map, s->pm_dist_map, pm->dist_map_len);
    memcpy(pm->mixing, s->pm_mixing, 8192);
}
static int decode_impl(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len, int skip_crc,
                       size_t *in_consumed, uint64_t *n_cmd_nibbles, uint64_t *n_lit_nibbles, int model_rev, dvo_cmdlist *rec) {
    *out_len = 0;
    if (in_len < 16) return DVO_NEEDS_MORE_INPUT;
    if (in[0] != 0xff || in[1] != 0xe5 || in[2] != 0x8c || in[3] != 0x9f) return DVO_FAILURE;
    int window = in[5];
    if (window < 10 || window >= 25) return DVO_FAILURE;
    uint8_t *cmdbuf = (uint8_t *)malloc(in_len + 16), *litbuf = (uint8_t *)malloc(in_len + 16);
    size_t cl, ll, consumed;
    int rc = dvo_demux(in + 16, in_len - 16, cmdbuf, &cl, litbuf, &ll, &consumed);
    if (rc != DVO_SUCCESS) { free(cmdbuf); free(litbuf); return rc; }
    size_t trailer = 16 + consumed;
    if (trailer + 8 > in_len) { free(cmdbuf); free(litbuf); return DVO_NEEDS_MORE_INPUT; }
    codec *s = (codec *)malloc(sizeof(codec));
    codec_init(s, window, 0);
    s->model_rev = model_rev; s->rec = rec; if (rec) rec->window = window;
    ans_dec_init(&s->cmd.d, cmdbuf, cl); ans_dec_init(&s->lit.d, litbuf, ll);
    s->rc.out = out; s->rc.out_cap = out_cap;
    uint8_t *scratch = NULL; size_t scratch_cap = 0;
    rc = DVO_SUCCESS;
    for (;;) {
        uint8_t t = code_and_blend(&s->cmd, 0, P(s->cc_priors, T_CC, CC_FullSelection, (uint32_t)s->last_4_states >> 4, 0, 0), SPEED_ROCKET);
        if (s->cmd.d.underflow) { rc = DVO_NEEDS_MORE_INPUT; break; }
        if (t == 0xf) break;
        s->n_cmds++;
        if (t == DVO_CMD_COPY) {
            next_state(s); s->last_4_states |= 64;
            uint32_t d = 0, nb = 0;
            rc = code_copy(s, &d, &nb); if (rc) break;
            obs_distance(s, d);
            if (rec) { dvo_cmd *c = cl_add(rec); c->type = t; c->a = d; c->b = nb; }
            rc = rc_copy(&s->rc, d, nb); if (rc) break;
        } else if (t == DVO_CMD_DICT) {
            next_state(s); s->last_4_states |= 192;
            uint32_t id = 0, sz = 0, tr = 0, fs = 0;
            rc = code_dict(s, &id, &sz, &tr, &fs); if (rc) break;
            if (rec) { dvo_cmd *c = cl_add(rec); c->type = t; c->a = id; c->b = sz; c->c = tr; c->d = fs; }
            rc = rc_dict(&s->rc, sz, id, tr, fs); if (rc) break;
        } else if (t == DVO_CMD_LITERAL) {
            next_state(s); s->last_4_states |= 128;
            uint32_t len = 0; int he = 0;
            rc = code_literal_len(s, &len, &he); if (rc) break;
            if (s->cmd.d.underflow) { rc = DVO_NEEDS_MORE_INPUT; break; }
            if ((uint64_t)len > (uint64_t)out_cap + 16) { rc = DVO_NEEDS_MORE_OUTPUT; break; }
            if (len > scratch_cap) { scratch_cap = len + 1024; scratch = (uint8_t *)realloc(scratch, scratch_cap); }
            memset(scratch, 0, len);
            code_literal_bytes(s, scratch, len);
            if (s->lit.d.underflow) { rc = DVO_NEEDS_MORE_INPUT; break; }
            if (rec) { size_t off = cl_add_lit(rec, scratch, len); dvo_cmd *c = cl_add(rec); c->type = t; c->a = (uint32_t)off; c->b = len; c->c = (uint32_t)he; }
            for (uint32_t i = 0; i < len; i++) rc_put(&s->rc, scratch[i]);
        } else if (t == DVO_CMD_BTYPE_L) {
            uint8_t bt = code_btype(s, 0, 0);
            uint8_t stride = code_and_blend(&s->cmd, 0, P(s->btype_priors, T_BT, BT_StrideNibble, 0, 0, 0), SPEED_SLOW);
            obs_btype(s, 0, bt);
            s->btype_last = bt; s->stride = stride; /* obs_literal_block_switch, interface.rs:289-292 */
            if (rec) { dvo_cmd *c = cl_add(rec); c->type = t; c->a = bt; c->b = stride; }
        } else if (t == DVO_CMD_BTYPE_C) {
            uint8_t bt = code_btype(s, 1, 0); obs_btype(s, 1, bt);
            if (rec) { dvo_cmd *c = cl_add(rec); c->type = t; c->a = bt; }
        } else if (t == DVO_CMD_BTYPE_D) {
            uint8_t bt = code_btype(s, 2, 0); obs_btype(s, 2, bt);
            if (rec) { dvo_cmd *c = cl_add(rec); c->type = t; c->a = bt; }
        } else if (t == DVO_CMD_PREDMODE) {
            rc = code_predmode(s, NULL); if (rc) break;
            if (rec) record_predmode(s);
        } else { rc = DVO_FAILURE; break; } /* CommandCodeOutOfBounds */
        if (s->cmd.d.underflow || s->lit.d.underflow) { rc = DVO_NEEDS_MORE_INPUT; break; }
        if (s->rc.overflow) { rc = DVO_NEEDS_MORE_OUTPUT; break; }
    }
    /* The reference asks for input at the nibble that cannot be refilled (drain_or_fill_static_buffer, codec/interface.rs:868-917)
     * and never decodes past it.  This restatement runs a command to its end with zero-filled states and looks at the underflow
     * flags afterwards: an error a command reports AFTER one of its coders ran dry is a consequence of the garbage that
     * followed, so the earlier event wins. */
    if ((rc == DVO_FAILURE || rc == DVO_NEEDS_MORE_OUTPUT) && (s->cmd.d.underflow || s->lit.d.underflow)) rc = DVO_NEEDS_MORE_INPUT;
    *out_len = s->rc.out_len;
    if (n_cmd_nibbles) *n_cmd_nibbles = s->cmd.d.n_syms;
    if (n_lit_nibbles) *n_lit_nibbles = s->lit.d.n_syms;
    if (rc == DVO_SUCCESS && s->rc.overflow) rc = DVO_NEEDS_MORE_OUTPUT;
    if (rc == DVO_SUCCESS) {
        /* trailer: LE32 crc32c(header..EOF marker) + "ans~" (codec/decoder.rs:186-213) */
        uint32_t crc = dvo_crc32c(0, in, trailer);
        const uint8_t *tr = in + trailer;
        uint8_t want[8] = {(uint8_t)crc, (uint8_t)(crc >> 8), (uint8_t)(crc >> 16), (uint8_t)(crc >> 24), 'a', 'n', 's', '~'};
        for (int i = 0; i < 8; i++) if (want[i] != tr[i] && (i >= 4 || !skip_crc)) { rc = DVO_FAILURE; break; }
    }
    if (in_consumed) *in_consumed = trailer + 8;
    free(scratch); codec_free(s); free(s); free(cmdbuf); free(litbuf);
    return rc;
}
int dvo_decode_ex(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len, int skip_crc,
                  size_t *in_consumed, uint64_t *n_cmd_nibbles, uint64_t *n_lit_nibbles) {
    return decode_impl(in, in_len, out, out_cap, out_len, skip_crc, in_consumed, n_cmd_nibbles, n_lit_nibbles, DVO_MODEL_CURRENT, NULL);
}
int dvo_decode(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len, int skip_crc) {
    return dvo_decode_ex(in, in_len, out, out_cap, out_len, skip_crc, NULL, NULL, NULL);
}
int dvo_decode_cmds(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len, int skip_crc,
                    int model_rev, dvo_cmdlist *cmds) {
    return decode_impl(in, in_len, out, out_cap, out_len, skip_crc, NULL, NULL, NULL, model_rev, cmds);
}

/* ------------------------------------------------------------------------------------------
 * whole-stream encode (divans_compressor.rs:126-174,276-427 ; codec/mod.rs:409-560)
 * ------------------------------------------------------------------------------------------ */
void dvo_options_default(dvo_options *o) {
    memset(o, 0, sizeof *o);
    o->window_size = 22; o->dynamic_context_mixing = 0; o->prior_depth = 0; o->use_context_map = 1; o->force_stride = 9;
}
/* Whether a stream can carry record c: every nibble the encoder would build from it is a nibble (0..15) that decodes back to
 * the record's value.  A record that fails this is refused before its type nibble is coded (include/divans_b200.h, DVCL):
 *  - type 1..7 (15 would end the stream, 0 and 8..14 fail the decode);
 *  - copy: distance 1 .. 2^30 - 1 (DistanceLastNib = bit length - 15 must be a nibble);
 *  - literal: length 1 .. 2^30 + 14 (length 0 codes as 2^15 and more; SizeLastNib = bit length of length - 15, minus 15);
 *  - dictionary: word size 4..24, word id below 2^round_up_mod_4(bits of the size), transform below 256 (121..255 are
 *    carried and fail the decode, DictTransformIndexUndefined);
 *  - block switch: type below 256, and a literal block switch's stride below 16 when the stride comes from the record;
 *  - PredictionMode: pred_mode below 16 (4..15 are carried and fail the decode), is_adv 0 or 1; mixing values: code_predmode. */
static int record_representable(const codec *s, const dvo_cmdlist *l, const dvo_cmd *c) {
    switch (c->type) {
    case DVO_CMD_COPY: return c->a != 0 && c->a < (1u << 30);
    case DVO_CMD_LITERAL: return c->b - 1u < (1u << 30) + 14u;
    case DVO_CMD_DICT: return c->b >= 4 && c->b <= 24 && c->c < 256 && (c->a >> round_up_mod_4(TB_SIZE_BITS[c->b])) == 0;
    case DVO_CMD_BTYPE_L: return c->a < 256 && (s->desired_force_stride != 9 || c->b < 16);
    case DVO_CMD_BTYPE_C: case DVO_CMD_BTYPE_D: return c->a < 256;
    case DVO_CMD_PREDMODE: return c->a < l->n_pms && l->pms[c->a].pred_mode < 16 && l->pms[c->a].is_adv < 2;
    default: return 0;
    }
}
int dvo_encode_cmds(const dvo_cmdlist *l, const dvo_options *o, uint8_t *out, size_t cap, size_t *out_len) {
    int window = o->window_size < 10 ? 10 : (o->window_size > 24 ? 24 : o->window_size);
    codec *s = (codec *)malloc(sizeof(codec));
    codec_init(s, window, 1);
    s->rc.out = NULL; s->rc.out_cap = 0;
    /* CrossCommandBookKeeping::new, codec/interface.rs:360-366 */
    int dcm = o->dynamic_context_mixing;
    if (o->force_stride != 0 && dcm == 0 && o->use_context_map) dcm = 1;
    s->desired_context_mixing = (uint8_t)dcm; s->desired_prior_depth = (uint8_t)o->prior_depth;
    s->desired_do_context_map = o->use_context_map; s->desired_force_stride = o->force_stride;
    s->have_desired_adapt = o->have_literal_adaptation;
    s->model_rev = o->model_rev;
    memcpy(s->desired_adapt, o->literal_adaptation, sizeof s->desired_adapt);
    int rc = DVO_SUCCESS;
    uint8_t *scratch = NULL; size_t scratch_cap = 0;
    for (size_t ci = 0; ci < l->n_cmds && rc == DVO_SUCCESS; ci++) {
        const dvo_cmd *c = &l->cmds[ci];
        if (!record_representable(s, l, c)) { rc = DVO_FAILURE; break; }
        code_and_blend(&s->cmd, (uint8_t)c->type, P(s->cc_priors, T_CC, CC_FullSelection, (uint32_t)s->last_4_states >> 4, 0, 0), SPEED_ROCKET);
        switch (c->type) {
        case DVO_CMD_COPY: {
            next_state(s); s->last_4_states |= 64;
            uint32_t d = c->a, nb = c->b;
            rc = code_copy(s, &d, &nb); if (rc) break;
            obs_distance(s, d);
            rc = rc_copy(&s->rc, d, nb);
        } break;
        case DVO_CMD_DICT: {
            next_state(s); s->last_4_states |= 192;
            uint32_t id = c->a, sz = c->b, tr = c->c, fs = 0;
            rc = code_dict(s, &id, &sz, &tr, &fs); if (rc) break;
            rc = rc_dict(&s->rc, sz, id, tr, fs); /* the coded command's final_size (dict.rs:163-166), not the IR's */
        } break;
        case DVO_CMD_LITERAL: {
            next_state(s); s->last_4_states |= 128;
            uint32_t len = c->b; int he = (int)c->c;
            rc = code_literal_len(s, &len, &he); if (rc) break;
            if (len > scratch_cap) { scratch_cap = len + 1024; scratch = (uint8_t *)realloc(scratch, scratch_cap); }
            memcpy(scratch, l->lits + c->a, len);
            code_literal_bytes(s, scratch, len);
            for (uint32_t i = 0; i < len; i++) rc_put(&s->rc, scratch[i]);
        } break;
        case DVO_CMD_BTYPE_L: {
            uint8_t bt = code_btype(s, 0, (uint8_t)c->a);
            uint8_t stride = (uint8_t)(s->desired_force_stride == 9 ? c->b : (uint32_t)s->desired_force_stride);
            stride = code_and_blend(&s->cmd, stride, P(s->btype_priors, T_BT, BT_StrideNibble, 0, 0, 0), SPEED_SLOW);
            obs_btype(s, 0, bt); s->btype_last = bt; s->stride = stride;
        } break;
        case DVO_CMD_BTYPE_C: { uint8_t bt = code_btype(s, 1, (uint8_t)c->a); obs_btype(s, 1, bt); } break;
        case DVO_CMD_BTYPE_D: { uint8_t bt = code_btype(s, 2, (uint8_t)c->a); obs_btype(s, 2, bt); } break;
        case DVO_CMD_PREDMODE: rc = code_predmode(s, &l->pms[c->a]); break;
        default: rc = DVO_FAILURE;
        }
    }
    if (rc == DVO_SUCCESS && (s->cmd.e.bad || s->lit.e.bad)) rc = DVO_FAILURE; /* the reference encoder panics here */
    if (rc == DVO_SUCCESS) {
        /* flush: end-of-stream nibble 0xf, close both coders, drain mux, EOF marker, trailer (codec/mod.rs:424-560) */
        code_and_blend(&s->cmd, 0xf, P(s->cc_priors, T_CC, CC_FullSelection, (uint32_t)s->last_4_states >> 4, 0, 0), SPEED_ROCKET);
        ans_enc_flush_chunk(&s->cmd.e); ans_enc_flush_chunk(&s->lit.e);
        bytevec v = {0};
        uint8_t hdr[16] = {0xff, 0xe5, 0x8c, 0x9f, 0, (uint8_t)window, 0}; /* make_header, divans_compressor.rs:126-131 */
        bv_push(&v, hdr, 16);
        mux_close(&v, s->cmd.e.out.p, s->cmd.e.out.n, s->lit.e.out.p, s->lit.e.out.n);
        uint32_t crc = dvo_crc32c(0, v.p, v.n);
        uint8_t tr[8] = {(uint8_t)crc, (uint8_t)(crc >> 8), (uint8_t)(crc >> 16), (uint8_t)(crc >> 24), 'a', 'n', 's', '~'};
        bv_push(&v, tr, 8);
        *out_len = v.n;
        if (v.n <= cap) memcpy(out, v.p, v.n); else rc = DVO_NEEDS_MORE_OUTPUT;
        bv_free(&v);
    }
    free(scratch); codec_free(s); free(s);
    return rc;
}

/* ---- command lists ---- */
void dvo_cmdlist_init(dvo_cmdlist *l) { memset(l, 0, sizeof *l); }
void dvo_cmdlist_free(dvo_cmdlist *l) { free(l->cmds); free(l->lits); free(l->pms); memset(l, 0, sizeof *l); }
static dvo_cmd *cl_add(dvo_cmdlist *l) {
    if (l->n_cmds == l->cap_cmds) { l->cap_cmds = l->cap_cmds ? l->cap_cmds * 2 : 64; l->cmds = (dvo_cmd *)realloc(l->cmds, l->cap_cmds * sizeof(dvo_cmd)); }
    dvo_cmd *c = &l->cmds[l->n_cmds++]; memset(c, 0, sizeof *c); return c;
}
static size_t cl_add_lit(dvo_cmdlist *l, const uint8_t *p, size_t n) {
    if (l->n_lits + n > l->cap_lits) { size_t nc = l->cap_lits ? l->cap_lits * 2 : 4096; while (nc < l->n_lits + n) nc *= 2; l->lits = (uint8_t *)realloc(l->lits, nc); l->cap_lits = nc; }
    size_t off = l->n_lits; if (p) memcpy(l->lits + off, p, n); l->n_lits += n; return off;
}
static dvo_predmode *cl_add_pm(dvo_cmdlist *l) {
    if (l->n_pms == l->cap_pms) { l->cap_pms = l->cap_pms ? l->cap_pms * 2 : 2; l->pms = (dvo_predmode *)realloc(l->pms, l->cap_pms * sizeof(dvo_predmode)); }
    dvo_predmode *p = &l->pms[l->n_pms++]; memset(p, 0, sizeof *p); return p;
}
static void internal_predmode(dvo_predmode *pm, int pred_mode, int mixing_value) {
    /* raw_to_cmd/mod.rs:116-143: 64-entry identity literal map, 4 distance entries, mixing values 4, speeds unset */
    memset(pm, 0, sizeof *pm);
    pm->pred_mode = (uint8_t)pred_mode; pm->has_speeds = 1;
    pm->lit_map_len = 64; for (int i = 0; i < 64; i++) pm->lit_map[i] = (uint8_t)(i & 0x3f);
    pm->dist_map_len = 4; for (int i = 0; i < 4; i++) pm->dist_map[i] = (uint8_t)(i & 3);
    memset(pm->mixing, mixing_value, 8192);
}
/* the literal-only list under the PredictionMode record of (pred_mode, mixing_value); dvo_encode_raw's is (LSB6, 4) */
static int encode_raw_record(const uint8_t *in, size_t n, const dvo_options *o, int pred_mode, int mixing_value, uint8_t *out, size_t cap,
                             size_t *out_len) {
    dvo_cmdlist l; dvo_cmdlist_init(&l);
    int window = o->window_size < 10 ? 10 : (o->window_size > 24 ? 24 : o->window_size);
    dvo_cmd *c = cl_add(&l); c->type = DVO_CMD_PREDMODE; c->a = 0;
    internal_predmode(cl_add_pm(&l), pred_mode, mixing_value);
    size_t ring = (size_t)1 << window;
    for (size_t pos = 0; pos < n;) { /* one Literal per ring-buffer fill, raw_to_cmd/mod.rs:55-104,144-181 */
        size_t chunk = n - pos < ring ? n - pos : ring;
        size_t off = cl_add_lit(&l, in + pos, chunk);
        c = cl_add(&l); c->type = DVO_CMD_LITERAL; c->a = (uint32_t)off; c->b = (uint32_t)chunk; c->c = 0;
        pos += chunk;
    }
    int rc = dvo_encode_cmds(&l, o, out, cap, out_len);
    dvo_cmdlist_free(&l);
    return rc;
}
int dvo_encode_raw(const uint8_t *in, size_t n, const dvo_options *o, uint8_t *out, size_t cap, size_t *out_len) {
    return encode_raw_record(in, n, o, 0, 4, out, cap, out_len);
}

/* deterministic greedy hash-chain LZ77 (ours; SURVEY 8d "Z" streams): min match 4, max match 2^16, no dictionary */
int dvo_lz77_cmds(const uint8_t *in, size_t n, int window, int pred_mode, int mixing_value, dvo_cmdlist *l) {
    dvo_cmd *c = cl_add(l); c->type = DVO_CMD_PREDMODE; c->a = (uint32_t)l->n_pms;
    internal_predmode(cl_add_pm(l), pred_mode, mixing_value);
    const size_t HB = 15; size_t hs = (size_t)1 << HB;
    int32_t *head = (int32_t *)malloc(hs * sizeof(int32_t)); int32_t *prev = (int32_t *)malloc((n + 1) * sizeof(int32_t));
    for (size_t i = 0; i < hs; i++) head[i] = -1;
    size_t maxdist = ((size_t)1 << window) - 16;
    size_t lit_start = 0, i = 0;
#define H4(p) ((((uint32_t)(p)[0] | ((uint32_t)(p)[1] << 8) | ((uint32_t)(p)[2] << 16) | ((uint32_t)(p)[3] << 24)) * 2654435761u) >> (32 - HB))
    while (i < n) {
        size_t best_len = 0, best_dist = 0;
        if (i + 4 <= n) {
            uint32_t h = H4(in + i);
            int32_t cand = head[h]; int chain = 16;
            while (cand >= 0 && chain-- > 0 && i - (size_t)cand <= maxdist) {
                size_t m = 0, lim = n - i; if (lim > 65535) lim = 65535;
                while (m < lim && in[cand + m] == in[i + m]) m++;
                if (m > best_len) { best_len = m; best_dist = i - (size_t)cand; }
                cand = prev[cand];
            }
        }
        if (best_len >= 4) {
            if (i > lit_start) { size_t off = cl_add_lit(l, in + lit_start, i - lit_start); c = cl_add(l); c->type = DVO_CMD_LITERAL; c->a = (uint32_t)off; c->b = (uint32_t)(i - lit_start); }
            c = cl_add(l); c->type = DVO_CMD_COPY; c->a = (uint32_t)best_dist; c->b = (uint32_t)best_len;
            for (size_t k = 0; k < best_len; k++) { if (i + 4 <= n) { uint32_t h = H4(in + i); prev[i] = head[h]; head[h] = (int32_t)i; } i++; }
            lit_start = i;
        } else {
            if (i + 4 <= n) { uint32_t h = H4(in + i); prev[i] = head[h]; head[h] = (int32_t)i; }
            i++;
        }
    }
    if (n > lit_start) { size_t off = cl_add_lit(l, in + lit_start, n - lit_start); c = cl_add(l); c->type = DVO_CMD_LITERAL; c->a = (uint32_t)off; c->b = (uint32_t)(n - lit_start); }
    free(head); free(prev);
    return DVO_SUCCESS;
}

int dvo_recode(const dvo_cmdlist *l, int window, uint8_t *out, size_t cap, size_t *out_len) {
    recoder r; memset(&r, 0, sizeof r);
    r.ring_len = 1u << window; r.ring = (uint8_t *)calloc(1, r.ring_len); r.out = out; r.out_cap = cap;
    int rc = DVO_SUCCESS;
    for (size_t i = 0; i < l->n_cmds && rc == DVO_SUCCESS; i++) {
        const dvo_cmd *c = &l->cmds[i];
        if (c->type == DVO_CMD_COPY) rc = rc_copy(&r, c->a, c->b);
        else if (c->type == DVO_CMD_DICT) rc = rc_dict(&r, c->b, c->a, c->c, c->d);
        else if (c->type == DVO_CMD_LITERAL) for (uint32_t k = 0; k < c->b; k++) rc_put(&r, l->lits[c->a + k]);
    }
    *out_len = r.out_len; if (r.overflow && rc == DVO_SUCCESS) rc = DVO_NEEDS_MORE_OUTPUT;
    free(r.ring); return rc;
}

/* ---- IR text (src/bin/divans.rs:191-483) ---- */
static int hexval(int ch) { if (ch >= '0' && ch <= '9') return ch - '0'; if (ch >= 'a' && ch <= 'f') return ch - 'a' + 10; if (ch >= 'A' && ch <= 'F') return ch - 'A' + 10; return -1; }
static const char *next_tok(const char *p, const char *end, const char **tok, size_t *tl) {
    /* split(' '): single spaces delimit, empty tokens possible */
    if (p > end) return NULL;
    const char *q = p; while (q < end && *q != ' ') q++;
    *tok = p; *tl = (size_t)(q - p);
    return q < end ? q + 1 : end + 1;
}
static int tok_is(const char *t, size_t tl, const char *s) { return strlen(s) == tl && memcmp(t, s, tl) == 0; }
static int tok_num(const char *t, size_t tl, long long *v) {
    if (tl == 0 || tl > 18) return 0;
    long long r = 0; size_t i = 0; int neg = 0;
    if (t[0] == '-') { neg = 1; i = 1; if (tl == 1) return 0; }
    for (; i < tl; i++) { if (t[i] < '0' || t[i] > '9') return 0; r = r * 10 + (t[i] - '0'); }
    *v = neg ? -r : r; return 1;
}
static int dvo_parse_ir_inner(const char *p, const char *tend, dvo_cmdlist *l, const char **toks, size_t *tls, int MAXTOK);
int dvo_parse_ir(const char *text, size_t n, dvo_cmdlist *l) {
    const char *p = text, *tend = text + n;
    const int MAXTOK = 40000;
    const char **toks = (const char **)malloc(sizeof(char *) * MAXTOK);
    size_t *tls = (size_t *)malloc(sizeof(size_t) * MAXTOK);
    int ret = dvo_parse_ir_inner(p, tend, l, toks, tls, MAXTOK);
    free(toks); free(tls);
    return ret;
}
static int dvo_parse_ir_inner(const char *p, const char *tend, dvo_cmdlist *l, const char **toks, size_t *tls, int MAXTOK) {
    while (p < tend) {
        const char *eol = (const char *)memchr(p, '\n', (size_t)(tend - p)); if (!eol) eol = tend;
        const char *le = eol; if (le > p && le[-1] == '\r') le--;
        const char *line = p; p = eol + 1;
        if (le == line) continue;
        int nt = 0;
        { const char *q = line; const char *t; size_t tl; while ((q = next_tok(q, le, &t, &tl)) != NULL && nt < MAXTOK) { toks[nt] = t; tls[nt] = tl; nt++; } }
        if (nt == 0) continue;
        if (tok_is(toks[0], tls[0], "window")) { long long v; if (nt > 1 && tok_num(toks[1], tls[1], &v)) l->window = (int)v; continue; }
        if (tok_is(toks[0], tls[0], "prediction")) {
            if (nt < 2) return DVO_FAILURE;
            dvo_cmd *c = cl_add(l); c->type = DVO_CMD_PREDMODE; c->a = (uint32_t)l->n_pms;
            dvo_predmode *pm = cl_add_pm(l);
            pm->has_speeds = 1;
            if (tok_is(toks[1], tls[1], "utf8")) pm->pred_mode = 2; else if (tok_is(toks[1], tls[1], "sign")) pm->pred_mode = 3;
            else if (tok_is(toks[1], tls[1], "lsb6")) pm->pred_mode = 0; else if (tok_is(toks[1], tls[1], "msb6")) pm->pred_mode = 1;
            else return DVO_FAILURE;
            for (int k = 2; k < nt; k++) {
                if (tok_is(toks[k], tls[k], "lcontextmap")) { for (int j = k + 1; j < nt; j++) { long long v; if (!tok_num(toks[j], tls[j], &v)) break; if (v < 0 || v > 255) return DVO_FAILURE; if (pm->lit_map_len < 16384) pm->lit_map[pm->lit_map_len++] = (uint8_t)v; } }
                else if (tok_is(toks[k], tls[k], "dcontextmap")) { for (int j = k + 1; j < nt; j++) { long long v; if (!tok_num(toks[j], tls[j], &v)) break; if (v < 0 || v > 255) return DVO_FAILURE; if (pm->dist_map_len < 1024) pm->dist_map[pm->dist_map_len++] = (uint8_t)v; } }
                else if (tok_is(toks[k], tls[k], "mixingvalues")) { uint32_t off = 0; for (int j = k + 1; j < nt; j++) { long long v; if (!tok_num(toks[j], tls[j], &v)) break; if (off >= 8192 || v < 0 || v > 8) return DVO_FAILURE; pm->mixing[off++] = (uint8_t)v; } }
                else {
                    static const char *keys[3][2] = {{"cmspeedinc", "cmspeedmax"}, {"stspeedinc", "stspeedmax"}, {"mxspeedinc", "mxspeedmax"}};
                    for (int w = 0; w < 3; w++) for (int im = 0; im < 2; im++) if (tok_is(toks[k], tls[k], keys[w][im])) {
                        uint16_t(*dst)[2] = w == 0 ? pm->cm_speed : (w == 1 ? pm->stride_speed : pm->combined_speed);
                        for (int j = 0; j < 2 && k + 1 + j < nt; j++) { long long v; if (!tok_num(toks[k + 1 + j], tls[k + 1 + j], &v)) break; if (v < 0 || v > 16384) return DVO_FAILURE; dst[j][im] = (uint16_t)v; }
                    }
                }
            }
            continue;
        }
        if (tok_is(toks[0], tls[0], "ctype") || tok_is(toks[0], tls[0], "ltype") || tok_is(toks[0], tls[0], "dtype")) {
            long long v; if (nt < 2 || !tok_num(toks[1], tls[1], &v)) return DVO_FAILURE;
            dvo_cmd *c = cl_add(l); c->a = (uint32_t)(uint8_t)v;
            c->type = toks[0][0] == 'c' ? DVO_CMD_BTYPE_C : (toks[0][0] == 'd' ? DVO_CMD_BTYPE_D : DVO_CMD_BTYPE_L);
            if (toks[0][0] == 'l' && nt >= 3) { long long sv; if (!tok_num(toks[2], tls[2], &sv) || sv > 8) return DVO_FAILURE; c->b = (uint32_t)sv; }
            continue;
        }
        if (tok_is(toks[0], tls[0], "copy")) {
            long long len, dist; if (nt < 4 || !tok_num(toks[1], tls[1], &len) || !tok_is(toks[2], tls[2], "from") || !tok_num(toks[3], tls[3], &dist)) return DVO_FAILURE;
            if (len == 0) continue;
            dvo_cmd *c = cl_add(l); c->type = DVO_CMD_COPY; c->a = (uint32_t)dist; c->b = (uint32_t)len; continue;
        }
        if (tok_is(toks[0], tls[0], "dict")) {
            long long flen; if (nt < 6 || !tok_num(toks[1], tls[1], &flen) || !tok_is(toks[2], tls[2], "word")) return DVO_FAILURE;
            const char *comma = (const char *)memchr(toks[3], ',', tls[3]); if (!comma) return DVO_FAILURE;
            long long wl, wi; if (!tok_num(toks[3], (size_t)(comma - toks[3]), &wl) || !tok_num(comma + 1, tls[3] - (size_t)(comma - toks[3]) - 1, &wi)) return DVO_FAILURE;
            int found = 0;
            for (int k = 5; k < nt; k++) if (tok_is(toks[k - 1], tls[k - 1], "func")) {
                long long tr; if (!tok_num(toks[k], tls[k], &tr)) return DVO_FAILURE;
                dvo_cmd *c = cl_add(l); c->type = DVO_CMD_DICT; c->a = (uint32_t)wi; c->b = (uint32_t)(uint8_t)wl; c->c = (uint32_t)(uint8_t)tr; c->d = (uint32_t)(uint8_t)flen; found = 1; break;
            }
            if (!found) return DVO_FAILURE;
            continue;
        }
        if (tok_is(toks[0], tls[0], "insert") || tok_is(toks[0], tls[0], "rndins")) {
            long long len; if (nt < 2 || !tok_num(toks[1], tls[1], &len)) return DVO_FAILURE;
            if (len == 0) continue;
            if (nt < 3) return DVO_FAILURE;
            const char *hx = toks[2]; size_t hl = tls[2];
            if (hl != (size_t)len * 2) return DVO_FAILURE;
            size_t off = cl_add_lit(l, NULL, (size_t)len);
            for (long long k = 0; k < len; k++) { int a = hexval(hx[2 * k]), b = hexval(hx[2 * k + 1]); if (a < 0 || b < 0) return DVO_FAILURE; l->lits[off + k] = (uint8_t)((a << 4) | b); }
            dvo_cmd *c = cl_add(l); c->type = DVO_CMD_LITERAL; c->a = (uint32_t)off; c->b = (uint32_t)len; c->c = tok_is(toks[0], tls[0], "rndins");
            continue;
        }
        return DVO_FAILURE;
    }
    return DVO_SUCCESS;
}

/* flat binary command list: see include/divans_b200.h "command list blob" */
size_t dvo_cmdlist_serialize(const dvo_cmdlist *l, uint8_t *out, size_t cap) {
    size_t pm_sz = 32 + 16384 + 1024 + 8192;
    size_t need = 32 + l->n_cmds * 20 + l->n_pms * pm_sz + l->n_lits;
    if (!out || cap < need) return need;
    uint8_t *p = out;
    uint32_t hdr[8] = {0x4c435644u /* "DVCL" */, 1, (uint32_t)l->n_cmds, (uint32_t)l->n_pms, (uint32_t)l->n_lits, (uint32_t)l->window, 0, 0};
    memcpy(p, hdr, 32); p += 32;
    for (size_t i = 0; i < l->n_cmds; i++) { uint32_t r[5] = {l->cmds[i].type, l->cmds[i].a, l->cmds[i].b, l->cmds[i].c, l->cmds[i].d}; memcpy(p, r, 20); p += 20; }
    for (size_t i = 0; i < l->n_pms; i++) {
        const dvo_predmode *m = &l->pms[i];
        uint8_t h[32]; memset(h, 0, 32);
        h[0] = m->pred_mode; h[1] = m->is_adv; h[2] = m->has_speeds;
        uint16_t sp[12]; for (int k = 0; k < 2; k++) for (int j = 0; j < 2; j++) { sp[k * 2 + j] = m->cm_speed[k][j]; sp[4 + k * 2 + j] = m->stride_speed[k][j]; sp[8 + k * 2 + j] = m->combined_speed[k][j]; }
        memcpy(h + 4, sp, 24);
        uint16_t ll = (uint16_t)m->lit_map_len, dl = (uint16_t)m->dist_map_len; memcpy(h + 28, &ll, 2); memcpy(h + 30, &dl, 2);
        memcpy(p, h, 32); p += 32;
        memcpy(p, m->lit_map, 16384); p += 16384; memcpy(p, m->dist_map, 1024); p += 1024; memcpy(p, m->mixing, 8192); p += 8192;
    }
    memcpy(p, l->lits, l->n_lits); p += l->n_lits;
    return (size_t)(p - out);
}

/* ---- threaded batch helpers for the CPU baseline ---- */
typedef struct {
    const uint8_t *in; const uint64_t *in_off, *in_len; uint8_t *out; const uint64_t *out_off, *out_cap; uint64_t *out_len; int32_t *status;
    size_t n; int skip_crc; volatile size_t *next; const dvo_options *o; int mode, lz77, pred_mode, mixing_value;
} batch_job;
static void *batch_worker(void *arg) {
    batch_job *j = (batch_job *)arg;
    for (;;) {
        size_t i = __sync_fetch_and_add(j->next, 1);
        if (i >= j->n) break;
        size_t ol = 0; int rc;
        if (j->mode == 0) rc = dvo_decode(j->in + j->in_off[i], j->in_len[i], j->out + j->out_off[i], j->out_cap[i], &ol, j->skip_crc);
        else if (!j->lz77)
            rc = encode_raw_record(j->in + j->in_off[i], j->in_len[i], j->o, j->pred_mode, j->mixing_value, j->out + j->out_off[i], j->out_cap[i], &ol);
        else {
            dvo_cmdlist l; dvo_cmdlist_init(&l);
            dvo_lz77_cmds(j->in + j->in_off[i], j->in_len[i], j->o->window_size, j->pred_mode, j->mixing_value, &l);
            rc = dvo_encode_cmds(&l, j->o, j->out + j->out_off[i], j->out_cap[i], &ol);
            dvo_cmdlist_free(&l);
        }
        j->out_len[i] = ol; j->status[i] = rc;
    }
    for (int i = 0; i < 2; i++) { free(tl_pool[i]); tl_pool[i] = NULL; }
    return NULL;
}
static int run_batch(batch_job *j, int n_threads) {
    if (n_threads < 1) n_threads = 1;
    if (n_threads > 256) n_threads = 256;
    volatile size_t next = 0; j->next = &next;
    if (!crc_table_ready) crc_init_table();
    pthread_t th[256];
    for (int t = 0; t < n_threads; t++) pthread_create(&th[t], NULL, batch_worker, j);
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
    j->next = NULL;   /* (the counter lives in this frame: no pointer to it survives the call) */
    int bad = 0; for (size_t i = 0; i < j->n; i++) if (j->status[i] != DVO_SUCCESS) bad++;
    return bad;
}
int dvo_decode_batch(const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                     const uint64_t *out_cap, uint64_t *out_len, int32_t *status, size_t n, int n_threads, int skip_crc) {
    batch_job j = {in, in_off, in_len, out, out_off, out_cap, out_len, status, n, skip_crc, NULL, NULL, 0, 0, 0, 0};
    return run_batch(&j, n_threads);
}
int dvo_encode_raw_batch(const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                         const uint64_t *out_cap, uint64_t *out_len, int32_t *status, size_t n, int n_threads, const dvo_options *o,
                         int lz77, int pred_mode, int mixing_value) {
    batch_job j = {in, in_off, in_len, out, out_off, out_cap, out_len, status, n, 0, NULL, o, 1, lz77, pred_mode, mixing_value};
    return run_batch(&j, n_threads);
}
