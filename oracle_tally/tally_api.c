/*
 * tally_api.c -- literal model selection, and the replay of serialised command lists, on top of the CPU oracle.
 * TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * oracle_tally/tally_py.py compiles this file appended to a copy of oracle/divans_oracle.c whose ans_enc_put has one hook
 * inserted (dvt_tally, below): while dvt_tally is set, every symbol the encoder would code adds the cost of its frequency to
 * *dvt_tally instead of being recorded.  So the walk is the oracle's encoder walk itself -- the same commands, priors and
 * end-of-stream nibble -- and only what happens to each (start, freq) differs.  This is the cost rule of the reference's
 * TallyingArithmeticEncoder (ir_optimize/statistics_tracking_codec.rs:20-42) in fixed point.
 *
 * The functions here see the oracle's static helpers (cl_add, internal_predmode, ...) because they share its translation unit.
 */

/* cost of a symbol of frequency f (1..32767 of 32768) in 1/65536 bit: 65536 * (15 - log2 f), the 16 fraction bits of log2 f by
 * repeated squaring of the mantissa.  Integer-only: the GPU library's table (divans_b200/csrc/dv_capi.cu, freq_cost) is the
 * same rule, so GPU and oracle costs are equal, not merely close.  f = 0 costs as f = 1. */
static uint32_t dvt_freq_cost(uint32_t f) {
    if (f == 0) f = 1;
    uint32_t e = 0;
    while ((f >> (e + 1)) != 0) e++;
    uint64_t x = (uint64_t)f << (31 - e);
    uint32_t frac = 0;
    for (int i = 0; i < 16; i++) {
        x = (x * x) >> 31;
        frac <<= 1;
        if (x >= ((uint64_t)1 << 32)) { x >>= 1; frac |= 1; }
    }
    return (15u << 16) - ((e << 16) | frac);
}

void dvo_cost_table(uint32_t *tab) { for (uint32_t f = 0; f < 32768; f++) tab[f] = dvt_freq_cost(f); }

/* the walk of dvo_encode_cmds without output: *cost = the sum of the costs of every coded nibble of both coders, the
 * end-of-stream nibble included; a list the encoder refuses returns its failure with *cost = UINT64_MAX */
int dvo_tally_cmds(const dvo_cmdlist *l, const dvo_options *o, uint64_t *cost) {
    uint8_t frame[4096];   /* the framing of two empty payloads: header, EOF marker, trailer */
    size_t n = 0;
    uint64_t t = 0;
    dvt_tally = &t;
    int rc = dvo_encode_cmds(l, o, frame, sizeof frame, &n);
    dvt_tally = NULL;
    *cost = rc == DVO_SUCCESS ? t : UINT64_MAX;
    return rc;
}

/* dvo_encode_raw's command list with the PredictionMode record of (pred_mode, mixing_value): one PredictionMode command, then
 * Literal commands of at most 2^window bytes (the GPU raw-mode encoder's list for the same options) */
static void dvt_raw_cmds(const uint8_t *in, size_t n, int window_size, int pred_mode, int mixing_value, dvo_cmdlist *l) {
    int window = window_size < 10 ? 10 : (window_size > 24 ? 24 : window_size);
    dvo_cmd *c = cl_add(l); c->type = DVO_CMD_PREDMODE; c->a = 0;
    internal_predmode(cl_add_pm(l), pred_mode, mixing_value);
    size_t ring = (size_t)1 << window;
    for (size_t pos = 0; pos < n;) {
        size_t chunk = n - pos < ring ? n - pos : ring;
        size_t off = cl_add_lit(l, in + pos, chunk);
        c = cl_add(l); c->type = DVO_CMD_LITERAL; c->a = (uint32_t)off; c->b = (uint32_t)chunk; c->c = 0;
        pos += chunk;
    }
}

int dvo_encode_raw_model(const uint8_t *in, size_t n, const dvo_options *o, int pred_mode, int mixing_value, uint8_t *out, size_t cap,
                         size_t *out_len) {
    dvo_cmdlist l; dvo_cmdlist_init(&l);
    dvt_raw_cmds(in, n, o->window_size, pred_mode, mixing_value, &l);
    int rc = dvo_encode_cmds(&l, o, out, cap, out_len);
    dvo_cmdlist_free(&l);
    return rc;
}

int dvo_tally_raw(const uint8_t *in, size_t n, const dvo_options *o, int pred_mode, int mixing_value, uint64_t *cost) {
    dvo_cmdlist l; dvo_cmdlist_init(&l);
    dvt_raw_cmds(in, n, o->window_size, pred_mode, mixing_value, &l);
    int rc = dvo_tally_cmds(&l, o, cost);
    dvo_cmdlist_free(&l);
    return rc;
}

/* cands = n_cands (pred_mode, mixing_value) pairs: *chosen = the argmin of their costs (ties to the lowest index; costs[c]
 * optional), and the stream encoded with it */
int dvo_encode_auto(const uint8_t *in, size_t n, const dvo_options *o, const int32_t *cands, uint32_t n_cands, uint8_t *out, size_t cap,
                    size_t *out_len, uint32_t *chosen, uint64_t *costs) {
    uint64_t best = UINT64_MAX; uint32_t arg = 0;
    for (uint32_t c = 0; c < n_cands; c++) {
        uint64_t t;
        dvo_tally_raw(in, n, o, cands[2 * c], cands[2 * c + 1], &t);
        if (costs) costs[c] = t;
        if (t < best) { best = t; arg = c; }
    }
    *chosen = arg;
    return dvo_encode_raw_model(in, n, o, cands[2 * arg], cands[2 * arg + 1], out, cap, out_len);
}

/* ---- command lists ----
 * A candidate (pred_mode, mixing_value) replaces every PredictionMode record of a list by the raw-mode record of that model
 * (internal_predmode); commands, literal pool and window are kept.  (-1, -1) is KEEP: the list's own records. */
static int dvt_is_keep(int pred_mode, int mixing_value) { return pred_mode == -1 && mixing_value == -1; }

int dvo_cmdlist_set_model(dvo_cmdlist *l, int pred_mode, int mixing_value) {
    if (dvt_is_keep(pred_mode, mixing_value)) return DVO_SUCCESS;
    if (pred_mode < 0 || pred_mode > 3 || mixing_value < 0 || mixing_value > 15) return DVO_FAILURE;
    for (size_t k = 0; k < l->n_pms; k++) internal_predmode(&l->pms[k], pred_mode, mixing_value);
    return DVO_SUCCESS;
}

/* record k's 8192 mixing values := mixing.  Values above 15 are refused (a mixing value is one nibble of the command coder);
 * the IR grammar stops at 8, so this is how a test writes values 9..15, or a mask of its own making, into a list */
int dvo_cmdlist_set_mixing(dvo_cmdlist *l, size_t k, const uint8_t *mixing) {
    if (k >= l->n_pms) return DVO_FAILURE;
    for (size_t e = 0; e < 8192; e++) if (mixing[e] > 15) return DVO_FAILURE;
    memcpy(l->pms[k].mixing, mixing, 8192);
    return DVO_SUCCESS;
}

/* calls fn on the list as coded under candidate (pred_mode, mixing_value): a shallow copy whose records are replaced */
static int dvt_with_model(const dvo_cmdlist *l, int pred_mode, int mixing_value, int (*fn)(const dvo_cmdlist *, void *), void *arg) {
    if (dvt_is_keep(pred_mode, mixing_value) || l->n_pms == 0) return fn(l, arg);
    dvo_cmdlist m = *l;
    m.pms = (dvo_predmode *)malloc(l->n_pms * sizeof(dvo_predmode));
    if (!m.pms) return DVO_FAILURE;
    m.cap_pms = l->n_pms;
    int rc = dvo_cmdlist_set_model(&m, pred_mode, mixing_value);
    if (rc == DVO_SUCCESS) rc = fn(&m, arg);
    free(m.pms);
    return rc;
}

typedef struct { const dvo_options *o; uint64_t *cost; uint8_t *out; size_t cap; size_t *out_len; } dvt_call;
static int dvt_tally_fn(const dvo_cmdlist *l, void *p) { dvt_call *c = (dvt_call *)p; return dvo_tally_cmds(l, c->o, c->cost); }
static int dvt_encode_fn(const dvo_cmdlist *l, void *p) { dvt_call *c = (dvt_call *)p; return dvo_encode_cmds(l, c->o, c->out, c->cap, c->out_len); }

/* dvo_encode_auto for a command list: *chosen = the argmin of the candidates' costs (ties to the lowest index; a candidate the
 * encoder refuses costs UINT64_MAX; costs[c] optional), and the list encoded under it */
int dvo_encode_cmds_auto(const dvo_cmdlist *l, const dvo_options *o, const int32_t *cands, uint32_t n_cands, uint8_t *out, size_t cap,
                         size_t *out_len, uint32_t *chosen, uint64_t *costs) {
    uint64_t best = UINT64_MAX; uint32_t arg = 0;
    for (uint32_t c = 0; c < n_cands; c++) {
        uint64_t t = UINT64_MAX;
        dvt_call call = {o, &t, NULL, 0, NULL};
        if (dvt_with_model(l, cands[2 * c], cands[2 * c + 1], dvt_tally_fn, &call) != DVO_SUCCESS) t = UINT64_MAX;
        if (costs) costs[c] = t;
        if (t < best) { best = t; arg = c; }
    }
    *chosen = arg;
    *out_len = 0;
    dvt_call call = {o, NULL, out, cap, out_len};
    return dvt_with_model(l, cands[2 * arg], cands[2 * arg + 1], dvt_encode_fn, &call);
}

/* ---- replaying a DVCL blob (include/divans_b200.h) ----
 * The CPU reference of divans_b200_replay_cmds_batch_*: dvo_recode's semantics (the oracle's ring, rc_copy, rc_dict and
 * dvo_dict_word) on the serialised form, with the blob's refusal rules applied where the library applies them -- the blob and
 * header first, then each record as the walk reaches it.  window 0: the header's window; either way clamped to 10..24.
 * Returns DVO_SUCCESS, DVO_NEEDS_MORE_OUTPUT (*out_len is still the exact length, out holds its first `cap` bytes) or
 * DVO_FAILURE (*out_len: the bytes of the commands before the refused one, 0 for a refused blob or header).  Past `cap` the
 * walk only counts bytes: nothing is written any more, so the ring's contents no longer matter. */
#define DVT_PM_RECORD_BYTES (32u + 16384u + 1024u + 8192u)
int dvo_recode_blob(const uint8_t *blob, size_t len, int window, uint8_t *out, size_t cap, size_t *out_len) {
    uint32_t h[8];
    *out_len = 0;
    if (len < 32) return DVO_FAILURE;
    memcpy(h, blob, 32);
    const uint64_t lit_base = 32ull + 20ull * h[2] + (uint64_t)DVT_PM_RECORD_BYTES * h[3];
    if (h[0] != 0x4c435644u || h[1] != 1u || lit_base + h[4] > len) return DVO_FAILURE;
    const uint32_t w = window != 0 ? (uint32_t)(window < 10 ? 10 : (window > 24 ? 24 : window)) : (h[5] < 10 ? 10 : (h[5] > 24 ? 24 : h[5]));
    recoder r; memset(&r, 0, sizeof r);
    r.ring_len = 1u << w; r.ring = (uint8_t *)calloc(1, r.ring_len); r.out = out; r.out_cap = cap;
    if (!r.ring) return DVO_FAILURE;
    const uint8_t *lits = blob + lit_base;
    int rc = DVO_SUCCESS;
    for (uint32_t i = 0; i < h[2] && rc == DVO_SUCCESS; i++) {
        uint32_t c[5];
        memcpy(c, blob + 32 + 20ull * i, 20);
        const size_t room = r.out_len < cap ? cap - r.out_len : 0;
        if (c[0] == DVO_CMD_LITERAL) {
            if ((uint64_t)c[1] + c[2] > h[4]) { rc = DVO_FAILURE; break; }
            const size_t take = c[2] < room ? c[2] : room;
            for (size_t k = 0; k < take; k++) rc_put(&r, lits[c[1] + k]);
            if (take < c[2]) { r.out_len += c[2] - take; r.overflow = 1; }
        } else if (c[0] == DVO_CMD_COPY) {
            const size_t take = c[2] < room ? c[2] : room;
            rc = rc_copy(&r, c[1], (uint32_t)take);   /* refuses a == 0 and a >= the ring before it writes anything */
            if (rc == DVO_SUCCESS && take < c[2]) { r.out_len += c[2] - take; r.overflow = 1; }
        } else if (c[0] == DVO_CMD_DICT) {
            rc = rc_dict(&r, c[2], c[1], c[3], c[4]);
        } else if (c[0] < DVO_CMD_COPY || c[0] > DVO_CMD_PREDMODE) {
            rc = DVO_FAILURE;
        }
    }
    *out_len = r.out_len;
    if (r.overflow && rc == DVO_SUCCESS) rc = DVO_NEEDS_MORE_OUTPUT;
    free(r.ring);
    return rc;
}

/* ---- per-context mixing values ----
 * The CPU reference of divans_b200_encode_mixmap_* / encode_cmds_mixmap_*.  While dvt_bins is set, ans_enc_put adds each
 * symbol's cost to the total and to bin dvt_bin -- the mixing-mask index code_lit_nibble read for the literal nibble being
 * coded -- or, for every other nibble (dvt_bin = -1), to *dvt_nobin.  So the bins and the "no bin" counter sum to the total. */
#define DVT_MIX 8192

/* dvo_tally_cmds with bins[8192] and *nobin (zeroed first) */
static int dvt_tally_bins(const dvo_cmdlist *l, const dvo_options *o, uint64_t *cost, uint64_t *bins, uint64_t *nobin) {
    memset(bins, 0, DVT_MIX * sizeof *bins); *nobin = 0;
    dvt_bins = bins; dvt_nobin = nobin; dvt_bin = -1;
    int rc = dvo_tally_cmds(l, o, cost);
    dvt_bins = NULL; dvt_nobin = NULL; dvt_bin = -1;
    return rc;
}

/* calls fn on the list with every PredictionMode record replaced by `rec` (a shallow copy; a list without records as given) */
static int dvt_with_record(const dvo_cmdlist *l, const dvo_predmode *rec, int (*fn)(const dvo_cmdlist *, void *), void *arg) {
    if (l->n_pms == 0) return fn(l, arg);
    dvo_cmdlist m = *l;
    m.pms = (dvo_predmode *)malloc(l->n_pms * sizeof(dvo_predmode));
    if (!m.pms) return DVO_FAILURE;
    m.cap_pms = l->n_pms;
    for (size_t k = 0; k < l->n_pms; k++) m.pms[k] = *rec;
    int rc = fn(&m, arg);
    free(m.pms);
    return rc;
}

typedef struct { const dvo_options *o; uint64_t *cost, *bins, *nobin; } dvt_bins_call;
static int dvt_bins_fn(const dvo_cmdlist *l, void *p) { dvt_bins_call *c = (dvt_bins_call *)p; return dvt_tally_bins(l, c->o, c->cost, c->bins, c->nobin); }

int dvo_tally_raw_bins(const uint8_t *in, size_t n, const dvo_options *o, int pred_mode, int mixing_value, uint64_t *cost, uint64_t *bins,
                       uint64_t *nobin) {
    dvo_cmdlist l; dvo_cmdlist_init(&l);
    dvt_raw_cmds(in, n, o->window_size, pred_mode, mixing_value, &l);
    int rc = dvt_tally_bins(&l, o, cost, bins, nobin);
    dvo_cmdlist_free(&l);
    return rc;
}

int dvo_tally_cmds_bins(const dvo_cmdlist *l, const dvo_options *o, int pred_mode, int mixing_value, uint64_t *cost, uint64_t *bins,
                        uint64_t *nobin) {
    if (dvt_is_keep(pred_mode, mixing_value)) { *cost = UINT64_MAX; return dvt_tally_bins(l, o, cost, bins, nobin); }
    dvo_predmode *rec = (dvo_predmode *)malloc(sizeof *rec);
    if (!rec) return DVO_FAILURE;
    internal_predmode(rec, pred_mode, mixing_value);
    dvt_bins_call call = {o, cost, bins, nobin};
    *cost = UINT64_MAX;
    int rc = dvt_with_record(l, rec, dvt_bins_fn, &call);
    free(rec);
    return rc;
}

/* The choice of include/divans_b200.h ("per-context mixing values") for the list `l`, every record replaced: uniform passes under
 * R(pred_mode, values[c]) with bins, the per-entry argmin (ties to the lowest c; failed passes take no part), the mixed pass, and
 * the encode under R(pred_mode, values[c*]) or M.  Outputs: *chosen (k = mixed), mixing[8192], cost[k + 1], bins[k * 8192]
 * (UINT64_MAX for a failed pass); each but chosen may be NULL. */
static int dvt_mixmap(const dvo_cmdlist *l, const dvo_options *o, int pred_mode, const int32_t *values, uint32_t k, uint8_t *out, size_t cap,
                      size_t *out_len, uint32_t *chosen, uint8_t *mixing, uint64_t *cost, uint64_t *bins) {
    dvo_predmode *rec = (dvo_predmode *)malloc(sizeof *rec), *mixed = (dvo_predmode *)malloc(sizeof *mixed);
    uint64_t *b = (uint64_t *)malloc(DVT_MIX * sizeof(uint64_t)), *best = (uint64_t *)malloc(DVT_MIX * sizeof(uint64_t));
    uint8_t *arg_e = (uint8_t *)calloc(DVT_MIX, 1);
    int rc = DVO_FAILURE;
    *out_len = 0;
    if (!rec || !mixed || !b || !best || !arg_e) goto done;
    for (uint32_t e = 0; e < DVT_MIX; e++) best[e] = UINT64_MAX;
    uint64_t u_best = UINT64_MAX; uint32_t arg = 0;
    for (uint32_t c = 0; c < k; c++) {
        uint64_t t = UINT64_MAX, nb = 0;
        internal_predmode(rec, pred_mode, values[c]);
        dvt_bins_call call = {o, &t, b, &nb};
        if (dvt_with_record(l, rec, dvt_bins_fn, &call) != DVO_SUCCESS) t = UINT64_MAX;
        if (cost) cost[c] = t;
        if (t < u_best) { u_best = t; arg = c; }
        for (uint32_t e = 0; e < DVT_MIX; e++) {
            if (t != UINT64_MAX && b[e] < best[e]) { best[e] = b[e]; arg_e[e] = (uint8_t)c; }
            if (bins) bins[(size_t)c * DVT_MIX + e] = t != UINT64_MAX ? b[e] : UINT64_MAX;
        }
    }
    internal_predmode(mixed, pred_mode, values[0]);
    for (uint32_t e = 0; e < DVT_MIX; e++) mixed->mixing[e] = (uint8_t)values[arg_e[e]];
    uint64_t x = UINT64_MAX;
    dvt_call xc = {o, &x, NULL, 0, NULL};
    if (dvt_with_record(l, mixed, dvt_tally_fn, &xc) != DVO_SUCCESS) x = UINT64_MAX;
    if (cost) cost[k] = x;
    const int use_mixed = x < u_best;   /* a tie keeps the uniform record */
    *chosen = use_mixed ? k : arg;
    if (!use_mixed) internal_predmode(rec, pred_mode, values[arg]);
    const dvo_predmode *fin = use_mixed ? mixed : rec;
    if (mixing) memcpy(mixing, fin->mixing, DVT_MIX);
    dvt_call ec = {o, NULL, out, cap, out_len};
    rc = dvt_with_record(l, fin, dvt_encode_fn, &ec);
done:
    free(rec); free(mixed); free(b); free(best); free(arg_e);
    return rc;
}

int dvo_encode_mixmap(const uint8_t *in, size_t n, const dvo_options *o, int pred_mode, const int32_t *values, uint32_t k, uint8_t *out,
                      size_t cap, size_t *out_len, uint32_t *chosen, uint8_t *mixing, uint64_t *cost, uint64_t *bins) {
    dvo_cmdlist l; dvo_cmdlist_init(&l);
    dvt_raw_cmds(in, n, o->window_size, pred_mode, values[0], &l);
    int rc = dvt_mixmap(&l, o, pred_mode, values, k, out, cap, out_len, chosen, mixing, cost, bins);
    dvo_cmdlist_free(&l);
    return rc;
}

int dvo_encode_cmds_mixmap(const dvo_cmdlist *l, const dvo_options *o, int pred_mode, const int32_t *values, uint32_t k, uint8_t *out,
                           size_t cap, size_t *out_len, uint32_t *chosen, uint8_t *mixing, uint64_t *cost, uint64_t *bins) {
    return dvt_mixmap(l, o, pred_mode, values, k, out, cap, out_len, chosen, mixing, cost, bins);
}

/* ---- command lists from DVCL blobs, and forged command nibbles ----
 * dvo_cmdlist_from_blob: the list a DVCL blob (include/divans_b200.h) holds, every field as it is, so that a test can hand the
 * oracle's encoder records the IR grammar cannot write (a word size of 3, a transform of 300, a type of 15).  FAILURE for a
 * blob whose header, records or pool do not fit, or a literal outside the pool (the encoder reads the pool unchecked).
 *
 * dvo_encode_cmds_forged: dvo_encode_cmds with command nibble at[i] (0 = the first command nibble) replaced by val[i]; the
 * hook in code_and_blend makes the replacement, so the encoder follows the forged nibble exactly as a decoder does, and every
 * nibble the walk builds after a forged one is taken mod 16.  A walk that fails after a forged nibble ends the stream there:
 * both coders are flushed, and the mux and the trailer written, so the stream is CRC-valid and fails at that nibble.
 * *n_nibbles: the command nibbles coded, the end-of-stream nibble included. */
static __thread size_t dvt_forge_i, dvt_forge_cnt;
static __thread const uint32_t *dvt_forge_at;
static __thread const uint8_t *dvt_forge_val;

static uint8_t dvt_forge_nib(uint8_t nib) {
    size_t i = dvt_forge_i++;
    for (size_t k = 0; k < dvt_forge_cnt; k++)
        if (dvt_forge_at[k] == i) { dvt_forge_hit = 1; return dvt_forge_val[k]; }
    return dvt_forge_hit ? (uint8_t)(nib & 15) : nib;
}

int dvo_cmdlist_from_blob(const uint8_t *b, size_t len, dvo_cmdlist *l) {
    uint32_t h[8];
    if (len < 32) return DVO_FAILURE;
    memcpy(h, b, 32);
    const uint64_t lit_base = 32ull + 20ull * h[2] + (uint64_t)DVT_PM_RECORD_BYTES * h[3];
    if (h[0] != 0x4c435644u || h[1] != 1u || lit_base + h[4] > len) return DVO_FAILURE;
    for (uint32_t i = 0; i < h[2]; i++) {
        uint32_t r[5];
        memcpy(r, b + 32 + 20ull * i, 20);
        if (r[0] == DVO_CMD_LITERAL && (uint64_t)r[1] + r[2] > h[4]) return DVO_FAILURE;
        dvo_cmd *c = cl_add(l); c->type = r[0]; c->a = r[1]; c->b = r[2]; c->c = r[3]; c->d = r[4];
    }
    for (uint32_t k = 0; k < h[3]; k++) {
        const uint8_t *p = b + 32 + 20ull * h[2] + (uint64_t)DVT_PM_RECORD_BYTES * k;
        dvo_predmode *m = cl_add_pm(l);
        memset(m, 0, sizeof *m);
        m->pred_mode = p[0]; m->is_adv = p[1]; m->has_speeds = p[2];
        uint16_t sp[12]; memcpy(sp, p + 4, 24);
        for (int i = 0; i < 2; i++) for (int j = 0; j < 2; j++) {
            m->cm_speed[i][j] = sp[i * 2 + j]; m->stride_speed[i][j] = sp[4 + i * 2 + j]; m->combined_speed[i][j] = sp[8 + i * 2 + j];
        }
        uint16_t ll, dl; memcpy(&ll, p + 28, 2); memcpy(&dl, p + 30, 2);
        m->lit_map_len = ll; m->dist_map_len = dl;
        memcpy(m->lit_map, p + 32, 16384); memcpy(m->dist_map, p + 32 + 16384, 1024); memcpy(m->mixing, p + 32 + 16384 + 1024, 8192);
    }
    if (h[4]) cl_add_lit(l, b + lit_base, h[4]);
    l->window = (int)h[5];
    return DVO_SUCCESS;
}

int dvo_encode_cmds_forged(const dvo_cmdlist *l, const dvo_options *o, const uint32_t *at, const uint8_t *val, size_t n, uint8_t *out,
                           size_t cap, size_t *out_len, uint64_t *n_nibbles) {
    dvt_forge_i = 0; dvt_forge_cnt = n; dvt_forge_hit = 0; dvt_forge_at = at; dvt_forge_val = val;
    dvt_forging = 1;
    *out_len = 0;
    int rc = dvo_encode_cmds(l, o, out, cap, out_len);
    dvt_forging = 0;
    *n_nibbles = dvt_forge_i;
    return rc;
}

/* ---- coverage ----
 * dvo_encode_cmds_cov: dvo_encode_cmds into a scratch buffer with every command nibble counted in cov[flat * 16 + nibble], where
 * flat is the prior's index in the concatenation of the codec's command prior tables (CC, LL, CP, DC, BT, PM: the layout of
 * PRIOR_TABLES in tally_py.py, whose total dvo_cov_size returns). */
size_t dvo_cov_size(void) {
    return prior_total(T_CC, NEL(T_CC)) + prior_total(T_LL, NEL(T_LL)) + prior_total(T_CP, NEL(T_CP)) + prior_total(T_DC, NEL(T_DC)) +
           prior_total(T_BT, NEL(T_BT)) + prior_total(T_PM, NEL(T_PM));
}

static void dvt_cov_add(const void *cdf, uint8_t nib) {
    const codec *s = (const codec *)dvt_codec;
    const dvo_cdf16 *p = (const dvo_cdf16 *)cdf;
    const dvo_cdf16 *base[6] = {s->cc_priors, s->lit_len_priors, s->copy_priors, s->dict_priors, s->btype_priors, s->pred_priors};
    const size_t n[6] = {prior_total(T_CC, NEL(T_CC)), prior_total(T_LL, NEL(T_LL)), prior_total(T_CP, NEL(T_CP)),
                         prior_total(T_DC, NEL(T_DC)), prior_total(T_BT, NEL(T_BT)), prior_total(T_PM, NEL(T_PM))};
    size_t off = 0;
    for (int t = 0; t < 6; t++) {
        if (p >= base[t] && p < base[t] + n[t]) { dvt_cov[(off + (size_t)(p - base[t])) * 16 + (nib & 15)]++; return; }
        off += n[t];
    }
}

int dvo_encode_cmds_cov(const dvo_cmdlist *l, const dvo_options *o, uint32_t *cov) {
    size_t cap = l->n_lits * 2 + l->n_cmds * 16 + ((size_t)1 << 20), n = 0;
    uint8_t *out = (uint8_t *)malloc(cap);
    if (!out) return DVO_FAILURE;
    dvt_cov = cov;
    int rc = dvo_encode_cmds(l, o, out, cap, &n);
    dvt_cov = NULL;
    free(out);
    return rc;
}

/* ---- literal speeds ----
 * The CPU reference of divans_b200_encode_speeds_* / encode_cmds_speeds_* (include/divans_b200.h, "literal speeds") for the list
 * `l`, records kept: uniform passes, the halves passes (high = bins [0, 4096), low = bins [4096, 8192), the mixing-mask index of
 * a high nibble being below 4096), the verify pass, and the encode under the chosen speeds.  values: k (inc, lim) pairs.
 * Outputs: chosen[3]; cost[k + 1] and halves[k * 2] (lo, hi per d), each may be NULL. */
static void dvt_set_speeds(dvo_options *o, const int16_t *values, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    const uint32_t idx[4] = {a, b, c, d};
    o->have_literal_adaptation = 1;
    for (int j = 0; j < 4; j++) { o->literal_adaptation[j].inc = values[2 * idx[j]]; o->literal_adaptation[j].lim = values[2 * idx[j] + 1]; }
}

static int dvt_speeds(const dvo_cmdlist *l, const dvo_options *o, const int16_t *values, uint32_t k, uint8_t *out, size_t cap,
                      size_t *out_len, uint32_t *chosen, uint64_t *cost, uint64_t *halves) {
    uint64_t *b = (uint64_t *)malloc(DVT_MIX * sizeof(uint64_t)), *lo = (uint64_t *)malloc(k * sizeof(uint64_t)),
             *hi = (uint64_t *)malloc(k * sizeof(uint64_t));
    int rc = DVO_FAILURE;
    *out_len = 0;
    if (!b || !lo || !hi) goto done;
    dvo_options w = *o;
    uint64_t u_best = UINT64_MAX; uint32_t cs = 0;
    for (uint32_t c = 0; c < k; c++) {
        uint64_t t = UINT64_MAX;
        dvt_set_speeds(&w, values, c, c, c, c);
        if (dvo_tally_cmds(l, &w, &t) != DVO_SUCCESS) t = UINT64_MAX;
        if (cost) cost[c] = t;
        if (t < u_best) { u_best = t; cs = c; }
    }
    const int tuned = o->dynamic_context_mixing >= 2 && k > 1 && u_best != UINT64_MAX;
    uint32_t ls = cs, hs = cs;
    uint64_t x = u_best;
    if (tuned) {
        uint64_t blo = UINT64_MAX, bhi = UINT64_MAX;
        for (uint32_t d = 0; d < k; d++) {
            uint64_t t = UINT64_MAX, nb = 0;
            dvt_set_speeds(&w, values, cs, cs, d, d);
            lo[d] = hi[d] = UINT64_MAX;
            if (dvt_tally_bins(l, &w, &t, b, &nb) == DVO_SUCCESS) {
                lo[d] = 0; hi[d] = 0;
                for (uint32_t e = 0; e < DVT_MIX / 2; e++) { hi[d] += b[e]; lo[d] += b[DVT_MIX / 2 + e]; }
                if (lo[d] < blo) { blo = lo[d]; ls = d; }
                if (hi[d] < bhi) { bhi = hi[d]; hs = d; }
            }
        }
        dvt_set_speeds(&w, values, cs, cs, ls, hs);
        if (dvo_tally_cmds(l, &w, &x) != DVO_SUCCESS) x = UINT64_MAX;
    }
    for (uint32_t d = 0; d < k && halves; d++) {
        halves[2 * d] = tuned ? lo[d] : UINT64_MAX;
        halves[2 * d + 1] = tuned ? hi[d] : UINT64_MAX;
    }
    if (cost) cost[k] = x;
    const int take = tuned && x < u_best;
    chosen[0] = cs; chosen[1] = take ? ls : cs; chosen[2] = take ? hs : cs;
    dvt_set_speeds(&w, values, chosen[0], chosen[0], chosen[1], chosen[2]);
    rc = dvo_encode_cmds(l, &w, out, cap, out_len);
done:
    free(b); free(lo); free(hi);
    return rc;
}

int dvo_encode_speeds(const uint8_t *in, size_t n, const dvo_options *o, int pred_mode, int mixing_value, const int16_t *values, uint32_t k,
                      uint8_t *out, size_t cap, size_t *out_len, uint32_t *chosen, uint64_t *cost, uint64_t *halves) {
    dvo_cmdlist l; dvo_cmdlist_init(&l);
    dvt_raw_cmds(in, n, o->window_size, pred_mode, mixing_value, &l);
    int rc = dvt_speeds(&l, o, values, k, out, cap, out_len, chosen, cost, halves);
    dvo_cmdlist_free(&l);
    return rc;
}

int dvo_encode_cmds_speeds(const dvo_cmdlist *l, const dvo_options *o, const int16_t *values, uint32_t k, uint8_t *out, size_t cap,
                           size_t *out_len, uint32_t *chosen, uint64_t *cost, uint64_t *halves) {
    return dvt_speeds(l, o, values, k, out, cap, out_len, chosen, cost, halves);
}

/* ---- LZ77 parses, and choosing one of k command lists by cost ----
 * dvo_lz77_cmds_parse: dvo_lz77_cmds under the parse of include/divans_b200.h ("the LZ77 parse"): best(i) is dvo_lz77_cmds's
 * match at i (the chain holds every position below i, none above), and the walk takes it when it is at least min_match long and
 * no lookahead defers it.  {4, 0} is dvo_lz77_cmds.  Outside min_match 4..32, lazy 0..2: DVO_FAILURE and `l` untouched. */
typedef struct { const uint8_t *in; size_t n, maxdist, ins; int32_t *head, *prev; size_t pos[4], len[4], dist[4]; } dvt_lz;

static uint32_t dvt_h4(const uint8_t *p) {
    return (((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24)) * 2654435761u) >> 17;
}

static size_t dvt_lz_best(dvt_lz *z, size_t i, size_t *dist) {
    if (z->pos[i & 3] == i) { *dist = z->dist[i & 3]; return z->len[i & 3]; }
    size_t best = 0, bd = 0;
    if (i + 4 <= z->n) {
        for (; z->ins < i; z->ins++)
            if (z->ins + 4 <= z->n) { uint32_t h = dvt_h4(z->in + z->ins); z->prev[z->ins] = z->head[h]; z->head[h] = (int32_t)z->ins; }
        int32_t cand = z->head[dvt_h4(z->in + i)]; int chain = 16;
        while (cand >= 0 && chain-- > 0 && i - (size_t)cand <= z->maxdist) {
            size_t m = 0, lim = z->n - i; if (lim > 65535) lim = 65535;
            while (m < lim && z->in[cand + m] == z->in[i + m]) m++;
            if (m > best) { best = m; bd = i - (size_t)cand; }
            cand = z->prev[cand];
        }
    }
    z->pos[i & 3] = i; z->len[i & 3] = best; z->dist[i & 3] = bd;
    *dist = bd;
    return best;
}

/* dict(i) of include/divans_b200.h ("dictionary words in the LZ77 parse"), restated without an index: every word of size 4..24
 * and id below 2^size_bits_by_length[size] is compared with the input; where one matches, every transform with an empty prefix
 * and the identity type is built by dvo_dict_word and compared.  The best is kept under the rule's order: longest, then lowest
 * transform, shortest size, lowest id.  Returns the length (0: none). */
static size_t dvt_dict_at(const uint8_t *in, size_t n, size_t i, uint32_t *id, uint32_t *size, uint32_t *transform) {
    size_t best = 0;
    uint8_t w[64];
    for (uint32_t s = 4; s <= 24; s++) {
        if (i + s > n) break;
        for (uint32_t wid = 0; wid < (1u << TB_SIZE_BITS[s]); wid++) {
            if (memcmp(TB_DICT + TB_OFFSETS[s] + (size_t)wid * s, in + i, s) != 0) continue;
            for (uint32_t t = 0; t < 121; t++) {
                const uint8_t *tr = TB_TRANSFORMS + 3 * t;
                if (TB_PS[TB_PSMAP[tr[0]]] != 0 || tr[1] != 0) continue;
                const int len = dvo_dict_word(s, wid, t, w);
                if (len < 0 || i + (size_t)len > n || memcmp(w, in + i, (size_t)len) != 0) continue;
                const int better = (size_t)len > best
                    || ((size_t)len == best && (t < *transform || (t == *transform && (s < *size || (s == *size && wid < *id)))));
                if (better) { best = (size_t)len; *id = wid; *size = s; *transform = t; }
            }
        }
    }
    return best;
}

typedef size_t (*dvt_dict_fn)(const uint8_t *in, size_t n, size_t i, uint32_t *id, uint32_t *size, uint32_t *transform);
static size_t dvt_words_at(const uint8_t *in, size_t n, size_t i, uint32_t *id, uint32_t *size, uint32_t *transform);

/* dvo_lz77_cmds_parse with dictionary words (dict_min 0 or 4..32; 0 is dvo_lz77_cmds_parse), found by dict_at.  At a position
 * the walk reaches and does not defer, a word of dict_min or more bytes that is longer than the copy there (0 below min_match)
 * is emitted as a Dictionary command. */
static int dvt_lz77_cmds(const uint8_t *in, size_t n, int window, int pred_mode, int mixing_value, int min_match, int lazy, int dict_min,
                         dvt_dict_fn dict_at, dvo_cmdlist *l) {
    if (min_match < 4 || min_match > 32 || lazy < 0 || lazy > 2) return DVO_FAILURE;
    if (dict_min != 0 && (dict_min < 4 || dict_min > 32)) return DVO_FAILURE;
    dvt_lz z; memset(&z, 0, sizeof z);
    z.in = in; z.n = n; z.maxdist = ((size_t)1 << window) - 16;
    z.head = (int32_t *)malloc(((size_t)1 << 15) * sizeof(int32_t)); z.prev = (int32_t *)malloc((n + 1) * sizeof(int32_t));
    if (!z.head || !z.prev) { free(z.head); free(z.prev); return DVO_FAILURE; }
    for (size_t k = 0; k < ((size_t)1 << 15); k++) z.head[k] = -1;
    for (int k = 0; k < 4; k++) z.pos[k] = SIZE_MAX;
    dvo_cmd *c = cl_add(l); c->type = DVO_CMD_PREDMODE; c->a = (uint32_t)l->n_pms;
    internal_predmode(cl_add_pm(l), pred_mode, mixing_value);
    size_t i = 0, lit_start = 0, d, d1;
    while (i < n) {
        const size_t L = dvt_lz_best(&z, i, &d);
        int take = L >= (size_t)min_match, deferred = 0;
        if (take && lazy >= 1 && L < 32) {
            deferred = dvt_lz_best(&z, i + 1, &d1) > L || (lazy == 2 && dvt_lz_best(&z, i + 2, &d1) > L + 1);
            take = !deferred;
        }
        uint32_t wid = 0, ws = 0, wt = 0;
        const size_t Ld = dict_min && !deferred ? dict_at(in, n, i, &wid, &ws, &wt) : 0;
        const int word = Ld >= (size_t)dict_min && Ld > (take ? L : 0);
        if (!take && !word) { i++; continue; }
        if (i > lit_start) {
            size_t off = cl_add_lit(l, in + lit_start, i - lit_start);
            c = cl_add(l); c->type = DVO_CMD_LITERAL; c->a = (uint32_t)off; c->b = (uint32_t)(i - lit_start);
        }
        c = cl_add(l);
        if (word) { c->type = DVO_CMD_DICT; c->a = wid; c->b = ws; c->c = wt; c->d = (uint32_t)Ld; i += Ld; }
        else { c->type = DVO_CMD_COPY; c->a = (uint32_t)d; c->b = (uint32_t)L; i += L; }
        lit_start = i;
    }
    if (n > lit_start) {
        size_t off = cl_add_lit(l, in + lit_start, n - lit_start);
        c = cl_add(l); c->type = DVO_CMD_LITERAL; c->a = (uint32_t)off; c->b = (uint32_t)(n - lit_start);
    }
    free(z.head); free(z.prev);
    return DVO_SUCCESS;
}

int dvo_lz77_cmds_dict_parse(const uint8_t *in, size_t n, int window, int pred_mode, int mixing_value, int min_match, int lazy, int dict_min,
                             dvo_cmdlist *l) {
    return dvt_lz77_cmds(in, n, window, pred_mode, mixing_value, min_match, lazy, dict_min, dvt_dict_at, l);
}

int dvo_lz77_cmds_parse(const uint8_t *in, size_t n, int window, int pred_mode, int mixing_value, int min_match, int lazy, dvo_cmdlist *l) {
    return dvo_lz77_cmds_dict_parse(in, n, window, pred_mode, mixing_value, min_match, lazy, 0, l);
}

/* dict(i) of include/divans_b200.h ("dictionary words under every transform in the LZ77 parse"), restated without an index:
 * every word of size 4..24 under every transform 0..120 whose prefix matches at i is built by dvo_dict_word and compared, when
 * its core (the word after the transform's omission) has 4 or more bytes.  Before the build, a word is filtered on where its
 * core starts, i + |prefix|: the core's first four bytes are the word's (from the omitted start on) unless a case transform
 * applies, and a case transform leaves a first byte below 0xc0 as its ASCII uppercase and any other as it is.  Returns the
 * length (0: none). */
static size_t dvt_words_at(const uint8_t *in, size_t n, size_t i, uint32_t *id, uint32_t *size, uint32_t *transform) {
    size_t best = 0;
    uint8_t w[64];
    int pre_ok[121];
    size_t pre_len[121], cores[121];   /* where the cores may start: i + the length of a prefix that matches */
    uint32_t n_cores = 0;
    for (uint32_t t = 0; t < 121; t++) {
        const uint8_t *prefix = TB_PS + TB_PSMAP[TB_TRANSFORMS[3 * t]];
        pre_len[t] = prefix[0];
        pre_ok[t] = i + prefix[0] + 4 <= n && memcmp(prefix + 1, in + i, prefix[0]) == 0;
        uint32_t k = 0;
        while (pre_ok[t] && k < n_cores && cores[k] != i + prefix[0]) k++;
        if (pre_ok[t] && k == n_cores) cores[n_cores++] = i + prefix[0];
    }
    for (uint32_t s = 4; s <= 24; s++) {
        for (uint32_t wid = 0; wid < (1u << TB_SIZE_BITS[s]); wid++) {
            const uint8_t *word = TB_DICT + TB_OFFSETS[s] + (size_t)wid * s;
            int any = 0;   /* the filter below, for any transform: skip the word when no core of it can start anywhere */
            for (uint32_t k = 0; k < n_cores && !any; k++) {
                const uint8_t *c = in + cores[k];
                any = (word[0] < 0xc0 && word[0] >= 'a' && word[0] <= 'z' ? word[0] ^ 32 : word[0]) == c[0];
                for (uint32_t skip = 0; skip <= 9 && skip + 4 <= s && !any; skip++) any = memcmp(word + skip, c, 4) == 0;
            }
            if (!any) continue;
            for (uint32_t t = 0; t < 121; t++) {
                if (!pre_ok[t]) continue;
                const uint32_t type = TB_TRANSFORMS[3 * t + 1];
                const uint32_t skip = type >= 12 ? type - 11 : 0, core = s - skip - (type <= 9 ? type : 0);
                const uint8_t *c = in + i + pre_len[t];
                if (skip > s || (int)core < 4) continue;
                if (type == 10 || type == 11) {
                    if ((word[0] < 0xc0 && word[0] >= 'a' && word[0] <= 'z' ? word[0] ^ 32 : word[0]) != c[0]) continue;
                } else if (memcmp(word + skip, c, 4) != 0) continue;
                const int len = dvo_dict_word(s, wid, t, w);
                if (len < 0 || i + (size_t)len > n || memcmp(w, in + i, (size_t)len) != 0) continue;
                const int better = (size_t)len > best
                    || ((size_t)len == best && (t < *transform || (t == *transform && (s < *size || (s == *size && wid < *id)))));
                if (better) { best = (size_t)len; *id = wid; *size = s; *transform = t; }
            }
        }
    }
    return best;
}

/* dvo_lz77_cmds_dict_parse with the candidate set of `transforms`: 0 the 44-member set (dvo_lz77_cmds_dict_parse), 1 every
 * transform (dvt_words_at). */
int dvo_lz77_cmds_words_parse(const uint8_t *in, size_t n, int window, int pred_mode, int mixing_value, int min_match, int lazy, int dict_min,
                              int transforms, dvo_cmdlist *l) {
    if (transforms != 0 && transforms != 1) return DVO_FAILURE;
    return dvt_lz77_cmds(in, n, window, pred_mode, mixing_value, min_match, lazy, dict_min, transforms ? dvt_words_at : dvt_dict_at, l);
}

/* The CPU reference of divans_b200_encode_cmds_choose_batch_device for one stream: costs[c] = dvo_tally_cmds of lists[c], each
 * under its own records (UINT64_MAX where the encoder refuses it), *chosen = their argmin (ties to the lowest index; 0 when all
 * fail), and lists[*chosen] encoded into out. */
int dvo_encode_cmds_choose(const dvo_cmdlist *const *lists, uint32_t k, const dvo_options *o, uint8_t *out, size_t cap, size_t *out_len,
                           uint32_t *chosen, uint64_t *costs) {
    uint64_t best = UINT64_MAX; uint32_t arg = 0;
    for (uint32_t c = 0; c < k; c++) {
        uint64_t t = UINT64_MAX;
        if (dvo_tally_cmds(lists[c], o, &t) != DVO_SUCCESS) t = UINT64_MAX;
        if (costs) costs[c] = t;
        if (t < best) { best = t; arg = c; }
    }
    *chosen = arg;
    *out_len = 0;
    return dvo_encode_cmds(lists[arg], o, out, cap, out_len);
}

/* ---- billing by coder state (include/divans_b200.h, "billing each stream's coding cost by coder state") ----
 * While dvt_rows is set, ans_enc_put also adds each symbol's cost and a count of one to row dvt_row of the bill: tally_py.py makes
 * every nibble-coding call of the encoder name the row of its own substate just before it codes, and ans_enc_put clears it.  A
 * nibble coded where no call named a row goes to row DVT_BILL_ROWS, and a walk with any such nibble is refused.  rows
 * [DVT_BILL_ROWS * 2]: (cost, nibbles) per row, all zero when the walk fails; *cost as dvo_tally_cmds. */
int dvo_bill_cmds(const dvo_cmdlist *l, const dvo_options *o, uint64_t *cost, uint64_t *rows) {
    uint64_t r[2 * (DVT_BILL_ROWS + 1)];
    memset(r, 0, sizeof r);
    dvt_rows = r; dvt_row = -1;
    int rc = dvo_tally_cmds(l, o, cost);
    dvt_rows = NULL; dvt_row = -1;
    if (rc == DVO_SUCCESS && r[2 * DVT_BILL_ROWS + 1] != 0) { rc = DVO_FAILURE; *cost = UINT64_MAX; }
    if (rc != DVO_SUCCESS) memset(r, 0, sizeof r);
    memcpy(rows, r, 2 * DVT_BILL_ROWS * sizeof *rows);
    return rc;
}

int dvo_bill_raw(const uint8_t *in, size_t n, const dvo_options *o, int pred_mode, int mixing_value, uint64_t *cost, uint64_t *rows) {
    dvo_cmdlist l; dvo_cmdlist_init(&l);
    dvt_raw_cmds(in, n, o->window_size, pred_mode, mixing_value, &l);
    int rc = dvo_bill_cmds(&l, o, cost, rows);
    dvo_cmdlist_free(&l);
    return rc;
}
