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
