/*
 * divans_oracle.h -- CPU restatement ("oracle") of the dropbox/divans entropy path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product
 * (divans_b200/, include/) never includes, links or calls anything in oracle/.
 *
 * Parity status: the reference is a Rust crate and no Rust toolchain exists in the build container, so this restatement cannot be
 * diffed against the real binary.  It IS pinned at whole-bitstream level by the one compressed stream the reference tree holds
 * (wasm/wasm.html:98-107, tests/golden/ref_wasm_example.divans): under model revision DVO_MODEL_WASM_2018 (below) the decoder
 * turns its 113 bytes into a CRC-valid English text and the encoder reproduces the 113 bytes byte for byte; the revision
 * differs from the mounted source in three named constructs of the PredictionMode / copy command coding, which are therefore
 * "parity unpinned" under DVO_MODEL_CURRENT (as are context-map value coding and dynamic context mixing >= 2, which the stream
 * does not use).  It is also pinned against every known-answer test the reference carries for this path (CRC32C, mux framing
 * vector, dictionary words, fast divide, f8 speed codec, IR->raw fixtures, ratio ceilings); see tests/test_oracle_kat.py.
 *
 * Every function cites the reference file:line it restates (paths relative to the
 * reference tree, dropbox/divans @ 23459c22).
 */
#ifndef DIVANS_ORACLE_H_
#define DIVANS_ORACLE_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- model revisions ----
 * DVO_MODEL_CURRENT   = the reference tree as mounted (dropbox/divans @ 23459c22).
 * DVO_MODEL_WASM_2018 = the build that produced the one compressed stream the reference tree holds
 *   (wasm/wasm.html:98-107, `_example_dv_file`, 113 bytes).  It differs from the current source in exactly two
 *   constructs of the PredictionMode command, both in codec/context_map.rs:
 *     (1) the context-map Mnemonic nibbles (:273) are coded with the prior that DynamicContextMixingSpeed, PriorDepth
 *         and ContextMapSpeedPalette[0] share, not with PredictionModePriorType::Mnemonic's own slots
 *         (codec/priors.rs:130);
 *     (2) every mixing value (:395-405) is coded with prior slot 16, also for index >= 256 (today: value[i-256] & 15).
 *   With these two the stream decodes to a CRC-valid plaintext; everything else (rANS, CDF arithmetic, command, literal,
 *   copy, dictionary coding, framing, CRC32C) is the same code in both revisions.  See tests/test_oracle_kat.py. */
#define DVO_MODEL_CURRENT 0
#define DVO_MODEL_WASM_2018 1

/* ---- result codes: reference src/ffi/interface.rs:8-12 ---- */
#define DVO_SUCCESS 0
#define DVO_NEEDS_MORE_INPUT 1
#define DVO_NEEDS_MORE_OUTPUT 2
#define DVO_FAILURE 3

/* ---- probability model: reference src/probability/frequentist_cdf.rs.  Compiled with -DDVO_FEATURE_BLEND (the second library
 * oracle/_build/libdivans_oracle_blend.so) the model is the reference's feature="blend" instead: BlendCDF16,
 * src/probability/blend_cdf.rs:109-208, selected for the whole crate by src/interface.rs:146-147.  A compile-time switch
 * there, a compile-time switch here: nothing in a stream says which model coded it.  Parity of the blend model: the
 * reference holds no stream coded with it; it is pinned by restating the four tests the reference runs on BlendCDF16
 * (probability/common_tests.rs:4-110 through blend_cdf.rs:213) -- tests/test_oracle_kat.py -- i.e. at property level only. ---- */
#ifdef DVO_FEATURE_BLEND
typedef struct { int16_t c[16]; int32_t mix_rate, count; } dvo_cdf16;
int16_t dvo_cdf_value(const dvo_cdf16 *c, uint8_t sym);    /* BaseCDF::cdf(), blend_cdf.rs:160-171 */
#else
typedef struct { int16_t c[16]; } dvo_cdf16;
#endif
typedef struct { int16_t inc, lim; } dvo_speed;
int dvo_feature_blend(void);                                /* 1 in the blend library */

void dvo_cdf_default(dvo_cdf16 *c);
void dvo_cdf_blend(dvo_cdf16 *c, uint8_t sym, dvo_speed s);
void dvo_cdf_average(const dvo_cdf16 *self, const dvo_cdf16 *other, int32_t mix_rate, dvo_cdf16 *out);
/* returns sym; writes start,freq (probability/interface.rs:136-198) */
uint8_t dvo_cdf_lookup(const dvo_cdf16 *c, int16_t cdf_offset, int16_t *start, int16_t *freq);
void dvo_cdf_sym_start_freq(const dvo_cdf16 *c, uint8_t sym, int16_t *start, int16_t *freq);
int32_t dvo_fast_divide(int32_t num, int16_t denom);        /* probability/numeric.rs:26-31 via LUT rule :14-17 */
uint8_t dvo_speed_to_u8(int16_t v);                         /* probability/interface.rs:566-575 */
int16_t dvo_u8_to_speed(uint8_t v);                         /* probability/interface.rs:577-585 */
uint32_t dvo_crc32c(uint32_t crc, const uint8_t *buf, size_t n); /* codec/crc32.rs:17-86 */

/* weights (codec/weights.rs) exposed for unit tests */
typedef struct { int32_t w[2]; uint8_t mixing_param; int16_t norm; } dvo_weights;
void dvo_weights_init(dvo_weights *w);
void dvo_weights_update(dvo_weights *w, int16_t p0, int16_t p1, int16_t weighted);
/* batch forms for the arithmetic tests: one update per case from (w0, w1) (mixing_param 1: not read by the update), and
 * symbol walks from the default CDF (trace: n_steps + 1 CDFs per walk, the state before each step, then the final one) */
void dvo_weights_update_batch(size_t n, const int32_t *w0, const int32_t *w1, const int16_t *p0, const int16_t *p1,
                              const int16_t *weighted, int32_t *out_w0, int32_t *out_w1, int16_t *out_norm);
/* one coded literal nibble per case at CDF level (plain, or mixing a context-map prior cdf2 with weights (w0, w1, norm)) */
void dvo_cdf_step_batch(size_t n, int mix, int enc, const int16_t *cdf, const int16_t *cdf2, const int32_t *wts,
                        const dvo_speed *speeds, const uint64_t *state, const uint8_t *sym_in, uint8_t *sym_out, int16_t *start_out,
                        int16_t *freq_out, uint64_t *state_out, int16_t *cdf_out, int16_t *cdf2_out, int32_t *wts_out);
void dvo_cdf_walk_batch(size_t n_walks, size_t n_steps, const dvo_speed *speeds, const uint8_t *syms, dvo_cdf16 *trace);

/* ---- commands (the IR): reference src/interface.rs (re-exported brotli::enc::interface types) ---- */
enum {
    DVO_CMD_COPY = 1, DVO_CMD_DICT = 2, DVO_CMD_LITERAL = 3, DVO_CMD_BTYPE_L = 4,
    DVO_CMD_BTYPE_C = 5, DVO_CMD_BTYPE_D = 6, DVO_CMD_PREDMODE = 7
}; /* numbering = the command-type nibble, codec/mod.rs:143-158 */

typedef struct {
    uint8_t pred_mode;            /* LSB6=0 MSB6=1 UTF8=2 SIGN=3 */
    uint8_t is_adv;               /* always 0 here */
    uint8_t has_speeds;           /* "has_context_speeds" on the encoder input */
    uint16_t cm_speed[2][2];      /* [low,high][inc,max] context-map prior speeds   (u16 values, f8 on the wire) */
    uint16_t stride_speed[2][2];
    uint16_t combined_speed[2][2];
    uint32_t lit_map_len;         /* literal context map entries to transmit */
    uint32_t dist_map_len;
    uint8_t lit_map[16384];
    uint8_t dist_map[1024];
    uint8_t mixing[8192];
} dvo_predmode;

typedef struct {
    uint32_t type;
    uint32_t a, b, c, d;
    /* copy: a=distance b=num_bytes
     * dict: a=word_id b=word_size c=transform d=final_size
     * literal: a=offset into literal pool, b=len, c=high_entropy
     * btype_*: a=block type, b=stride (literal only)
     * predmode: a=index into predmode pool */
} dvo_cmd;

typedef struct {
    dvo_cmd *cmds; size_t n_cmds, cap_cmds;
    uint8_t *lits; size_t n_lits, cap_lits;
    dvo_predmode *pms; size_t n_pms, cap_pms;
    int window;                  /* from "window N" line; 0 if absent */
} dvo_cmdlist;

void dvo_cmdlist_init(dvo_cmdlist *l);
void dvo_cmdlist_free(dvo_cmdlist *l);
/* IR text grammar: reference src/bin/divans.rs:191-483 */
int dvo_parse_ir(const char *text, size_t n, dvo_cmdlist *out);
/* serialise a cmdlist to a flat binary blob (the format the CUDA encoder consumes; see include/divans_b200.h) */
size_t dvo_cmdlist_serialize(const dvo_cmdlist *l, uint8_t *out, size_t cap);

/* ---- encoder options: reference src/interface.rs:444-484 ---- */
typedef struct {
    int window_size;             /* 10..24, default 22 */
    int dynamic_context_mixing;  /* default per caller; FFI default Some(1); CLI/internal unwrap_or(0) */
    int prior_depth;             /* unwrap_or(0) */
    int use_context_map;         /* bool */
    int force_stride;            /* 0..8, 9 = UseBrotliRec (default) */
    int have_literal_adaptation; /* Option<[Speed;4]> */
    dvo_speed literal_adaptation[4];
    int model_rev;               /* DVO_MODEL_CURRENT (0, what dvo_options_default sets) or DVO_MODEL_WASM_2018 */
} dvo_options;
void dvo_options_default(dvo_options *o);

/* ---- whole-stream entry points ---- */
/* decode a complete .divans buffer (header..trailer). returns DVO_SUCCESS / DVO_FAILURE /
 * DVO_NEEDS_MORE_INPUT (truncated) / DVO_NEEDS_MORE_OUTPUT (out_cap too small). */
int dvo_decode(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len, int skip_crc);
/* like dvo_decode but also reports how many input bytes form the stream (header..trailer) */
int dvo_decode_ex(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len,
                  int skip_crc, size_t *in_consumed, uint64_t *n_cmd_nibbles, uint64_t *n_lit_nibbles);
/* decode with an explicit model revision; when `cmds` is non-NULL the decoded commands are appended to it (an
 * initialised dvo_cmdlist), so that a stream can be re-encoded with dvo_encode_cmds */
int dvo_decode_cmds(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len, int skip_crc,
                    int model_rev, dvo_cmdlist *cmds);
/* encode a command list */
int dvo_encode_cmds(const dvo_cmdlist *l, const dvo_options *o, uint8_t *out, size_t cap, size_t *out_len);
/* the reference's internal literal-only compressor (raw_to_cmd/mod.rs:105-181): one PredictionMode
 * command then Literal commands of at most (1<<window) bytes */
int dvo_encode_raw(const uint8_t *in, size_t n, const dvo_options *o, uint8_t *out, size_t cap, size_t *out_len);
/* deterministic greedy hash-chain LZ77 front end (ours, SURVEY 8d "Z" encoding) producing a cmdlist */
int dvo_lz77_cmds(const uint8_t *in, size_t n, int window, int pred_mode, int mixing_value, dvo_cmdlist *out);
/* IR -> raw replay through the ring buffer only (reference `recode`, src/bin/divans.rs:1108, cmd_to_raw/mod.rs) */
int dvo_recode(const dvo_cmdlist *l, int window, uint8_t *out, size_t cap, size_t *out_len);

/* per-coder payload extraction (for encoder parity tests): demux a .divans buffer */
int dvo_demux(const uint8_t *in, size_t in_len, uint8_t *cmd, size_t *cmd_len, uint8_t *lit, size_t *lit_len,
              size_t *consumed);
/* mux known-answer helper: serialise one stream's bytes with the flush policy at close (mux.rs:445-561) */
size_t dvo_mux_single(int stream_id, const uint8_t *data, size_t n, uint8_t *out, size_t cap);

/* dictionary word + transform (cmd_to_raw/mod.rs:284-309); returns final length or -1 */
int dvo_dict_word(uint32_t word_size, uint32_t word_id, uint32_t transform, uint8_t *out37);

/* threaded batch decode for the CPU baseline: streams[i] = in + in_off[i], len in_len[i] */
int dvo_decode_batch(const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len,
                     uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                     int32_t *status, size_t n_streams, int n_threads, int skip_crc);
int dvo_encode_raw_batch(const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len,
                         uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                         int32_t *status, size_t n_streams, int n_threads, const dvo_options *o, int lz77,
                         int pred_mode, int mixing_value);
#ifdef __cplusplus
}
#endif
#endif
