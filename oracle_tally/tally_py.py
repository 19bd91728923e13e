"""ctypes binding of the oracle's literal model selection (oracle_tally/tally_api.c).

TEST INFRASTRUCTURE: imported only by tests/ and tools/.  Nothing under divans_b200/ may import this module.

build() writes oracle_tally/_build/divans_oracle_tally.c: oracle/divans_oracle.c (read, never modified) with one hook in
ans_enc_put -- while a tally is running, each symbol adds the cost of its frequency to the tally instead of being recorded --
and a second one at the literal nibble's mixing-mask read -- the index becomes the bin of that nibble's cost --
and the billing hook -- each nibble-coding call of the encoder names its row of the bill (BILL_ROWS) just before it codes, and
ans_enc_put adds the symbol's cost to that row --
and three forging hooks -- every command nibble the encoder codes passes through dvt_forge_nib, a command-type nibble other than
the record's type ends the walk, and a walk that fails after a forged nibble is still flushed and framed --
followed by tally_api.c, and compiles it twice, with the reference's default probability model and with feature="blend", as
the oracle's own Makefile does.  Every function of the oracle is in these libraries unchanged while no forged encode runs; only
the tally entry points, dvo_cmdlist_set_mixing (a test's own mixing values in a list), dvo_recode_blob (the CPU reference of
the library's command-list replay, on the serialised blob), dvo_cmdlist_from_blob, dvo_encode_cmds_forged, dvo_lz77_cmds_parse
(the LZ77 generator under a parse), dvo_lz77_cmds_dict_parse (the same with dictionary words), dvo_lz77_cmds_words_parse (with
dictionary words under every transform), dvo_encode_cmds_choose (one of k command lists chosen by cost) and dvo_bill_cmds /
dvo_bill_raw (the cost billed by coder state) are new.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_ORACLE_C = os.path.join(_ROOT, "oracle", "divans_oracle.c")
_API_C = os.path.join(_HERE, "tally_api.c")
_TABLES = os.path.join(_ROOT, "divans_b200", "csrc", "brotli_tables.bin")
_BUILD = os.path.join(_HERE, "_build")
_SRC = os.path.join(_BUILD, "divans_oracle_tally.c")

SUCCESS, NEEDS_MORE_INPUT, NEEDS_MORE_OUTPUT, FAILURE = 0, 1, 2, 3
TALLY_FAILED = (1 << 64) - 1   # the cost of a stream the encoder refuses

# the hook: the first two lines of the oracle's ans_enc_put, and the same with the tally inserted after its frequency guard
_PUT = ("static inline void ans_enc_put(ans_enc *e, int16_t start, int16_t freq) {\n"
        "    if (freq <= 0) { e->bad = 1; freq = 1; start = 0; } /* only reachable after a stream-supplied speed wrapped an i16 counter */\n")
_PUT_TALLIED = _PUT + ("    if (dvt_tally) {   /* (oracle_tally) */\n"
                       "        const uint32_t dvt_c = dvt_freq_cost((uint32_t)freq);\n"
                       "        *dvt_tally += dvt_c;\n"
                       "        if (dvt_bins) { if (dvt_bin >= 0) dvt_bins[dvt_bin] += dvt_c; else *dvt_nobin += dvt_c; }\n"
                       "        if (dvt_rows) { const int32_t r = dvt_row >= 0 ? dvt_row : DVT_BILL_ROWS; dvt_rows[2 * r] += dvt_c; dvt_rows[2 * r + 1]++; }\n"
                       "        dvt_bin = -1; dvt_row = -1; e->n_syms++; return;\n"
                       "    }\n")
# the second hook: a literal nibble's mixing-mask index becomes the bin of the nibble coded next (ans_enc_put clears it)
_MM = "    uint8_t mm_opts = s->mixing_mask[mmi];\n"
_MM_TALLIED = _MM + "    dvt_bin = (int32_t)mmi;   /* (oracle_tally) */\n"
# the forging hooks (dvo_encode_cmds_forged): every command nibble passes through dvt_forge_nib; the command-type nibble the
# encoder codes must be the record's type, or the walk fails; and a walk that fails after a forged nibble is flushed and framed
_CAB = ("static inline uint8_t code_and_blend(coder *k, uint8_t nib, dvo_cdf16 *cdf, dvo_speed sp) {\n"
        "    nib = code_nibble(k, nib, cdf, NULL);\n")
_CAB_FORGED = ("static inline uint8_t code_and_blend(coder *k, uint8_t nib, dvo_cdf16 *cdf, dvo_speed sp) {\n"
               "    if (k->encoding && dvt_forging) nib = dvt_forge_nib(nib);   /* (oracle_tally) */\n"
               "    nib = code_nibble(k, nib, cdf, NULL);\n"
               "    if (k->encoding && dvt_cov) dvt_cov_add(cdf, nib);   /* (oracle_tally) coverage */\n")
# the coverage hook: the encoder's codec, so that a prior pointer maps back to its table and flat index
_INIT = "    codec_init(s, window, 1);\n"
_INIT_COV = _INIT + "    dvt_codec = s;   /* (oracle_tally) */\n"
_TYPE = ("        code_and_blend(&s->cmd, (uint8_t)c->type, P(s->cc_priors, T_CC, CC_FullSelection, (uint32_t)s->last_4_states >> 4, 0, 0), SPEED_ROCKET);\n"
         "        switch (c->type) {\n")
_TYPE_FORGED = ("        if (code_and_blend(&s->cmd, (uint8_t)c->type, P(s->cc_priors, T_CC, CC_FullSelection, (uint32_t)s->last_4_states >> 4, 0, 0), SPEED_ROCKET) != c->type) {\n"
                "            rc = DVO_FAILURE; break;   /* (oracle_tally) a forged command type: the walk ends */\n"
                "        }\n"
                "        switch (c->type) {\n")
_FLUSH = ("    if (rc == DVO_SUCCESS) {\n"
          "        /* flush: end-of-stream nibble 0xf, close both coders, drain mux, EOF marker, trailer (codec/mod.rs:424-560) */\n"
          "        code_and_blend(&s->cmd, 0xf, P(s->cc_priors, T_CC, CC_FullSelection, (uint32_t)s->last_4_states >> 4, 0, 0), SPEED_ROCKET);\n")
_FLUSH_FORGED = ("    const int dvt_cut = rc != DVO_SUCCESS && dvt_forging && dvt_forge_hit;   /* (oracle_tally) failed after a forged nibble */\n"
                 "    if (rc == DVO_SUCCESS || dvt_cut) {\n"
                 "        /* flush: end-of-stream nibble 0xf, close both coders, drain mux, EOF marker, trailer (codec/mod.rs:424-560) */\n"
                 "        if (!dvt_cut) code_and_blend(&s->cmd, 0xf, P(s->cc_priors, T_CC, CC_FullSelection, (uint32_t)s->last_4_states >> 4, 0, 0), SPEED_ROCKET);\n")
# a forged literal length never reads past the list's pool: the walk fails there instead (and the stream is cut)
_LIT = "            memcpy(scratch, l->lits + c->a, len);\n"
_LIT_FORGED = ("            if (dvt_forging && (uint64_t)c->a + len > l->n_lits) { rc = DVO_FAILURE; break; }   /* (oracle_tally) */\n"
               + _LIT)
_PREFIX = ("/* generated by oracle_tally/tally_py.py from oracle/divans_oracle.c and oracle_tally/tally_api.c: do not edit */\n"
           "#include <stdint.h>\n"
           "static __thread uint64_t *dvt_tally;   /* set: the encoder's symbols are costed, not coded */\n"
           "static __thread uint64_t *dvt_bins, *dvt_nobin;   /* set: each cost also goes to bin dvt_bin, or to *dvt_nobin */\n"
           "static __thread int32_t dvt_bin = -1;   /* the mixing-mask index of the literal nibble being coded, or -1 */\n"
           "static uint32_t dvt_freq_cost(uint32_t f);\n"
           "static __thread int dvt_forging;   /* set: dvo_encode_cmds_forged is running */\n"
           "static __thread int dvt_forge_hit;   /* a forged nibble has been coded */\n"
           "static uint8_t dvt_forge_nib(uint8_t nib);\n"
           "static __thread uint32_t *dvt_cov;   /* set: every coded command nibble counts in dvt_cov[flat prior * 16 + nibble] */\n"
           "static __thread void *dvt_codec;   /* the codec of the running encode */\n"
           "static void dvt_cov_add(const void *cdf, uint8_t nib);\n"
           "#define DVT_BILL_ROWS %d   /* the bill's rows; one more collects a nibble coded where no call named its row */\n"
           "static __thread uint64_t *dvt_rows;   /* set: each cost also goes to row dvt_row of the bill (cost, nibbles) */\n"
           "static __thread int32_t dvt_row = -1;   /* the row of the nibble being coded, named by its coding call, or -1 */\n"
           "#line 1 \"oracle/divans_oracle.c\"\n")


# The bill's rows (include/divans_b200.h, "billing each stream's coding cost by coder state"), and which of the oracle's nibble-coding
# calls codes each: its own prior types (the P() type of a code_and_blend call of the command coder) mapped onto the rows.  A call
# whose prior names no row, or two, stops the build.
BILL_ROWS = ["CMD_TYPE", "LIT_HI", "LIT_LO", "LL_COUNT_SMALL", "LL_SIZE_BEG", "LL_SIZE_LAST", "LL_MANT", "CP_COUNT_SMALL", "CP_COUNT_BEG",
             "CP_COUNT_LAST", "CP_COUNT_MANT", "CP_MNEMONIC", "CP_DIST_BEG", "CP_DIST_LAST", "CP_DIST_MANT", "DC_SIZE_BEG", "DC_SIZE_LAST",
             "DC_INDEX", "DC_TR_HI", "DC_TR_LO", "BT_MNEMONIC", "BT_FIRST", "BT_SECOND", "BT_STRIDE", "PM_MODE", "PM_MIX", "PM_DEPTH",
             "PM_SPEED", "PM_MAP_MNEMONIC", "PM_MAP_FIRST", "PM_MAP_SECOND", "PM_MIXVAL"]
_ROW_OF_PRIOR = {
    "CC_FullSelection,": "CMD_TYPE",
    "LL_CountSmall,": "LL_COUNT_SMALL", "LL_SizeBegNib,": "LL_SIZE_BEG", "LL_SizeLastNib,": "LL_SIZE_LAST", "LL_SizeMantissaNib,": "LL_MANT",
    "CP_CountSmall,": "CP_COUNT_SMALL", "CP_CountBegNib,": "CP_COUNT_BEG", "CP_CountLastNib,": "CP_COUNT_LAST",
    "CP_CountMantissaNib,": "CP_COUNT_MANT", "CP_DistanceMnemonic,": "CP_MNEMONIC", "CP_DistanceBegNib,": "CP_DIST_BEG",
    "CP_DistanceLastNib,": "CP_DIST_LAST", "CP_DistanceMantissaNib,": "CP_DIST_MANT",
    "DC_SizeBegNib,": "DC_SIZE_BEG", "DC_SizeLastNib,": "DC_SIZE_LAST", "DC_Index,": "DC_INDEX",
    "DC_Transform, 0,": "DC_TR_HI", "DC_Transform, 1,": "DC_TR_LO",
    "BT_Mnemonic,": "BT_MNEMONIC", "BT_FirstNibble,": "BT_FIRST", "BT_SecondNibble,": "BT_SECOND", "BT_StrideNibble,": "BT_STRIDE",
    "PM_Only,": "PM_MODE", "PM_DynamicContextMixingSpeed,": "PM_MIX", "PM_PriorDepth,": "PM_DEPTH", "PM_ContextMapSpeedPalette,": "PM_SPEED",
    "mn_prior,": "PM_MAP_MNEMONIC", "PM_FirstNibble,": "PM_MAP_FIRST", "PM_SecondNibble,": "PM_MAP_SECOND",
    "PM_PriorMixingValue,": "PM_MIXVAL",
}
_CMD_CALL = "code_and_blend(&s->cmd, "
_LIT_CALL = "code_nibble(&s->lit, "   # the literal nibbles (code_lit_nibble): high or low by its is_high


def _bill_hooked(src):
    """``src`` with every nibble-coding call of the encoder naming its bill row first: code_and_blend((dvt_row = r, &s->cmd), ...)"""
    out = []
    for line in src.split("\n"):
        if _CMD_CALL in line:
            assert line.count(_CMD_CALL) == 1, line
            rows = {r for k, r in _ROW_OF_PRIOR.items() if k in line.split(_CMD_CALL, 1)[1]}
            if len(rows) != 1:
                raise RuntimeError("oracle_tally: no single bill row for the oracle's call: " + line.strip())
            line = line.replace(_CMD_CALL, "code_and_blend((dvt_row = %d, &s->cmd), " % BILL_ROWS.index(rows.pop()))
        elif _LIT_CALL in line:
            line = line.replace(_LIT_CALL, "code_nibble((dvt_row = is_high ? %d : %d, &s->lit), " % (BILL_ROWS.index("LIT_HI"), BILL_ROWS.index("LIT_LO")))
        out.append(line)
    return "\n".join(out)


def _lib_path(blend):
    return os.path.join(_BUILD, "libdivans_oracle_tally%s.so" % ("_blend" if blend else ""))


def build(force=False):
    srcs = [_ORACLE_C, _API_C, __file__]
    libs = [_lib_path(False), _lib_path(True)]
    if not force and all(os.path.exists(p) for p in libs) and \
            min(os.path.getmtime(p) for p in libs) >= max(os.path.getmtime(s) for s in srcs):
        return
    oracle = open(_ORACLE_C).read()
    if oracle.count(_PUT) != 1:
        raise RuntimeError("oracle_tally: ans_enc_put of oracle/divans_oracle.c is not the one the tally hook was written for")
    if oracle.count(_MM) != 1:
        raise RuntimeError("oracle_tally: the mixing-mask read of oracle/divans_oracle.c is not the one the bin hook was written for")
    for pat, what in ((_CAB, "code_and_blend"), (_TYPE, "the command-type nibble of dvo_encode_cmds"), (_FLUSH, "the flush of dvo_encode_cmds"),
                      (_LIT, "the literal copy of dvo_encode_cmds"), (_INIT, "the codec_init of dvo_encode_cmds")):
        if oracle.count(pat) != 1:
            raise RuntimeError("oracle_tally: %s of oracle/divans_oracle.c is not the one the forging hook was written for" % what)
    os.makedirs(_BUILD, exist_ok=True)
    hooked = oracle.replace(_PUT, _PUT_TALLIED).replace(_MM, _MM_TALLIED)
    hooked = hooked.replace(_CAB, _CAB_FORGED).replace(_TYPE, _TYPE_FORGED).replace(_FLUSH, _FLUSH_FORGED).replace(_LIT, _LIT_FORGED).replace(_INIT, _INIT_COV)
    if hooked.count(_LIT_CALL) != 2:
        raise RuntimeError("oracle_tally: the literal nibbles of oracle/divans_oracle.c are not the ones the billing hook was written for")
    hooked = _bill_hooked(hooked)
    with open(_SRC + ".tmp", "w") as f:
        f.write(_PREFIX % len(BILL_ROWS) + hooked + '\n#line 1 "oracle_tally/tally_api.c"\n' + open(_API_C).read())
    os.replace(_SRC + ".tmp", _SRC)
    cc = os.environ.get("CC", "gcc")
    flags = ["-O3", "-march=x86-64-v2", "-fwrapv", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-pthread", "-shared",
             "-I", os.path.join(_ROOT, "oracle"), '-DDVO_TABLES_PATH="%s"' % _TABLES]
    for blend, out in ((False, libs[0]), (True, libs[1])):
        subprocess.check_call([cc] + flags + (["-DDVO_FEATURE_BLEND=1"] if blend else []) + ["-o", out + ".tmp", _SRC])
        os.replace(out + ".tmp", out)


class Speed(ctypes.Structure):
    _fields_ = [("inc", ctypes.c_int16), ("lim", ctypes.c_int16)]


class Options(ctypes.Structure):   # dvo_options, oracle/divans_oracle.h
    _fields_ = [
        ("window_size", ctypes.c_int), ("dynamic_context_mixing", ctypes.c_int), ("prior_depth", ctypes.c_int),
        ("use_context_map", ctypes.c_int), ("force_stride", ctypes.c_int), ("have_literal_adaptation", ctypes.c_int),
        ("literal_adaptation", Speed * 4), ("model_rev", ctypes.c_int),
    ]


_libs = {}


def lib(blend=False):
    if blend not in _libs:
        build()
        L = ctypes.CDLL(_lib_path(blend))
        vp, szp, op = ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(Options)
        u64p = ctypes.POINTER(ctypes.c_uint64)
        L.dvo_options_default.argtypes = [op]
        L.dvo_cost_table.argtypes = [vp]
        L.dvo_encode_raw_model.argtypes = [vp, ctypes.c_size_t, op, ctypes.c_int, ctypes.c_int, vp, ctypes.c_size_t, szp]
        L.dvo_tally_raw.argtypes = [vp, ctypes.c_size_t, op, ctypes.c_int, ctypes.c_int, u64p]
        L.dvo_encode_auto.argtypes = [vp, ctypes.c_size_t, op, vp, ctypes.c_uint32, vp, ctypes.c_size_t, szp,
                                      ctypes.POINTER(ctypes.c_uint32), vp]
        L.dvo_cmdlist_set_model.argtypes = [vp, ctypes.c_int, ctypes.c_int]
        L.dvo_cmdlist_set_mixing.argtypes = [vp, ctypes.c_size_t, vp]
        L.dvo_encode_cmds_auto.argtypes = [vp, op, vp, ctypes.c_uint32, vp, ctypes.c_size_t, szp, ctypes.POINTER(ctypes.c_uint32), vp]
        L.dvo_tally_raw_bins.argtypes = [vp, ctypes.c_size_t, op, ctypes.c_int, ctypes.c_int, u64p, vp, u64p]
        L.dvo_tally_cmds_bins.argtypes = [vp, op, ctypes.c_int, ctypes.c_int, u64p, vp, u64p]
        L.dvo_encode_mixmap.argtypes = [vp, ctypes.c_size_t, op, ctypes.c_int, vp, ctypes.c_uint32, vp, ctypes.c_size_t, szp,
                                        ctypes.POINTER(ctypes.c_uint32), vp, vp, vp]
        L.dvo_encode_cmds_mixmap.argtypes = [vp, op, ctypes.c_int, vp, ctypes.c_uint32, vp, ctypes.c_size_t, szp,
                                             ctypes.POINTER(ctypes.c_uint32), vp, vp, vp]
        L.dvo_recode_blob.argtypes = [vp, ctypes.c_size_t, ctypes.c_int, vp, ctypes.c_size_t, szp]
        L.dvo_encode_speeds.argtypes = [vp, ctypes.c_size_t, op, ctypes.c_int, ctypes.c_int, vp, ctypes.c_uint32, vp, ctypes.c_size_t, szp,
                                        vp, vp, vp]
        L.dvo_encode_cmds_speeds.argtypes = [vp, op, vp, ctypes.c_uint32, vp, ctypes.c_size_t, szp, vp, vp, vp]
        L.dvo_cmdlist_from_blob.argtypes = [vp, ctypes.c_size_t, vp]
        L.dvo_cov_size.restype = ctypes.c_size_t
        L.dvo_encode_cmds_cov.argtypes = [vp, op, vp]
        L.dvo_encode_cmds_forged.argtypes = [vp, op, vp, vp, ctypes.c_size_t, vp, ctypes.c_size_t, szp, u64p]
        L.dvo_tally_cmds.argtypes = [vp, op, u64p]
        L.dvo_bill_cmds.argtypes = [vp, op, u64p, vp]
        L.dvo_bill_raw.argtypes = [vp, ctypes.c_size_t, op, ctypes.c_int, ctypes.c_int, u64p, vp]
        L.dvo_lz77_cmds_parse.argtypes = [vp, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
        L.dvo_lz77_cmds_dict_parse.argtypes = [vp, ctypes.c_size_t] + [ctypes.c_int] * 6 + [vp]
        L.dvo_lz77_cmds_words_parse.argtypes = [vp, ctypes.c_size_t] + [ctypes.c_int] * 7 + [vp]
        L.dvo_encode_cmds_choose.argtypes = [vp, ctypes.c_uint32, op, vp, ctypes.c_size_t, szp, ctypes.POINTER(ctypes.c_uint32), vp]
        assert L.dvo_feature_blend() == int(blend)
        _libs[blend] = L
    return _libs[blend]


def options(blend=False, literal_adaptation=None, **kw):
    """dvo_options: the oracle's defaults, then the keyword arguments (oracle_py.options takes the same names)"""
    o = Options()
    lib(blend).dvo_options_default(ctypes.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    if literal_adaptation is not None:
        o.have_literal_adaptation = 1
        for i, (a, b) in enumerate(literal_adaptation):
            o.literal_adaptation[i].inc, o.literal_adaptation[i].lim = a, b
    return o


def _u8(b):
    return np.frombuffer(bytes(b), np.uint8) if len(b) else np.zeros(1, np.uint8)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def cost_table():
    """the cost of a symbol of each frequency 0..32767, in 1/65536 bit (dvo_cost_table)"""
    t = np.empty(32768, np.uint32)
    lib().dvo_cost_table(_p(t))
    return t


def encode_raw_model(data, pred_mode, mixing_value, blend=False, **kw):
    """(rc, stream or None): the oracle's raw-mode encoding with the literal model (pred_mode, mixing_value)"""
    d = _u8(data)
    cap = len(data) + len(data) // 2 + 65536
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    rc = lib(blend).dvo_encode_raw_model(_p(d), len(data), ctypes.byref(options(blend, **kw)), pred_mode, mixing_value, _p(out), cap,
                                         ctypes.byref(n))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None


def tally_raw(data, pred_mode=0, mixing_value=4, blend=False, **kw):
    """(rc, cost): the cost-only walk of encode_raw_model, in 1/65536 bit (TALLY_FAILED where the encoder refuses the stream)"""
    d = _u8(data)
    c = ctypes.c_uint64(0)
    rc = lib(blend).dvo_tally_raw(_p(d), len(data), ctypes.byref(options(blend, **kw)), pred_mode, mixing_value, ctypes.byref(c))
    return rc, c.value


def encode_auto(data, cands, blend=False, **kw):
    """(rc, stream or None, chosen, costs): the candidate (pred_mode, mixing_value) of the lowest cost, ties to the lowest
    index, and the stream encoded with it"""
    d = _u8(data)
    cv = np.ascontiguousarray(np.array(cands, np.int32).reshape(-1, 2))
    costs = np.zeros(cv.shape[0], np.uint64)
    cap = len(data) + len(data) // 2 + 65536
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    ch = ctypes.c_uint32(0)
    rc = lib(blend).dvo_encode_auto(_p(d), len(data), ctypes.byref(options(blend, **kw)), _p(cv), cv.shape[0], _p(out), cap,
                                    ctypes.byref(n), ctypes.byref(ch), _p(costs))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None, ch.value, costs


KEEP = (-1, -1)   # the candidate that keeps a command list's own PredictionMode records


def cmdlist_set_model(cmds, pred_mode, mixing_value):
    """Replace every PredictionMode record of ``cmds`` (an oracle_py / oracle_blend Commands: from_ir, lz77, decode_cmds) in
    place by the raw-mode record of (pred_mode, mixing_value); KEEP leaves it as it is.  Returns the oracle's status."""
    return lib().dvo_cmdlist_set_model(ctypes.addressof(cmds.c), pred_mode, mixing_value)


def cmdlist_set_mixing(cmds, k, mixing):
    """Write the 8192 mixing values ``mixing`` (0..15) into PredictionMode record ``k`` of ``cmds`` in place.  Returns the
    oracle's status: FAILURE, and nothing written, for a value above 15 or a record the list does not have."""
    m = np.ascontiguousarray(mixing, np.uint8)
    assert m.size == MIX_ENTRIES
    return lib().dvo_cmdlist_set_mixing(ctypes.addressof(cmds.c), k, _p(m))


def encode_cmds_auto(cmds, cands, blend=False, **kw):
    """(rc, stream or None, chosen, costs): the candidate (pred_mode, mixing_value, or KEEP) under which the command list
    ``cmds`` costs least, ties to the lowest index, and the list encoded under it.  ``cmds`` is not modified."""
    cv = np.ascontiguousarray(np.array(cands, np.int32).reshape(-1, 2))
    costs = np.zeros(cv.shape[0], np.uint64)
    cap = int(cmds.c.n_lits) * 2 + int(cmds.c.n_cmds) * 16 + (1 << 20)
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    ch = ctypes.c_uint32(0)
    rc = lib(blend).dvo_encode_cmds_auto(ctypes.addressof(cmds.c), ctypes.byref(options(blend, **kw)), _p(cv), cv.shape[0], _p(out), cap,
                                         ctypes.byref(n), ctypes.byref(ch), _p(costs))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None, ch.value, costs


def recode_blob(blob, window=0, cap=None):
    """(rc, out_len, bytes): the DVCL blob ``blob`` replayed to raw bytes through the oracle's ring (dvo_recode_blob), with the
    refusal rules of the library's replay.  ``window`` 0 takes the header's window; ``cap`` (default: the exact length, found by
    a first call with cap 0) bounds the bytes written.  rc 2: out_len is the exact length and ``bytes`` its first ``cap`` bytes;
    rc 3: the list is refused, out_len counts the bytes before the refused command."""
    b = np.frombuffer(bytes(blob), np.uint8) if not isinstance(blob, np.ndarray) else np.ascontiguousarray(blob, np.uint8)
    src = b if b.size else np.zeros(1, np.uint8)
    n = ctypes.c_size_t(0)
    if cap is None:
        lib().dvo_recode_blob(_p(src), b.size, int(window), None, 0, ctypes.byref(n))
        cap = n.value
    out = np.zeros(max(1, cap), np.uint8)
    rc = lib().dvo_recode_blob(_p(src), b.size, int(window), _p(out), cap, ctypes.byref(n))
    return rc, n.value, out[: min(n.value, cap)].tobytes()


MIX_ENTRIES = 8192


def tally_raw_bins(data, pred_mode=0, mixing_value=4, blend=False, **kw):
    """(rc, cost, bins [8192] u64, nobin): tally_raw with each literal nibble's cost also summed into the bin of its mixing-mask
    index, and every other nibble's into ``nobin``; bins.sum() + nobin == cost"""
    d = _u8(data)
    c, nb = ctypes.c_uint64(0), ctypes.c_uint64(0)
    bins = np.zeros(MIX_ENTRIES, np.uint64)
    rc = lib(blend).dvo_tally_raw_bins(_p(d), len(data), ctypes.byref(options(blend, **kw)), pred_mode, mixing_value, ctypes.byref(c),
                                       _p(bins), ctypes.byref(nb))
    return rc, c.value, bins, nb.value


def tally_cmds_bins(cmds, pred_mode, mixing_value, blend=False, **kw):
    """tally_raw_bins for the command list ``cmds`` with every PredictionMode record replaced by that of (pred_mode,
    mixing_value), or KEEP: the list's own records; ``cmds`` is not modified"""
    c, nb = ctypes.c_uint64(0), ctypes.c_uint64(0)
    bins = np.zeros(MIX_ENTRIES, np.uint64)
    rc = lib(blend).dvo_tally_cmds_bins(ctypes.addressof(cmds.c), ctypes.byref(options(blend, **kw)), pred_mode, mixing_value,
                                        ctypes.byref(c), _p(bins), ctypes.byref(nb))
    return rc, c.value, bins, nb.value


def _mixmap_out(k):
    return (np.zeros(MIX_ENTRIES, np.uint8), np.zeros(k + 1, np.uint64), np.zeros(k * MIX_ENTRIES, np.uint64))


def encode_mixmap(data, pred_mode, values, blend=False, **kw):
    """(rc, stream or None, chosen, mixing [8192], cost [k + 1], bins [k, 8192]): the per-context mixing values of
    divans_b200_encode_mixmap_batch_host for one raw buffer"""
    d = _u8(data)
    v = np.ascontiguousarray(values, np.int32)
    mixing, cost, bins = _mixmap_out(v.size)
    cap = len(data) + len(data) // 2 + 65536
    out = np.empty(cap, np.uint8)
    n, ch = ctypes.c_size_t(0), ctypes.c_uint32(0)
    rc = lib(blend).dvo_encode_mixmap(_p(d), len(data), ctypes.byref(options(blend, **kw)), pred_mode, _p(v), v.size, _p(out), cap,
                                      ctypes.byref(n), ctypes.byref(ch), _p(mixing), _p(cost), _p(bins))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None, ch.value, mixing, cost, bins.reshape(v.size, MIX_ENTRIES)


def encode_cmds_mixmap(cmds, pred_mode, values, blend=False, **kw):
    """encode_mixmap for the command list ``cmds`` (every PredictionMode record replaced; ``cmds`` is not modified)"""
    v = np.ascontiguousarray(values, np.int32)
    mixing, cost, bins = _mixmap_out(v.size)
    cap = int(cmds.c.n_lits) * 2 + int(cmds.c.n_cmds) * 16 + (1 << 20)
    out = np.empty(cap, np.uint8)
    n, ch = ctypes.c_size_t(0), ctypes.c_uint32(0)
    rc = lib(blend).dvo_encode_cmds_mixmap(ctypes.addressof(cmds.c), ctypes.byref(options(blend, **kw)), pred_mode, _p(v), v.size, _p(out),
                                           cap, ctypes.byref(n), ctypes.byref(ch), _p(mixing), _p(cost), _p(bins))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None, ch.value, mixing, cost, bins.reshape(v.size, MIX_ENTRIES)


def from_blob(oracle, blob):
    """the oracle_py / oracle_blend Commands of DVCL blob ``blob``, every field as the blob holds it (dvo_cmdlist_from_blob), or
    None for a blob whose header, records or literals do not fit"""
    cl = oracle.Commands()
    b = _u8(blob)
    return cl if lib().dvo_cmdlist_from_blob(_p(b), len(blob), ctypes.addressof(cl.c)) == SUCCESS else None


def encode_forged(cmds, forge=(), blend=False, cap=None, **kw):
    """(rc, stream, n_nibbles): the oracle's encoding of ``cmds`` with each (k, v) of ``forge`` making command nibble k (0 = the
    first) the value v (dvo_encode_cmds_forged).  ``stream`` is the encoded stream, also for rc 3 when the walk failed after a
    forged nibble (the stream then ends there), else b"".  n_nibbles: the command nibbles coded, the end-of-stream one included."""
    at = np.ascontiguousarray([k for k, _ in forge] or [0], np.uint32)
    val = np.ascontiguousarray([v for _, v in forge] or [0], np.uint8)
    cap = cap or int(cmds.c.n_lits) * 2 + int(cmds.c.n_cmds) * 16 + (1 << 20)
    out = np.empty(cap, np.uint8)
    n, nn = ctypes.c_size_t(0), ctypes.c_uint64(0)
    rc = lib(blend).dvo_encode_cmds_forged(ctypes.addressof(cmds.c), ctypes.byref(options(blend, **kw)), _p(at), _p(val), len(forge),
                                           _p(out), cap, ctypes.byref(n), ctypes.byref(nn))
    return rc, out[: n.value].tobytes(), nn.value


# ---- coverage of the command coder's priors (dvo_encode_cmds_cov) ----
# the prior tables of oracle/divans_oracle.c (codec/priors.rs:12-133) in the order dvo_cov_size concatenates them: (table,
# [(type, dims)]); a flat index is the offset of its table plus the type's offset plus i0 + d0 * (i1 + d1 * i2)
PRIOR_TABLES = [
    ("CC", [("FullSelection", (16, 1)), ("EndIndicator", (1, 256))]),
    ("LL", [("CountSmall", (256, 16)), ("SizeBegNib", (256,)), ("SizeLastNib", (256,)), ("SizeMantissaNib", (256,))]),
    ("CP", [("DistanceBegNib", (256, 64)), ("DistanceMnemonic", (256, 2)), ("DistanceLastNib", (256, 1)), ("DistanceMantissaNib", (256, 5)),
            ("CountSmall", (256, 64)), ("CountBegNib", (256, 64)), ("CountLastNib", (256, 64)), ("CountMantissaNib", (256, 64))]),
    ("DC", [("SizeBegNib", (256,)), ("SizeLastNib", (256,)), ("Index", (256, 5)), ("Transform", (2, 25))]),
    ("BT", [("Mnemonic", (3,)), ("FirstNibble", (3,)), ("SecondNibble", (3,)), ("StrideNibble", (1,))]),
    ("PM", [("Only", (1,)), ("LiteralSpeed", (1,)), ("FirstNibble", (2,)), ("SecondNibble", (2,)), ("Mnemonic", (4,)),
            ("PriorMixingValue", (17,)), ("ContextMapSpeedPalette", (4,))]),
]


def prior_of(flat):
    """(table, type, (i0, i1)) of flat prior index ``flat`` (the P() indices of the oracle's code_and_blend call)"""
    for table, ents in PRIOR_TABLES:
        for typ, dims in ents:
            n = int(np.prod(dims))
            if flat < n:
                return table, typ, (flat % dims[0], flat // dims[0])
            flat -= n
    raise IndexError(flat)


def cov_size():
    n = int(lib().dvo_cov_size())
    assert n == sum(int(np.prod(d)) for _, e in PRIOR_TABLES for _, d in e), "PRIOR_TABLES differs from the oracle's"
    return n


def coverage(cmd_lists, **kw):
    """counts [n_priors, 16]: how often each command nibble was coded under each prior over the oracle's encodings of the
    command lists ``cmd_lists`` (oracle_py Commands) with options ``kw``; every encode must succeed"""
    cov = np.zeros((cov_size(), 16), np.uint32)
    for cl in cmd_lists:
        rc = lib().dvo_encode_cmds_cov(ctypes.addressof(cl.c), ctypes.byref(options(**kw)), _p(cov))
        assert rc == SUCCESS, rc
    return cov


def coverage_pairs(cov):
    """{(table, type): {(i0, i1): set of nibbles}} of the nonzero entries of ``cov``"""
    out = {}
    for flat, nib in zip(*np.nonzero(cov)):
        t, typ, idx = prior_of(int(flat))
        out.setdefault((t, typ), {}).setdefault(idx, set()).add(int(nib))
    return out


def _speed_to_u8(x):   # the stream's f8 speed code (probability/interface.rs), on an i16
    u = x & 0xffff
    length = u.bit_length()
    mant = 0
    if x != 0:
        rem = ((x - (1 << (length - 1))) + 0x8000) % 0x10000 - 0x8000
        r3 = (((rem << 3) & 0xffff) ^ 0x8000) - 0x8000
        mant = (r3 >> (length - 1)) & 0xff
    return ((length << 3) | mant) & 0xff


def _u8_to_speed(d):
    if d < 8:
        return 0
    lv = (d >> 3) - 1
    rem = ((((d & 7) << lv) & 0xffff) ^ 0x8000) - 0x8000
    return (((1 << lv) | (rem >> 3)) & 0xffff ^ 0x8000) - 0x8000


def speed_ok(inc, lim):
    """whether (inc, lim) is a speed the speeds calls accept: unchanged by the f8 round trip, and unable to wrap an i16 prior"""
    rt = all(_u8_to_speed(_speed_to_u8(x)) == x for x in (inc, lim))
    return rt and inc >= 0 and lim >= 0 and lim + inc + 16 <= 0x7fff and 4 * (inc + 16) <= 0x7fff


def _speeds_args(values):
    v = np.ascontiguousarray(values, np.int16).reshape(-1, 2)
    if not 1 <= v.shape[0] <= 16 or not all(speed_ok(int(a), int(b)) for a, b in v):
        raise ValueError("speeds: 1..16 speeds that survive the f8 round trip and cannot wrap an i16 prior are required")
    k = v.shape[0]
    return v, k, np.zeros(3, np.uint32), np.zeros(k + 1, np.uint64), np.zeros(2 * k, np.uint64)


def encode_speeds(data, pred_mode, mixing_value, values, blend=False, **kw):
    """(rc, stream or None, chosen [3], cost [k + 1], halves [k, 2]): the literal speeds of divans_b200_encode_speeds_batch_host for
    one raw buffer under the literal model (pred_mode, mixing_value); ``values`` are (inc, lim) pairs"""
    d = _u8(data)
    v, k, ch, cost, halves = _speeds_args(values)
    cap = len(data) + len(data) // 2 + 65536
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    rc = lib(blend).dvo_encode_speeds(_p(d), len(data), ctypes.byref(options(blend, **kw)), pred_mode, mixing_value, _p(v), k, _p(out), cap,
                                      ctypes.byref(n), _p(ch), _p(cost), _p(halves))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None, ch, cost, halves.reshape(k, 2)


def encode_cmds_speeds(cmds, values, blend=False, **kw):
    """encode_speeds for the command list ``cmds`` (its records kept, the speeds overriding theirs)"""
    v, k, ch, cost, halves = _speeds_args(values)
    cap = int(cmds.c.n_lits) * 2 + int(cmds.c.n_cmds) * 16 + (1 << 20)
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    rc = lib(blend).dvo_encode_cmds_speeds(ctypes.addressof(cmds.c), ctypes.byref(options(blend, **kw)), _p(v), k, _p(out), cap,
                                           ctypes.byref(n), _p(ch), _p(cost), _p(halves))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None, ch, cost, halves.reshape(k, 2)


# ---- LZ77 parses (include/divans_b200.h, "the LZ77 parse") and the choice among k command lists ----
def tally_cmds(cmds, blend=False, **kw):
    """(rc, cost): the cost-only walk of the oracle's encoder over the command list ``cmds`` under its own records (dvo_tally_cmds;
    TALLY_FAILED where the encoder refuses it)"""
    c = ctypes.c_uint64(0)
    rc = lib(blend).dvo_tally_cmds(ctypes.addressof(cmds.c), ctypes.byref(options(blend, **kw)), ctypes.byref(c))
    return rc, c.value


def lz77_parse(oracle, data, min_match=4, lazy=0, window=16, pred_mode=2, mixing_value=4):
    """the oracle_py Commands of dvo_lz77_cmds_parse for ``data`` under the parse (min_match, lazy), or None for a parse outside
    min_match 4..32, lazy 0..2 (the list is then untouched)"""
    cl = oracle.Commands()
    d = _u8(data)
    rc = lib().dvo_lz77_cmds_parse(_p(d), len(data), window, pred_mode, mixing_value, min_match, lazy, ctypes.addressof(cl.c))
    return cl if rc == SUCCESS else None


def lz77_dict_parse(oracle, data, min_match=4, lazy=0, dict_min=0, window=16, pred_mode=2, mixing_value=4):
    """the oracle_py Commands of dvo_lz77_cmds_dict_parse for ``data`` under the parse (min_match, lazy, dict_min), or None for a
    parse outside min_match 4..32, lazy 0..2, dict_min 0 or 4..32 (the list is then untouched)"""
    cl = oracle.Commands()
    d = _u8(data)
    rc = lib().dvo_lz77_cmds_dict_parse(_p(d), len(data), window, pred_mode, mixing_value, min_match, lazy, dict_min, ctypes.addressof(cl.c))
    return cl if rc == SUCCESS else None


def lz77_words_parse(oracle, data, min_match=4, lazy=0, dict_min=0, transforms=0, window=16, pred_mode=2, mixing_value=4):
    """the oracle_py Commands of dvo_lz77_cmds_words_parse for ``data`` under the parse (min_match, lazy, dict_min, transforms),
    or None for a parse outside min_match 4..32, lazy 0..2, dict_min 0 or 4..32, transforms 0 or 1 (the list is then untouched)"""
    cl = oracle.Commands()
    d = _u8(data)
    rc = lib().dvo_lz77_cmds_words_parse(_p(d), len(data), window, pred_mode, mixing_value, min_match, lazy, dict_min, transforms,
                                         ctypes.addressof(cl.c))
    return cl if rc == SUCCESS else None


def encode_cmds_choose(lists, blend=False, **kw):
    """(rc, stream or None, chosen, costs [k]): the command list of ``lists`` (oracle_py Commands) that costs least under its own
    records, ties to the lowest index, encoded (dvo_encode_cmds_choose)"""
    k = len(lists)
    ptrs = (ctypes.c_void_p * k)(*[ctypes.addressof(c.c) for c in lists])
    costs = np.zeros(k, np.uint64)
    cap = max(int(c.c.n_lits) * 2 + int(c.c.n_cmds) * 16 for c in lists) + (1 << 20)
    out = np.empty(cap, np.uint8)
    n, ch = ctypes.c_size_t(0), ctypes.c_uint32(0)
    rc = lib(blend).dvo_encode_cmds_choose(ptrs, k, ctypes.byref(options(blend, **kw)), _p(out), cap, ctypes.byref(n), ctypes.byref(ch),
                                           _p(costs))
    return rc, out[: n.value].tobytes() if rc == SUCCESS else None, ch.value, costs


# ---- billing by coder state (include/divans_b200.h) ----
def bill_cmds(cmds, blend=False, **kw):
    """(rc, cost, rows [len(BILL_ROWS), 2] u64): tally_cmds with each nibble's cost and a count of one added to the row of the
    encoder substate that coded it (dvo_bill_cmds); rows.sum(axis=0)[0] == cost, and all zeros where the encoder refuses the list"""
    c = ctypes.c_uint64(0)
    rows = np.zeros((len(BILL_ROWS), 2), np.uint64)
    rc = lib(blend).dvo_bill_cmds(ctypes.addressof(cmds.c), ctypes.byref(options(blend, **kw)), ctypes.byref(c), _p(rows))
    return rc, c.value, rows


def bill_raw(data, pred_mode=0, mixing_value=4, blend=False, **kw):
    """bill_cmds for the raw buffer ``data`` coded as tally_raw codes it (dvo_bill_raw)"""
    d = _u8(data)
    c = ctypes.c_uint64(0)
    rows = np.zeros((len(BILL_ROWS), 2), np.uint64)
    rc = lib(blend).dvo_bill_raw(_p(d), len(data), ctypes.byref(options(blend, **kw)), pred_mode, mixing_value, ctypes.byref(c), _p(rows))
    return rc, c.value, rows
