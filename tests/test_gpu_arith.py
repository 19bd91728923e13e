"""The arithmetic under the CDF model and the rANS coders, tested as functions over whole input domains (-m gpu).

Whole-stream tests only reach the values their streams happen to produce.  These call the product's own device functions
through the test-only probe library (tests/probe/dv_probe.cu, built next to libdivans_b200.so) and compare them with exact
references: the reference's CDF division restated in 64-bit integers (tests/probe/numeric_ref.h, itself checked against the
oracle by tests/test_arith_domains.py), exact integer division, and the oracle's weight update.  Each test prints how many
cases it ran.  One test sends a stream that codes a CDF element above its max through the encoder and all three decode
layouts (tests/regimes.py c_over_max).  The step tests at the end run one coding step of each nibble core and of the fast
loops' pieces per case, at CDF level, against the oracle's dvo_cdf_step_batch."""
import ctypes
import os

import numpy as np
import pytest

import regimes as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_LIB = os.path.join(ROOT, "divans_b200", "lib", "libdivans_b200_probe.so")
MODE_CDF_DIV, MODE_CDF_DIV_POS, MODE_DIVQ = 0, 1, 2


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE_LIB), "%s is missing: build() makes it (make -C divans_b200/csrc)" % PROBE_LIB
    L = ctypes.CDLL(PROBE_LIB)
    vp = ctypes.c_void_p
    L.dvp_div_sweep.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp]
    L.dvp_rcp15_table.argtypes = [vp]
    L.dvp_div_u15.argtypes = [vp, vp, ctypes.c_size_t, vp, vp]
    L.dvp_weights.argtypes = [ctypes.c_int, ctypes.c_size_t, vp, vp]
    L.dvp_speed_gate.argtypes = [vp]
    L.dvp_step.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint32] + [vp] * 14
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def sweep(probe, mode, d_lo, d_hi):
    counts = np.zeros(3, np.uint64)
    ex = np.zeros((64, 4), np.int32)
    n_ex, ms = ctypes.c_int(0), ctypes.c_float(0)
    assert probe.dvp_div_sweep(mode, d_lo, d_hi, _p(counts), _p(ex), ctypes.byref(n_ex), ctypes.byref(ms)) == 0
    return dict(mismatches=int(counts[0]), cases=int(counts[1]), c_over_max=int(counts[2]),
                examples=[tuple(int(v) for v in r) for r in ex[:min(n_ex.value, 64)]], seconds=ms.value / 1e3)


def _report(what, r):
    print("%s: %d cases (%d with c > max) in %.3f s, %d mismatches %s" % (
        what, r["cases"], r["c_over_max"], r["seconds"], r["mismatches"], r["examples"][:8]))


def test_cdf_div_equals_the_reference_division_on_the_whole_i16_domain(probe):
    """cdf_div(c, max) for every c and max in i16 (2^32 pairs), including c > max: the i16 counters of a prior wrap under
    stream-supplied speeds, and a CDF element can then exceed the max by far (quotients up to 2^30)"""
    r = sweep(probe, MODE_CDF_DIV, -32768, 32768)
    _report("cdf_div vs numeric.rs", r)
    assert r["cases"] == 1 << 32
    assert r["c_over_max"] == sum(32767 - d for d in range(1, 32768))
    assert r["mismatches"] == 0, "(c, max, got, want): %s" % r["examples"]


def test_cdf_div_pos_is_exact_for_every_c_up_to_max(probe):
    """the division of the encoder's literal fast loop: 0 <= c <= max < 2^15"""
    r = sweep(probe, MODE_CDF_DIV_POS, 1, 32768)
    _report("cdf_div_pos", r)
    assert r["cases"] == sum(d + 1 for d in range(1, 32768))
    assert r["mismatches"] == 0, "(c, max, got, want): %s" % r["examples"]


def test_divq_with_recip32_is_exact_for_every_c_up_to_max(probe):
    """the v2 fast loops' and mixing loop's division: divq(c, recip32(d), d) for 0 <= c <= d, 16 <= d < 2^15 (a max below 16
    cannot occur under the speeds those loops take: tests/test_arith_domains.py)"""
    r = sweep(probe, MODE_DIVQ, 16, 32768)
    _report("divq(recip32)", r)
    assert r["cases"] == sum(d + 1 for d in range(16, 32768))
    assert r["mismatches"] == 0, "(c, d, got, want): %s" % r["examples"]
    small = sweep(probe, MODE_DIVQ, 1, 16)         # outside recip32's stated range: reported, not asserted
    _report("divq(recip32), 1 <= d < 16 (outside its range)", small)


def test_rcp15_table_and_div_by_u15(probe):
    """the reverse rANS pass divides a state st < 2^63 by a frequency f in 1..32767 through M[f] = floor((2^64 - 1) / f)"""
    tab = np.zeros(32768, np.uint64)
    assert probe.dvp_rcp15_table(_p(tab)) == 0
    want = [0] + [(2 ** 64 - 1) // f for f in range(1, 32768)]
    assert tab[1:].tolist() == want[1:]
    rng = np.random.default_rng(15)
    f = np.arange(1, 32768, dtype=np.uint64)
    top = np.uint64(2 ** 63 - 1)
    cols = [np.full(f.size, 2 ** 31, np.uint64), f * np.uint64(1 << 48) - np.uint64(1), np.full(f.size, top, np.uint64)]
    kmax = (top - np.uint64(1)) // f                # k * f + 1 <= 2^63 - 1
    for j in range(16):
        k = np.maximum(np.uint64(1), (kmax // np.uint64(15)) * np.uint64(j))
        for dk in (-1, 0, 1):
            cols.append((k * f).astype(np.uint64) + np.uint64(dk) if dk >= 0 else k * f - np.uint64(1))
    for _ in range(64):
        cols.append(rng.integers(0, 2 ** 63, f.size, dtype=np.uint64))
    x = np.concatenate(cols)
    ff = np.tile(f, len(cols)).astype(np.uint32)
    assert (x < np.uint64(2 ** 63)).all()
    q, r = np.zeros(x.size, np.uint64), np.zeros(x.size, np.uint32)
    assert probe.dvp_div_u15(_p(x), _p(ff), x.size, _p(q), _p(r)) == 0
    fq = ff.astype(np.uint64)
    bad = np.nonzero((q != x // fq) | (r.astype(np.uint64) != x % fq))[0]
    print("div_by_u15: %d cases over every f in 1..32767" % x.size)
    assert bad.size == 0, [(int(x[i]), int(ff[i]), int(q[i]), int(r[i])) for i in bad[:8]]


WEIGHT_EDGES = [1, 2, (1 << 24) - 1, 1 << 24, (1 << 24) + 1, 0x7EFFFFFF, 0x7F000000, 0x7FFFFFFF, 0x00FFFFFF, 0x01000000, 12345]


def _weight_cases(rng, n, f_lo):
    """n x (w0, w1, f_cm, f_nb, weighted): weights log-uniform over [1, 2^31) plus the fix_weights edges, frequencies in
    f_lo..32767 plus their edges"""
    w = np.exp2(rng.uniform(0, 31, (n, 2))).astype(np.int64).clip(1, 2 ** 31 - 1)
    pick = rng.random((n, 2)) < 0.1
    w[pick] = rng.choice(WEIGHT_EDGES, int(pick.sum()))
    f = rng.integers(f_lo, 32768, (n, 3))
    fe = rng.random((n, 3)) < 0.05
    f[fe] = rng.choice([x for x in (f_lo, f_lo + 1, -1, 0, 1, 2, 16384, 32766, 32767) if x >= f_lo], int(fe.sum()))
    grid = np.array([(a, b, c, d, e) for a in WEIGHT_EDGES for b in WEIGHT_EDGES for c in (f_lo, 1, 32767)
                     for d in (f_lo, 32767) for e in (max(f_lo, 1), 16384, 32767)], np.int64)
    return np.concatenate([np.concatenate([w, f], 1), grid]).astype(np.int32)


def _gpu_weights(probe, variant, cases):
    out = np.zeros((cases.shape[0], 3), np.int32)
    assert probe.dvp_weights(variant, cases.shape[0], _p(np.ascontiguousarray(cases)), _p(out)) == 0
    return out


def _oracle_weights(oracle, cases):
    o0, o1, on = oracle.weights_update_batch(cases[:, 0], cases[:, 1], cases[:, 2], cases[:, 3], cases[:, 4])
    return np.stack([o0, o1, on.astype(np.int32) & 0xFFFF], 1)


def test_weights_update_equals_the_oracle(probe, oracle):
    """weights_update (generic cores): any i16 frequency, wrapped ones included"""
    cases = _weight_cases(np.random.default_rng(7), 10 ** 7, -32768)
    got, want = _gpu_weights(probe, 0, cases), _oracle_weights(oracle, cases)
    bad = np.nonzero((got != want).any(1))[0]
    print("weights_update: %d cases" % cases.shape[0])
    assert bad.size == 0, [(cases[i].tolist(), got[i].tolist(), want[i].tolist()) for i in bad[:8]]


def test_weights_update32_equals_weights_update_where_it_claims(probe, oracle):
    """weights_update32 (v2 mixing loop) claims equality with weights_update for coded frequencies in 1..32767"""
    cases = _weight_cases(np.random.default_rng(8), 10 ** 7, 1)
    got32, got = _gpu_weights(probe, 1, cases), _gpu_weights(probe, 0, cases)
    want = _oracle_weights(oracle, cases)
    print("weights_update32: %d cases" % cases.shape[0])
    bad = np.nonzero((got32 != got).any(1) | (got32 != want).any(1))[0]
    assert bad.size == 0, [(cases[i].tolist(), got32[i].tolist(), want[i].tolist()) for i in bad[:8]]


def test_speed_is_small_on_every_i16_pair(probe):
    """the product's gate equals its restatement (the four comparisons, tests/regimes.py speed_is_small) on every packed
    i16 (inc, lim): per inc, the number of accepted lim and the least and greatest of them"""
    out = np.zeros((65536, 3), np.int32)
    assert probe.dvp_speed_gate(_p(out)) == 0
    lim = np.arange(-32768, 32768, dtype=np.int64)      # ascending
    want = np.zeros((65536, 3), np.int64)
    want[:, 1], want[:, 2] = 1 << 20, -(1 << 20)
    for row in range(65536):
        inc = row - 65536 if row >= 32768 else row
        if not (inc >= 0 and 4 * (inc + 16) <= 0x7FFF):  # comparisons on inc alone: no lim passes
            continue
        ok = np.nonzero((lim >= 0) & (lim + inc + 16 <= 0x7FFF))[0]
        if ok.size:
            want[row] = (ok.size, lim[ok[0]], lim[ok[-1]])
    # spot-check the vectorised restatement against the scalar one
    for inc, l in [(0, 0), (8175, 0), (8176, 0), (0, 0x7FEF), (0, 0x7FF0), (-1, 5), (5, -1), (8175, 0x7FFF - 16 - 8175)]:
        row = inc & 0xFFFF
        assert R.speed_is_small(inc, l) == bool(want[row, 0] and want[row, 1] <= l <= want[row, 2])
    bad = np.nonzero((out != want).any(1))[0]
    print("speed_is_small: %d pairs, %d accepted" % (1 << 32, int(out[:, 0].sum())))
    assert bad.size == 0, [(int(r), out[r].tolist(), want[r].tolist()) for r in bad[:8]]


@pytest.mark.parametrize("variant", sorted(R.C_OVER_MAX_OPTIONS))
def test_c_over_max_regime_matches_the_oracle(engine, engine16, oracle, variant):
    """one literal prior driven into a state with an element far above its max, then coded at that element: the GPU
    encoder's bytes equal the oracle's, and every decode layout returns the oracle's status and bytes"""
    import divans_b200
    cl, stream = R.c_over_max(oracle, variant)
    got = engine.encode([cl.serialize()], divans_b200.encode_options(**R.C_OVER_MAX_OPTIONS[variant]), cmds=True)
    assert got[0] == stream, "GPU encoder output differs from the oracle's"
    cap = len(R.C_OVER_MAX_BYTES) + 64
    rc, ref = oracle.decode(stream, out_cap=cap)
    for layout, eng in (("16 lanes", engine), ("8 lanes", engine16)):
        st, out = eng.decode([stream], [cap])[0]
        assert (st, out) == (rc, ref), "%s: status %d, oracle %d" % (layout, st, rc)


# ---------------------------------------------------------------------------------------------------------------------
# One coding step at CDF level: the cores as the engine calls them (the probe's dvp_step), against the oracle's
# dvo_cdf_step_batch (code_lit_nibble, codec/literal.rs:154-259, with the rANS step of ans.rs:230-244)
# ---------------------------------------------------------------------------------------------------------------------
V2_16, V2_8, R1_ENC, FAST_16, FAST_8, FAST_MIX_16 = 0, 1, 3, 4, 5, 6   # dv_probe.cu StepVariant
GEN = 0xA5C3                                             # a nonzero generation: the fast pieces store its bits as tags
HIGH_WORDS = [1, 1 << 16, (1 << 31) - 1, 1 << 47]


def _f8_pairs(oracle, small):
    sp = sorted(set(int(oracle.lib().dvo_u8_to_speed(v)) for v in range(256)))
    return np.array([(a, b) for a in sp for b in sp if R.speed_is_small(a, b) == small or not small], np.int16)


@pytest.fixture(scope="module")
def step_states(oracle):
    """walk states per speed class: 'wide' = every f8 pair, 'small' = the speed_is_small ones (monotone CDFs).  Each state
    comes with the speed its walk ran under: every state is reachable by construction.  Returns
    {class: (cdf (n, 16), speed (n, 2), number of c > max states kept)}"""
    from test_arith_domains import walk_syms
    rng = np.random.default_rng(31)
    out = {}
    for cls in ("wide", "small"):
        pairs = _f8_pairs(oracle, cls == "small")
        pick = pairs[rng.integers(0, len(pairs), 2048)]
        tr = oracle.cdf_walks(pick, walk_syms(rng, len(pick), 96))
        cdf = tr.reshape(-1, 16).astype(np.int16)
        spd = np.repeat(pick, tr.shape[1], axis=0)
        c32 = cdf.astype(np.int64)
        over = ((c32 > c32[:, 15:16]) & (c32[:, 15:16] > 0)).any(1)
        sel = np.concatenate([rng.choice(np.nonzero(~over)[0], 4096, replace=False), np.nonzero(over)[0]])
        out[cls] = (cdf[sel], spd[sel], int(over.sum()))
    return out


def _edge_vectors(rng):
    v = []
    for m in (-32768, -1, 0, 1, 2, 3, 0x7FFF):
        for _ in range(8):
            c = np.sort(rng.integers(-32768, 32768, 16)); c[15] = m; v.append(c)
    for e in (0, 1, 3, 64, 0x7FFF, -1, -32768):
        v.append(np.full(16, e))
    for k in range(15):
        c = np.arange(16) % 2; c[k] = 0x7FFF; c[15] = 1; v.append(c)
    return np.array(v, np.int16)


@pytest.fixture(scope="module")
def weight_states(oracle):
    """(w0, w1, norm) states of a long walk of weight updates, plus the fix_weights boundary (weights at 2^24 - 1, 2^24 and
    0x7f000000, the last update's norm)"""
    rng = np.random.default_rng(32)
    w = np.array([1, 1, 1 << 14], np.int32)
    states = []
    f = rng.integers(1, 32768, (20000, 3))
    for k in range(20000):
        o0, o1, on = oracle.weights_update_batch([w[0]], [w[1]], [f[k, 0]], [f[k, 1]], [f[k, 2]])
        w = np.array([o0[0], o1[0], int(on[0]) & 0xFFFF], np.int32)
        states.append(w)
    s = np.array(states)
    edges = [(a, b, int(s[i % len(s), 2])) for i, (a, b) in enumerate(
        [(a, b) for a in ((1 << 24) - 1, 1 << 24, 0x7F000000, 1) for b in ((1 << 24) - 1, 1 << 24, 0x7F000000, 5)])]
    return np.concatenate([s, np.array(edges, np.int32)])


def _cases(rng, cdf, spd, cm_spd_pairs, weights, enc, full_offsets=64, offsets=256):
    """cross product of states and offsets (decode: `full_offsets` states take all 32768, every state `offsets` random
    ones) or of states and the 16 symbols (encode); high state words from HIGH_WORDS and random"""
    n = len(cdf)
    if enc:
        idx, sym = np.repeat(np.arange(n), 16), np.tile(np.arange(16), n)
        state = np.zeros(idx.size, np.uint64)
    else:
        idx = np.concatenate([np.repeat(np.arange(min(full_offsets, n)), 32768), np.repeat(np.arange(n), offsets)])
        off = np.concatenate([np.tile(np.arange(32768), min(full_offsets, n)), rng.integers(0, 32768, n * offsets)])
        hw = np.array(HIGH_WORDS + [int(x) for x in rng.integers(1, 1 << 48, 60)], np.uint64)
        state = (hw[rng.integers(0, hw.size, idx.size)] << np.uint64(15)) | off.astype(np.uint64)
        sym = np.zeros(idx.size, np.int32)
    m = idx.size
    other = rng.integers(0, n, m)                          # the context-map prior: another state
    cmsp = cm_spd_pairs[rng.integers(0, len(cm_spd_pairs), m)]
    return dict(cdf=cdf[idx], cdf2=cdf[other], spd=np.stack([spd[idx], cmsp], 1), state=state, sym=sym,
                wts=weights[rng.integers(0, len(weights), m)])


def _run_step(probe, variant, mix, c):
    n = c["cdf"].shape[0]
    pk = (c["spd"][:, :, 0].astype(np.int32) & 0xFFFF) | (c["spd"][:, :, 1].astype(np.int32) << 16)
    o = dict(sym=np.zeros(n, np.int32), start=np.zeros(n, np.int32), freq=np.zeros(n, np.int32), status=np.zeros(n, np.int32),
             state=np.zeros(n, np.uint64), cdf=np.zeros((n, 16), np.int16), cdf2=np.zeros((n, 16), np.int16),
             wts=np.zeros((n, 3), np.int32))
    args = [np.ascontiguousarray(c[k], t) for k, t in (("cdf", np.int16), ("cdf2", np.int16), ("wts", np.int32))]
    args += [np.ascontiguousarray(pk), np.ascontiguousarray(c["state"], np.uint64), np.ascontiguousarray(c["sym"], np.int32)]
    assert probe.dvp_step(variant, n, int(mix), GEN, *[_p(a) for a in args],
                          *[_p(o[k]) for k in ("sym", "start", "freq", "status", "state", "cdf", "cdf2", "wts")]) == 0
    return o


def _check_step(probe, oracle, variant, mix, c, what):
    enc = variant == R1_ENC
    got = _run_step(probe, variant, mix, c)
    ref = oracle.cdf_steps(c["cdf"], c["spd"], state=None if enc else c["state"], sym=c["sym"] if enc else None,
                           cdf2=c["cdf2"] if mix else None, wts=c["wts"] if mix else None)
    bad = got["sym"] != ref["sym"]
    fast = variant in (FAST_16, FAST_8, FAST_MIX_16)
    if enc:
        bad |= (got["start"] != ref["start"]) | (got["freq"] != ref["freq"])
        bad |= got["status"] != np.where(ref["freq"] <= 0, 3, 0)       # enc_log refuses a frequency <= 0
    else:
        want = ref["state"]
        if variant == FAST_MIX_16:                                      # renormalised with a zero word
            want = np.where(want < np.uint64(1 << 31), want << np.uint64(32), want)
        bad |= got["state"] != want
    gc = got["cdf"]
    if fast:
        tags = ((GEN >> np.arange(16)) & 1).astype(np.int32) << 15
        bad |= ((gc.astype(np.int32) & 0x8000) != tags).any(1)
        gc = (gc.astype(np.int32) & 0x7FFF).astype(np.int16)
    bad |= (gc != ref["cdf"]).any(1)
    if mix:
        bad |= (got["cdf2"] != ref["cdf2"]).any(1) | (got["wts"] != ref["wts"]).any(1)
    c32 = c["cdf"].astype(np.int64)
    n_over = int(((c32 > c32[:, 15:16]) & (c32[:, 15:16] > 0)).any(1).sum())
    print("%s: %d cases, %d with c > max, %d mismatches" % (what, len(bad), n_over, int(bad.sum())))
    i = np.nonzero(bad)[0][:4]
    assert not bad.any(), [dict(cdf=c["cdf"][k].tolist(), state=int(c["state"][k]), sym=(int(got["sym"][k]), int(ref["sym"][k])),
                                got_cdf=got["cdf"][k].tolist(), want_cdf=ref["cdf"][k].tolist()) for k in i]


def test_walk_states_reach_c_over_max_with_quotients_above_2_24(step_states):
    cdf, _spd, n_over = step_states["wide"]
    c = cdf.astype(np.int64)
    m = c[:, 15:16]
    q = np.where((c > m) & (m > 0), (np.clip(c, 0, None) << 15) // np.maximum(m, 1), 0)
    print("wide walks: %d states with c > max kept, largest quotient %d" % (n_over, int(q.max())))
    assert n_over > 100 and (q >= 1 << 24).any()
    assert step_states["small"][2] == 0, "a c > max state under speed_is_small speeds"


@pytest.mark.parametrize("mix", [False, True], ids=["plain", "mixing"])
@pytest.mark.parametrize("variant", [V2_16, V2_8, R1_ENC], ids=["v2_16", "v2_8", "r1_encode"])
def test_generic_core_step_equals_the_oracle(probe, oracle, step_states, weight_states, variant, mix):
    """nibble_core_v2<16> / <8> (untagged) and the round-1 core's encoder step (nibble_core_enc, with the enc_log refusal) on walk
    states under every f8 speed pair, the c > max states those walks reach, and edge vectors"""
    rng = np.random.default_rng(40 + variant + 8 * mix)
    cdf, spd, _ = step_states["wide"]
    pairs = _f8_pairs(oracle, False)
    edges = _edge_vectors(rng)
    cdf = np.concatenate([cdf, edges])
    spd = np.concatenate([spd, pairs[rng.integers(0, len(pairs), len(edges))]])
    c = _cases(rng, cdf, spd, pairs, weight_states, variant == R1_ENC)
    _check_step(probe, oracle, variant, mix, c, "core %d %s" % (variant, "mixing" if mix else "plain"))


@pytest.mark.parametrize("variant", [FAST_16, FAST_8, FAST_MIX_16], ids=["fast_16", "fast_8", "mix_16"])
def test_fast_loop_pieces_equal_the_oracle(probe, oracle, step_states, weight_states, variant):
    """search_v2 + rans_advance_v2 + blend_store_v2 (16 and 8 lanes) and mixv_search + mixv_finish (16 lanes) on walk states
    under speed_is_small speeds, storing with the tag bits of a nonzero generation"""
    rng = np.random.default_rng(50 + variant)
    cdf, spd, _ = step_states["small"]
    c = _cases(rng, cdf, spd, _f8_pairs(oracle, True), weight_states, False)
    _check_step(probe, oracle, variant, variant == FAST_MIX_16, c, "fast piece %d" % variant)
