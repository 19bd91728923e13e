"""GPU tests (-m gpu) of mixing values 0..15 and per-context mixing masks (tests/mixing_values.py) against the CPU oracle: the
v2 decoder on both lane layouts and with the lanes chosen by batch size, one-warp contexts where per-context and uniform
streams are warp-mates, the blend decoder, the command-list and raw encoders, encode_auto, encode_mixmap at the edges of its
candidate list, and PredictionMode records whose bytes no stream can carry."""
import itertools

import numpy as np
import pytest

import divans_b200
import mixing_values as V
import regimes as R
import test_gpu_encode_auto as A
import test_gpu_encode_cmds_auto as C
import test_gpu_encode_mixmap as X
from irfuzz import random_ir
from oracle_tally import tally_py as T

pytestmark = pytest.mark.gpu

PMB = divans_b200.PM_RECORD_BYTES
MIX_AT = 32 + 16384 + 1024      # the mixing values inside a PredictionMode record
PLAIN = ["lsb6", "msb6", "utf8", "sign", "dcm2", "mix2_flat"]   # regimes.py streams of one uniform value
BLEND = divans_b200.FLAG_CDF_BLEND


# The contexts of this file are its own, 64 slots each, and closed when the file is done.  A context's arena and scratch only
# grow (a decode takes one 16 MiB slot per resident stream) and stay allocated until it closes: run on the session's engines,
# these batches would leave them holding memory that later tests of the session need.
@pytest.fixture(scope="module")
def small():
    """16 lanes per stream: the decoder of two streams per warp, the encoders and decode_cmds"""
    eng = divans_b200.Engine(0, 64, 16)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def small8():
    """8 lanes per stream: the decoder of four streams per warp"""
    eng = divans_b200.Engine(0, 64, 8)
    yield eng
    eng.close()


def _cases(O, names, dcms=V.DCMS):
    return [(n, d, V.build(n, O, d)) for n in names for d in dcms]


def _decode_check(eng, O, cases, flags, what, cmds_eng):
    """one launch; every status 0 and every byte the oracle's; then decode_cmds on `cmds_eng`: the records carry the masks
    that were built"""
    if not cases:
        return
    res = eng.decode([c.stream for _, _, c in cases], [c.cap for _, _, c in cases], flags)
    for (name, dcm, c), (st, out) in zip(cases, res):
        assert st == 0 and out == c.raw, "%s: %s dcm %d: status %d, %s" % (what, name, dcm, st, "bytes differ" if st == 0 else "")
    res = cmds_eng.decode_cmds([c.stream for _, _, c in cases], [c.cap for _, _, c in cases], flags)
    for (name, dcm, c), (st, out, blob) in zip(cases, res):
        want = np.stack(V.command_list(name, O)[1])
        assert st == 0 and out == c.raw and (V.masks_of(blob) == want).all(), "%s: %s dcm %d: decoded masks differ" % (what, name, dcm)


def _split_wasm(cases):
    return [x for x in cases if x[0] != "wasm_2018"], [x for x in cases if x[0] == "wasm_2018"]


# ---------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes", ["16", "8", "auto"])
def test_decode_every_stream(oracle, small, small8, lanes):
    """every stream under dynamic mixing 0/1/2 in one batch (more streams than slots: the slots are reused), the same batch
    reversed and one shorter, on each lane layout and on a context that picks its layout by batch size"""
    eng = {"16": small, "8": small8}.get(lanes) or divans_b200.Engine(0, 64, 0)
    try:
        cur, wasm = _split_wasm(_cases(oracle, V.ALL))
        _decode_check(eng, oracle, cur, 0, "batch", small)
        _decode_check(eng, oracle, cur[::-1][1:], 0, "odd batch, reversed", small)
        _decode_check(eng, oracle, wasm, divans_b200.FLAG_MODEL_WASM_2018, "WASM_2018", small)
    finally:
        if lanes == "auto":
            eng.close()


@pytest.mark.parametrize("layout", [(2, 16), (4, 8)])
def test_one_warp_mates(oracle, layout):
    """one warp: each per-context stream next to each uniform 9..15 stream and each plain regime, in both orders (8 lanes:
    the pair twice), so that a warp-mate's lit_cfg >= 0 never lets the fast loops take a per-context stream"""
    g, lanes = layout
    eng = divans_b200.Engine(0, g, lanes)
    try:
        for dcm in (1, 2):
            per = _cases(oracle, V.PER_CONTEXT, [dcm])
            mates = _cases(oracle, V.UNIFORM_NAMES, [dcm]) + [(n, 0, R.build(n, oracle)) for n in PLAIN]
            for p, u in itertools.product(per, mates):
                for pair in ([p, u], [u, p]):
                    batch = pair * (g // 2)
                    res = eng.decode([c.stream for _, _, c in batch], [c.cap for _, _, c in batch])
                    for (name, d, c), (st, out) in zip(batch, res):
                        assert st == 0 and out == c.raw, "%s + %s (dcm %d): %s" % (pair[0][0], pair[1][0], dcm, name)
        assert eng.last_lanes() == lanes
    finally:
        eng.close()


@pytest.mark.parametrize("lanes", ["16", "8"])
def test_blend_decoder(oracle_blend, small, small8, lanes):
    _decode_check(small if lanes == "16" else small8, oracle_blend, _cases(oracle_blend, V.BLEND_TWINS), BLEND, "blend", small)


# ---------------------------------------------------------------------------------------------------------------------
# encode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("blend", [False, True])
@pytest.mark.parametrize("dcm", V.DCMS)
def test_encode_cmds_matches_oracle(small, oracle, oracle_blend, blend, dcm):
    O = oracle_blend if blend else oracle
    names = V.BLEND_TWINS if blend else V.ALL
    for wasm in (False, True):
        group = [n for n in names if (n == "wasm_2018") == wasm]
        if not group:
            continue
        o = divans_b200.encode_options(cdf_model=int(blend), **V.encode_options(group[0], dcm))
        blobs = [V.command_list(n, O)[0].serialize() for n in group]
        want = [V.build(n, O, dcm).stream for n in group]
        host = small.encode(blobs, o, cmds=True)
        dev, _, _ = C._auto_device(small, blobs, o, plain=True)
        for n, h, d, w in zip(group, host, dev, want):
            assert h == w, "%s: host stream differs from the oracle's" % n
            assert d[0] == 0 and d[2] == w, "%s: device stream differs from the oracle's" % n


def _raws():
    return [V.mode_input(m, 2500, 141000 + 1000 * k) for k, m in enumerate(V.MODES)] + [V.records(2000, 2, 7)]


@pytest.mark.parametrize("dcm", [1, 2])
@pytest.mark.parametrize("mode", range(4))
def test_raw_encoder_values_9_to_15(small, oracle, mode, dcm):
    """the raw encoder's one PredictionMode record with literal_mixing_value 9..15 (mixing-value priors 9..15 from entry 256
    on, the clamped stride of mm_cfg) equals dvo_encode_raw_batch"""
    from test_gpu_encode import _oracle_raw
    raws = _raws()
    kw = dict(window_size=16, dynamic_context_mixing=dcm)
    for v in V.UNIFORM:
        got = small.encode(raws, divans_b200.encode_options(literal_pred_mode=mode, literal_mixing_value=v, **kw))
        ref = _oracle_raw(oracle, raws, kw, mode, v)
        assert [(0, g) for g in got] == ref, (mode, v)


def test_encode_auto_with_values_9_to_15(small, oracle):
    cands = [(m, v) for m in range(4) for v in (9, 12, 15)] + [(0, 4), (2, 8), (1, 11), (3, 13)]
    for dcm in (1, 2):
        kw = dict(window_size=16, dynamic_context_mixing=dcm)
        A._check_batch(small, oracle, _raws(), divans_b200.encode_options(**kw), kw, False, cands)


# ---------------------------------------------------------------------------------------------------------------------
# encode_mixmap at the edges of its candidate list
# ---------------------------------------------------------------------------------------------------------------------
SCRAMBLED16 = [12, 3, 15, 8, 0, 9, 5, 14, 1, 11, 6, 2, 13, 7, 4, 10]
EDGE_VALUES = {"k16": SCRAMBLED16, "k1_9": [9], "k1_2": [2], "dup_4_4": [4, 4], "dup_9_13": [9, 13]}


def _tie_rule(mixing, values):
    """values 8..15 code literals identically, so their bins tie: a mixed map holds none of them but the first in the list"""
    first = next((v for v in values if v >= 8), None)
    assert not np.isin(mixing, [v for v in range(8, 16) if v != first]).any(), np.unique(mixing)


def _mixmap_lists(oracle):
    return [V.command_list(n, oracle)[0] for n in ("all16_lsb6", "switch", "halves_3_15")] + \
        [oracle.Commands.from_ir(random_ir(oracle, 9300 + s, n_cmds=50, window=16, text=R.text())) for s in range(2)]


@pytest.mark.parametrize("values", list(EDGE_VALUES))
@pytest.mark.parametrize("call", ["host", "device"])
@pytest.mark.parametrize("cmds", [False, True])
def test_mixmap_candidate_edges(small, oracle, values, call, cmds):
    vals = EDGE_VALUES[values]
    k = len(vals)
    okw = dict(window_size=16, dynamic_context_mixing=2 if values == "k16" else 1)
    opts = divans_b200.encode_options(literal_pred_mode=0, **okw)
    lists = _mixmap_lists(oracle) if cmds else None
    inputs = [cl.serialize() for cl in lists] if cmds else X._raws()
    res = (X._host if call == "host" else X._device)(small, inputs, opts, cmds, vals)
    mixed = 0
    for i, x in enumerate(inputs):
        want = T.encode_cmds_mixmap(lists[i], 0, vals, **okw) if cmds else T.encode_mixmap(x, 0, vals, **okw)
        X._check(res[i], want, "%s %s %d" % (values, call, i))
        st, ln, out, ch, mixing, cost, bins = res[i]
        if k == 1:
            assert ch == 0 and (mixing == vals[0]).all()
        if ch < k:   # a uniform choice: the plain encoder's stream with that value
            plain = divans_b200.encode_options(literal_pred_mode=0, literal_mixing_value=vals[ch], **okw)
            assert out == (C._plain_host(small, [C._rewrite(x, (0, vals[ch]))], plain)[0][2] if cmds else small.encode([x], plain)[0])
        if ch == k:
            mixed += 1
            _tie_rule(mixing, vals)
        if values == "dup_4_4":   # the second 4 never wins an entry nor the uniform choice
            assert (bins[0] == bins[1]).all() and ch != 1
    if values == "k16":
        assert mixed, "no input took a mixed record"


# ---------------------------------------------------------------------------------------------------------------------
# PredictionMode records no stream can carry
# ---------------------------------------------------------------------------------------------------------------------
def _hostile_lists(oracle):
    return [oracle.Commands.from_ir(random_ir(oracle, 9400 + s, n_cmds=40, window=16, text=R.text())) for s in range(4)]


def _records_at(blob):
    h = np.frombuffer(bytes(blob[:32]), np.uint32)
    at = 32 + 20 * int(h[2])
    return [at + k * PMB for k in range(int(h[3]))]


def _rewrite(blob, fn):
    b = np.frombuffer(bytes(blob), np.uint8).copy()
    for at in _records_at(blob):
        fn(b[at:at + PMB])
    return b.tobytes()


def _entries(oracle, cl):
    """(a mask entry some literal is coded with, one none is) of the list's own records"""
    rc, _, bins, _ = T.tally_cmds_bins(cl, *T.KEEP, window_size=16)
    assert rc == 0
    return int(np.argmax(bins)), int(np.flatnonzero(bins == 0)[0])


def _hostile_blobs(oracle):
    out = []
    for cl in _hostile_lists(oracle):
        blob = cl.serialize()
        vis, unvis = _entries(oracle, cl)
        for v in (16, 17, 31, 200, 255):
            for e, where in ((vis, "visited"), (unvis, "unvisited")):
                def f(r, e=e, v=v):
                    r[MIX_AT + e] = v
                out.append(("mixing %d %s" % (v, where), _rewrite(blob, f), True))
        for a in (2, 255):
            out.append(("is_adv %d" % a, _rewrite(blob, lambda r, a=a: r.__setitem__(1, a)), True))
        for p in (4, 16, 255):
            out.append(("pred_mode %d" % p, _rewrite(blob, lambda r, p=p: r.__setitem__(0, p)), True))
        for off, n in ((28, 16385), (28, 65535), (30, 1025)):
            def f(r, off=off, n=n):
                r[off:off + 2] = np.frombuffer(np.uint16(n).tobytes(), np.uint8)
            out.append(("map length @%d = %d" % (off, n), _rewrite(blob, f), True))
    return out


def _fuzzed_blobs(oracle, n=48, seed=77):
    """random bytes written inside the PredictionMode records -- the mode, is_adv, has_speeds, the map lengths, the maps and the
    mixing values (not the speeds: a stream-supplied speed may wrap a counter, and such a stream need not decode to its input)"""
    rng = np.random.default_rng(seed)
    lists = _hostile_lists(oracle)
    out = []
    for i in range(n):
        blob = lists[i % len(lists)].serialize()
        b = np.frombuffer(blob, np.uint8).copy()
        recs = _records_at(blob)
        for _ in range(int(rng.integers(1, 5))):
            at = recs[int(rng.integers(0, len(recs)))]
            field = int(rng.integers(0, 5))
            off = [int(rng.integers(0, 3)), 28 + int(rng.integers(0, 4)), 32 + int(rng.integers(0, 16384)),
                   32 + 16384 + int(rng.integers(0, 1024)), MIX_AT + int(rng.integers(0, 8192))][field]
            b[at + off] = int(rng.integers(0, 256)) if field != 4 or rng.random() < 0.5 else int(rng.integers(0, 16))
        out.append(("fuzz %d" % i, b.tobytes(), False))
    return out


def _roundtrip_or_refused(engine, oracle, blobs, results, what, must_refuse):
    """status 3, or status 0 with a stream that the GPU and the oracle decode to the list's replay; and (must_refuse) status
    3 for every record of _hostile_blobs"""
    good = []
    for (name, blob, hostile), (st, stream) in zip(blobs, results):
        assert st in (0, 3), "%s: %s: status %d" % (what, name, st)
        if st == 0:
            rc, n, replay = T.recode_blob(blob)
            assert rc == 0
            good.append((name, stream, replay))
    if good:
        res = engine.decode([s for _, s, _ in good], [len(r) + 64 for _, _, r in good])
        for (name, s, replay), (st, out) in zip(good, res):
            assert oracle.decode(s, out_cap=len(replay) + 64) == (0, replay), "%s: %s: status 0, but the oracle decodes other bytes" % (what, name)
            assert st == 0 and out == replay, "%s: %s: status 0, but the GPU decodes other bytes" % (what, name)
    for (name, _, hostile), (st, _) in zip(blobs, results):
        assert st == 3 or not (must_refuse and hostile), "%s: %s: status %d" % (what, name, st)


@pytest.mark.parametrize("kind", ["hostile", "fuzz"])
def test_unrepresentable_records_are_refused(small, oracle, kind):
    blobs = _hostile_blobs(oracle) if kind == "hostile" else _fuzzed_blobs(oracle)
    bl = [b for _, b, _ in blobs]
    o = divans_b200.encode_options(window_size=16)
    host = C._plain_host(small, bl, o)
    _roundtrip_or_refused(small, oracle, blobs, [(s, x) for s, _, x in host], "encode_cmds host", True)
    dev, _, _ = C._auto_device(small, bl, o, plain=True)
    _roundtrip_or_refused(small, oracle, blobs, [(s, x) for s, _, x in dev], "encode_cmds device", True)
    auto, chosen, cost = C._auto_host(small, bl, o, [C.KEEP])
    _roundtrip_or_refused(small, oracle, blobs, [(s, x) for s, _, x in auto], "encode_cmds_auto KEEP", True)
    for (name, _, hostile), (st, _, _), c in zip(blobs, auto, cost):
        assert (st == 3) == (c[0] == T.TALLY_FAILED), "%s: status %d, KEEP cost %d" % (name, st, c[0])
    mm = X._host(small, bl, divans_b200.encode_options(window_size=16, literal_pred_mode=0), True)
    _roundtrip_or_refused(small, oracle, blobs, [(x[0], x[2]) for x in mm], "encode_cmds_mixmap", False)
