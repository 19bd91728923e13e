"""GPU tests (-m gpu) of the state a v2 decoder slot carries from stream to stream and from launch to launch, and of which
streams share a warp (DESIGN.md "Slot state of the v2 decoder").

The lever is a one-warp engine: Engine(0, 2, 16) is one warp with two slots, Engine(0, 4, 8) one warp with four.  A batch of
exactly 2 (or 4) streams makes them warp-mates; a longer batch sends every stream through the same few slots, one after
another.  Identical streams finish together and fetch together, so `[A] * G + [B] * G` gives every slot A, then B.  The slot
header readout (Engine.slot_header) asserts that each test hit its case: the generation of every slot, the lockstep split,
and the flags set or cleared.  Every byte and every status is checked against the CPU oracle."""
import itertools

import numpy as np
import pytest

import regimes as R

pytestmark = pytest.mark.gpu

LAYOUTS = {"16lanes_2slots": (2, 16), "8lanes_4slots": (4, 8)}


@pytest.fixture(params=list(LAYOUTS))
def warp(request):
    """a fresh one-warp engine (every slot header starts at zero); .groups = its slots"""
    import divans_b200
    g, lanes = LAYOUTS[request.param]
    eng = divans_b200.Engine(0, g, lanes)
    eng.groups = g
    yield eng
    eng.close()


def _check(eng, oracle, cases, what=""):
    """one launch of `cases`; every status equals the oracle's, every successful output its bytes"""
    flags = 0
    for c in cases:
        flags |= c.flags
    res = eng.decode([c.stream for c in cases], [c.cap for c in cases], flags)
    for i, ((st, out), c) in enumerate(zip(res, cases)):
        rc, ref = oracle.decode(c.stream, out_cap=c.cap, skip_crc=bool(flags))
        assert rc == c.status, (what, i)
        assert st == rc, "%s: stream %d: status %d, oracle %d" % (what, i, st, rc)
        if rc == 0:
            assert out == ref, "%s: stream %d: first diff at %d" % (
                what, i, next((k for k in range(min(len(out), len(ref))) if out[k] != ref[k]), min(len(out), len(ref))))
    return res


def _headers(eng):
    return [eng.slot_header(i) for i in range(eng.groups)]


def _in_every_slot(eng, oracle, seq, what=""):
    """one launch in which every slot decodes seq[0], then seq[1], ...; asserts the lockstep split through the generation
    counters and returns the slot headers after the launch"""
    before = [h[0] for h in _headers(eng)] if eng.launch_count else [0] * eng.groups
    _check(eng, oracle, [c for c in seq for _ in range(eng.groups)], what)
    after = _headers(eng)
    assert [h[0] - b for h, b in zip(after, before)] == [len(seq)] * eng.groups, (what, before, after)
    assert all(h[0] & 0xFFFF for h in after)
    return after


@pytest.fixture(scope="module")
def cases(oracle):
    return {n: R.build(n, oracle) for n in R.ALL}


# ---------------------------------------------------------------------------------------------------------------------
# warp composition
# ---------------------------------------------------------------------------------------------------------------------
def test_every_pair_of_regimes_as_warp_mates(oracle, cases):
    """Two groups of one 16-lane warp: the literal fast loops run only when both agree (T2S only if both are LSB6/MSB6, the
    mix loop only if both mix, else the generic path), and a group out of work rides along as a dummy.  Every unordered
    pair, each as a 2-stream batch on a one-warp engine."""
    import divans_b200
    eng = divans_b200.Engine(0, 2, 16)
    try:
        for a, b in itertools.combinations_with_replacement(R.ALL, 2):
            _check(eng, oracle, [cases[a], cases[b]], "%s + %s" % (a, b))
        assert eng.last_lanes() == 16
    finally:
        eng.close()


def test_seeded_quads_of_regimes_as_warp_mates(oracle, cases):
    """Four groups of one 8-lane warp: 80 seeded four-stream combinations of the regimes."""
    import divans_b200
    rng = np.random.default_rng(2024)
    eng = divans_b200.Engine(0, 4, 8)
    try:
        for _ in range(80):
            pick = [R.ALL[int(k)] for k in rng.integers(0, len(R.ALL), 4)]
            _check(eng, oracle, [cases[n] for n in pick], " + ".join(pick))
        assert eng.last_lanes() == 8
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# slot succession
# ---------------------------------------------------------------------------------------------------------------------
def test_generation_tags_separate_successive_streams(warp, oracle):
    """Generation tags: literal priors are never re-initialised; a prior written by stream A carries A's generation and
    reads as the default CDF for the next stream B in the slot.  A and B touch the same priors (LSB6 text), in one launch
    and across two launches (header word 0 survives the launch)."""
    a, b = R.build("lsb6", oracle, 0), R.build("lsb6", oracle, 1)
    h = _in_every_slot(warp, oracle, [a, b], "one launch")
    assert [x[0] for x in h] == [2] * warp.groups
    _in_every_slot(warp, oracle, [a], "launch 2")
    h = _in_every_slot(warp, oracle, [b], "launch 3")
    assert [x[0] for x in h] == [4] * warp.groups


@pytest.mark.parametrize("launches", [1, 3])
def test_generation_wrap_wipes_the_literal_tables(warp, oracle, launches):
    """Generation wrap: header word 0 counts the streams of a slot; when its low 16 bits wrap to 0 the slot's literal tables
    are wiped and generation 0 is skipped.  Poison stream P (2 KB LSB6 text) adapts the hot priors under generation 1, then
    65534 empty streams run through every slot, then P's twin R gets generation 1 again: without the wipe it would read P's
    priors as its own."""
    G = warp.groups
    p, r, e = R.build("lsb6", oracle, 0), R.build("lsb6", oracle, 1), R.build("empty", oracle)
    n_empty = 65534 * G
    seq = [p] * G + [e] * n_empty + [r] * G
    streams = [np.frombuffer(c.stream, np.uint8) for c in (p, e, r)]
    soff = np.cumsum([0] + [((s.size + 15) // 16) * 16 for s in streams])
    blob = np.zeros(int(soff[-1]) + 16, np.uint8)
    for s, o in zip(streams, soff):
        blob[int(o):int(o) + s.size] = s
    kind = np.array([0] * G + [1] * n_empty + [2] * G)
    in_off = soff[kind].astype(np.uint64)                # the empty streams alias one copy of the input
    in_len = np.array([s.size for s in streams], np.uint64)[kind]
    cap = np.array([c.cap for c in seq], np.uint64)
    out_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
    bounds = [(0, len(seq))] if launches == 1 else [(0, G), (G, G + n_empty), (G + n_empty, len(seq))]
    out = np.zeros(int(cap.sum()), np.uint8)
    status = np.full(len(seq), -1, np.int32)
    out_len = np.zeros(len(seq), np.uint64)
    seen = []
    for lo, hi in bounds:
        ol, st = warp.decode_batch_host(blob, in_off[lo:hi], in_len[lo:hi], out, out_off[lo:hi], cap[lo:hi])
        out_len[lo:hi], status[lo:hi] = ol, st
        seen.append(_headers(warp))
        assert all(h[0] & 0xFFFF for h in seen[-1]), seen[-1]
    if launches == 3:
        assert [h[0] for h in seen[0]] == [1] * G and [h[0] for h in seen[1]] == [65535] * G
    # 65536 streams per slot and the skipped generation 0: R decoded under generation 1, like P
    assert [h[0] for h in seen[-1]] == [65537] * G and [h[1] for h in seen[-1]] == [0] * G
    assert (status == 0).all() and (out_len[G:G + n_empty] == 0).all()
    for i in list(range(G)) + list(range(len(seq) - G, len(seq))):
        c = seq[i]
        got = out[int(out_off[i]):int(out_off[i] + out_len[i])].tobytes()
        assert got == c.raw, "stream %d: first diff at %d" % (i, next((k for k in range(min(len(got), len(c.raw))) if got[k] != c.raw[k]), -1))


def test_untagged_flag_after_wide_speed_stream(warp, oracle):
    """Header word 1, set by v2_make_untagged: a stream that switches to wide speeds mid-stream leaves untagged 16-bit
    priors; the next v2 stream in the slot must wipe the tables before it trusts tags."""
    h = _in_every_slot(warp, oracle, [R.build("wide_midstream", oracle)], "wide")
    assert [x[1] for x in h] == [1] * warp.groups
    h = _in_every_slot(warp, oracle, [R.build("lsb6", oracle)], "after wide")
    assert [x[1] for x in h] == [0] * warp.groups
    _in_every_slot(warp, oracle, [R.build("wide_speeds", oracle), R.build("msb6", oracle), R.build("wide_midstream", oracle),
                                  R.build("lsb6", oracle, 1)], "one launch")


def test_untagged_flag_after_gpu_encode_with_wide_speeds(warp, oracle):
    """Header word 1, set by the encoder's model pass with wide speeds: the encoder shares the arena of its context, and the
    next v2 decode in the same slot must not read its 16-bit priors as tagged ones."""
    import divans_b200
    raws = [R.text()[i * 3000: i * 3000 + 2500] for i in range(4)]       # 4 streams: the encoder's block of slots
    wide = divans_b200.encode_options(literal_adaptation=[(16, 8192), (16, 8192), R.WIDE, R.WIDE])
    enc = warp.encode(raws, wide)
    for s, r in zip(enc, raws):
        rc, ref = oracle.decode(s, out_cap=len(r) + 64)
        assert rc == 0 and ref == r
    assert [h[1] for h in _headers(warp)] == [1] * warp.groups
    h = _in_every_slot(warp, oracle, [R.build("lsb6", oracle)], "after encode")
    assert [x[1] for x in h] == [0] * warp.groups


def test_untagged_flag_after_blend_decode(warp, oracle, oracle_blend):
    """Header word 1, set by reset_slot for a blend-model stream (its priors keep a step count in the sign bits): the next
    default-model v2 stream in the slot must wipe the tables."""
    import divans_b200
    raw = R.text()[5000:8000]
    bs = oracle_blend.encode_raw(raw)
    res = warp.decode([bs] * 4, [len(raw) + 64] * 4, divans_b200.FLAG_CDF_BLEND)   # 4 streams: the blend kernel's block of slots
    assert all(st == 0 and out == raw for st, out in res)
    assert [h[1] for h in _headers(warp)] == [1] * warp.groups
    h = _in_every_slot(warp, oracle, [R.build("lsb6", oracle), R.build("dcm2", oracle)], "after blend")
    assert [x[1] for x in h] == [0] * warp.groups


def _corrupt_map_stream(oracle):
    """bt256 with a bit flipped early in its command payload: the 16384-byte context map is only partly right and the stream
    fails before its first literal"""
    base = R.build("bt256", oracle).stream
    cmd = oracle.demux(base)[0]
    at = base.find(cmd[64:96])
    rng = np.random.default_rng(5)
    for _ in range(2000):
        b = bytearray(base)
        b[at + int(rng.integers(len(cmd) // 8, len(cmd) // 2))] ^= 1 << int(rng.integers(0, 8))
        rc, _, st = oracle.decode(bytes(b), out_cap=1 << 16, skip_crc=True, stats=True)
        if rc in (1, 3) and st["lit_nibbles"] == 0:
            return R.Case(bytes(b), None, R.SKIP_CRC, rc, 1 << 16)
    raise AssertionError("no corruption found")


def test_context_map_high_water_mark(warp, oracle):
    """Header word 2: reset_slot_v2 zeroes only as many literal-context-map bytes as earlier streams wrote.  After the
    256-block-type stream (a full 16384-byte map, no zero entry) the stream without a PredictionMode command must see a zero
    map; also after a corrupted 256-block-type stream that fails partway through."""
    bt, nopm = R.build("bt256", oracle), R.build("no_predmode", oracle)
    h = _in_every_slot(warp, oracle, [bt], "bt256")
    assert [x[2] for x in h] == [16384] * warp.groups
    h = _in_every_slot(warp, oracle, [nopm], "no predmode")
    assert [x[2] for x in h] == [0] * warp.groups
    _in_every_slot(warp, oracle, [bt, nopm, bt, R.build("no_predmode", oracle, 1)], "one launch")
    bad = _corrupt_map_stream(oracle)
    h = _in_every_slot(warp, oracle, [bad], "corrupt bt256")
    assert all(x[2] > 64 for x in h), h
    _in_every_slot(warp, oracle, [nopm], "after corrupt bt256")
    _in_every_slot(warp, oracle, [bad, nopm], "corrupt, one launch")


def test_stale_mixing_mask(warp, oracle):
    """Header word 3: the mixing mask is zeroed lazily (v2_mix_before_use) by a literal that arrives before any
    PredictionMode command.  After a stream with per-context mixing values, the stream without PredictionMode must read
    mixing value 0 everywhere."""
    mix, nopm = R.build("per_context_mix", oracle), R.build("no_predmode", oracle)
    h = _in_every_slot(warp, oracle, [mix], "mix")
    assert [x[3] for x in h] == [1] * warp.groups
    h = _in_every_slot(warp, oracle, [nopm], "no predmode")
    assert [x[3] for x in h] == [0] * warp.groups
    _in_every_slot(warp, oracle, [mix, nopm, R.build("dcm2", oracle), R.build("no_predmode", oracle, 1)], "one launch")


def test_context_mixing_priors_are_defaulted_per_stream(warp, oracle):
    """LIT_CM: the context-map priors of dynamic context mixing are defaulted once per stream behind bitmaps[64]; a second
    mixing stream with different text must not inherit the first one's."""
    _in_every_slot(warp, oracle, [R.build("dcm2", oracle, 0), R.build("dcm2", oracle, 1)], "one launch")
    _in_every_slot(warp, oracle, [R.build("dcm2", oracle, 2)], "next launch")


@pytest.mark.parametrize("failing", R.FAILING)
def test_good_stream_after_failure(warp, oracle, failing):
    """A stream that fails (payload runs dry: status 1, output region too small: 2, invalid command after literals: 3)
    leaves its slot in whatever state it reached; the next stream in the slot must decode exactly."""
    _in_every_slot(warp, oracle, [R.build(failing, oracle), R.build("lsb6", oracle), R.build(failing, oracle),
                                  R.build("dcm2", oracle)], failing)
