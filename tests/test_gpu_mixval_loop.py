"""GPU tests (-m gpu) of the v2 decoder's converged loop over the mixing values of a PredictionMode command (dv2_core.cuh,
mixval_fast_v2), on both lane layouts.  Every byte and every status is compared with the CPU oracle.  One-warp engines (as in
tests/test_gpu_slot_state.py) decide which streams share a warp and which streams follow each other in a slot."""
import itertools
import json
import os

import pytest

import mixval_regimes as M
import regimes as R

pytestmark = pytest.mark.gpu

LANES = [16, 8]
ONE_WARP = {16: 2, 8: 4}           # slots of a one-warp engine


def _decode_check(eng, oracle, cases, what="", flags=0):
    for c in cases:
        flags |= c.flags
    res = eng.decode([c.stream for c in cases], [c.cap for c in cases], flags)
    for i, ((st, out), c) in enumerate(zip(res, cases)):
        rc, ref = oracle.decode(c.stream, out_cap=c.cap, skip_crc=bool(flags & R.SKIP_CRC))
        assert rc == c.status, (what, i)
        assert st == rc, "%s: stream %d: status %d, oracle %d" % (what, i, st, rc)
        if rc == 0:
            assert out == ref, "%s: stream %d: first diff at %d" % (
                what, i, next((k for k in range(min(len(out), len(ref))) if out[k] != ref[k]), min(len(out), len(ref))))


@pytest.fixture(scope="module")
def mix_cases(oracle):
    return ([M.random_mix(oracle, v) for v in range(4)] + [M.multi_pm(oracle, v) for v in range(2)] +
            [M.chunk_at(oracle, at) for at in M.CHUNK_AT] + [M.late_pm(oracle, v) for v in range(4)])


@pytest.mark.parametrize("lanes", LANES)
def test_mixing_values_match_the_oracle(oracle, mix_cases, lanes):
    """random per-value priors, several PredictionMode commands per stream, the chunk restart at mixing values 0, 1, 255,
    256, 8190 and 8191 (both parities of the run), warp-mates that reach the values at different nibbles; an odd batch
    leaves a group without work (a dummy in the loop)"""
    import divans_b200
    eng = divans_b200.Engine(0, 0, lanes)
    try:
        _decode_check(eng, oracle, mix_cases, "batch")
        _decode_check(eng, oracle, mix_cases[:-1][::-1], "odd batch, reversed")
        for at in M.CHUNK_AT:                                   # alone: the stream's own group and a dummy
            _decode_check(eng, oracle, [M.chunk_at(oracle, at)], "chunk at %d" % at)
        assert eng.last_lanes() == lanes
    finally:
        eng.close()


@pytest.mark.parametrize("lanes", LANES)
def test_warp_mates_in_other_regimes(oracle, lanes):
    """one warp: every stream of the loop next to every regime of tests/regimes.py, and next to each other at different
    offsets (16 lanes: pairs; 8 lanes: the pair twice), and odd batches of three"""
    import divans_b200
    g = ONE_WARP[lanes]
    mine = [M.random_mix(oracle, 0), M.multi_pm(oracle, 0), M.chunk_at(oracle, 256), M.late_pm(oracle, 2)]
    eng = divans_b200.Engine(0, g, lanes)
    try:
        for a, name in itertools.product(mine, R.ALL):
            b = R.build(name, oracle)
            _decode_check(eng, oracle, ([a, b] * (g // 2)), name)
            _decode_check(eng, oracle, [b, a, b], name + ", odd")
        for a, b in itertools.combinations(mine + [M.late_pm(oracle, 0)], 2):
            _decode_check(eng, oracle, [a, b] * (g // 2), "pair")
    finally:
        eng.close()


def _wasm_golden():
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    vec = open(os.path.join(d, "ref_wasm_example.divans"), "rb").read()
    return vec, json.load(open(os.path.join(d, "ref_wasm_example.json")))


@pytest.mark.parametrize("lanes", LANES)
def test_wasm_2018_mixing_values(oracle, lanes):
    """model revision WASM_2018 codes every mixing value with slot 16: the reference-held stream, an oracle-encoded stream
    with random values, and the same commands encoded by the GPU encoder"""
    import divans_b200
    vec, meta = _wasm_golden()
    cl, stream, raw = M.wasm_2018(oracle)
    eng = divans_b200.Engine(0, 0, lanes)
    try:
        gpu = eng.encode([cl.serialize()], divans_b200.encode_options(window_size=16, model_rev=divans_b200.MODEL_WASM_2018), cmds=True)[0]
        assert gpu == stream
        rc, want, _ = oracle.decode_cmds(vec, model_rev=oracle.MODEL_WASM_2018)
        assert rc == 0 and len(want) == meta["plain_len"]
        streams = [vec, stream, gpu, vec, stream]
        wants = [want, raw, raw, want, raw]
        res = eng.decode(streams, [len(w) + 64 for w in wants], divans_b200.FLAG_MODEL_WASM_2018)
        for i, ((st, out), w) in enumerate(zip(res, wants)):
            assert st == 0 and out == w, i
    finally:
        eng.close()


@pytest.mark.parametrize("lanes", LANES)
def test_corrupt_mixing_values_then_a_good_stream(oracle, lanes):
    """payloads truncated or bit-flipped inside the mixing values: the oracle's status, no hang; the next stream in the same
    slot decodes exactly"""
    import divans_b200
    g = ONE_WARP[lanes]
    bad = [M.truncated(oracle, f) for f in (0.1, 0.5, 0.9)] + [M.bitflip(oracle, s) for s in range(4)]
    good = [M.random_mix(oracle, 1), R.build("lsb6", oracle)]
    eng = divans_b200.Engine(0, g, lanes)
    try:
        for b in bad:
            _decode_check(eng, oracle, [b] * g + [good[0]] * g + [b] * g + [good[1]] * g, "slot succession")
            _decode_check(eng, oracle, [b, good[0]] * (g // 2) + [b], "warp-mates")
    finally:
        eng.close()


@pytest.mark.parametrize("lanes", LANES)
def test_mixing_mask_flag_set_by_the_loop(oracle, lanes):
    """Header word 3 (the mixing mask holds a stream's values): the loop writes value 0 of the mask and must set it, so that
    a later stream without a PredictionMode command zeroes the mask before its first literal"""
    import divans_b200
    g = ONE_WARP[lanes]
    mix, nopm = M.random_mix(oracle, 0), R.build("no_predmode", oracle)
    eng = divans_b200.Engine(0, g, lanes)
    try:
        _decode_check(eng, oracle, [mix] * g, "mix")
        assert [eng.slot_header(i)[3] for i in range(g)] == [1] * g
        _decode_check(eng, oracle, [nopm] * g, "no predmode")
        _decode_check(eng, oracle, [mix] * g + [nopm] * g, "one launch")
    finally:
        eng.close()
