"""CPU checks of the mixing-value stream builders (tests/mixval_regimes.py): each stream decodes on the oracle as stated and
has the property the GPU tests of the mixing-value loop rely on."""
import pytest

import mixval_regimes as M
import regimes as R


def _describe(oracle, c):
    rc, out, cl = oracle.decode_cmds(c.stream, out_cap=c.cap, skip_crc=bool(c.flags))
    cmds, pms = R.commands(cl)
    _, _, st = oracle.decode(c.stream, out_cap=c.cap, skip_crc=bool(c.flags), stats=True)
    return rc, out, cmds, pms, st


def test_random_mixing_values_switch_the_prior(oracle):
    mv = M.mixing_values(100)
    switches = sum((mv[i - 256] & 15) != (mv[i - 255] & 15) for i in range(256, 8191))
    assert switches > 7000 and mv[255] != mv[256] and mv[8190] != mv[8191]
    for v in range(2):
        rc, out, cmds, pms, st = _describe(oracle, M.random_mix(oracle, v))
        assert rc == 0 and [c[0] for c in cmds] == [R.PREDMODE, R.LITERAL]
        assert list(pms[0]["mixing"]) == M.mixing_values(100 + v)


def test_several_prediction_modes_with_literals_between(oracle):
    rc, out, cmds, pms, st = _describe(oracle, M.multi_pm(oracle))
    assert [c[0] for c in cmds] == [R.PREDMODE, R.LITERAL] * 3
    assert [p["mode"] for p in pms] == [0, 1, 2] and set(pms[1]["mixing"]) == {4} and len(set(pms[2]["mixing"])) == 9


def test_late_prediction_mode(oracle):
    for v in range(3):
        rc, out, cmds, pms, st = _describe(oracle, M.late_pm(oracle, v))
        assert [c[0] for c in cmds] == [R.LITERAL] * (v + 1) + [R.PREDMODE, R.LITERAL]


@pytest.mark.parametrize("at", M.CHUNK_AT)
def test_chunk_restart_falls_on_the_named_mixing_value(oracle, at):
    c = M.chunk_at(oracle, at)
    rc, out, cmds, pms, st = _describe(oracle, c)
    assert rc == 0 and cmds[-2][0] == R.PREDMODE and cmds[-1][0] == R.LITERAL and len(pms) >= 2
    tail = M.cmd_nibbles(oracle, [R.insert(c.raw[-900:])])
    before = st["cmd_nibbles"] - 1 - tail - 8192 - M._pm_head(oracle)      # symbols before the last PredictionMode command
    assert before + M._pm_head(oracle) + at == 65535


def test_corrupt_streams_fail_inside_the_mixing_values(oracle):
    for c in [M.truncated(oracle, f) for f in (0.1, 0.5, 0.9)] + [M.bitflip(oracle, s) for s in range(4)]:
        rc, out, cmds, pms, st = _describe(oracle, c)
        assert rc == c.status != 0 and st["lit_nibbles"] == 0


def test_wasm_2018_stream_needs_its_model_revision(oracle):
    cl, stream, raw = M.wasm_2018(oracle)
    rc, plain, _ = oracle.decode_cmds(stream, model_rev=oracle.MODEL_WASM_2018)
    assert rc == 0 and plain == raw
    assert stream != cl.encode(oracle.options(window_size=16))
