"""CPU checks of the regime builders (tests/regimes.py): each stream decodes on the oracle to its input or to its stated
status, and really is the regime its name says -- command kinds, PredictionMode commands, speeds, mixing values, literal
lengths and nibble counts -- so that the GPU tests built on them cannot quietly lose the case they were written to hit."""
import pytest

import regimes as R


def _describe(oracle, c):
    rc, out, cl = oracle.decode_cmds(c.stream, out_cap=c.cap, skip_crc=bool(c.flags))
    cmds, pms = R.commands(cl)
    _, _, st = oracle.decode(c.stream, out_cap=c.cap, skip_crc=bool(c.flags), stats=True)
    return rc, out, cmds, pms, st


def _kinds(cmds):
    return [c[0] for c in cmds]


def _lits(cmds):
    return [c[2] for c in cmds if c[0] == R.LITERAL]


@pytest.mark.parametrize("name", R.ALL)
def test_regime_decodes_as_stated(oracle, name):
    c = R.build(name, oracle)
    rc, ref = oracle.decode(c.stream, out_cap=c.cap, skip_crc=bool(c.flags))
    assert rc == c.status
    if c.status == 0:
        assert ref == c.raw
    else:
        assert c.raw is None
    assert R.build(name, oracle, 1).stream != c.stream or name in ("empty", "out_cap_small")   # variants are different streams


@pytest.mark.parametrize("name,mode", [("lsb6", 0), ("msb6", 1), ("utf8", 2), ("sign", 3)])
def test_plain_literal_regimes(oracle, name, mode):
    rc, out, cmds, pms, st = _describe(oracle, R.build(name, oracle))
    assert _kinds(cmds) == [R.PREDMODE, R.LITERAL] and _lits(cmds) == [2048]
    assert len(pms) == 1 and pms[0]["mode"] == mode and set(pms[0]["mixing"]) == {4}
    assert all(R.speed_is_small(*s) for s in pms[0]["speeds"])
    assert pms[0]["lit_map"] == bytes(range(64))
    assert st["lit_nibbles"] == 4096


def test_mixing_regimes(oracle):
    for name, mv in (("dcm2", {4}), ("mix2_flat", {2})):
        rc, out, cmds, pms, st = _describe(oracle, R.build(name, oracle))
        assert _kinds(cmds) == [R.PREDMODE, R.LITERAL] and _lits(cmds) == [3000] and set(pms[0]["mixing"]) == mv
    rc, out, cmds, pms, st = _describe(oracle, R.build("per_context_mix", oracle))
    assert _kinds(cmds) == [R.PREDMODE, R.LITERAL] and len(set(pms[0]["mixing"])) == 9   # lit_cfg < 0: the generic path
    # dynamic context mixing is not in the decoded command list: it shows as a different stream for the same literals
    c = R.build("dcm2", oracle)
    assert c.stream != R._raw_mode(oracle, c.raw, 0, 4)


def test_wide_speed_regimes(oracle):
    rc, out, cmds, pms, st = _describe(oracle, R.build("wide_speeds", oracle))
    assert _kinds(cmds) == [R.PREDMODE, R.LITERAL]
    assert not all(R.speed_is_small(*s) for s in pms[0]["speeds"])
    rc, out, cmds, pms, st = _describe(oracle, R.build("wide_midstream", oracle))
    assert _kinds(cmds) == [R.PREDMODE, R.LITERAL, R.PREDMODE, R.LITERAL] and _lits(cmds) == [1500, 1500]
    assert all(R.speed_is_small(*s) for s in pms[0]["speeds"]) and not all(R.speed_is_small(*s) for s in pms[1]["speeds"])


def test_short_literal_regime(oracle):
    rc, out, cmds, pms, st = _describe(oracle, R.build("short_literals", oracle))
    lits = _lits(cmds)
    assert len(lits) == 150 and max(lits) == 11 and min(lits) == 1
    assert _kinds(cmds).count(R.COPY) == 50 and len(pms) == 1 and pms[0]["mode"] == 1


def test_lit_quirk_regime(oracle):
    c = R.build("lit_quirk_w10", oracle)
    assert c.stream[5] == 10                            # window 10 in the header: a 1024-byte ring
    rc, out, cmds, pms, st = _describe(oracle, c)
    starts = [p for p, n in R.literal_starts(cmds)]
    assert starts == [0, 1027, 2055, 3073] and all((p & 1023) < 8 for p in starts)
    assert all(n >= 12 for n in _lits(cmds))


def test_chunk_restart_regime(oracle):
    rc, out, cmds, pms, st = _describe(oracle, R.build("chunk_restart", oracle))
    assert _kinds(cmds) == [R.PREDMODE, R.LITERAL] and st["lit_nibbles"] == 80000 > 65536


def test_switch_regimes(oracle):
    rc, out, cmds, pms, st = _describe(oracle, R.build("switches", oracle))
    assert [p["mode"] for p in pms] == [0, 2, 0]
    assert _kinds(cmds).count(R.BTYPE_L) == 4 and len(_lits(cmds)) == 7
    assert all(len(p["lit_map"]) == 192 for p in pms)
    rc, out, cmds, pms, st = _describe(oracle, R.build("bt256", oracle))
    assert len(pms) == 1 and len(pms[0]["lit_map"]) == 16384 and 0 not in pms[0]["lit_map"]
    assert [c[1] for c in cmds if c[0] == R.BTYPE_L] == [255, 17, 128, 254, 3]


def test_no_predmode_and_empty_regimes(oracle):
    rc, out, cmds, pms, st = _describe(oracle, R.build("no_predmode", oracle))
    assert pms == [] and _kinds(cmds) == [R.LITERAL, R.COPY, R.LITERAL]
    rc, out, cmds, pms, st = _describe(oracle, R.build("empty", oracle))
    assert cmds == [] and out == b"" and st["lit_nibbles"] == 0


def test_failing_regimes(oracle):
    for name, want in (("corrupt_status1", 1), ("corrupt_status3", 3), ("out_cap_small", 2)):
        c = R.build(name, oracle)
        rc, out, cmds, pms, st = _describe(oracle, c)
        assert rc == c.status == want
        if want != 2:                                   # the failure comes after the decoder went through literal bytes
            assert c.flags == R.SKIP_CRC and st["lit_nibbles"] > 1000
