"""CPU checks of the regime builders (tests/regimes.py): each stream decodes on the oracle to its input or to its stated
status, and really is the regime its name says -- command kinds, PredictionMode commands, speeds, mixing values, literal
lengths and nibble counts -- so that the GPU tests built on them cannot quietly lose the case they were written to hit."""
import numpy as np
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


# ---- the command lists behind the regimes, the framing edges and the re-muxer ----
@pytest.mark.parametrize("name", R.GOOD)
def test_regime_command_list_reencodes_to_its_stream(oracle, name):
    """The GPU encoder tests send command_list(name) under encode_options(name); the oracle must turn that pair back into
    exactly build(name).stream, so the encoder and decoder tests cannot drift apart."""
    cl = R.command_list(name, oracle)
    assert cl.encode(oracle.options(**R.encode_options(name))) == R.build(name, oracle).stream


def _edge_property(oracle, name):
    _cl, raw, stream = R.edge(name, oracle)
    rc, out, st = oracle.decode(stream, out_cap=len(raw) + 64, stats=True)
    assert rc == 0 and out == raw
    cmd, lit = oracle.demux(stream)
    return dict(cmd_payload=len(cmd), lit_payload=len(lit), cmd_nibbles=st["cmd_nibbles"], lit_nibbles=st["lit_nibbles"])


@pytest.mark.parametrize("name", R.EDGE_NAMES)
def test_framing_edge_has_its_property(oracle, name):
    prop, want = R.EDGES[name][3]
    got = _edge_property(oracle, name)
    if prop == "both_over":
        assert got["cmd_payload"] > want and got["lit_payload"] > want, got
    else:
        assert got[prop] == want, got
    cl, raw, stream = R.edge(name, oracle)
    assert cl.encode(oracle.options(**R.edge_options(name))) == stream


def test_framing_edges_cover_the_mux_codes(oracle):
    """the mux writes a one-byte record code for a 4096- or 16384-byte payload, and 65536-byte records before a tail; the
    edges put each payload exactly on these sizes (and the command coder's final chunk at 1 symbol)"""
    lit = sorted(R.EDGES[n][3][1] for n in R.EDGE_NAMES if R.EDGES[n][3][0] == "lit_payload")
    cmd = sorted(R.EDGES[n][3][1] for n in R.EDGE_NAMES if R.EDGES[n][3][0] == "cmd_payload")
    nib = sorted(R.EDGES[n][3][1] for n in R.EDGE_NAMES if R.EDGES[n][3][0] == "cmd_nibbles")
    assert lit == [4096, 16384, 65536, 65536 + 4096, 65536 + 16384, 131072]
    assert cmd == [4096, 16384] and nib == [65535, 65536, 65537]
    stream = R.edge("lit16384", oracle)[2]
    at = stream.find(oracle.demux(stream)[1][:64])
    assert stream[at - 1] == 0x21   # literal coder, code k = 2: one header byte


def test_regimes_under_the_blend_model(oracle_blend):
    """tests/test_gpu_blend_regimes.py builds every regime with the blend oracle: each decodes to its input or its stated
    status there too, and each good regime's command list re-encodes to its stream"""
    for name in R.ALL:
        c = R.build(name, oracle_blend)
        rc, out = oracle_blend.decode(c.stream, out_cap=c.cap, skip_crc=bool(c.flags))
        assert rc == c.status and (c.status != 0 or out == c.raw), name
    for name in R.GOOD:
        cl = R.command_list(name, oracle_blend)
        assert cl.encode(oracle_blend.options(**R.encode_options(name))) == R.build(name, oracle_blend).stream, name
    assert [R.build(n, oracle_blend).status for n in R.FAILING] == [1, 3, 2]


@pytest.mark.parametrize("name", R.EDGE_NAMES)
def test_blend_framing_edge_has_its_property(oracle_blend, name):
    """BLEND_EDGES: the properties of EDGES under the blend model, whose payloads are longer for the same input"""
    assert list(R.edges(oracle_blend)) == R.EDGE_NAMES and R.edges(oracle_blend)[name][3] == R.EDGES[name][3]
    src, off, n, prop = R.BLEND_EDGES[name]
    cl, raw, stream = R.edge(name, oracle_blend)
    got = R.edge_measure(oracle_blend, src, off, n)
    assert R.edge_has_property(got, prop), got
    assert cl.encode(oracle_blend.options(**R.edge_options(name, oracle_blend))) == stream
    rc, out = oracle_blend.decode(stream, out_cap=len(raw) + 64)
    assert rc == 0 and out == raw


def test_blend_edges_reach_the_mux_codes_of_the_default_edges(oracle, oracle_blend):
    """each blend edge has the record chain of its default twin: the same one-byte codes of the same coders, the same
    three-byte records, in the same order (the sizes of the three-byte records differ)"""
    shape = lambda stream: [(c, k) if k is not None else (c, None) for c, _n, k in R.record_chain(stream)]
    for name in R.EDGE_NAMES:
        d, b = R.edge(name, oracle)[2], R.edge(name, oracle_blend)[2]
        assert R.mux_records(oracle, d, R.record_chain(d)) == d and R.mux_records(oracle_blend, b, R.record_chain(b)) == b
        assert shape(b) == shape(d), name
        assert {k for _c, _n, k in R.record_chain(b)} - {None} == {k for _c, _n, k in R.record_chain(d)} - {None}
    # the blend model moves the payload edges: the default parameters miss the property under it
    for name in ("lit4096", "cmd4096"):
        src, off, n, prop = R.EDGES[name]
        assert not R.edge_has_property(R.edge_measure(oracle_blend, src, off, n), prop)


@pytest.mark.parametrize("lay", R.LAYOUTS)
def test_remuxed_stream_decodes_on_the_oracle(oracle, lay):
    """a new record chain over the same payloads decodes to the same bytes; each layout has the shape it is named for"""
    for name in ("lit16384", "cmd4096", "both_over"):
        _cl, raw, stream = R.edge(name, oracle)
        lens = tuple(len(p) for p in oracle.demux(stream))
        plan = R.layout(lay, lens, seed=3)
        s2 = R.mux_records(oracle, stream, plan)
        assert s2 != stream or lay == "codes"      # (codes on a 16384-byte payload: the mux's own layout)
        rc, out = oracle.decode(s2, out_cap=len(raw) + 64)
        assert rc == 0 and out == raw, (name, lay)
        assert oracle.demux(s2) == oracle.demux(stream)
        if lay == "one_byte":
            assert all(n == 1 for _c, n, _k in plan)
        if lay == "lit_first":
            assert [c for c, _n, _k in plan] == sorted((c for c, _n, _k in plan), reverse=True)
        if lay == "align16":
            assert {o % 16 for o in R.record_starts(plan)} == set(range(16))
        if lay == "codes" and name == "both_over":
            assert {k for _c, _n, k in plan} == {1, 2, 3, None}
        if lay == "random" and name == "both_over":
            assert len({n for _c, n, _k in plan}) > 10 and len({c for c, _n, _k in plan[:20]}) == 2


@pytest.mark.parametrize("variant", sorted(R.C_OVER_MAX_OPTIONS))
def test_c_over_max_regime_codes_an_element_above_the_max(oracle, variant):
    """the oracle encoder accepts the list (every coded frequency > 0), the stream decodes on the oracle, every high nibble
    takes one prior, and the last one is coded at an element above that prior's max with a quotient >= 2^24"""
    cl, stream = R.c_over_max(oracle, variant)
    cmds, pms = R.commands(cl)
    assert [c[0] for c in cmds] == [R.PREDMODE, R.LITERAL] and pms[0]["lit_map"] == bytes(64)
    assert set(pms[0]["mixing"]) == {0}
    rc, out = oracle.decode(stream, out_cap=len(R.C_OVER_MAX_BYTES) + 64)
    assert rc == 0 and len(out) == len(R.C_OVER_MAX_BYTES)
    walk = R.c_over_max_walk(oracle)
    over = [(k, int(h)) for k, h in enumerate(np.frombuffer(R.C_OVER_MAX_BYTES, np.uint8) >> 4)
            if 0 < walk[k, 15] < walk[k, h] <= 0x7FFF]
    assert over, "no high nibble is coded at an element above the max"
    k, h = over[-1]
    assert k == len(R.C_OVER_MAX_BYTES) - 1
    assert (int(walk[k, h]) << 15) // int(walk[k, 15]) >= 1 << 24
