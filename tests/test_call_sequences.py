"""CPU checks of the call catalogue (tests/call_catalogue.py) behind tests/test_gpu_call_sequences.py: every kind's inputs
reach what its row claims, and its oracle result is what the kind is meant to show."""
import pytest

import call_catalogue as C
import regimes as R


@pytest.fixture(scope="module")
def cat(oracle, oracle_blend, golden):
    return C.catalogue(oracle, oracle_blend, golden)


def _pms(oracle, stream, cap):
    rc, _, cl = oracle.decode_cmds(stream, out_cap=cap, skip_crc=True)
    return rc, R.commands(cl)


def test_every_kind_has_an_oracle_result(cat):
    for name, k in cat.items():
        e = k.expect(2)
        assert len(e) == 2 * len(k.unit) and e[0] == e[1], name


def test_decode_unit_is_the_regimes_it_names(cat, oracle):
    """the failing regimes fail and the others decode; the unit starts with the stream without a PredictionMode command and
    ends with two raw-mode streams (64-entry literal map), so every slot ends in the same header state"""
    k = cat["dec"]
    for (name, _), c, (rc, out) in zip(C.DEC_UNIT, k.unit, k.unit_expect):
        assert rc == (c.status if name in R.FAILING else 0), name
        assert (rc != 0) == (name in R.FAILING), name
    rc, (cmds, pms) = _pms(oracle, k.unit[0].stream, k.unit[0].cap)
    assert rc == 0 and pms == [] and any(t == R.LITERAL for t, *_ in cmds)
    for c in k.unit[-2:]:
        rc, (_, pms) = _pms(oracle, c.stream, c.cap)
        assert rc == 0 and len(pms) == 1 and len(pms[0]["lit_map"]) == 64
    rc, (_, pms) = _pms(oracle, k.unit[1].stream, k.unit[1].cap)          # bt256: the high-water mark goes past 64 bytes
    assert max(len(p["lit_map"]) for p in pms) == 16384


def test_wide_speed_kinds_are_outside_speed_is_small(oracle):
    assert [R.speed_is_small(*s) for s in C.WIDE_OPTS["literal_adaptation"]] == [True, True, False, False]
    import irfuzz
    assert any(not R.speed_is_small(*s) for s in irfuzz.random_f8_speeds(oracle, 4))


def test_command_list_kinds(cat, oracle):
    """enc_cmds: a list whose literal map is 16384 bytes, one without a PredictionMode command, and one every encoder refuses;
    enc_nopm: lists without PredictionMode commands only"""
    from oracle_tally import tally_py as T
    lists = [T.from_blob(oracle, b) for b in cat["enc_cmds"].unit]
    maps = [max([len(p["lit_map"]) for p in R.commands(cl)[1]] or [0]) for cl in lists[:-1]]
    assert 16384 in maps and 0 in maps
    assert [s for s, _ in cat["enc_cmds"].unit_expect][-1] == 3
    assert all(R.commands(T.from_blob(oracle, b))[1] == [] for b in cat["enc_nopm"].unit)


def test_choose_and_replay_units(cat):
    """choose: stream 1 has a refused list and picks another, stream 3 has only refused lists and fails; replay: one refused
    list between good ones"""
    e = cat["choose_dev"].unit_expect
    assert e[1][0] == 0 and e[1][2] != 0 and e[1][3][0] == (1 << 64) - 1
    assert e[3][0] != 0 and e[0][0] == 0 and e[2][0] == 0
    assert [s for s, _ in cat["replay"].unit_expect] == [0, 0, 3, 0, 0]


def test_blend_unit_uses_mixing_0_and_2(cat, oracle_blend):
    for c, m in zip(cat["dec_blend"].unit, (0, 2)):
        rc, out = oracle_blend.decode(c.stream, out_cap=c.cap)
        assert rc == 0 and out == c.raw


def test_slots_used():
    """one-warp engines: the default decode uses its warp's slots, the encoder and the blend decoder whole blocks of four"""
    assert C.slots_used("v2", 2, 16, 24) == 2 and C.slots_used("v2", 4, 8, 48) == 4
    assert C.slots_used("rec", 4, 8, 16) == 4 and C.slots_used("rec", 2, 16, 8) == 2
    assert C.slots_used("enc", 2, 16, 1) == 4 and C.slots_used("blend", 2, 16, 4) == 4
    assert C.slots_used("v2", 8, 0, 2) == 2 and C.slots_used("enc", 8, 0, 8) == 8


def test_header_model_rejects_what_a_broken_build_leaves():
    """the model refuses the headers that the broken builds of DESIGN.md section 3 leave behind"""
    class K:
        gens, phases = 0, [("enc", 4, 1, C.RAW_HDR)]
    before = [[3, 0, 64, 1]] * 4
    C.check_headers(K, 1, before, [[3, 1, 64, 1]] * 4, 2, 16)
    for bad in ([[3, 0, 64, 1]] * 4, [[3, 1, 0, 1]] * 4, [[0, 1, 64, 1]] * 4):
        with pytest.raises(AssertionError):
            C.check_headers(K, 1, before, bad, 2, 16)

    class N:
        gens, phases = 0, [("enc", 2, "keep", C.NOPM_HDR)]
    with pytest.raises(AssertionError):
        C.check_headers(N, 2, before, [[3, 0, 0, 1]] * 4, 2, 16)
    C.check_headers(N, 2, before, [[3, 0, 0, 0]] * 4, 2, 16)
