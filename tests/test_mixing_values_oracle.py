"""CPU checks that each stream of tests/mixing_values.py is what its name says: it round-trips through the oracle, its records
carry the masks that were built, and (tallied under the list's own records) its literals are coded under the values it is
meant to exercise.  Also the oracle hook that writes those masks, dvo_cmdlist_set_mixing."""
import numpy as np
import pytest

import mixing_values as V
import mixval_regimes as M
import regimes as R
from oracle_tally import tally_py as T


def _decoded_masks(oracle, name, case):
    rc, out, cl = oracle.decode_cmds(case.stream, out_cap=case.cap, model_rev=V.encode_options(name).get("model_rev", 0))
    assert rc == 0 and out == case.raw
    return V.masks_of(cl.serialize()), cl


@pytest.mark.parametrize("dcm", V.DCMS)
@pytest.mark.parametrize("name", V.ALL)
def test_round_trip_and_masks(oracle, name, dcm):
    case = V.build(name, oracle, dcm)
    cl, masks, raw = V.command_list(name, oracle)
    assert case.raw == raw
    got, dec = _decoded_masks(oracle, name, case)
    assert (got == np.stack(masks)).all(), name
    assert dec.encode(oracle.options(**V.encode_options(name, dcm))) == case.stream   # the decoded list codes the same stream


@pytest.mark.parametrize("dcm", V.DCMS)
@pytest.mark.parametrize("name", V.BLEND_TWINS)
def test_blend_twins_round_trip(oracle_blend, name, dcm):
    case = V.build(name, oracle_blend, dcm)
    got, _ = _decoded_masks(oracle_blend, name, case)
    assert (got == np.stack(V.command_list(name, oracle_blend)[1])).all()


def _visited(oracle, name, blend=False):
    cl, masks, _ = V.command_list(name, oracle)
    rc, cost, bins, nobin = T.tally_cmds_bins(cl, *T.KEEP, blend=blend, **V.encode_options(name))
    assert rc == 0 and int(bins.sum()) + nobin == cost
    return masks, bins > 0


@pytest.mark.parametrize("name", V.ALL16 + V.HALF_NAMES)
def test_every_value_codes_literals_in_both_halves(oracle, name):
    masks, vis = _visited(oracle, name)
    want = list(range(16)) if name.startswith("all16_") else [int(x) for x in name.split("_")[1:]]
    for half, what in ((V.HIGH, "high"), (V.LOW, "low")):
        seen = set(masks[0][half][vis[half]].tolist())
        assert seen == (set(want) if name.startswith("all16_") else {want[0] if half == V.HIGH else want[1]}), (name, what, seen)
    if name.startswith("all16_"):
        assert vis[V.HIGH].reshape(16, 256)[:, 64:].any() and vis[V.LOW].reshape(16, 256)[:, 64:].any(), "no context above 63"


def test_one_entry(oracle):
    masks, vis = _visited(oracle, "one_entry")
    odd = np.flatnonzero(masks[0] != 4)
    assert odd.tolist() == [V.one_entry_index(oracle)] and vis[odd[0]] and odd[0] < 4096
    masks, vis = _visited(oracle, "one_entry_unvisited")
    odd = np.flatnonzero(masks[0] != 4)
    assert odd.tolist() == [V.UNVISITED] and not vis[odd[0]]


def test_switch(oracle):
    """four records -- uniform 12, all16, uniform 4, a mask rich in 2 and 3 -- each followed by literals of 1..11 and of 12 or
    more bytes"""
    cl, masks, _ = V.command_list("switch", oracle)
    assert [len(set(m.tolist())) for m in masks] == [1, 16, 1, 3] and masks[0][0] == 12 and masks[2][0] == 4
    cmds, _ = R.commands(cl)
    lens = [b for ty, a, b, c, d in cmds if ty == R.LITERAL]
    assert min(lens) == 1 and any(1 < n < 12 for n in lens) and any(n >= 12 for n in lens)


@pytest.mark.parametrize("name", V.UNIFORM_NAMES)
def test_uniform_masks_code_through_their_own_prior(oracle, name):
    """every value from entry 256 on is coded with the prior of the value 256 entries back (mixval_prior): slot v.  The
    literal cost differs from the same input under value 4 (values 9..15 are configurations of their own)"""
    v = int(name.split("_")[1])
    masks, vis = _visited(oracle, name)
    assert (masks[0] == v).all() and vis.any()
    cl, _, _ = V.command_list(name, oracle)
    assert T.tally_cmds_bins(cl, *T.KEEP, window_size=16)[1] != T.tally_cmds_bins(cl, int(R.commands(cl)[1][0]["mode"]), 4,
                                                                                   window_size=16)[1]


@pytest.mark.parametrize("at", M.CHUNK_AT)
def test_chunk_at_keeps_its_position(oracle, at):
    """the last record's values rewritten: command symbol 65535 still falls at mixing value `at`"""
    mine = oracle.decode(V.build("chunk_at_%d" % at, oracle).stream, out_cap=1 << 20, stats=True)[2]["cmd_nibbles"]
    base = oracle.decode(M.chunk_at(oracle, at).stream, out_cap=1 << 20, stats=True)[2]["cmd_nibbles"]
    assert mine == base
    assert (V.command_list("chunk_at_%d" % at, oracle)[1][-1] > 8).any()


def test_set_mixing_refuses_values_above_15(oracle):
    cl, masks, _ = V.command_list("uniform_9_lsb6", oracle)
    before = cl.serialize()
    for e, bad in ((0, 16), (4095, 17), (4096, 31), (8191, 255)):
        m = masks[0].copy()
        m[e] = bad
        assert T.cmdlist_set_mixing(cl, 0, m) == T.FAILURE
        assert cl.serialize() == before
    assert T.cmdlist_set_mixing(cl, 1, masks[0]) == T.FAILURE      # no record 1
    assert T.cmdlist_set_mixing(cl, 0, np.full(8192, 15, np.uint8)) == T.SUCCESS
    assert (V.masks_of(cl.serialize()) == 15).all()
