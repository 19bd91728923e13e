"""The CPU oracle's literal model selection for command lists (oracle_tally): dvo_cmdlist_set_model and dvo_encode_cmds_auto."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from divans_b200 import synth  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _text(n, seed=3):
    blob, off, ln = synth.text_streams(1, n, seed=seed)
    return blob.tobytes()


def _records(n, width, seed=5):
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return (np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n]).tobytes()


def test_set_model(oracle):
    """the replacing record is the raw-mode record: an LZ77 list generated with one model and set to another is the list
    generated with the other; KEEP changes nothing; out-of-range models are refused"""
    text = _text(20000)
    c = oracle.Commands.lz77(text, window=16, pred_mode=2, mixing_value=4)
    before = c.serialize()
    assert T.cmdlist_set_model(c, *T.KEEP) == T.SUCCESS and c.serialize() == before
    for bad in ((4, 4), (0, 16), (-1, 4), (0, -1)):
        assert T.cmdlist_set_model(c, *bad) == T.FAILURE and c.serialize() == before
    assert T.cmdlist_set_model(c, 0, 5) == T.SUCCESS
    assert c.serialize() == oracle.Commands.lz77(text, window=16, pred_mode=0, mixing_value=5).serialize()


def _with_model(oracle, ir, pm, mv):
    c = oracle.Commands.from_ir(ir)
    assert T.cmdlist_set_model(c, pm, mv) == T.SUCCESS
    return c


def test_one_candidate_is_the_rewritten_list(oracle):
    """every PredictionMode record is replaced, whatever the list's own records hold (three records of another mode, with
    speeds and full maps); the list passed in is not modified"""
    import regimes as R
    pm = R.pm_line("msb6", lmap=[(i * 37) % 256 for i in range(256)], mix=[(i * 7) % 9 for i in range(8192)])
    ir = "window 16 0 0 0\n" + "\n".join([pm, "insert 600 " + _text(600).hex(), pm, "insert 300 " + _text(300, 4).hex(), pm,
                                         "copy 200 from 600 ctx 0"]) + "\n"
    c = oracle.Commands.from_ir(ir)
    before = c.serialize()
    for cand in [(0, 4), (2, 7), (3, 5), (1, 1), T.KEEP]:
        rc, got, chosen, costs = T.encode_cmds_auto(c, [cand], window_size=16)
        want = _with_model(oracle, ir, *cand).encode(oracle.options(window_size=16))
        assert rc == 0 and chosen == 0 and got == want, cand
        assert oracle.decode(got)[1] == oracle.decode(c.encode(oracle.options(window_size=16)))[1]
    assert c.serialize() == before


def test_selection_and_ties(oracle):
    """4-byte records: the stride model (2, 7) beats the generator's own (2, 4); KEEP and a candidate equal to the list's own
    records cost the same, and the lower index wins"""
    c = oracle.Commands.lz77(_records(20000, 4), window=16, pred_mode=2, mixing_value=4)
    rc, got, chosen, costs = T.encode_cmds_auto(c, [T.KEEP, (0, 4), (2, 7)], window_size=16)
    assert rc == 0 and chosen == 2 and costs[2] < costs[0] / 1.5, costs
    assert got == _lz_with(oracle, _records(20000, 4), 2, 7)
    for cands in ([T.KEEP, (2, 4)], [(2, 4), T.KEEP]):
        rc, got, chosen, costs = T.encode_cmds_auto(c, cands, window_size=16)
        assert costs[0] == costs[1] and chosen == 0
        assert got == c.encode(oracle.options(window_size=16))


def _lz_with(oracle, data, pm, mv):
    return oracle.Commands.lz77(data, window=16, pred_mode=pm, mixing_value=mv).encode(oracle.options(window_size=16))


def test_literal_only_list_is_encode_auto(oracle):
    """a stream stored by the raw encoder, decoded to its list and re-coded under the candidates, is encode_auto of its input:
    the list is the raw encoder's own (one PredictionMode command, literal commands of 2^window bytes)"""
    cands = [(0, 4), (2, 8), (2, 5), (2, 1), (2, 7), (3, 5)]
    for data, w in ((_text(30000), 16), (_records(5000, 4), 10), (b"", 16)):
        stream = oracle.encode_raw(data, oracle.options(window_size=w))
        rc, raw, cl = oracle.decode_cmds(stream)
        assert rc == 0 and raw == data
        a = T.encode_cmds_auto(cl, cands, window_size=w)
        b = T.encode_auto(data, cands, window_size=w)
        assert a[0] == b[0] == 0 and a[2] == b[2] and (a[3] == b[3]).all() and a[1] == b[1]

