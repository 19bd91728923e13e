"""The CPU oracle's literal model selection (oracle_tally): the cost-only walk (dvo_tally_raw) and dvo_encode_auto."""
import lzma
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from divans_b200 import synth  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _text(n, seed=3):
    blob, off, ln = synth.text_streams(1, n, seed=seed)
    return blob.tobytes()


def _records(n, width, seed=5):
    """records of `width` bytes whose columns drift independently: byte i is predicted by byte i - width, not by byte i - 1"""
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return (np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n]).tobytes()


def _fixtures(oracle):
    rc, alice = oracle.decode(open(os.path.join(GOLDEN, "alice29_literal_only.divans"), "rb").read(), out_cap=1 << 20)
    assert rc == 0
    ir = lzma.decompress(open(os.path.join(GOLDEN, "asyoulik.ir.xz"), "rb").read())
    rc, ayl = oracle.Commands.from_ir(ir).recode(22)
    assert rc == 0
    return {"alice29": alice, "asyoulik": ayl, "text": _text(70000), "records4": _records(50000, 4)}


def test_cost_table(oracle):
    t = T.cost_table().astype(np.int64)
    f = np.arange(1, 32768)
    exact = 65536 * (15 - np.log2(f))
    assert t[0] == t[1] == 15 << 16
    d = t[1:] - exact
    assert (d >= 0).all() and (d < 1.001).all()      # log2 f with 16 fraction bits, truncated: the cost rounds up by under one unit
    assert (np.diff(t[1:]) <= 0).all()               # a likelier symbol never costs more


@pytest.mark.parametrize("window", [10, 22])
def test_one_candidate_is_encode_raw(oracle, window):
    data = _text(5000)
    for pm, mv in [(0, 4), (2, 7), (3, 5), (1, 1)]:
        rc, ref = T.encode_raw_model(data, pm, mv, window_size=window)
        assert rc == 0
        rc, got, chosen, costs = T.encode_auto(data, [(pm, mv)], window_size=window)
        assert rc == 0 and chosen == 0 and got == ref
        assert costs[0] == T.tally_raw(data, pm, mv, window_size=window)[1]
    # (0, 4) is the reference's internal compressor, literal commands of at most 2^window bytes included
    assert T.encode_raw_model(data, 0, 4, window_size=window)[1] == oracle.encode_raw(data, oracle.options(window_size=window))


def test_tally_bound(oracle):
    """0 <= payload bytes - cost / 8 <= 16 x rANS chunks (each 65536-symbol chunk of a coder starts with 16 bytes of state)"""
    for name, data in _fixtures(oracle).items():
        for pm, mv in [(0, 4), (2, 1), (2, 7)]:
            rc, stream = T.encode_raw_model(data, pm, mv)
            assert rc == 0
            cmd, lit = oracle.demux(stream)
            _, _, st = oracle.decode(stream, out_cap=len(data) + 64, stats=True)
            chunks = math.ceil(st["cmd_nibbles"] / 65536) + math.ceil(st["lit_nibbles"] / 65536)
            cost_bytes = T.tally_raw(data, pm, mv)[1] / 65536 / 8
            gap = len(cmd) + len(lit) - cost_bytes
            assert 0 <= gap <= 16 * chunks, (name, pm, mv, gap, chunks)


def test_selection(oracle):
    data = _records(20000, 4)
    rc, _, chosen, costs = T.encode_auto(data, [(0, 4), (2, 7), (2, 5)])
    assert rc == 0 and chosen == 1, costs         # (2, 7): the byte four back is the stride byte
    rc, _, chosen, _ = T.encode_auto(data, [(2, 5), (0, 4), (2, 7)])
    assert chosen == 2
    # ties go to the lowest index: the same model twice, and two models that cost the same under mixing value 4
    text = _text(3000)
    for cands in ([(0, 4), (0, 4)], [(1, 4), (0, 4)], [(0, 4), (1, 4)]):
        rc, got, chosen, costs = T.encode_auto(text, cands)
        assert costs[0] == costs[1] and chosen == 0
        assert got == T.encode_raw_model(text, *cands[0])[1]


def test_empty_and_tiny(oracle):
    for data in (b"", b"x", b"ab"):
        rc, got, chosen, costs = T.encode_auto(data, [(0, 4), (2, 1)])
        assert rc == 0 and got == T.encode_raw_model(data, *[(0, 4), (2, 1)][chosen])[1]
        assert oracle.decode(got)[1] == data
