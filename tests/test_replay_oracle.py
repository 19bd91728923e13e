"""The CPU reference of the GPU replay (oracle_tally: dvo_recode_blob): a serialised command list replays to what the oracle's
own recode gives, every refusal rule of divans_b200_replay_cmds_batch_* holds on a hand-built blob, and a blob whose pool
would reach past its end is refused before its pool is read.  No GPU."""
import lzma
import os

import numpy as np
import pytest

from divans_b200 import synth

import dvcl
from dvcl import COPY, DICT, LIT, PREDMODE, BT_L, blob
from irfuzz import random_ir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def T():
    from oracle_tally import tally_py
    tally_py.build()
    return tally_py


def _ir_fixtures(oracle):
    c1 = oracle.Commands.from_ir(open(os.path.join(GOLD, "ends_with_truncated_dictionary.ir"), "rb").read())
    c2 = oracle.Commands.from_ir(lzma.decompress(open(os.path.join(GOLD, "asyoulik.ir.xz"), "rb").read()))
    return [c1, c2]


def test_ir_fixtures_equal_recode(oracle, T):
    for c in _ir_fixtures(oracle):
        w = c.window or 22
        rc, ref = c.recode(w)
        assert rc == 0 and len(ref) > 0
        # the header window of these lists is 0 (clamped to 10 by window 0), so the window is passed, as recode takes it
        assert T.recode_blob(c.serialize(), w) == (0, len(ref), ref)


@pytest.mark.parametrize("window", [10, 14, 16, 22, 24])
def test_random_ir_equals_recode(oracle, T, window):
    text = synth.text_corpus(1 << 16)
    for seed in range(6):
        c = oracle.Commands.from_ir(random_ir(oracle, 7000 + 31 * window + seed, n_cmds=150, window=window, text=text))
        rc, ref = c.recode(window)
        assert rc == 0
        b = c.serialize()
        assert T.recode_blob(b, window) == (0, len(ref), ref)
        assert T.recode_blob(b, 0) == (0, len(ref), ref)   # the IR's `window` line is the header window
        # status 2: the exact length, the first cap bytes
        for cap in (0, len(ref) // 2, len(ref) - 1):
            assert T.recode_blob(b, window, cap) == (2, len(ref), ref[:cap])


@pytest.mark.parametrize("case", dvcl.refusal_cases(), ids=lambda c: c[0])
def test_refusal_rules(T, case):
    name, b, window, out_len = case
    rc, n, got = T.recode_blob(b, window, cap=64)
    assert (rc, n) == (3, out_len), name
    assert got == b"abc"[:out_len]


def test_refusal_takes_precedence_over_output_size(T):
    b = blob([(LIT, 0, 8, 0, 0), (COPY, 0, 5, 0, 0)], b"abcdefgh")
    assert T.recode_blob(b, 0, cap=2) == (3, 8, b"ab")


def test_pool_past_the_blob_is_not_read(T):
    # the pool the header states reaches 4 bytes past the blob; the bytes that follow it in memory are not part of it
    lits = b"0123456789"
    b = blob([(LIT, 0, 12, 0, 0)], lits, n_lits=12)
    buf = np.full(len(b) + 64, 0xEE, np.uint8)
    buf[:len(b)] = np.frombuffer(b, np.uint8)
    rc, n, got = T.recode_blob(buf[:len(b)], 0, cap=64)
    assert (rc, n, got) == (3, 0, b"")
    # a literal record whose offset reaches past the pool the header states, inside a larger buffer
    b = blob([(LIT, 8, 4, 0, 0)], lits)
    buf = np.full(len(b) + 64, 0xEE, np.uint8)
    buf[:len(b)] = np.frombuffer(b, np.uint8)
    assert T.recode_blob(buf[:len(b)], 0, cap=64) == (3, 0, b"")


def test_commands_by_hand(T):
    lits = b"abcd"
    cases = [
        ([(LIT, 0, 4, 0, 0), (COPY, 1, 5, 0, 0)], b"abcdddddd"),                # distance 1: a run
        ([(LIT, 0, 4, 0, 0), (COPY, 3, 7, 0, 0)], b"abcdbcdbcdb"),              # overlapping period 3
        ([(COPY, 4, 3, 0, 0), (LIT, 0, 2, 0, 0)], b"\0\0\0ab"),                 # before position 0: zeros
        ([(LIT, 0, 2, 0, 0), (COPY, 5, 6, 0, 0)], b"ab\0\0\0ab\0"),            # partly before position 0
        ([(PREDMODE, 0, 0, 0, 0), (BT_L, 1, 2, 0, 0), (LIT, 1, 2, 0, 0)], b"bc"),
        ([(DICT, 0, 4, 0, 4)], None),                                             # d == length: accepted
        ([], b""),
    ]
    for cmds, want in cases:
        rc, n, got = T.recode_blob(blob(cmds, lits, window=10), 0)
        assert rc == 0
        if want is not None:
            assert got == want, cmds
        else:
            assert n == 4
