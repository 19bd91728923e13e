"""The CPU oracle's literal speeds (oracle_tally): the halves the rule relies on, and dvo_encode_speeds / dvo_encode_cmds_speeds."""
import itertools
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from divans_b200 import synth  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_encode_mixmap_oracle as MX  # noqa: E402

VALUES = [(16, 8192), (32, 4096), (64, 16384), (128, 16384), (512, 16384), (1664, 16384)]
MUD = (16, 8192)
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="module")
def texts(oracle):
    """8 KiB of alice29 (from the golden stream) and of the bench corpus's synthetic text"""
    rc, raw = oracle.decode(open(os.path.join(GOLDEN, "alice29_literal_only.divans"), "rb").read(), out_cap=1 << 20)[:2]
    assert rc == 0
    blob, off, ln = synth.text_streams(1, 8192, seed=3)
    return [raw[:8192], blob.tobytes()]


def _halves(d, sp, mode=2, **kw):
    rc, cost, bins, nobin = T.tally_raw_bins(d, mode, 4, literal_adaptation=sp, **kw)
    b = bins.astype(np.uint64)
    return rc, cost, int(b[4096:].sum()), int(b[:4096].sum()), nobin


@pytest.mark.parametrize("dcm", [0, 1, 2])
def test_halves_sum_to_tally(texts, dcm):
    for d in texts:
        rc, cost, lo, hi, nobin = _halves(d, [(64, 16384), MUD, (32, 4096), (512, 16384)], dynamic_context_mixing=dcm)
        assert rc == 0 and lo + hi + nobin == cost == T.tally_raw(d, 2, 4, dynamic_context_mixing=dcm,
                                                                   literal_adaptation=[(64, 16384), MUD, (32, 4096), (512, 16384)])[1]


@pytest.mark.parametrize("name", sorted(MX._corpora()))
def test_separability(texts, name):
    """on the per-context mixing tests' corpora and the fixture text: at dcm 2 the low nibbles' cost does not move with S3, nor
    the high nibbles' with S2; at dcm 0/1 the literals ignore S2 and S3"""
    s0 = (64, 16384)
    for d in [MX._corpora()[name]] + (texts if name == "text" else []):
        for mode in (0, 2):
            base = _halves(d, [s0, s0, MUD, MUD], mode, dynamic_context_mixing=2, window_size=10)
            for s in VALUES[1:]:
                assert _halves(d, [s0, s0, MUD, s], mode, dynamic_context_mixing=2, window_size=10)[2] == base[2]
                assert _halves(d, [s0, s0, s, MUD], mode, dynamic_context_mixing=2, window_size=10)[3] == base[3]
            for dcm in (0, 1):
                b = _halves(d, [s0, s0, MUD, MUD], mode, dynamic_context_mixing=dcm, window_size=10)
                for s in VALUES[1:]:
                    h = _halves(d, [s0, s0, s, s], mode, dynamic_context_mixing=dcm, window_size=10)
                    assert (h[2], h[3]) == (b[2], b[3])


def test_tuned_pair_is_exhaustive_minimum(texts):
    """k <= 4: the tuned (l*, h*) minimises the literal cost over all k^2 (S2, S3) pairs for the chosen S0"""
    vals = VALUES[:4]
    for d in texts:
        rc, out, ch, cost, halves = T.encode_speeds(d, 2, 4, vals, dynamic_context_mixing=2)
        s0 = vals[ch[0]]
        lits = {}
        for a, b in itertools.product(range(4), repeat=2):
            r = _halves(d, [s0, s0, vals[a], vals[b]], dynamic_context_mixing=2)
            lits[(a, b)] = r[2] + r[3]
        l_star, h_star = int(np.argmin(halves[:, 0])), int(np.argmin(halves[:, 1]))
        assert lits[(l_star, h_star)] == min(lits.values())


@pytest.mark.parametrize("dcm", [1, 2])
def test_mud_alone_is_the_plain_encoder(texts, dcm):
    for d in texts:
        rc, out, ch, cost, halves = T.encode_speeds(d, 2, 4, [MUD], dynamic_context_mixing=dcm)
        assert rc == 0 and list(ch) == [0, 0, 0]
        assert out == T.encode_raw_model(d, 2, 4, dynamic_context_mixing=dcm)[1]


@pytest.mark.parametrize("dcm,mode", [(1, 2), (2, 2), (2, 0)])
def test_streams_decode_and_never_cost_more(oracle, texts, dcm, mode):
    for d in texts + [b"", b"x", bytes(range(256)) * 9]:
        rc, out, ch, cost, halves = T.encode_speeds(d, mode, 4, VALUES, dynamic_context_mixing=dcm)
        assert rc == 0 and oracle.decode(out, out_cap=len(d) + 64)[1] == d
        k = len(VALUES)
        want = T.tally_raw(d, mode, 4, dynamic_context_mixing=dcm,
                           literal_adaptation=[VALUES[ch[0]], VALUES[ch[0]], VALUES[ch[1]], VALUES[ch[2]]])[1]
        assert want == min(cost[k], min(cost[:k])) <= min(cost[:k])   # the verify pass is taken only when it is cheaper


def test_real_text_gains(texts):
    rc, out, ch, cost, halves = T.encode_speeds(texts[0], 2, 4, VALUES, dynamic_context_mixing=2)
    assert min(cost) < cost[0]


def test_out_of_domain_values_are_refused():
    # (16384, 16384) survives the f8 round trip but could wrap an i16 prior
    assert T._u8_to_speed(T._speed_to_u8(16384)) == 16384 and not T.speed_ok(16384, 16384)
    for vals in ([], [(1000, 16384)], [(-1, 1024)], [(16, 32767)], [(16384, 16384)], [MUD] * 17):
        with pytest.raises(ValueError):
            T.encode_speeds(b"abc", 2, 4, vals if vals else np.zeros((0, 2), np.int16))
    assert all(T.speed_ok(*v) for v in VALUES)
