"""CPU halves of the arithmetic domain tests (tests/test_gpu_arith.py holds the GPU halves).

* The in-kernel reference of the CDF division (tests/probe/numeric_ref.h, probability/numeric.rs restated in 64-bit
  integers), compiled for the host with g++, must equal the oracle's dvo_fast_divide on every (c, max) of i16 x i16: the GPU
  sweep of cdf_div is only as good as this reference.
* The fast-loop speed gate (dv_engine.cuh speed_is_small) claims that with the speeds it accepts no adaptive value can leave
  [0, 0x7fff], and DESIGN section 2 relies on a CDF step never falling below 3 under them (so a coded frequency is >= 2) and on
  the max never falling below 16 (recip32 / divq need 16 <= max).  Checked on the max recurrence of every accepted i16 pair,
  and on seeded symbol walks (the oracle's dvo_cdf_blend) under every accepted pair of f8 speeds."""
import os
import subprocess

import numpy as np
import pytest

import regimes

HERE = os.path.dirname(os.path.abspath(__file__))
PROBE = os.path.join(HERE, "probe")


@pytest.fixture(scope="module")
def arith_host(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("arith_host") / "arith_host")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-I", PROBE, "-o", exe,
                           os.path.join(PROBE, "arith_host.cpp"), "-ldl"])
    return exe


def test_numeric_reference_equals_oracle_fast_divide_on_the_i16_domain(arith_host, oracle):
    out = subprocess.run([arith_host, "divide", oracle._LIB_PATH], check=True, capture_output=True, text=True).stdout
    cases, bad = map(int, out.split()[-2:])
    print("numeric.rs restatement vs dvo_fast_divide: %d cases, %d mismatches" % (cases, bad))
    assert cases == 1 << 32
    assert bad == 0, out


def test_speed_gate_keeps_the_max_recurrence_inside_i16(arith_host):
    out = subprocess.run([arith_host, "gate"], check=True, capture_output=True, text=True).stdout
    accepted, lowest, highest = map(int, out.split())
    print("speed gate: %d accepted i16 (inc, lim) pairs, values in [%d, %d]" % (accepted, lowest, highest))
    # the accepted pairs: inc in 0..8175 (4 * (inc + 16) <= 0x7fff), lim in 0..0x7fff - 16 - inc
    assert accepted == sum(0x7FFF - 16 - inc + 1 for inc in range(0, 8176))
    assert 16 <= lowest and highest <= 0x7FFF     # max >= 16: what recip32 / divq need (dv2_core.cuh)


def f8_speeds(oracle):
    """every distinct speed value an f8 byte decodes to (probability/interface.rs:577-585)"""
    return sorted(set(int(oracle.lib().dvo_u8_to_speed(v)) for v in range(256)))


def walk_syms(rng, n, steps):
    """symbol runs: a walk keeps one of a few symbols for a while, so that single elements climb far"""
    hot = rng.integers(0, 16, (n, 3))
    pick = rng.integers(0, 3, (n, steps))
    noise = rng.integers(0, 16, (n, steps))
    return np.where(rng.random((n, steps)) < 0.8, np.take_along_axis(hot, pick, 1), noise).astype(np.uint8)


def test_small_f8_speeds_keep_every_cdf_step_at_least_3(oracle):
    sp = f8_speeds(oracle)
    pairs = np.array([(a, b) for a in sp for b in sp if regimes.speed_is_small(a, b)], np.int16)
    rng = np.random.default_rng(20)
    # each walk runs long enough for its max to climb from the default to lim about four times (rescales), 256 to 8192 steps:
    # walks of one length are run together
    lens = np.clip(4 * (pairs[:, 1].astype(np.int64) + 64) // np.maximum(pairs[:, 0], 1) + 256, 256, 8192)
    lens = 1 << np.ceil(np.log2(lens)).astype(np.int64)
    states = 0
    for steps in np.unique(lens):
        group = pairs[lens == steps]
        per = max(1, (1 << 21) // int(steps))
        for k in range(0, len(group), per):
            chunk = group[k:k + per]
            tr = oracle.cdf_walks(chunk, walk_syms(rng, len(chunk), int(steps))).astype(np.int32)
            steps_ = np.diff(np.concatenate([np.zeros(tr.shape[:2] + (1,), np.int32), tr], axis=2), axis=2)
            assert tr.min() >= 0 and tr.max() <= 0x7FFF
            assert steps_.min() >= 3, "a CDF step below 3 under small speeds"
            assert tr[:, :, 15].min() >= 16, "a max below 16 under small speeds (recip32 needs 16 <= d)"
            states += tr.shape[0] * tr.shape[1]
    print("small f8 speed pairs: %d, walk states: %d" % (len(pairs), states))
    assert len(pairs) > 1000
