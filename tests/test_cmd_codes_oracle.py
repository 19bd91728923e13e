"""CPU tests of the command-code catalogue (tests/cmd_codes.py): every list round-trips on the oracle, every forged stream fails
or succeeds as the decoder's rules say, the copy-count shift rule of CountLastNib 14 / 15, and the records no stream can carry
are refused by the oracle's encoder."""
import numpy as np
import pytest

import cmd_codes as K
import dvcl as D
from oracle_tally import tally_py as T


def _window(blob):
    return int(np.frombuffer(blob[20:24], np.uint32)[0])


@pytest.mark.parametrize("name", list(K.BUILDERS))
def test_catalogue_round_trips(oracle, name):
    """the oracle encodes the list, decodes it back to the same records, and the bytes equal the replay of the list"""
    blob = K.blob_of(name)
    cl = T.from_blob(oracle, blob)
    w = _window(blob)
    rc, stream, _ = T.encode_forged(cl, window_size=w)
    assert rc == 0, name
    rc_r, n, replay = T.recode_blob(blob)
    assert rc_r == 0
    rc_d, out, dec = oracle.decode_cmds(stream, out_cap=n + 64)
    assert rc_d == 0 and out == replay
    assert T.recode_blob(dec.serialize()) == (0, n, replay)
    got = np.frombuffer(dec.serialize()[32:32 + 20 * dec.n_cmds], np.uint32).reshape(-1, 5)
    want = np.frombuffer(blob[32:32 + 20 * cl.n_cmds], np.uint32).reshape(-1, 5)
    assert got.shape == want.shape
    # canonical form: the decoded list holds each literal at its own pool offset, block switches carry no stride but L's,
    # and copies / switches leave c, d at 0
    assert (got[:, 0] == want[:, 0]).all()
    for t, cols in ((D.COPY, [1, 2]), (D.DICT, [1, 2, 3, 4]), (D.LIT, [2, 3]), (D.BT_L, [1, 2]), (D.BT_C, [1]), (D.BT_D, [1])):
        m = want[:, 0] == t
        assert (got[m][:, cols] == want[m][:, cols]).all(), (name, t)


def test_distances_reach_every_mnemonic():
    K.distances()   # asserts every code 0..15 is the one the encoder picks for some copy


def test_huge_count_is_status_2(oracle):
    blob = K.huge_count()
    rc, stream, _ = T.encode_forged(T.from_blob(oracle, blob), window_size=16)
    assert rc == 0 and stream == open(K.HUGE_COUNT_STREAM, "rb").read()   # the GPU tests' fixture
    st, out = oracle.decode(stream, out_cap=1 << 16)
    assert st == 2 and len(out) == 1 << 16
    assert T.recode_blob(blob, cap=1 << 16)[:2] == (2, 10 + (1 << 31) - 1)


def _count_of(stream, oracle):
    rc, _, dec = oracle.decode_cmds(stream, out_cap=1 << 20)
    recs = np.frombuffer(dec.serialize()[32:32 + 20 * dec.n_cmds], np.uint32).reshape(-1, 5)
    return rc, int(recs[2, 2]) if len(recs) > 2 and recs[2, 0] == D.COPY else None


def test_forged_streams(oracle):
    """every forged stream is CRC-valid and gets the status its entry states; a failure leaves the output of the commands
    before the forged one"""
    res = K.forged(T, oracle)
    assert len(res) == len(K.forged_cases())
    for name, _, st, data, want in res:
        assert st == want, "%s: status %d, stated %d" % (name, st, want)
    by = {name: (st, data) for name, _, st, data, _ in res}
    for v in [0] + list(range(8, 16)):
        assert len(by["cmd nibble %d" % v][1]) == 600
    for p in range(4, 16):
        assert by["pred_mode %d" % p] == (3, b"")


@pytest.mark.parametrize("last, mant, count", [
    (14, [0] * 8, 1), (14, [0] * 7 + [9], 9), (14, [0] * 6 + [1, 9], 0x19),
    (15, [0] * 9, 2), (15, [3] + [0] * 7 + [5], 7), (15, [0] * 8 + [9], 11), (15, [15] + [0] * 8, 15), (15, [0, 1] + [0] * 7, 2 | (1 << 28))])
def test_count_last_nibble_shifts_mod_32(oracle, last, mant, count):
    """CountLastNib 14 / 15 shift the leading bit by 32 / 33 and the first mantissa nibble by 28 / 32: every shift count is
    taken mod 32, as the reference's release build does -- so the leading bit is 1 << 0 / 1 << 1 and nibble 15's first
    mantissa lands in the low bits"""
    base = K._base()
    k0 = K.nibble_at(T, oracle, base, 2)
    forge = [(k0 + 3, last)] + [(k0 + 4 + i, m) for i, m in enumerate(mant)]
    rc, stream, _ = T.encode_forged(T.from_blob(oracle, base), forge, window_size=K.BASE_WINDOW)
    if count >= 1 << 20:   # too long for the output: status 2, the copy never lands
        assert oracle.decode(stream, out_cap=1 << 20)[0] == 2
        return
    assert _count_of(stream, oracle) == (0, count)


# ---------------------------------------------------------------------------------------------------------------------
# records no stream can carry
# ---------------------------------------------------------------------------------------------------------------------
def test_unrepresentable_records_are_refused_by_the_oracle(oracle):
    """status 0 decodes to the list's replay; a record no stream carries is refused (status 3) before any nibble of it"""
    for name, blob, carried in D.limit_cases() + D.long_literal_cases():
        cl = T.from_blob(oracle, blob)
        if cl is None:   # a literal outside the pool: refused by the blob loader
            assert not carried or "literal" in name
            continue
        rc, stream, _ = T.encode_forged(cl, window_size=16)
        if not carried:
            assert rc == 3, name
        if rc == 0:
            rc_r, n, replay = T.recode_blob(blob)
            assert rc_r == 0, name
            assert oracle.decode(stream, out_cap=n + 64) == (0, replay), name


# ---------------------------------------------------------------------------------------------------------------------
# coverage of the command coder's priors (oracle_tally.coverage: every code_and_blend(&s->cmd, ...) of the oracle's encoder)
# ---------------------------------------------------------------------------------------------------------------------
ALL = set(range(16))
# (table, prior type) -> (the nibbles an encoder can write into a status-0 stream, {nibble: why it is left out})
EXPECTED = {
    ("CC", "FullSelection"): (set(range(1, 8)) | {15}, {0: "no command has type 0", **{n: "types 8..14 are no command" for n in range(8, 15)}}),
    ("LL", "CountSmall"): (ALL, {}),
    ("LL", "SizeBegNib"): (ALL, {}),
    ("LL", "SizeLastNib"): (set(range(6)), {n: "literals of 2^(n + 14) + 15 bytes and more: left out for size" for n in range(6, 16)}),
    ("LL", "SizeMantissaNib"): (ALL, {}),
    ("CP", "CountSmall"): (ALL, {}),
    ("CP", "CountBegNib"): (ALL, {}),
    ("CP", "CountLastNib"): (set(range(8)), {**{n: "copies of 2^(n + 18) bytes and more: left out for size" for n in range(8, 14)},
                                             14: "a count of 33 bits: no u32 count", 15: "a count of 34 bits: no u32 count"}),
    ("CP", "CountMantissaNib"): (ALL, {}),
    ("CP", "DistanceMnemonic"): (ALL, {}),
    ("CP", "DistanceBegNib"): (ALL, {}),
    ("CP", "DistanceLastNib"): (set(range(10)), {n: "a distance of %d bits: not below the largest ring, 2^24" % (n + 15) for n in range(10, 16)}),
    ("CP", "DistanceMantissaNib"): (ALL, {}),
    ("DC", "SizeBegNib"): (ALL, {}),
    ("DC", "SizeLastNib"): (set(range(6)), {n: "word size %d: above 24" % (n + 19) for n in range(6, 16)}),
    ("DC", "Index"): (ALL, {}),
    ("DC", "Transform"): (ALL, {}),
    ("BT", "Mnemonic"): (ALL, {}),
    ("BT", "FirstNibble"): (ALL, {}),
    ("BT", "SecondNibble"): (ALL, {}),
    ("BT", "StrideNibble"): (ALL, {}),
    ("PM", "Only"): (set(range(4)), {n: "pred_mode %d: PredictionModeOutOfBounds" % n for n in range(4, 16)}),
    ("PM", "Mnemonic"): (ALL, {}),
    ("PM", "FirstNibble"): (ALL, {}),
    ("PM", "SecondNibble"): (ALL, {}),
}
# (the speed palette, the mixing values and the PredictionMode mixing nibble are the mixing-value tests' subject:
# tests/mixing_values.py; the catalogue claims nothing of them)


@pytest.fixture(scope="module")
def coverage(oracle):
    cov = np.zeros((T.cov_size(), 16), np.uint32)
    for _, blob in K.lists():
        cov += T.coverage([T.from_blob(oracle, blob)], window_size=_window(blob))
    return T.coverage_pairs(cov)


def test_prior_of_inverts_the_layout():
    n = T.cov_size()
    assert T.prior_of(0) == ("CC", "FullSelection", (0, 0))
    assert T.prior_of(n - 1) == ("PM", "ContextMapSpeedPalette", (3, 0))
    assert T.prior_of(16 + 256) == ("LL", "CountSmall", (0, 0))


@pytest.mark.parametrize("site", list(EXPECTED))
def test_catalogue_reaches_every_nibble(coverage, site):
    """the catalogue codes every nibble an encoder can write under each command prior, and no other"""
    can, why = EXPECTED[site]
    assert can | set(why) == ALL and not can & set(why)
    got = set().union(*coverage.get(site, {}).values())
    assert got == can, (site, sorted(can - got), sorted(got - can))


def _indices(coverage, site, k):
    return {idx[k] for idx in coverage[site]}


def test_catalogue_reaches_every_prior_index(coverage):
    """the prior indices the catalogue claims: every CTYPE slab 0..255 (literal length, copy count, dictionary size) and every
    distance prior 0..255 (mnemonic, mantissa, dictionary index); every CountSmall index, first-mantissa index, mnemonic
    index, transform prior, last-two-commands state and block-switch kind"""
    every = set(range(256))
    for site in (("LL", "CountSmall"), ("CP", "CountSmall"), ("DC", "SizeBegNib"), ("CP", "CountBegNib")):
        assert _indices(coverage, site, 0) >= (every if site != ("CP", "CountBegNib") else {0}), site
    for site in (("CP", "DistanceMnemonic"), ("CP", "DistanceMantissaNib"), ("DC", "Index")):
        assert _indices(coverage, site, 0) == every, (site, sorted(every - _indices(coverage, site, 0))[:10])
    assert _indices(coverage, ("CP", "CountSmall"), 1) == set(range(16))
    assert _indices(coverage, ("CP", "CountMantissaNib"), 1) == set(range(5))
    assert _indices(coverage, ("CP", "DistanceMantissaNib"), 1) == set(range(5))
    assert _indices(coverage, ("DC", "Index"), 1) == set(range(5))
    assert _indices(coverage, ("CP", "DistanceMnemonic"), 1) == {0, 1}
    assert {i for i in coverage[("DC", "Transform")] if i[0] == 0} == {(0, h) for h in range(2, 13)}   # size >> 1
    assert _indices(coverage, ("CC", "FullSelection"), 0) == set(range(16))
    assert _indices(coverage, ("BT", "Mnemonic"), 0) == {0, 1, 2}
    assert _indices(coverage, ("PM", "Mnemonic"), 0) == {0, 1}
