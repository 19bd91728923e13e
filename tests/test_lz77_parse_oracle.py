"""LZ77 parses on the CPU (include/divans_b200.h, "the LZ77 parse"): the oracle's dvo_lz77_cmds_parse, the library's host
generator divans_b200_lz77_cmds_batch_parse, and the oracle's choice of one of k command lists by cost (dvo_encode_cmds_choose)."""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import divans_b200  # noqa: E402
from divans_b200 import synth  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402

MIN_MATCHES = (4, 5, 6, 7, 8, 12, 16, 32)


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _records(n, width, seed=5):
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return (np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n]).tobytes()


def _alice(oracle):
    rc, alice = oracle.decode(open(os.path.join(ROOT, "tests", "golden", "alice29_literal_only.divans"), "rb").read(), out_cap=1 << 20)
    assert rc == 0
    return alice


def _corpora(oracle):
    rng = np.random.default_rng(3)
    return {
        "empty": b"", "short": b"abcabcabcab", "run": bytes(5000), "text": synth.text_corpus(40000, seed=2)[:40000],
        "periodic": bytes(rng.integers(0, 256, 7, dtype=np.uint8)) * 3000, "records4": _records(30000, 4),
        "random": rng.integers(0, 256, 20000, dtype=np.uint8).tobytes(), "small_alphabet": rng.integers(0, 3, 20000, dtype=np.uint8).tobytes(),
        "alice29": _alice(oracle),
    }


def _records_of(blob):
    h = np.frombuffer(blob[:32], np.uint32)
    return np.frombuffer(blob[32:32 + 20 * int(h[2])], np.uint32).reshape(-1, 5)


def test_default_parse_is_the_oracle_generator(oracle):
    """{4, 0} is dvo_lz77_cmds on every corpus, windows 10..24"""
    for name, data in _corpora(oracle).items():
        for w in (10, 16, 24):
            assert T.lz77_parse(oracle, data, 4, 0, window=w).serialize() == oracle.Commands.lz77(data, window=w).serialize(), (name, w)


def test_every_parse_replays_to_its_input(oracle):
    """every parse in the domain: the host generator's list replays (dvo_recode_blob) to the input, every copy is at least
    min_match long, its commands are the oracle's, and lz77_blob_cap holds it"""
    cs = _corpora(oracle)
    raws = [cs[k] for k in ("text", "records4", "small_alphabet", "periodic", "short", "empty")]
    blob, off, ln = divans_b200._pack(raws)
    for mm in range(4, 33):
        for lz in range(3):
            out, bo, bl = divans_b200.lz77_cmds_batch(blob, off, ln, 16, 2, 4, parse=(mm, lz))
            assert (bl <= divans_b200.lz77_blob_cap(ln)).all()
            for r, o, n in zip(raws, bo, bl):
                b = out[int(o):int(o + n)].tobytes()
                rc, _, got = T.recode_blob(b)
                assert rc == 0 and got == r, (mm, lz, len(r))
                rec = _records_of(b)
                assert (rec[rec[:, 0] == 1, 2] >= mm).all()
                want = _records_of(T.lz77_parse(oracle, r, mm, lz).serialize())
                cp = want[:, 0] == 1
                assert (rec[:, 0] == want[:, 0]).all() and (rec[cp, 1:3] == want[cp, 1:3]).all() and (rec[~cp, 2] == want[~cp, 2]).all()


def test_lazy_parses_differ_from_greedy(oracle):
    """on text, each lazy step changes the list and makes fewer commands than greedy at the same minimum, and each replays"""
    data = _alice(oracle)
    lists = [T.lz77_parse(oracle, data, 6, lz) for lz in range(3)]
    blobs = [cl.serialize() for cl in lists]
    assert len(set(blobs)) == 3
    assert lists[2].n_cmds < lists[0].n_cmds and lists[1].n_cmds < lists[0].n_cmds
    for b in blobs:
        rc, _, got = T.recode_blob(b, window=16)
        assert rc == 0 and got == data


def test_out_of_domain_parses_are_refused(oracle):
    data = synth.text_corpus(5000, seed=4)[:5000]
    blob, off, ln = divans_b200._pack([data])
    for bad in ((3, 0), (33, 0), (4, 3), (4, -1), (0, 0), (-4, 1)):
        assert T.lz77_parse(oracle, data, *bad) is None
        with pytest.raises(ValueError):
            divans_b200.lz77_cmds_batch(blob, off, ln, parse=bad)


def test_host_parse_none_is_the_plain_call():
    data = [synth.text_corpus(30000, seed=6)[:30000], b"", b"xyzxyzxyz"]
    blob, off, ln = divans_b200._pack(data)
    a = divans_b200.lz77_cmds_batch(blob, off, ln)
    b = divans_b200.lz77_cmds_batch(blob, off, ln, parse=(4, 0))
    assert all((x == y).all() for x, y in zip(a, b))


@pytest.mark.parametrize("blend", [False, True])
def test_oracle_chooser_is_the_argmin_of_the_tallies(oracle, blend):
    """dvo_encode_cmds_choose: costs are dvo_tally_cmds of each list, the choice their argmin (ties to the lowest index), and the
    stream the chosen list's encoding"""
    cs = _corpora(oracle)
    parses = divans_b200.DEFAULT_LZ77_PARSES + [(32, 0), (4, 0)]
    for name in ("text", "records4", "alice29", "empty", "random"):
        lists = [T.lz77_parse(oracle, cs[name], mm, lz) for mm, lz in parses]
        kw = dict(window_size=16, dynamic_context_mixing=1)
        rc, stream, chosen, costs = T.encode_cmds_choose(lists, blend=blend, **kw)
        want = [T.tally_cmds(cl, blend=blend, **kw)[1] for cl in lists]
        assert rc == 0 and list(costs) == want
        assert chosen == int(np.argmin(want)) and costs[-1] == costs[0] and chosen != len(parses) - 1
        assert stream == T.encode_cmds_choose([lists[chosen]], blend=blend, **kw)[1]


def test_oracle_chooser_skips_a_failing_list(oracle):
    """a list the encoder refuses (copies farther than a 2^10 window) costs UINT64_MAX; when every list fails, the choice is 0
    and the call fails"""
    data = synth.text_corpus(30000, seed=8)[:30000]
    good = T.lz77_parse(oracle, data, 6, 1, window=10)
    bad = T.lz77_parse(oracle, data, 4, 0, window=20)
    kw = dict(window_size=10)
    assert T.tally_cmds(bad, **kw)[0] != T.SUCCESS and T.tally_cmds(good, **kw)[0] == T.SUCCESS
    rc, _, chosen, costs = T.encode_cmds_choose([bad, good], **kw)
    assert rc == 0 and chosen == 1 and costs[0] == T.TALLY_FAILED
    rc, _, chosen, costs = T.encode_cmds_choose([bad, bad], **kw)
    assert rc != 0 and chosen == 0 and (costs == T.TALLY_FAILED).all()


def test_prototypes_in_header():
    h = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    for name in ("divans_b200_lz77_cmds_batch_parse", "divans_b200_lz77_cmds_batch_device_parse", "divans_b200_encode_cmds_choose_batch_device"):
        assert re.search(r"DivansResult\s+%s\(" % name, h), name
        assert name in divans_b200.BATCH_SYMBOLS
    assert "typedef struct {\n    int32_t min_match;" in h
    assert divans_b200.DEFAULT_LZ77_PARSES[0] == (4, 0)
    assert all(4 <= m <= 32 and 0 <= z <= 2 for m, z in divans_b200.DEFAULT_LZ77_PARSES)
