"""Dictionary words under every transform in the LZ77 parse on the CPU (include/divans_b200.h, "dictionary words under every
transform in the LZ77 parse"): the library's host generator divans_b200_lz77_cmds_batch_words against the oracle's
dvo_lz77_cmds_words_parse, which builds every transform of every word with the decoder's dvo_dict_word and has no index;
transforms 0 against the _dict call; refusals; and the oracle's choice between lists with and without every transform."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import divans_b200  # noqa: E402
from divans_b200 import synth  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402
import lz77_dict_corpora as C  # noqa: E402
import lz77_words_corpora as W  # noqa: E402


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _alice(oracle):
    rc, alice = oracle.decode(open(os.path.join(ROOT, "tests", "golden", "alice29_literal_only.divans"), "rb").read(), out_cap=1 << 20)
    assert rc == 0
    return alice


def _records(n, width, seed=5):
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return (np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n]).tobytes()


def _small():
    """the inputs every parse of the domain runs on: words under prefixed, capitalised, upper-cased and truncated forms"""
    rng = np.random.default_rng(7)
    return [W.forms_buffer(10, 4), W.forms_buffer(6, 5, types=(10, 11)), W.forms_buffer(6, 6, types=range(12, 21)), b"",
            b"abc", rng.integers(0, 256, 40, dtype=np.uint8).tobytes()] + W.forms_at_end()[::37] + W.short_cores()[:2]


def _large(oracle):
    """the inputs sampled parses run on"""
    rng = np.random.default_rng(3)
    return {"text": synth.text_corpus(8000, seed=2)[:8000], "alice29": _alice(oracle)[:8192], "forms": W.forms_buffer(300),
            "random": rng.integers(0, 256, 6000, dtype=np.uint8).tobytes(), "records4": _records(6000, 4)}


def _decode(oracle, stream, cap, blend):
    if blend:
        from oracle import oracle_blend as oracle
    return oracle.decode(stream, out_cap=cap)


def _host(raws, parse, window=16):
    blob, off, ln = divans_b200._pack(raws)
    out, boff, blen = divans_b200.lz77_cmds_batch(blob, off, ln, window, 2, 4, parse=parse)
    assert (blen <= divans_b200.lz77_blob_cap(ln)).all()
    return [out[int(o):int(o + n)].tobytes() for o, n in zip(boff, blen)]


def _same_commands(blob, ref):
    """the host's records equal the oracle's, except a Literal's offset (the host's pool is the raw stream, the oracle's its own)"""
    rec, want = C.records_of(blob), C.records_of(ref)
    lit = want[:, 0] == 3
    return rec.shape == want.shape and (rec[~lit] == want[~lit]).all() and (rec[lit, :1] == want[lit, :1]).all() and \
        (rec[lit, 2] == want[lit, 2]).all()


def test_transforms_zero_is_the_dict_parse(oracle):
    """transforms 0 gives the _dict call's lists byte for byte for every parse of the domain, and the oracle's too"""
    raws = _small() + [synth.text_corpus(3000, seed=9)[:3000], C.word_buffer(40, 3)]
    for mm in range(4, 33):
        for lz in range(3):
            for dm in [0] + list(range(4, 33)):
                assert _host(raws, (mm, lz, dm, 0)) == _host(raws, (mm, lz, dm)), (mm, lz, dm)
    for parse in ((4, 0, 4), (6, 2, 6), (7, 1, 0)):
        for r in raws:
            assert T.lz77_words_parse(oracle, r, *parse, 0).serialize() == T.lz77_dict_parse(oracle, r, *parse).serialize()


def test_every_parse_on_small_inputs(oracle):
    """every parse of the domain with transforms 1: the host's list is the oracle's record for record, replays to its input, and
    its words are the decoder's at their positions, each with a core of 4 or more bytes"""
    raws = _small()
    for mm in range(4, 33):
        for lz in range(3):
            for dm in [0] + list(range(4, 33)):
                got = _host(raws, (mm, lz, dm, 1))
                for r, b in zip(raws, got):
                    assert _same_commands(b, T.lz77_words_parse(oracle, r, mm, lz, dm, 1).serialize()), ((mm, lz, dm), len(r))
                    rc, _, back = T.recode_blob(b)
                    assert rc == 0 and back == r
                    assert dm or not W.check_words(b, r)
                    rec = C.records_of(b)
                    assert (rec[rec[:, 0] == 1, 2] >= mm).all() and (rec[rec[:, 0] == 2, 4] >= max(dm, 1)).all()
                if dm == 0:
                    assert got == _host(raws, (mm, lz))


SAMPLED = ((4, 0, 4, 1), (6, 2, 6, 1), (7, 2, 4, 1), (5, 1, 12, 1), (32, 0, 4, 1), (10, 2, 32, 1))


@pytest.mark.parametrize("name", ["text", "alice29", "forms", "random", "records4", "edges"])
def test_sampled_parses_on_larger_inputs(oracle, name):
    raws = W.forms_at_end() + W.short_cores() if name == "edges" else [_large(oracle)[name]]
    for parse in SAMPLED:
        for data, b in zip(raws, _host(raws, parse)):
            assert _same_commands(b, T.lz77_words_parse(oracle, data, *parse).serialize()), (name, parse, len(data))
            rc, _, back = T.recode_blob(b)
            assert rc == 0 and back == data
            W.check_words(b, data)


def test_each_transform_type_and_prefix_is_chosen():
    """a buffer of words under every transform takes words of every type and every prefix; alice29's text takes prefixed and
    capitalised forms that the 44-member set cannot; random bytes take none"""
    tr = C.tables()[3]
    forms = W.forms_buffer(1500, 8)
    got = W.check_words(_host([forms], (32, 0, 4, 1))[0], forms)
    assert {tr[t][1] for _, t in got} == set(W.TYPES)
    assert {tr[t][0] for _, t in got} == {p for p, _, _ in tr}
    # each type alone, back to back: the word's own type is chosen for many of them
    for typ in W.TYPES:
        buf = W.forms_buffer(40, 20 + typ, types=(typ,))
        got = W.check_words(_host([buf], (32, 0, 4, 1))[0], buf)
        assert sum(tr[t][1] == typ for _, t in got) >= 10, typ
    text = synth.text_corpus(6000, seed=3)[:6000]
    rng = np.random.default_rng(1)
    rnd = rng.integers(0, 256, 20000, dtype=np.uint8).tobytes()
    g, r = _host([text, rnd], (7, 2, 4, 1))
    assert any(tr[t][0] != b"" or tr[t][1] != 0 for _, t in W.check_words(g, text)) and not W.check_words(r, rnd)


def test_a_core_shorter_than_four_bytes_is_never_taken():
    """a word that an omission leaves with fewer than 4 bytes is not a candidate, even where nothing else matches"""
    raws = W.short_cores()
    for parse in ((4, 0, 4, 1), (32, 2, 4, 1)):
        for r, b in zip(raws, _host(raws, parse)):
            W.check_words(b, r)   # (asserts every core has 4 or more bytes)
    # the same bytes with a core of 4 are taken: omit-last-1 of a 5-byte word, alone
    tr = C.tables()[3]
    t = next(t for t in range(121) if tr[t] == (b"", 1, b""))
    w = W.transformed(5, 3, t)
    assert len(W.check_words(_host([w], (32, 0, 4, 1))[0], w)) == 1


def test_out_of_domain_parses_are_refused(oracle):
    data = synth.text_corpus(3000, seed=4)[:3000]
    blob, off, ln = divans_b200._pack([data])
    for bad in ((4, 0, 4, 2), (4, 0, 4, -1), (4, 0, 0, 2), (4, 0, 3, 1), (4, 0, 33, 1), (3, 0, 4, 1), (4, 3, 4, 1)):
        assert T.lz77_words_parse(oracle, data, *bad) is None, bad
        with pytest.raises(ValueError, match="transforms 0 or 1"):
            divans_b200.lz77_cmds_batch(blob, off, ln, parse=bad)
    # the C call itself writes nothing
    L = divans_b200.load_library()
    boff, blen, total = np.zeros(1, np.uint64), np.zeros(1, np.uint64), ctypes.c_size_t(7)
    p = lambda a: a.ctypes.data
    for bad in ((4, 0, 4, 2), (4, 0, 0, -1), (4, 0, 3, 1), (33, 0, 4, 0)):
        ps = divans_b200.Lz77WordsParse(*bad)
        rc = L.divans_b200_lz77_cmds_batch_words(1, p(blob), p(off), p(ln), 16, 2, 4, None, 0, p(boff), p(blen), ctypes.byref(total), 1,
                                                 ctypes.byref(ps))
        assert rc == divans_b200.DIVANS_FAILURE and total.value == 7 and blen[0] == 0
    rc = L.divans_b200_lz77_cmds_batch_words(1, p(blob), p(off), p(ln), 16, 2, 4, None, 0, p(boff), p(blen), ctypes.byref(total), 1, None)
    assert rc == divans_b200.DIVANS_FAILURE


def test_lists_decode_through_the_oracle(oracle):
    """lists with words under every transform encode and decode through the oracle to their inputs"""
    data = _large(oracle)
    for name in ("text", "alice29", "forms"):
        raw = data[name]
        b = _host([raw], (7, 2, 4, 1))[0]
        stream = T.from_blob(oracle, b).encode(oracle.options(window_size=16, dynamic_context_mixing=1))
        rc, back = oracle.decode(stream, out_cap=len(raw) + 64)
        assert rc == 0 and back == raw, name


@pytest.mark.parametrize("blend", [False, True])
def test_oracle_chooser_over_word_and_dict_lists(oracle, blend):
    """dvo_encode_cmds_choose over DEFAULT_LZ77_WORD_PARSES' lists: the argmin of the tallies, and every chosen stream decodes"""
    data = _large(oracle)
    parses = divans_b200.DEFAULT_LZ77_WORD_PARSES
    kw = dict(window_size=16, dynamic_context_mixing=1)
    for name in ("alice29", "forms", "random"):
        raw = data[name]
        lists = [T.lz77_words_parse(oracle, raw, *(tuple(p) + (0, 0))[:4]) for p in parses]
        rc, stream, chosen, costs = T.encode_cmds_choose(lists, blend=blend, **kw)
        want = [T.tally_cmds(cl, blend=blend, **kw)[1] for cl in lists]
        assert rc == 0 and list(costs) == want and chosen == int(np.argmin(want))
        rc, back = _decode(oracle, stream, len(raw) + 64, blend)
        assert rc == 0 and back == raw


def test_default_word_parses_and_prototypes():
    h = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    for name in ("divans_b200_lz77_cmds_batch_words", "divans_b200_lz77_cmds_batch_device_words"):
        assert re.search(r"DivansResult\s+%s\(" % name, h), name
        assert name in divans_b200.BATCH_SYMBOLS
    assert "int32_t transforms;" in h and "} divans_b200_lz77_words_parse;" in h
    d, base = divans_b200.DEFAULT_LZ77_WORD_PARSES, divans_b200.DEFAULT_LZ77_DICT_PARSES
    assert d[:len(base)] == base and len(d) <= 16
    assert all(len(p) == 4 and 4 <= p[0] <= 32 and 0 <= p[1] <= 2 and 4 <= p[2] <= 32 and p[3] == 1 for p in d[len(base):])
    assert base == divans_b200.DEFAULT_LZ77_PARSES + [(7, 2, 4), (10, 2, 4)]
