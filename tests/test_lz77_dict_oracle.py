"""Dictionary words in the LZ77 parse on the CPU (include/divans_b200.h, "dictionary words in the LZ77 parse"): the library's
host generator divans_b200_lz77_cmds_batch_dict against the oracle's dvo_lz77_cmds_dict_parse, which searches every word
under every transform of the set without an index; refusals; and the oracle's choice between lists with and without words."""
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
    """the inputs every parse of the domain runs on"""
    rng = np.random.default_rng(7)
    return [C.word_buffer(12, 4) + C.words_at_end()[1], b"", b"abc", rng.integers(0, 256, 60, dtype=np.uint8).tobytes()] + \
        C.words_at_end()[:4] + C.words_cut_short()[:3]


def _edges():
    """words at and one byte short of the stream's end, and cut short, under the parses the larger inputs sample"""
    return C.words_at_end() + C.words_cut_short() + [b"a", b"ab"]


def _large(oracle):
    """the inputs sampled parses run on (the oracle searches the whole dictionary at every position it reaches)"""
    rng = np.random.default_rng(3)
    return {"text": synth.text_corpus(12000, seed=2)[:12000], "alice29": _alice(oracle)[:16384], "words": C.word_buffer(400),
            "random": rng.integers(0, 256, 8000, dtype=np.uint8).tobytes(), "records4": _records(8000, 4)}


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


def test_transform_set_from_tables():
    """the set is derived from the tables: 44 transforms with an empty prefix and the identity type"""
    s = C.transform_set()
    assert len(s) == 44
    assert [t for t, _ in s[:6]] == [0, 1, 5, 8, 10, 14]
    assert [x for _, x in s[:4]] == [b"", b" ", b" the ", b" of "] and max(len(x) for _, x in s) == 7


def test_dict_min_zero_is_the_parse(oracle):
    """dict_min 0 gives the (min_match, lazy) parse's lists byte for byte, on the host and the oracle, for every (min_match, lazy)"""
    raws = _small() + [synth.text_corpus(6000, seed=9)[:6000]]
    for mm in range(4, 33):
        for lz in range(3):
            assert _host(raws, (mm, lz, 0)) == _host(raws, (mm, lz)), (mm, lz)
            for r in raws[:8] + raws[-1:]:
                assert T.lz77_dict_parse(oracle, r, mm, lz, 0).serialize() == T.lz77_parse(oracle, r, mm, lz).serialize(), (mm, lz)


def test_every_parse_on_small_inputs(oracle):
    """every parse of the domain: the host's list is the oracle's record for record, replays to its input, and its words are
    words of the set at their positions"""
    raws = _small()
    for mm in range(4, 33):
        for lz in range(3):
            for dm in [0] + list(range(4, 33)):
                got = _host(raws, (mm, lz, dm))
                for r, b in zip(raws, got):
                    assert _same_commands(b, T.lz77_dict_parse(oracle, r, mm, lz, dm).serialize()), ((mm, lz, dm), len(r))
                    rc, _, back = T.recode_blob(b)
                    assert rc == 0 and back == r
                    nw = C.check_words(b, r)
                    assert dm or nw == 0
                    rec = C.records_of(b)
                    assert (rec[rec[:, 0] == 1, 2] >= mm).all() and (rec[rec[:, 0] == 2, 4] >= max(dm, 1)).all()


SAMPLED = ((4, 0, 4), (6, 2, 6), (7, 2, 8), (5, 1, 12), (32, 0, 4), (10, 2, 32))


@pytest.mark.parametrize("name", ["text", "alice29", "words", "random", "records4", "edges"])
def test_sampled_parses_on_larger_inputs(oracle, name):
    raws = _edges() if name == "edges" else [_large(oracle)[name]]
    for parse in SAMPLED:
        for data, b in zip(raws, _host(raws, parse)):
            assert _same_commands(b, T.lz77_dict_parse(oracle, data, *parse).serialize()), (name, parse, len(data))
            rc, _, back = T.recode_blob(b)
            assert rc == 0 and back == data
            C.check_words(b, data)


def test_words_appear_where_they_should():
    """the word-built buffer takes many words; random bytes take none; alice29 takes some"""
    words = C.word_buffer(400)
    rng = np.random.default_rng(11)
    rnd = rng.integers(0, 256, 20000, dtype=np.uint8).tobytes()
    for parse in ((4, 0, 4), (6, 2, 6), (32, 2, 4)):
        w, r = _host([words, rnd], parse)
        assert C.check_words(w, words) >= 100 and C.check_words(r, rnd) == 0
    assert C.check_words(_host([words], (32, 0, 24))[0], words) > 0
    assert C.check_words(_host([words], (4, 0, 32))[0], words) == 0   # (no transformed word is longer than 31 bytes)


def test_words_at_the_end_and_cut_short():
    """a word that ends the stream is taken; one cut a byte short is not taken as that word"""
    for parse in ((4, 0, 4), (4, 2, 4)):
        for r, b in zip(C.words_at_end(), _host(C.words_at_end(), parse)):
            C.check_words(b, r)
        w = C.word(9, 5) + b" "
        assert C.check_words(_host([w], parse)[0], w) == 1 and C.records_of(_host([w], parse)[0])[-1, 0] == 2
        assert C.records_of(_host([w[:-1]], parse)[0])[-1, 4] != len(w)


def test_deferred_position_takes_no_word():
    """a position a lazy parse defers (its copy is shorter than the next position's) stays a literal even where a longer word
    starts; with lazy 0 the same position takes the word"""
    w = C.word(6, 120)   # a word of the dictionary
    tail = w[1:] + b" and ZZZZZZZZZZZZQQ"
    data = b"#" + w[:4] + b"%%" + tail + b"////" + w + b" and ZZZZZZZZZZZZQQ"
    i = data.rindex(w + b" and ")
    for lz, word_at_i in ((0, True), (1, False), (2, False)):
        b = _host([data], (4, lz, 4))[0]
        pos, at = 0, None
        for t, a, bb, c, d in C.records_of(b):
            if pos == i:
                at = t
            pos += int(bb) if t in (1, 3) else int(d) if t == 2 else 0
            if t == 3 and pos > i and at is None:
                at = 3   # i falls inside a literal run
        assert (at == 2) == word_at_i, (lz, at)


def test_out_of_domain_parses_are_refused(oracle):
    data = synth.text_corpus(3000, seed=4)[:3000]
    blob, off, ln = divans_b200._pack([data])
    for bad in ((4, 0, 1), (4, 0, 2), (4, 0, 3), (4, 0, 33), (4, 0, -1), (3, 0, 4), (4, 3, 4)):
        assert T.lz77_dict_parse(oracle, data, *bad) is None, bad
        with pytest.raises(ValueError, match="dict_min 0 or 4..32"):
            divans_b200.lz77_cmds_batch(blob, off, ln, parse=bad)
    # the C call itself, with a nonzero reserved field too, writes nothing
    L = divans_b200.load_library()
    boff, blen, total = np.zeros(1, np.uint64), np.zeros(1, np.uint64), ctypes.c_size_t(7)
    p = lambda a: a.ctypes.data
    for bad in ((4, 0, 3, 0), (4, 0, 33, 0), (4, 0, 4, 1), (4, 0, 0, 1)):
        ps = divans_b200.Lz77DictParse(*bad)
        rc = L.divans_b200_lz77_cmds_batch_dict(1, p(blob), p(off), p(ln), 16, 2, 4, None, 0, p(boff), p(blen), ctypes.byref(total), 1,
                                                ctypes.byref(ps))
        assert rc == divans_b200.DIVANS_FAILURE and total.value == 7 and blen[0] == 0
    rc = L.divans_b200_lz77_cmds_batch_dict(1, p(blob), p(off), p(ln), 16, 2, 4, None, 0, p(boff), p(blen), ctypes.byref(total), 1, None)
    assert rc == divans_b200.DIVANS_FAILURE


@pytest.mark.parametrize("blend", [False, True])
def test_oracle_chooser_over_dict_and_plain_lists(oracle, blend):
    """dvo_encode_cmds_choose over lists with and without words: the argmin of the tallies, and every chosen stream decodes"""
    data = _large(oracle)
    parses = divans_b200.DEFAULT_LZ77_DICT_PARSES
    kw = dict(window_size=16, dynamic_context_mixing=1)
    for name in ("text", "alice29", "words", "random"):
        raw = data[name]
        lists = [T.lz77_dict_parse(oracle, raw, *(tuple(p) + (0,))[:3]) for p in parses]
        rc, stream, chosen, costs = T.encode_cmds_choose(lists, blend=blend, **kw)
        want = [T.tally_cmds(cl, blend=blend, **kw)[1] for cl in lists]
        assert rc == 0 and list(costs) == want and chosen == int(np.argmin(want))
        if name == "words":
            assert len(parses[chosen]) == 3 and parses[chosen][2] != 0
        rc, back = _decode(oracle, stream, len(raw) + 64, blend)
        assert rc == 0 and back == raw


def test_default_dict_parses_and_prototypes():
    h = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    for name in ("divans_b200_lz77_cmds_batch_dict", "divans_b200_lz77_cmds_batch_device_dict"):
        assert re.search(r"DivansResult\s+%s\(" % name, h), name
        assert name in divans_b200.BATCH_SYMBOLS
    assert "typedef struct {\n    int32_t min_match;   /* 4..32: the shortest match emitted as a copy */\n    int32_t lazy;" in h
    assert "int32_t dict_min;" in h
    d = divans_b200.DEFAULT_LZ77_DICT_PARSES
    assert d[:len(divans_b200.DEFAULT_LZ77_PARSES)] == divans_b200.DEFAULT_LZ77_PARSES and len(d) <= 16
    assert all(len(p) == 3 and 4 <= p[0] <= 32 and 0 <= p[1] <= 2 and 4 <= p[2] <= 32 for p in d[len(divans_b200.DEFAULT_LZ77_PARSES):])
    assert divans_b200.DEFAULT_LZ77_PARSES == [(4, 0), (7, 2), (10, 2), (6, 2)]
