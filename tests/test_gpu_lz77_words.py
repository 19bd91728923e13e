"""Dictionary words under every transform in the LZ77 parse on the GPU: divans_b200_lz77_cmds_batch_device_words against the
host generator (divans_b200_lz77_cmds_batch_words) byte for byte, transforms 0 against the _dict call, statuses and refusals,
and Engine.compress_device(parses=DEFAULT_LZ77_WORD_PARSES)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import divans_b200  # noqa: E402
import lz77_dict_corpora as C  # noqa: E402
import lz77_words_corpora as W  # noqa: E402
from test_gpu_lz77_dict import _device, _fixtures, _host, _on_device, _streams, _text  # noqa: E402

gpu = pytest.mark.gpu
PARSES = [(4, 0, 4, 1), (4, 1, 5, 1), (4, 2, 4, 1), (6, 2, 6, 1), (7, 2, 4, 1), (10, 2, 4, 1), (8, 1, 10, 1), (16, 0, 24, 1),
          (32, 2, 4, 1), (6, 2, 32, 1), (7, 1, 0, 1)]


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="module")
def eng():
    """a context of its own with 64 resident streams"""
    import torch
    e = divans_b200.Engine(0, 64, 16)
    yield e
    e.close()
    torch.cuda.empty_cache()


def _straddling(seed=5):
    """transformed words under every transform, starting at every position 0..31 of a 32-position window, with copies around
    them, and words that end the stream"""
    rng = np.random.default_rng(seed)
    size_bits = C.tables()[0]
    raws = []
    for at in range(32):
        t = (at * 4 + seed) % 121
        size = 24 if W.core_len(4 + at % 21, t) < 4 else 4 + at % 21
        w = W.transformed(size, int(rng.integers(0, 1 << size_bits[size])), t)
        head = bytes(rng.integers(128, 256, 32 + at, dtype=np.uint8))
        raws += [head + w + head[:12] + w, head + w, (head + w)[:-1], head[:at] + w + w[:at % 7]]
    return raws


def _corpora(oracle):
    rng = np.random.default_rng(9)
    raws = [b"", b"a", b"ab", b"abc"] + [_text(n, n) for n in (4, 5, 31, 32, 33, 63, 64, 65, 1000)]
    raws += [W.forms_buffer(400), W.forms_buffer(3000, 8), rng.integers(0, 256, 20000, dtype=np.uint8).tobytes(), bytes(5000)]
    raws += W.forms_at_end() + W.short_cores() + _straddling()
    return raws + _fixtures(oracle) + [_text(70000, 3)]


def _agree(eng, raws, parse, window=16):
    want = _host(raws, parse, window)
    got = _device(eng, raws, parse, window)
    for i, ((s, l, region), w, r) in enumerate(zip(got, want, raws)):
        assert s == 0 and l == len(w), "%s stream %d (%d bytes): status %d, blob_len %d, host %d" % (parse, i, len(r), s, l, len(w))
        if region[:l] != w:
            k = int(np.nonzero(np.frombuffer(region[:l], np.uint8) != np.frombuffer(w, np.uint8))[0][0])
            raise AssertionError("%s stream %d (%d bytes): blob differs from the host's at byte %d" % (parse, i, len(r), k))
    return want


@gpu
@pytest.mark.parametrize("parse", PARSES, ids=["%d,%d,%d,%d" % p for p in PARSES])
def test_device_equals_host(eng, oracle, parse):
    want = _agree(eng, _corpora(oracle), parse)
    if 4 <= parse[2] <= 16:
        assert W.check_words(want[13], W.forms_buffer(400))


@gpu
@pytest.mark.parametrize("window", [10, 16, 24])
def test_windows(eng, oracle, window):
    raws = [_text(min(1 << (window + 1), 1 << 20), window), W.forms_buffer(2000, window)] + _straddling(window) + _fixtures(oracle)
    for parse in ((4, 0, 4, 1), (6, 2, 6, 1), (7, 1, 8, 1)):
        _agree(eng, raws, parse, window)


@gpu
def test_transforms_zero_is_the_dict_call(eng, oracle):
    raws = _corpora(oracle) + [C.word_buffer(400)]
    for parse in ((4, 0, 4), (6, 2, 6), (7, 1, 0), (10, 2, 4)):
        a = [g[2][:g[1]] for g in _device(eng, raws, parse + (0,))]
        b = [g[2][:g[1]] for g in _device(eng, raws, parse)]
        assert a == b, parse


@gpu
def test_batch_larger_than_the_warps(eng):
    """300 streams through the 64-slot context's warps in one launch"""
    rng = np.random.default_rng(4)
    raws = [W.forms_buffer(int(rng.integers(0, 200)), k) if k % 2 else _text(int(rng.integers(0, 9000)), k) for k in range(300)]
    _agree(eng, raws, (6, 2, 6, 1))


@gpu
def test_statuses_and_refusals(eng):
    """status 2 with the exact size, a misaligned region and in_len > max_in_len refused (status 3), as for the _dict call"""
    raws = [W.forms_buffer(300), b"", _text(7000, 3)]
    parse = (5, 1, 5, 1)
    want = _host(raws, parse)
    for caps in ([0] * 3, [len(w) - 1 for w in want], [len(w) for w in want]):
        for (s, l, region), w, c in zip(_device(eng, raws, parse, caps=caps), want, caps):
            assert l == len(w)
            assert (s == 2) if c < len(w) else (s == 0 and region[:l] == w)
    caps = divans_b200.lz77_blob_cap(np.array([len(r) for r in raws], np.uint64))
    b1 = ((64 + int(caps[0]) + 64) & ~15) + 2   # not 4-byte aligned
    boff = [64, b1, (b1 + int(caps[1]) + 64) & ~15]
    got = _device(eng, raws, parse, caps=caps, boff=boff)
    assert [g[0] for g in got] == [0, 3, 0] and got[1][1] == 0
    got = _device(eng, raws, parse, max_in=6999)
    assert [g[0] for g in got] == [0, 0, 3] and got[2][1] == 0
    for bad in ((4, 0, 4, 2), (4, 0, 4, -1), (4, 0, 3, 1), (3, 0, 4, 1), (4, 3, 4, 1)):
        with pytest.raises(divans_b200.DivansError, match="transforms 0 or 1"):
            _device(eng, [_text(1000)], bad)


@gpu
def test_compress_device_word_parses(eng, oracle):
    """compress_device(parses=DEFAULT_LZ77_WORD_PARSES): every stream decodes on the GPU and the oracle to its input, and no
    stream's chosen cost is above its cost under DEFAULT_LZ77_DICT_PARSES, whose lists are still candidates"""
    rng = np.random.default_rng(2)
    raws = [W.forms_buffer(int(rng.integers(1, 300)), k) for k in range(12)] + [_text(n, n) for n in (0, 100, 4096, 16384)]
    raws += W.forms_at_end()[:8] + _fixtures(oracle)[:1] + [rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()]
    raws += [f[k:k + 2048] for f in _fixtures(oracle) for k in range(0, 40000, 5000)]
    d_in, off, ln = _on_device(raws)
    opts = divans_b200.encode_options(window_size=16)
    parses = divans_b200.DEFAULT_LZ77_WORD_PARSES
    d_new, new_off, new_len, st, chosen, pcost = eng.compress_device(d_in, off, ln, opts=opts, parses=parses)
    got = _streams(d_new, new_off, new_len)
    assert (st == 0).all()
    for i, r in enumerate(raws):
        rc, back = oracle.decode(got[i], out_cap=len(r) + 64)
        assert rc == 0 and back == r, "stream %d" % i
    dec = eng.decode(got, [len(r) + 64 for r in raws])
    assert all(s == 0 and b == r for (s, b), r in zip(dec, raws))
    z = eng.compress_device(d_in, off, ln, opts=opts, parses=divans_b200.DEFAULT_LZ77_DICT_PARSES)
    k0 = len(divans_b200.DEFAULT_LZ77_DICT_PARSES)
    assert (z[3] == 0).all() and (pcost[:, :k0] == z[5]).all()
    assert (pcost.min(1) <= z[5].min(1)).all()
    assert any(len(parses[c]) == 4 for c in chosen)
