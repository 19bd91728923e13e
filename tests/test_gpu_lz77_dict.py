"""Dictionary words in the LZ77 parse on the GPU: divans_b200_lz77_cmds_batch_device_dict against the host generator
(divans_b200_lz77_cmds_batch_dict) byte for byte, its statuses and refusals, and Engine.compress_device(parses=
DEFAULT_LZ77_DICT_PARSES) against the oracle's choice."""
import lzma
import os
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

gpu = pytest.mark.gpu
PARSES = [(4, 0, 4), (4, 1, 5), (4, 2, 4), (5, 0, 6), (6, 2, 6), (7, 2, 8), (8, 1, 10), (10, 2, 12), (12, 0, 16), (16, 1, 24),
          (32, 2, 4), (32, 0, 31), (6, 2, 32), (7, 1, 0)]
CANARY = 0x5A
G = 64


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


def _text(n, seed=1):
    return synth.text_corpus(n, seed=seed)[:n] if n else b""


def _fixtures(oracle):
    g = os.path.join(ROOT, "tests", "golden")
    rc, alice = oracle.decode(open(os.path.join(g, "alice29_literal_only.divans"), "rb").read(), out_cap=1 << 20)
    assert rc == 0
    rc, ayl = oracle.Commands.from_ir(lzma.decompress(open(os.path.join(g, "asyoulik.ir.xz"), "rb").read())).recode(22)
    assert rc == 0
    return [alice, ayl]


def _host(raws, parse, window=16):
    blob, off, ln = divans_b200._pack(raws)
    out, boff, blen = divans_b200.lz77_cmds_batch(blob, off, ln, window, 2, 4, parse=parse)
    return [out[int(o):int(o + l)].tobytes() for o, l in zip(boff, blen)]


def _u64(a):
    import torch
    return torch.from_numpy(np.array(a, np.uint64).reshape(-1).view(np.int64)).to("cuda:0")


def _device(eng, raws, parse, window=16, caps=None, boff=None, max_in=None):
    """lz77_cmds_batch_device under `parse`, guard bytes around every region: [(status, blob_len, region bytes)]"""
    import torch
    n = len(raws)
    blob, off, ln = divans_b200._pack(raws)
    caps = divans_b200.lz77_blob_cap(ln) if caps is None else np.array(caps, np.uint64)
    if boff is None:
        boff, pos = [], G
        for c in caps:
            boff.append(pos)
            pos = (pos + int(c) + G + 15) & ~15
    else:
        pos = max(int(b) + int(c) for b, c in zip(boff, caps)) + G
    d_in = torch.from_numpy(blob).to("cuda:0")
    d_blobs = torch.full((pos,), CANARY, dtype=torch.uint8, device="cuda:0")
    m = [_u64(off), _u64(ln), _u64(boff), _u64(caps)]
    d_len = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda:0")
    d_st = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda:0")
    torch.cuda.current_stream().synchronize()
    mx = (int(ln.max()) if n else 0) if max_in is None else max_in
    eng.lz77_cmds_batch_device(n, d_in.data_ptr(), m[0].data_ptr(), m[1].data_ptr(), mx, window, 2, 4, d_blobs.data_ptr(), m[2].data_ptr(),
                               m[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), parse=parse)
    eng.synchronize()
    o = d_blobs.cpu().numpy()
    mask = np.ones(o.size, bool)
    for a, c in zip(boff, caps):
        mask[int(a):int(a) + int(c)] = False
    assert (o[mask] == CANARY).all(), "a byte outside the blob regions changed"
    st, bl = d_st.cpu().numpy()[:n], d_len.cpu().numpy()[:n].view(np.uint64)
    return [(int(s), int(l), o[int(a):int(a) + int(c)].tobytes()) for s, l, a, c in zip(st, bl, boff, caps)]


def _agree(eng, raws, parse, window=16, what=""):
    want = _host(raws, parse, window)
    got = _device(eng, raws, parse, window)
    for i, ((s, l, region), w, r) in enumerate(zip(got, want, raws)):
        assert s == 0 and l == len(w), "%s %s stream %d (%d bytes): status %d, blob_len %d, host %d" % (what, parse, i, len(r), s, l, len(w))
        if region[:l] != w:
            k = int(np.nonzero(np.frombuffer(region[:l], np.uint8) != np.frombuffer(w, np.uint8))[0][0])
            raise AssertionError("%s %s stream %d (%d bytes): blob differs from the host's at byte %d" % (what, parse, i, len(r), k))
    return want


def _straddling(seed=5):
    """transformed words that start at every position 0..31 of a 32-position window, so they cross its edge, with copies and
    lazy deferrals around them, and words that end the stream"""
    rng = np.random.default_rng(seed)
    sfx = [s for _, s in C.transform_set()]
    size_bits = C.tables()[0]
    raws = []
    for at in range(32):
        size = 4 + at % 21
        w = C.word(size, int(rng.integers(0, 1 << size_bits[size]))) + sfx[at % len(sfx)]
        head = bytes(rng.integers(128, 256, 32 + at, dtype=np.uint8))
        raws += [head + w + head[:12] + w, head + w, (head + w)[:-1], head[:at] + w + w[:at % 7]]
    return raws


def _corpora(oracle):
    rng = np.random.default_rng(9)
    raws = [b"", b"a", b"ab", b"abc"] + [_text(n, n) for n in (4, 5, 31, 32, 33, 63, 64, 65, 1000)]
    raws += [C.word_buffer(400), C.word_buffer(3000, 8), rng.integers(0, 256, 20000, dtype=np.uint8).tobytes(), bytes(5000)]
    raws += C.words_at_end() + C.words_cut_short() + _straddling()
    return raws + _fixtures(oracle) + [_text(70000, 3)]


@gpu
@pytest.mark.parametrize("parse", PARSES, ids=["%d,%d,%d" % p for p in PARSES])
def test_device_equals_host(eng, oracle, parse):
    want = _agree(eng, _corpora(oracle), parse)
    if 4 <= parse[2] <= 16:   # (the word buffer holds few transformed words of more than 16 bytes)
        assert C.check_words(want[13], C.word_buffer(400)) > 0


@gpu
@pytest.mark.parametrize("window", [10, 16, 24])
def test_windows(eng, oracle, window):
    raws = [_text(min(1 << (window + 1), 1 << 20), window), C.word_buffer(2000, window)] + _straddling(window) + _fixtures(oracle)
    for parse in ((4, 0, 4), (6, 2, 6), (7, 1, 8)):
        _agree(eng, raws, parse, window)


@gpu
def test_dict_min_zero_is_the_parse_call(eng, oracle):
    raws = _corpora(oracle)
    for mm, lz in ((4, 0), (6, 2), (7, 1)):
        a = [g[2][:g[1]] for g in _device(eng, raws, (mm, lz, 0))]
        b = [g[2][:g[1]] for g in _device(eng, raws, (mm, lz))]
        assert a == b


@gpu
def test_batch_larger_than_the_warps(eng, oracle):
    """300 streams through the 64-slot context's warps in one launch"""
    rng = np.random.default_rng(4)
    raws = [C.word_buffer(int(rng.integers(0, 200)), k) if k % 2 else _text(int(rng.integers(0, 9000)), k) for k in range(300)]
    _agree(eng, raws, (6, 2, 6))


@gpu
def test_statuses_and_refusals(eng):
    """status 2 with the exact size, a misaligned region and in_len > max_in_len refused (status 3), as for the _parse call"""
    raws = [C.word_buffer(300), b"", _text(7000, 3)]
    parse = (5, 1, 5)
    want = _host(raws, parse)
    for caps in ([0] * 3, [len(w) - 1 for w in want], [len(w) for w in want]):
        for (s, l, region), w, c in zip(_device(eng, raws, parse, caps=caps), want, caps):
            assert l == len(w)
            assert (s == 2) if c < len(w) else (s == 0 and region[:l] == w)
    caps = divans_b200.lz77_blob_cap(np.array([len(r) for r in raws], np.uint64))
    b1 = ((G + int(caps[0]) + G) & ~15) + 2   # not 4-byte aligned
    boff = [G, b1, (b1 + int(caps[1]) + G) & ~15]
    got = _device(eng, raws, parse, caps=caps, boff=boff)
    assert [g[0] for g in got] == [0, 3, 0] and got[1][1] == 0
    got = _device(eng, raws, parse, max_in=6999)
    assert [g[0] for g in got] == [0, 0, 3] and got[2][1] == 0
    for bad in ((4, 0, 3), (4, 0, 33), (4, 0, -1), (3, 0, 4), (4, 3, 4)):
        with pytest.raises(divans_b200.DivansError, match="dict_min 0 or 4..32"):
            _device(eng, [_text(1000)], bad)


def _on_device(raws):
    import torch
    blob, off, ln = divans_b200._pack(raws)
    return torch.from_numpy(blob).to("cuda:0"), off, ln


def _streams(d_new, off, ln):
    h = d_new.cpu().numpy()
    return [h[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]


@gpu
def test_compress_device_dict_parses(eng, oracle):
    """compress_device(parses=DEFAULT_LZ77_DICT_PARSES): the oracle's choice among the oracle's lists, streams equal to the oracle
    chooser's, decoding on the GPU and the oracle; no stream larger than under DEFAULT_LZ77_PARSES"""
    rng = np.random.default_rng(2)
    raws = [C.word_buffer(int(rng.integers(1, 300)), k) for k in range(12)] + [_text(n, n) for n in (0, 100, 4096, 16384)]
    raws += C.words_at_end()[:8] + _fixtures(oracle)[:1] + [rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()]
    d_in, off, ln = _on_device(raws)
    opts = divans_b200.encode_options(window_size=16)
    parses = divans_b200.DEFAULT_LZ77_DICT_PARSES
    d_new, new_off, new_len, st, chosen, pcost = eng.compress_device(d_in, off, ln, opts=opts, parses=parses)
    got = _streams(d_new, new_off, new_len)
    assert (st == 0).all()
    for i, r in enumerate(raws):
        lists = [T.lz77_dict_parse(oracle, r, *(tuple(p) + (0,))[:3]) for p in parses]
        rc, stream, ch, costs = T.encode_cmds_choose(lists, window_size=16)
        assert rc == 0 and ch == chosen[i] and list(costs) == list(pcost[i]) and stream == got[i], "stream %d" % i
        rc, back = oracle.decode(got[i], out_cap=len(r) + 64)
        assert rc == 0 and back == r
    dec = eng.decode(got, [len(r) + 64 for r in raws])
    assert all(s == 0 and b == r for (s, b), r in zip(dec, raws))
    # DEFAULT_LZ77_PARSES stay candidates: no stream's chosen cost is higher.  (The choice is by tallied cost, so a stream of a
    # few hundred bytes may still come out a few bytes longer, by the coder's flush.)
    z = eng.compress_device(d_in, off, ln, opts=opts, parses=divans_b200.DEFAULT_LZ77_PARSES)
    k0 = len(divans_b200.DEFAULT_LZ77_PARSES)
    assert (z[3] == 0).all() and (pcost[:, :k0] == z[5]).all()
    assert (pcost.min(1) <= z[5].min(1)).all() and int(new_len.sum()) <= int(z[2].sum())
    assert (new_len <= z[2] + 8).all()
    assert any(len(parses[c]) == 3 for c in chosen)
