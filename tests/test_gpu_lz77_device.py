"""Generating LZ77 command lists on the GPU (divans_b200_lz77_cmds_batch_device, Engine.compress_device).  The reference of every
check is the library's host generator, divans_b200_lz77_cmds_batch: status, blob_len and blob bytes must be equal, and bytes
around every blob region must not change.  The first three tests need no GPU."""
import os
import re

import numpy as np
import pytest

import divans_b200
from divans_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
CANARY = 0x5A
G = 64          # guard bytes around every blob region


def test_prototype_in_header():
    h = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    m = re.search(r"DivansResult\s+divans_b200_lz77_cmds_batch_device\(([^;]*)\);", h)
    assert m
    assert [a.strip() for a in " ".join(m.group(1).split()).split(",")] == [
        "divans_b200_ctx *ctx", "size_t n", "const uint8_t *d_in", "const uint64_t *d_in_off", "const uint64_t *d_in_len",
        "uint64_t max_in_len", "int32_t window", "int32_t pred_mode", "int32_t mixing_value", "uint8_t *d_blobs",
        "const uint64_t *d_blob_off", "const uint64_t *d_blob_cap", "uint64_t *d_blob_len", "int32_t *d_status", "void *cuda_stream"]


def _max_cmds(n):
    return 3 + 2 * (n // 5)


def _dense(reps, seed):
    """1-byte literal + 4-byte copy, over and over: a byte, then a 4-gram seen before, each (byte, 4-gram) and (4-gram, byte)
    pair new, so that no copy covers more than the 4-gram"""
    rng = np.random.default_rng(seed)
    grams = [rng.integers(0, 256, 4, dtype=np.uint8).tobytes() for _ in range(8)]
    out = bytearray(b"".join(g + b"\xff" for g in grams))
    for r in range(reps):
        out += bytes([(r // 8) % 255]) + grams[r % 8]
    return bytes(out)


def test_blob_cap_bounds_oracle_commands(oracle):
    """lz77_blob_cap bounds the command count of the oracle's LZ77 (the host generator's commands), on inputs built to have
    the most commands and on random ones; and the host generator's blobs fit it"""
    rng = np.random.default_rng(5)
    cases = [_dense(r, s) for s in range(4) for r in (1, 7, 100, 2000)]
    cases += [b"a" + b"bcde" * k for k in range(1, 40)]
    cases += [rng.integers(0, 3, int(rng.integers(0, 60)), dtype=np.uint8).tobytes() for _ in range(3000)]
    cases += [rng.integers(0, 256, int(rng.integers(0, 5000)), dtype=np.uint8).tobytes() for _ in range(50)]
    cases += [bytes(n) for n in range(12)]
    densest = 0.0
    for c in cases:
        k = oracle.Commands.lz77(c, window=16).n_cmds
        assert k <= _max_cmds(len(c)), (len(c), k)
        if len(c) > 1000:
            densest = max(densest, k / _max_cmds(len(c)))
    assert densest > 0.9   # the constructed inputs come close to the bound: it is not loose
    blob, off, ln = divans_b200._pack(cases)
    _, _, blen = divans_b200.lz77_cmds_batch(blob, off, ln, 16, 2, 4)
    assert (blen <= divans_b200.lz77_blob_cap(ln)).all()
    assert (divans_b200.lz77_blob_cap(ln) - blen).min() >= 0


def test_symbol_listed():
    assert "divans_b200_lz77_cmds_batch_device" in divans_b200.BATCH_SYMBOLS


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    """a context of its own, at most 64 streams resident (a 1 GiB slot arena when it encodes): the session's contexts hold most
    of the GPU, and closing this one returns its arena, logs and scratch to the tests that follow"""
    import torch
    e = divans_b200.Engine(0, 64, 16)
    yield e
    e.close()
    torch.cuda.empty_cache()   # (the blob and output tensors of compress_device)


def _host(raws, window=16, pm=2, mv=4):
    blob, off, ln = divans_b200._pack(raws)
    out, boff, blen = divans_b200.lz77_cmds_batch(blob, off, ln, window, pm, mv)
    return [out[int(o):int(o + l)].tobytes() for o, l in zip(boff, blen)]


def _device(eng, raws, window=16, pm=2, mv=4, caps=None, shift=None, max_in_len=None, lens=None):
    """lz77_cmds_batch_device with guard bytes around every blob region: [(status, blob_len, region bytes)].  `shift[i]` moves
    region i off 4-byte alignment; `lens` overrides the lengths passed."""
    import torch
    n = len(raws)
    blob, off, ln = divans_b200._pack(raws)
    lens = ln if lens is None else np.array(lens, np.uint64)
    caps = divans_b200.lz77_blob_cap(ln) if caps is None else np.array(caps, np.uint64)
    shift = [0] * n if shift is None else shift
    boff, pos = [], G
    for c, s in zip(caps, shift):
        boff.append(pos + s)
        pos = (pos + s + int(c) + G + 15) & ~15
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.array(a, np.uint64).reshape(-1).view(np.int64)).to(dev)
    d_in = torch.from_numpy(blob).to(dev)
    d_blobs = torch.full((pos,), CANARY, dtype=torch.uint8, device=dev)
    d_meta = [u64(off), u64(lens), u64(boff), u64(caps)]
    d_len = torch.full((max(n, 1),), -1, dtype=torch.int64, device=dev)
    d_st = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    torch.cuda.current_stream().synchronize()
    mx = int(lens.max()) if max_in_len is None else max_in_len
    eng.lz77_cmds_batch_device(n, d_in.data_ptr(), d_meta[0].data_ptr(), d_meta[1].data_ptr(), mx, window, pm, mv, d_blobs.data_ptr(),
                               d_meta[2].data_ptr(), d_meta[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr())
    eng.synchronize()
    o = d_blobs.cpu().numpy()
    mask = np.ones(o.size, bool)
    for a, c in zip(boff, caps):
        mask[a:a + int(c)] = False
    assert (o[mask] == CANARY).all(), "a byte outside the blob regions changed"
    st, bl = d_st.cpu().numpy()[:n], d_len.cpu().numpy()[:n].view(np.uint64)
    return [(int(s), int(l), o[a:a + int(c)].tobytes()) for s, l, a, c in zip(st, bl, boff, caps)]


def _agree(eng, raws, window=16, pm=2, mv=4, what=""):
    want = _host(raws, window, pm, mv)
    got = _device(eng, raws, window, pm, mv)
    for i, ((s, l, region), w) in enumerate(zip(got, want)):
        assert s == 0, "%s stream %d (%d bytes): status %d" % (what, i, len(raws[i]), s)
        assert l == len(w), "%s stream %d (%d bytes): blob_len %d, host %d" % (what, i, len(raws[i]), l, len(w))
        if region[:l] != w:
            a = np.frombuffer(region[:l], np.uint8)
            k = int(np.nonzero(a != np.frombuffer(w, np.uint8))[0][0])
            raise AssertionError("%s stream %d (%d bytes): blob differs from the host's at byte %d" % (what, i, len(raws[i]), k))
    return want


def _text(n, seed=1):
    return synth.text_corpus(n, seed=seed)[:n] if n else b""


def _h4(words):
    return (words.astype(np.uint64) * np.uint64(2654435761) & np.uint64(0xffffffff)) >> np.uint64(17)


# ---------------------------------------------------------------------------------------------------------------------
# byte-exact lists
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_short_lengths(eng):
    raws = [b"", b"a", b"abc", b"abcd", b"abcde", b"aaaa", b"aaaaa", b"abab", b"ababa", bytes(5)]
    _agree(eng, raws, what="short")


@gpu
def test_text_around_the_copy_limit(eng):
    """text of 65535..65537 bytes and 1 MiB, and runs where copies longer than 65535 bytes are split"""
    raws = [_text(65535), _text(65536), _text(65537), _text(1 << 20, 3), bytes(1 << 20), b"xy" * (1 << 19), _text(200000, 4) * 3]
    _agree(eng, raws, what="long")


@gpu
@pytest.mark.parametrize("w", [10, 12, 16, 22, 24])
def test_windows_and_maxdist(eng, w):
    """a repeat at distance exactly 2^w - 16 is a candidate, one at 2^w - 15 is not"""
    rng = np.random.default_rng(w)
    raws, dists = [], ((1 << w) - 16, (1 << w) - 15, (1 << w) - 17)
    for d in dists:
        a = np.zeros(d + 64, np.uint8)   # a run of zeros between: the repeat is the first candidate of its 4-grams
        a[:48] = a[d:d + 48] = rng.integers(1, 256, 48, dtype=np.uint8)
        raws.append(a.tobytes())
    raws.append(_text(min(1 << (w + 1), 1 << 21), w))
    _agree(eng, raws, window=w, what="window %d" % w)
    # (the inputs test the boundary: the host generator takes the repeats at 2^w - 16 and 2^w - 17, not the one at 2^w - 15)
    for b, d, taken in zip(_host(raws[:3], window=w), dists, (True, False, True)):
        rec = np.frombuffer(b[32:32 + 20 * int(np.frombuffer(b[8:12], np.uint32)[0])], np.uint32).reshape(-1, 5)
        assert bool(((rec[:, 0] == 1) & (rec[:, 1] == d)).any()) == taken


@gpu
def test_periodic_and_random(eng):
    rng = np.random.default_rng(9)
    raws = [bytes([7]) * 5000, bytes([0]) * 70000]
    for p in (2, 3, 4, 7):
        rec = rng.integers(0, 256, p, dtype=np.uint8).tobytes()
        raws.append(rec * (40000 // p))
        raws.append((rec * (20000 // p))[:-1] + b"!" + rec * 500)
    raws += [rng.integers(0, 256, k, dtype=np.uint8).tobytes() for k in (100, 4096, 100000)]
    raws += [rng.integers(0, 4, 30000, dtype=np.uint8).tobytes()]
    _agree(eng, raws, what="patterns")


@gpu
def test_chain_cap_and_ties(eng):
    """more than 16 distinct 4-grams in one hash bucket, repeated with endings from a small alphabet: long chains (the cap of
    16 candidates) and many candidates of equal length (the tie goes to the newest)"""
    rng = np.random.default_rng(17)
    w = rng.integers(0, 1 << 32, 1 << 22, dtype=np.uint64).astype(np.uint32)
    h = _h4(w)
    counts = np.bincount(h.astype(np.int64), minlength=1 << 15)
    bucket = int(np.argmax(counts))
    grams = np.unique(w[h == bucket])[:40]
    assert grams.size > 16
    gb = [int(g).to_bytes(4, "little") for g in grams]
    raws = []
    for s in range(4):
        r = np.random.default_rng(s)
        out = bytearray()
        for _ in range(6000):
            out += gb[int(r.integers(0, len(gb) if s < 2 else 20))] + bytes(int(x) for x in r.integers(0, 2 + s, int(r.integers(0, 4))))
        raws.append(bytes(out))
    # one gram over and over, then each of the others: every position of the bucket has a full chain
    raws.append(b"".join(gb[k % len(gb)] for k in range(20000)))
    _agree(eng, raws, what="chains")


@gpu
def test_pred_mode_and_mixing_value(eng):
    raws = [_text(3000, 5), b"", _text(70000, 6)]
    for pm, mv in ((0, 0), (1, 7), (3, 15), (2, 4), (7, 200), (-2, 260)):
        _agree(eng, raws, pm=pm, mv=mv, what="pm %d mv %d" % (pm, mv))


def _batch(seed, n):
    rng = np.random.default_rng(seed)
    corpus = np.frombuffer(synth.text_corpus(1 << 22, seed=seed), np.uint8)
    raws = []
    for i in range(n):
        k = int(rng.choice([0, 1, 3, 4, 5, 31, 32, 33]) if i % 10 == 0 else rng.integers(0, 20000))
        if i % 3 == 0:
            raws.append(rng.integers(0, 256 if i % 2 else 6, k, dtype=np.uint8).tobytes())
        else:
            o = int(rng.integers(0, corpus.size - k))
            raws.append(corpus[o:o + k].tobytes())
    return raws


@gpu
def test_random_batch(eng):
    _agree(eng, _batch(23, 3000), what="batch")


@gpu
def test_random_batch_two_warps():
    """the same streams on two warps: each warp takes many streams of different lengths in turn, and a head table entry left
    by the previous stream would be a wrong candidate"""
    e = divans_b200.Engine(0, 2, 16)
    try:
        _agree(e, _batch(23, 3000), what="two warps")
        _agree(e, [_text(40000, 8), _text(40000, 8)[:30000], b"", _text(40000, 8)[7:]], what="two warps, shared text")
    finally:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# statuses and refusals
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_region_too_small(eng):
    raws = [_text(5000, 2), b"", _text(70000, 3)]
    want = _host(raws)
    for caps in ([0] * 3, [len(w) - 1 for w in want], [len(w) for w in want]):
        got = _device(eng, raws, caps=caps)
        for (s, l, region), w, c in zip(got, want, caps):
            assert l == len(w)
            if c < len(w):
                assert s == 2
            else:
                assert s == 0 and region == w


@gpu
def test_refusals(eng):
    raws = [_text(1000, 2), _text(2000, 3), _text(3000, 4), _text(500, 5)]
    want = _host(raws)
    got = _device(eng, raws, shift=[1, 0, 2, 3])
    assert [g[:2] for g in got] == [(3, 0), (0, len(want[1])), (3, 0), (3, 0)]
    assert got[1][2][:got[1][1]] == want[1]
    got = _device(eng, raws, max_in_len=2000)
    assert [g[0] for g in got] == [0, 0, 3, 0] and got[2][1] == 0
    assert [g[2][:g[1]] for g in got if g[0] == 0] == [want[0], want[1], want[3]]
    for w in (9, 25):
        with pytest.raises(divans_b200.DivansError):
            _device(eng, raws, window=w)


@gpu
def test_replay_of_gpu_lists_gives_the_inputs(eng):
    import torch
    raws = _batch(31, 200) + [_text(1 << 20, 9)]
    got = _device(eng, raws)
    blobs = [r[2][:r[1]] for r in got]
    blob, off, ln = divans_b200._pack(blobs)
    out_off, total = divans_b200._regions([len(r) for r in raws])
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.array(a, np.uint64).reshape(-1).view(np.int64)).to(dev)
    d_b, d_o, d_l, d_oo, d_oc = torch.from_numpy(blob).to(dev), u64(off), u64(ln), u64(out_off), u64([len(r) for r in raws])
    d_out = torch.zeros(max(total, 1), dtype=torch.uint8, device=dev)
    d_len = torch.zeros(len(raws), dtype=torch.int64, device=dev)
    d_st = torch.full((len(raws),), -1, dtype=torch.int32, device=dev)
    torch.cuda.current_stream().synchronize()
    eng.replay_cmds_batch_device(len(raws), d_b.data_ptr(), d_o.data_ptr(), d_l.data_ptr(), d_out.data_ptr(), d_oo.data_ptr(), d_oc.data_ptr(),
                                 d_len.data_ptr(), d_st.data_ptr(), 0)
    eng.synchronize()
    o, st = d_out.cpu().numpy(), d_st.cpu().numpy()
    assert (st == 0).all()
    for r, a in zip(raws, out_off):
        assert o[int(a):int(a) + len(r)].tobytes() == r


# ---------------------------------------------------------------------------------------------------------------------
# compress_device
# ---------------------------------------------------------------------------------------------------------------------
def _on_device(raws):
    import torch
    blob, off, ln = divans_b200._pack(raws)
    return torch.from_numpy(blob).to("cuda:0"), off, ln


def _streams(d_new, off, ln):
    h = d_new.cpu().numpy()
    return [h[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]


@gpu
def test_compress_device_equals_host_route(eng):
    raws = _batch(41, 300) + [_text(65536, 10), _text(65537, 11)]
    d_in, off, ln = _on_device(raws)
    host = _host(raws, 16)
    opts = divans_b200.encode_options(window_size=16)
    want = eng.encode(host, opts, cmds=True)
    d_new, new_off, new_len, st = eng.compress_device(d_in, off, ln, opts=opts)
    assert (st == 0).all()
    got = _streams(d_new, new_off, new_len)
    assert got == want
    # opts None: each list coded with its header window, here 16
    d2, o2, l2, st2 = eng.compress_device(d_in, off, ln)
    assert (st2 == 0).all() and _streams(d2, o2, l2) == want
    # the streams decode to the inputs
    dec = eng.decode(got, [len(r) + 64 for r in raws])
    assert all(s == 0 and b == r for (s, b), r in zip(dec, raws))
    # another generator window and literal model
    host12 = _host(raws[:50], 12, 0, 7)
    o12 = divans_b200.encode_options(window_size=12, dynamic_context_mixing=2)
    d3, o3, l3, st3 = eng.compress_device(d_in, off[:50], ln[:50], window=12, pred_mode=0, mixing_value=7, opts=o12)
    assert (st3 == 0).all() and _streams(d3, o3, l3) == eng.encode(host12, o12, cmds=True)


@gpu
def test_compress_device_candidates(eng):
    raws = _batch(43, 120)
    d_in, off, ln = _on_device(raws)
    cands = [divans_b200.LITERAL_MODEL_KEEP] + divans_b200.DEFAULT_LITERAL_MODELS
    opts = divans_b200.encode_options(window_size=16)
    want = eng.encode_cmds_auto(_host(raws), opts, cands)
    d_new, new_off, new_len, st, chosen, cost = eng.compress_device(d_in, off, ln, opts=opts, candidates=cands)
    assert (st == 0).all() and cost.shape == (len(raws), len(cands))
    assert _streams(d_new, new_off, new_len) == [b for _, b, _ in want]
    assert list(chosen) == [c for _, _, c in want]


@gpu
def test_compress_device_sub_batches_and_streams(eng):
    import torch
    raws = _batch(47, 100)
    d_in, off, ln = _on_device(raws)
    one = eng.compress_device(d_in, off, ln)
    assert eng.last_compress_sub_batches == 1
    many = eng.compress_device(d_in, off, ln, sub_batch=7)
    assert eng.last_compress_sub_batches == 15
    assert (one[3] == 0).all() and (many[3] == 0).all()
    assert _streams(one[0], one[1], one[2]) == _streams(many[0], many[1], many[2])
    # ordered after the work of a caller's stream
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_new, new_off, new_len, st = eng.compress_device(d_in, off[:3], ln[:3], stream=s)
        h = d_new.cpu()
    assert (st == 0).all()
    assert _streams(h, new_off, new_len) == _streams(one[0], one[1], one[2])[:3]


@gpu
def test_compress_4096_text_streams_in_one_call(eng):
    """4096 x 64 KiB of text in one call on an 80 GB H100 (the encoder runs in as many sub-batches as its logs need); a sample
    of the streams equals the host route's.  The call holds the raw bytes, blob regions of lz77_blob_cap and the output next
    to the contexts' buffers, about 4 GiB in all."""
    import torch
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info(0)[0]
    if free < (8 << 30):
        pytest.skip("needs 8 GiB free next to the other contexts of this process; %.1f GiB are" % (free / 2 ** 30))
    blob, off, ln = synth.text_streams(4096, 65536)
    d_in = torch.from_numpy(np.ascontiguousarray(blob)).to("cuda:0")
    d_new, new_off, new_len, st = eng.compress_device(d_in, off, ln)
    assert (st == 0).all()
    idx = list(range(0, 4096, 97))
    raws = [blob[int(off[i]):int(off[i] + ln[i])].tobytes() for i in idx]
    want = eng.encode(_host(raws), divans_b200.encode_options(window_size=16), cmds=True)
    h = d_new.cpu().numpy()
    assert [h[int(new_off[i]):int(new_off[i] + new_len[i])].tobytes() for i in idx] == want
