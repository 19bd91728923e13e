"""LZ77 parses on the GPU and the choice of one of k command lists per stream by coding cost:
divans_b200_lz77_cmds_batch_device_parse against the host generator (divans_b200_lz77_cmds_batch_parse) and the oracle
(dvo_lz77_cmds_parse); divans_b200_encode_cmds_choose_batch_device against the oracle's tallies and against
encode_cmds_batch_device of the chosen list; Engine.compress_device(parses=...) against the host route."""
import lzma
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import divans_b200  # noqa: E402
from divans_b200 import synth  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402

gpu = pytest.mark.gpu
MIN_MATCHES = (4, 5, 6, 7, 8, 12, 16, 32)
PARSES = [(m, z) for m in MIN_MATCHES for z in range(3)]
CANARY = 0x5A
G = 64


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="module")
def eng():
    """a context of its own with 64 resident streams: the n * k pairs of a choice run through its slots in waves"""
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


def _host(raws, parse, window=16, pm=2, mv=4):
    blob, off, ln = divans_b200._pack(raws)
    out, boff, blen = divans_b200.lz77_cmds_batch(blob, off, ln, window, pm, mv, parse=parse)
    return [out[int(o):int(o + l)].tobytes() for o, l in zip(boff, blen)]


def _u64(a):
    import torch
    return torch.from_numpy(np.array(a, np.uint64).reshape(-1).view(np.int64)).to("cuda:0")


def _device(eng, raws, parse, window=16, caps=None):
    """lz77_cmds_batch_device under `parse`, guard bytes around every region: [(status, blob_len, region bytes)]"""
    import torch
    n = len(raws)
    blob, off, ln = divans_b200._pack(raws)
    caps = divans_b200.lz77_blob_cap(ln) if caps is None else np.array(caps, np.uint64)
    boff, pos = [], G
    for c in caps:
        boff.append(pos)
        pos = (pos + int(c) + G + 15) & ~15
    d_in = torch.from_numpy(blob).to("cuda:0")
    d_blobs = torch.full((pos,), CANARY, dtype=torch.uint8, device="cuda:0")
    m = [_u64(off), _u64(ln), _u64(boff), _u64(caps)]
    d_len = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda:0")
    d_st = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda:0")
    torch.cuda.current_stream().synchronize()
    eng.lz77_cmds_batch_device(n, d_in.data_ptr(), m[0].data_ptr(), m[1].data_ptr(), int(ln.max()) if n else 0, window, 2, 4,
                               d_blobs.data_ptr(), m[2].data_ptr(), m[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), parse=parse)
    eng.synchronize()
    o = d_blobs.cpu().numpy()
    mask = np.ones(o.size, bool)
    for a, c in zip(boff, caps):
        mask[a:a + int(c)] = False
    assert (o[mask] == CANARY).all(), "a byte outside the blob regions changed"
    st, bl = d_st.cpu().numpy()[:n], d_len.cpu().numpy()[:n].view(np.uint64)
    return [(int(s), int(l), o[a:a + int(c)].tobytes()) for s, l, a, c in zip(st, bl, boff, caps)]


def _records_of(blob):
    h = np.frombuffer(blob[:32], np.uint32)
    return np.frombuffer(blob[32:32 + 20 * int(h[2])], np.uint32).reshape(-1, 5)


def _agree(eng, oracle, raws, parse, window=16, what=""):
    """device blobs == host blobs, and the host's commands == the oracle's (the oracle's literal pool is its own)"""
    want = _host(raws, parse, window)
    got = _device(eng, raws, parse, window)
    for i, ((s, l, region), w, r) in enumerate(zip(got, want, raws)):
        assert s == 0 and l == len(w), "%s %s stream %d (%d bytes): status %d, blob_len %d, host %d" % (what, parse, i, len(r), s, l, len(w))
        if region[:l] != w:
            k = int(np.nonzero(np.frombuffer(region[:l], np.uint8) != np.frombuffer(w, np.uint8))[0][0])
            raise AssertionError("%s %s stream %d (%d bytes): blob differs from the host's at byte %d" % (what, parse, i, len(r), k))
        rec, ref = _records_of(w), _records_of(T.lz77_parse(oracle, r, *parse, window=window).serialize())
        cp = ref[:, 0] == 1
        assert rec.shape == ref.shape and (rec[:, 0] == ref[:, 0]).all() and (rec[cp, 1:3] == ref[cp, 1:3]).all() \
            and (rec[~cp, 2] == ref[~cp, 2]).all(), "%s %s stream %d: commands differ from the oracle's" % (what, parse, i)
        assert (rec[cp, 2] >= parse[0]).all()
    return want


def _edges(seed=5):
    """inputs whose copies and lookaheads end on 32-position window edges: text and periodic data of every length around the
    multiples of 32, and repeats placed so that a match starts at positions 29..31 of a window"""
    rng = np.random.default_rng(seed)
    t = _text(4096, seed)
    raws = [t[:n] for n in list(range(28, 100)) + [126, 127, 128, 129, 130, 159, 160, 161, 191, 192, 193]]
    for p in (3, 5, 31, 33):
        rec = rng.integers(0, 256, p, dtype=np.uint8).tobytes()
        raws += [(rec * (300 // p + 2))[:n] for n in (62, 63, 64, 65, 66, 95, 96, 97)]
    for at in range(26, 36):
        base = bytearray(rng.integers(0, 256, 200, dtype=np.uint8).tobytes())
        word = base[:12]
        base[at + 32:at + 32 + 12] = word                 # a 12-byte repeat starting near a window's end
        base[at + 33:at + 33 + 14] = base[40:54]          # and a longer one a byte later (a lazy deferral)
        raws.append(bytes(base))
    return raws


@gpu
@pytest.mark.parametrize("parse", PARSES, ids=["%d,%d" % p for p in PARSES])
def test_device_equals_host_and_oracle(eng, oracle, parse):
    rng = np.random.default_rng(parse[0] * 3 + parse[1])
    raws = [b""] + [_text(n, n) for n in range(1, 41)] + _edges()
    raws += [bytes(5000), bytes([7]) * 70000, b"ab" * 20000, rng.integers(0, 4, 30000, dtype=np.uint8).tobytes(),
             rng.integers(0, 256, 20000, dtype=np.uint8).tobytes(), _text(200000, 3)]
    raws += [rng.integers(0, 256, 11, dtype=np.uint8).tobytes() * 3000]
    raws += _fixtures(oracle)
    _agree(eng, oracle, raws, parse)


@gpu
@pytest.mark.parametrize("window", [10, 12, 14, 16, 18, 20, 22, 24])
def test_windows(eng, oracle, window):
    raws = [_text(min(1 << (window + 1), 1 << 20), window), _text(70000, 2)] + _edges(window)
    for parse in ((4, 0), (5, 1), (7, 2), (32, 2)):
        _agree(eng, oracle, raws, parse, window)


@gpu
def test_region_too_small(eng):
    raws = [_text(5000, 2), b"", _text(70000, 3)]
    for parse in ((6, 1), (7, 2)):
        want = _host(raws, parse)
        for caps in ([0] * 3, [len(w) - 1 for w in want], [len(w) for w in want]):
            for (s, l, region), w, c in zip(_device(eng, raws, parse, caps=caps), want, caps):
                assert l == len(w)
                assert (s == 2) if c < len(w) else (s == 0 and region[:l] == w)


@gpu
def test_out_of_domain_parse_is_refused(eng):
    for bad in ((3, 0), (33, 1), (4, 3), (8, -1)):
        with pytest.raises(divans_b200.DivansError, match="outside min_match 4..32"):
            _device(eng, [_text(1000)], bad)


# ---------------------------------------------------------------------------------------------------------------------
# choosing one of k command lists
# ---------------------------------------------------------------------------------------------------------------------
def _choose(eng, lists, max_raw, opts, choose_only=False):
    """lists[i][c]: list c of stream i.  encode_cmds_choose_batch_device -> (status, streams, chosen, cost [n, k])"""
    import torch
    n, k = len(lists), len(lists[0])
    flat = [lists[i][c] for c in range(k) for i in range(n)]   # candidate-major
    blob, off, ln = divans_b200._pack(flat)
    max_blob = int(ln.max())
    cap = divans_b200._encoded_cap(np.array([max(len(b) for b in row) for row in lists], np.uint64))
    out_off, total = divans_b200._regions(cap)
    d_b = torch.from_numpy(blob).to("cuda:0")
    m = [_u64(off), _u64(ln), _u64(out_off), _u64(cap)]
    d_out = torch.zeros(total, dtype=torch.uint8, device="cuda:0")
    d_len = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda:0")
    d_ch = torch.full((n,), -1, dtype=torch.int32, device="cuda:0")
    d_cost = torch.zeros(n * k, dtype=torch.int64, device="cuda:0")
    torch.cuda.current_stream().synchronize()
    eng.encode_cmds_choose_batch_device(n, k, d_b.data_ptr(), m[0].data_ptr(), m[1].data_ptr(), max_blob, max_raw,
                                        None if choose_only else d_out.data_ptr(), m[2].data_ptr(), m[3].data_ptr(), d_len.data_ptr(),
                                        d_st.data_ptr(), d_ch.data_ptr(), d_cost.data_ptr(), opts)
    eng.synchronize()
    st, ln_, o = d_st.cpu().numpy(), d_len.cpu().numpy().view(np.uint64), d_out.cpu().numpy()
    streams = [o[int(a):int(a + l)].tobytes() for a, l in zip(out_off, ln_)]
    return st, streams, d_ch.cpu().numpy().view(np.uint32), d_cost.cpu().numpy().view(np.uint64).reshape(n, k), max_blob


def _plain(eng, blobs, max_blob, max_raw, opts):
    """encode_cmds_batch_device of the lists `blobs` with the given capacities -> (status, streams)"""
    import torch
    n = len(blobs)
    blob, off, ln = divans_b200._pack(blobs)
    cap = divans_b200._encoded_cap(ln)
    out_off, total = divans_b200._regions(cap)
    d_b = torch.from_numpy(blob).to("cuda:0")
    m = [_u64(off), _u64(ln), _u64(out_off), _u64(cap)]
    d_out = torch.zeros(total, dtype=torch.uint8, device="cuda:0")
    d_len = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda:0")
    torch.cuda.current_stream().synchronize()
    eng.encode_cmds_batch_device(n, d_b.data_ptr(), m[0].data_ptr(), m[1].data_ptr(), max_blob, max_raw, d_out.data_ptr(), m[2].data_ptr(),
                                 m[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), opts)
    eng.synchronize()
    st, ln_, o = d_st.cpu().numpy(), d_len.cpu().numpy().view(np.uint64), d_out.cpu().numpy()
    return st, [o[int(a):int(a + l)].tobytes() for a, l in zip(out_off, ln_)]


def _check_choice(eng, oracle, lists, raws, opts, blend=False, okw=None, expect_ok=None):
    """chosen and cost equal the oracle's, each stream equals encode_cmds_batch_device of its chosen list, and decodes to its raw"""
    max_raw = max(len(r) for r in raws)
    st, streams, chosen, cost, max_blob = _choose(eng, lists, max_raw, opts)
    okw = okw or {}
    for i, row in enumerate(lists):
        want = [T.tally_cmds(T.from_blob(oracle, b), blend=blend, **okw)[1] for b in row]
        assert list(cost[i]) == want, "stream %d: costs differ from the oracle's" % i
        assert chosen[i] == int(np.argmin(want)), "stream %d" % i
    pst, pstreams = _plain(eng, [row[c] for row, c in zip(lists, chosen)], max_blob, max_raw, opts)
    assert list(st) == list(pst)
    assert [s for s, x in zip(streams, st) if x == 0] == [s for s, x in zip(pstreams, pst) if x == 0]
    if expect_ok is not None:
        assert list(st == 0) == list(expect_ok)
    ok = [i for i in range(len(raws)) if st[i] == 0]
    flags = divans_b200.FLAG_CDF_BLEND if blend else 0
    dec = eng.decode([streams[i] for i in ok], [len(raws[i]) + 64 for i in ok], flags)
    assert all(s == 0 and b == raws[i] for (s, b), i in zip(dec, ok))
    # the choice alone: the same chosen and cost
    _, _, ch2, co2, _ = _choose(eng, lists, max_raw, opts, choose_only=True)
    assert (ch2 == chosen).all() and (co2 == cost).all()
    return st, streams, chosen, cost


def _mixed_raws(oracle, n=40, seed=3):
    rng = np.random.default_rng(seed)
    raws = []
    for i in range(n):
        k = int(rng.integers(0, 30000))
        raws.append(_text(k, i) if i % 3 else rng.integers(0, 6 if i % 2 else 256, k, dtype=np.uint8).tobytes())
    return raws + _fixtures(oracle) + [b""]


@gpu
@pytest.mark.parametrize("blend", [False, True], ids=["frequentist", "blend"])
def test_choose_generated_lists(eng, oracle, blend):
    """the device generator's lists under DEFAULT_LZ77_PARSES (and one more): 3 x 16 + ... pairs on 64 slots, in waves"""
    raws = _mixed_raws(oracle)
    parses = divans_b200.DEFAULT_LZ77_PARSES + [(32, 0)]
    per = [[g[2][:g[1]] for g in _device(eng, raws, p)] for p in parses]
    lists = [[per[c][i] for c in range(len(parses))] for i in range(len(raws))]
    opts = divans_b200.encode_options(window_size=16, dynamic_context_mixing=1, cdf_model=int(blend))
    _check_choice(eng, oracle, lists, raws, opts, blend, dict(window_size=16, dynamic_context_mixing=1))


@gpu
def test_choose_host_and_ir_lists(eng, oracle):
    """lists from any source: host-generated lists next to the IR fixture's own list and a literal-only list"""
    g = os.path.join(ROOT, "tests", "golden")
    ir = lzma.decompress(open(os.path.join(g, "asyoulik.ir.xz"), "rb").read())
    ir_blob, _ = divans_b200.ir_to_cmds(ir)
    rc, ayl = oracle.Commands.from_ir(ir).recode(22)
    raws = [ayl, _text(50000, 4), _text(3000, 5)]
    lists = []
    for r in raws:
        row = [b for p in ((4, 0), (7, 2)) for b in _host([r], p, window=22)]
        row.append(ir_blob if r is ayl else _host([r], (12, 1), window=22)[0])
        lists.append(row)
    opts = divans_b200.encode_options(window_size=22)
    _check_choice(eng, oracle, lists, raws, opts, okw=dict(window_size=22))


@gpu
def test_choose_with_failing_lists(eng, oracle):
    """a list with copies farther than the 2^10 window fails: a stream whose lists all fail fails as the plain call does on list 0
    (chosen 0, every cost UINT64_MAX), next to streams with one failing and one good list, and streams with good ones only"""
    raws = [_text(30000, k) for k in range(6)]
    far = [_host([r], (4, 0), window=20)[0] for r in raws]
    near = [_host([r], (6, 1), window=10)[0] for r in raws]
    lists = [[far[0], far[0]], [far[1], near[1]], [near[2], far[2]], [near[3], near[3]], [far[4], far[4]], [near[5], far[5]]]
    opts = divans_b200.encode_options(window_size=10)
    st, _, chosen, cost = _check_choice(eng, oracle, lists, raws, opts, okw=dict(window_size=10),
                                        expect_ok=[False, True, True, True, False, True])
    assert chosen[0] == 0 and chosen[4] == 0 and (cost[[0, 4]] == T.TALLY_FAILED).all()
    assert list(chosen[[1, 2]]) == [1, 0]


@gpu
def test_choose_refusals(eng):
    import torch
    d = torch.zeros(64, dtype=torch.int64, device="cuda:0")
    p = d.data_ptr()
    for k in (0, 17):
        with pytest.raises(divans_b200.DivansError, match="1..16 command lists"):
            eng.encode_cmds_choose_batch_device(1, k, p, p, p, 100, 100, p, p, p, p, p, p, p)
    with pytest.raises(divans_b200.DivansError, match="d_chosen is required"):
        eng.encode_cmds_choose_batch_device(1, 2, p, p, p, 100, 100, p, p, p, p, p, None, p)


# ---------------------------------------------------------------------------------------------------------------------
# compress_device(parses=...)
# ---------------------------------------------------------------------------------------------------------------------
def _on_device(raws):
    import torch
    blob, off, ln = divans_b200._pack(raws)
    return torch.from_numpy(blob).to("cuda:0"), off, ln


def _streams(d_new, off, ln):
    h = d_new.cpu().numpy()
    return [h[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]


def _host_route(eng, oracle, raws, parses, opts, okw, candidates=None):
    """generate every parse's list on the host, choose by the oracle's tally, encode the chosen lists (encode_cmds_auto with
    candidates) -> (streams, chosen parse, parse costs)"""
    per = [_host(raws, p) for p in parses]
    cost = np.array([[T.tally_cmds(T.from_blob(oracle, per[c][i]), **okw)[1] for c in range(len(parses))] for i in range(len(raws))],
                    np.uint64)
    ch = cost.argmin(1)
    lists = [per[c][i] for i, c in enumerate(ch)]
    if candidates is None:
        return eng.encode(lists, opts, cmds=True), ch, cost
    res = eng.encode_cmds_auto(lists, opts, candidates)
    return [b for _, b, _ in res], ch, cost, [c for _, _, c in res]


@gpu
def test_compress_device_parses_equals_host_route(eng, oracle):
    raws = _mixed_raws(oracle, 60, 9) + [_text(65536, 10)]
    d_in, off, ln = _on_device(raws)
    opts = divans_b200.encode_options(window_size=16)
    parses = divans_b200.DEFAULT_LZ77_PARSES
    want, ch, cost = _host_route(eng, oracle, raws, parses, opts, dict(window_size=16))
    d_new, new_off, new_len, st, chosen, pcost = eng.compress_device(d_in, off, ln, opts=opts, parses=parses)
    assert (st == 0).all() and (chosen == ch).all() and (pcost == cost).all()
    got = _streams(d_new, new_off, new_len)
    assert got == want
    dec = eng.decode(got, [len(r) + 64 for r in raws])
    assert all(s == 0 and b == r for (s, b), r in zip(dec, raws))
    # sub-batches give the same streams
    d2, o2, l2, st2, ch2, co2 = eng.compress_device(d_in, off, ln, opts=opts, parses=parses, sub_batch=7)
    assert eng.last_compress_sub_batches == (len(raws) + 6) // 7
    assert (st2 == 0).all() and (ch2 == ch).all() and _streams(d2, o2, l2) == want
    # the plain call is unchanged by the new keyword
    z = eng.compress_device(d_in, off, ln, opts=opts)
    assert len(z) == 4 and _streams(z[0], z[1], z[2]) == eng.encode(_host(raws, (4, 0)), opts, cmds=True)


@gpu
def test_compress_device_parses_and_candidates(eng, oracle):
    raws = _mixed_raws(oracle, 30, 11)
    d_in, off, ln = _on_device(raws)
    opts = divans_b200.encode_options(window_size=16)
    cands = [divans_b200.LITERAL_MODEL_KEEP] + divans_b200.DEFAULT_LITERAL_MODELS
    parses = divans_b200.DEFAULT_LZ77_PARSES
    want, ch, cost, mch = _host_route(eng, oracle, raws, parses, opts, dict(window_size=16), cands)
    d_new, new_off, new_len, st, chosen, mcost, pch, pcost = eng.compress_device(d_in, off, ln, opts=opts, candidates=cands, parses=parses)
    assert (st == 0).all() and (pch == ch).all() and (pcost == cost).all() and list(chosen) == mch
    assert mcost.shape == (len(raws), len(cands))
    assert _streams(d_new, new_off, new_len) == want


@gpu
def test_compress_device_parses_no_larger_than_greedy(eng, oracle):
    """on the synthetic text and the fixtures, the chosen streams total no more bytes than the (4, 0) streams, and with the
    parse costs (4, 0) is never cheaper than the choice"""
    blob, off, ln = synth.text_streams(64, 65536)
    raws = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)] + _fixtures(oracle)
    d_in, off, ln = _on_device(raws)
    z = eng.compress_device(d_in, off, ln)
    c = eng.compress_device(d_in, off, ln, parses=divans_b200.DEFAULT_LZ77_PARSES)
    assert (z[3] == 0).all() and (c[3] == 0).all()
    assert int(c[2].sum()) <= int(z[2].sum())
    assert (c[5][np.arange(len(raws)), c[4]] <= c[5][:, 0]).all()
    dec = eng.decode(_streams(c[0], c[1], c[2]), [len(r) + 64 for r in raws])
    assert all(s == 0 and b == r for (s, b), r in zip(dec, raws))
