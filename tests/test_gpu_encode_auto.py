"""encode_auto on the GPU: the cost-only model pass against the oracle's tally, the selection, and the streams it encodes."""
import numpy as np
import pytest

import divans_b200
from divans_b200 import synth
from oracle_tally import tally_py as T

pytestmark = pytest.mark.gpu

CANDS = divans_b200.DEFAULT_LITERAL_MODELS


def _records(n, width, seed):
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n].tobytes()


def _mixed():
    """text, UTF-8 text, records of 2 / 4 / 8 bytes, Bernoulli bits, random bytes, empty and 1-byte streams, and lengths
    around 2^10 (window 10: one, two and three literal commands)"""
    blob, off, ln = synth.text_streams(4, 3000, seed=9)
    text = [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)]
    cyr = b"".join(chr(0x430 + (c % 26)).encode() if 97 <= c < 123 else bytes([c]) for c in text[1])[:3000]
    bern = synth.bernoulli_streams(1, 2000, 0.2, seed=4)[0].tobytes()
    rnd = np.random.default_rng(2).integers(0, 256, 2000, dtype=np.uint8).tobytes()
    return [text[0], cyr, _records(3000, 2, 1), _records(3000, 4, 2), _records(3000, 8, 3), bern, rnd, b"", b"Q",
            text[2][:1023], text[3][:1025], (text[2] + text[3])[:2049]]


def _check_batch(engine, O, raws, opts, okw, blend, cands=CANDS):
    """O: the oracle of the probability model (for decoding); okw: its encoder options"""
    blob, off, ln, out, ooff, ocap = _layout(raws)
    out_len, status, chosen, cost = engine.encode_auto_batch_host(blob, off, ln, out, ooff, ocap, opts, cands)
    for i, r in enumerate(raws):
        ref = np.array([T.tally_raw(r, pm, mv, blend, **okw)[1] for pm, mv in cands], np.uint64)
        assert (cost[i] == ref).all(), "stream %d (%d bytes): GPU cost %s, oracle %s" % (i, len(r), cost[i], ref)
        assert chosen[i] == int(np.argmin(ref)), i
        rc, want, och, _ = T.encode_auto(r, cands, blend, **okw)
        assert rc == 0 and och == chosen[i] and status[i] == 0
        got = out[int(ooff[i]):int(ooff[i] + out_len[i])].tobytes()
        assert got == want, "stream %d: auto-encoded stream differs from the oracle's" % i
        assert O.decode(got, out_cap=len(r) + 64)[1] == r
    return out_len, status, chosen, cost, [out[int(o):int(o + n)].tobytes() for o, n in zip(ooff, out_len)]


def _layout(raws):
    in_len = np.array([len(r) for r in raws], np.uint64)
    pad = (in_len + np.uint64(15)) & ~np.uint64(15)
    off = np.concatenate([[0], np.cumsum(pad)[:-1]]).astype(np.uint64)
    blob = np.zeros(int(pad.sum()) + 16, np.uint8)
    for r, o in zip(raws, off):
        blob[int(o):int(o) + len(r)] = np.frombuffer(r, np.uint8)
    ocap = (in_len + in_len // np.uint64(2) + np.uint64(70000 + 255)) & ~np.uint64(255)
    ooff = np.concatenate([[0], np.cumsum(ocap)[:-1]]).astype(np.uint64)
    return blob, off, in_len, np.zeros(int(ocap.sum()), np.uint8), ooff, ocap


@pytest.mark.parametrize("blend,dcm", [(False, 0), (False, 1), (False, 2), (True, 0), (True, 1), (True, 2)])
def test_cost_and_streams_match_oracle(engine, oracle, oracle_blend, blend, dcm):
    O = oracle_blend if blend else oracle
    raws = _mixed()
    opts = divans_b200.encode_options(window_size=10, dynamic_context_mixing=dcm, cdf_model=int(blend))
    _, _, chosen, _, streams = _check_batch(engine, O, raws, opts, dict(window_size=10, dynamic_context_mixing=dcm), blend)
    # each stream is the plain encoder's with the chosen candidate
    for c in sorted(set(chosen.tolist())):
        idx = [i for i in range(len(raws)) if chosen[i] == c]
        pm, mv = CANDS[c]
        plain = engine.encode([raws[i] for i in idx], divans_b200.encode_options(window_size=10, dynamic_context_mixing=dcm,
                                                                                 cdf_model=int(blend), literal_pred_mode=pm,
                                                                                 literal_mixing_value=mv))
        assert plain == [streams[i] for i in idx]
    if not blend:   # and the GPU decoder reads them back
        res = engine.decode(streams, [len(r) + 64 for r in raws])
        assert [(s, o) for s, o in res] == [(0, r) for r in raws]
    else:
        res = engine.decode(streams, [len(r) + 64 for r in raws], divans_b200.FLAG_CDF_BLEND)
        assert [(s, o) for s, o in res] == [(0, r) for r in raws]
    assert len(set(chosen.tolist())) > 2   # the mixed batch really picks different models


def test_device_matches_host(engine):
    import torch
    raws = _mixed()
    blob, off, ln, out, ooff, ocap = _layout(raws)
    opts = divans_b200.encode_options(window_size=10)
    h_len, h_st, h_ch, h_cost = engine.encode_auto_batch_host(blob, off, ln, out, ooff, ocap, opts)
    n, C = len(raws), len(CANDS)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
    d_in = torch.from_numpy(blob).cuda()
    d_off, d_len, d_oo, d_cap = t(off), t(ln), t(ooff), t(ocap)
    d_out = torch.zeros(out.size, dtype=torch.uint8, device="cuda")
    d_ol = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int32, device="cuda")
    d_ch = torch.full((n,), 99, dtype=torch.int32, device="cuda")
    d_cost = torch.zeros(n * C, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    engine.encode_auto_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()), d_out.data_ptr(), d_oo.data_ptr(),
                                    d_cap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), d_ch.data_ptr(), d_cost.data_ptr(), opts, None,
                                    s.cuda_stream)
    torch.cuda.synchronize()
    assert (d_st.cpu().numpy() == h_st).all() and (d_ol.cpu().numpy().view(np.uint64) == h_len).all()
    assert (d_ch.cpu().numpy().view(np.uint32) == h_ch).all()
    assert (d_cost.cpu().numpy().view(np.uint64).reshape(n, C) == h_cost).all()
    o = d_out.cpu().numpy()
    for i in range(n):
        a, b = int(ooff[i]), int(ooff[i] + h_len[i])
        assert o[a:b].tobytes() == out[a:b].tobytes()
    # without a cost matrix
    d_ch.fill_(99)
    engine.encode_auto_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()), d_out.data_ptr(), d_oo.data_ptr(),
                                    d_cap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), d_ch.data_ptr(), None, opts, None, s.cuda_stream)
    torch.cuda.synchronize()
    assert (d_ch.cpu().numpy().view(np.uint32) == h_ch).all()


def test_more_pairs_than_slots_and_slot_reuse(engine):
    """a context with 32 slots: 20 streams x 8 candidates run through them five times over; a plain encode before and a
    decode in between leave no state behind"""
    small = divans_b200.Engine(0, 32, 16)
    try:
        blob, off, ln = synth.text_streams(20, 1500, seed=21)
        raws = [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)]
        raws[3::4] = [_records(1500, 4, k) for k in range(5)]
        opts = divans_b200.encode_options(window_size=10)
        small.encode([r[::-1] for r in raws], divans_b200.encode_options(literal_pred_mode=3, literal_mixing_value=9))
        ref = engine.encode_auto(raws, opts)
        got = small.encode_auto(raws, opts)
        assert got == ref
        assert [s for s, _, _ in got] == [0] * len(raws)
        assert small.decode([b for _, b, _ in got], [len(r) + 64 for r in raws]) == [(0, r) for r in raws]
        assert small.encode_auto(raws, opts) == ref
        assert [c for _, _, c in ref] == [T.encode_auto(r, CANDS, window_size=10)[2] for r in raws]
    finally:
        small.close()


def test_status_contract(engine):
    raws = _mixed()[:5]
    blob, off, ln, out, ooff, ocap = _layout(raws)
    full_len, st, chosen, _ = engine.encode_auto_batch_host(blob, off, ln, out, ooff, ocap)
    assert (st == 0).all()
    ocap2 = ocap.copy()
    ocap2[1] = full_len[1] - 1
    out2 = np.zeros_like(out)
    l2, st2, ch2, _ = engine.encode_auto_batch_host(blob, off, ln, out2, ooff, ocap2)
    assert st2[1] == divans_b200.DIVANS_NEEDS_MORE_OUTPUT and l2[1] == full_len[1]
    assert (ch2 == chosen).all() and [s for i, s in enumerate(st2) if i != 1] == [0] * 4
    # invalid candidate lists are refused before any work; an empty batch succeeds
    for bad in ([], [(0, 4)] * 17, [(4, 4)], [(0, 16)], [(-1, 4)], [(0, -1)]):
        with pytest.raises(divans_b200.DivansError):
            engine.encode_auto_batch_host(blob, off, ln, out2, ooff, ocap, None, bad)
    e = np.zeros(0, np.uint64)
    l0, s0, c0, k0 = engine.encode_auto_batch_host(blob, e, e, out2, e, e)
    assert l0.size == s0.size == c0.size == k0.size == 0
    assert engine.encode_auto([]) == []
