"""Per-context mixing values on the GPU (encode_mixmap / encode_cmds_mixmap): the binned cost pass, the per-entry choice, the
mixed pass and the streams, against the CPU oracle (oracle_tally: dvo_encode_mixmap, dvo_encode_cmds_mixmap)."""
import numpy as np
import pytest

import divans_b200
import test_gpu_encode_auto as A
import test_gpu_encode_cmds_auto as C
from oracle_tally import tally_py as T

pytestmark = pytest.mark.gpu

VALUES = divans_b200.DEFAULT_MIXING_VALUES
K = len(VALUES)


def _raws():
    """A._mixed() (text, UTF-8, 2/4/8-byte records, bits, random, empty, 1 byte, lengths around 2^10) and text then records"""
    r = A._mixed()
    return r + [r[0][:1500] + A._records(1500, 4, 7), A._records(1200, 2, 8) + A._records(1200, 8, 9)]


def _check(got, want, name):
    (st, ln, out, ch, mixing, cost, bins) = got
    rc, wout, wch, wmix, wcost, wbins = want
    assert (cost == wcost).all(), "%s: GPU cost %s, oracle %s" % (name, cost, wcost)
    assert (bins == wbins).all(), "%s: bins differ at %s" % (name, np.argwhere(bins != wbins)[:4].tolist())
    assert ch == wch and (mixing == wmix).all(), name
    assert rc == st == 0 and out == wout, "%s: stream differs from the oracle's" % name


def _host(eng, blobs, opts, cmds, values=VALUES):
    buf, off, ln, out, ooff, ocap = C._host_layout(blobs)
    fn = eng.encode_cmds_mixmap_batch_host if cmds else eng.encode_mixmap_batch_host
    out_len, st, chosen, mixing, cost, bins = fn(buf, off, ln, out, ooff, ocap, opts, values, bins=True)
    return [(int(st[i]), int(out_len[i]), out[int(ooff[i]):int(ooff[i] + out_len[i])].tobytes(), int(chosen[i]), mixing[i], cost[i],
             bins[i]) for i in range(len(blobs))]


def _device(eng, blobs, opts, cmds, values=VALUES):
    import torch
    n, k = len(blobs), len(values)
    buf, off, ln, out, ooff, ocap = C._host_layout(blobs)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    i64 = lambda a: dev(np.asarray(a, np.uint64).view(np.int64))
    d_in, d_off, d_len, d_out, d_ooff, d_ocap = dev(buf), i64(off), i64(ln), dev(out), i64(ooff), i64(ocap)
    d_olen, d_st = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d_ch = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_mix = torch.zeros(n * 8192, dtype=torch.uint8, device="cuda")
    d_cost = torch.zeros(n * (k + 1), dtype=torch.int64, device="cuda")
    d_bins = torch.zeros(n * k * 8192, dtype=torch.int64, device="cuda")
    outs = dict(d_chosen=d_ch.data_ptr(), d_mixing=d_mix.data_ptr(), d_cost=d_cost.data_ptr(), d_bins=d_bins.data_ptr(), opts=opts, values=values)
    if cmds:
        eng.encode_cmds_mixmap_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()),
                                            max(C._replay_len(b) for b in blobs) + 1, d_out.data_ptr(), d_ooff.data_ptr(), d_ocap.data_ptr(),
                                            d_olen.data_ptr(), d_st.data_ptr(), **outs)
    else:
        eng.encode_mixmap_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()), d_out.data_ptr(),
                                       d_ooff.data_ptr(), d_ocap.data_ptr(), d_olen.data_ptr(), d_st.data_ptr(), **outs)
    eng.synchronize()
    o, olen, st = d_out.cpu().numpy(), d_olen.cpu().numpy(), d_st.cpu().numpy()
    mix, cost = d_mix.cpu().numpy().reshape(n, 8192), d_cost.cpu().numpy().view(np.uint64).reshape(n, k + 1)
    bins = d_bins.cpu().numpy().view(np.uint64).reshape(n, k, 8192)
    ch = d_ch.cpu().numpy()
    return [(int(st[i]), int(olen[i]), o[int(ooff[i]):int(ooff[i] + olen[i])].tobytes(), int(ch[i]), mix[i], cost[i], bins[i])
            for i in range(n)]


@pytest.mark.parametrize("blend,dcm", [(False, 0), (False, 1), (False, 2), (True, 0), (True, 1), (True, 2)])
@pytest.mark.parametrize("call", ["host", "device"])
def test_raw_matches_oracle(engine, oracle, oracle_blend, blend, dcm, call):
    O = oracle_blend if blend else oracle
    raws = _raws()
    okw = dict(window_size=10, dynamic_context_mixing=dcm)
    opts = divans_b200.encode_options(cdf_model=int(blend), literal_pred_mode=2, **okw)
    res = (_host if call == "host" else _device)(engine, raws, opts, False)
    for i, r in enumerate(raws):
        want = T.encode_mixmap(r, 2, VALUES, blend, **okw)
        _check(res[i], want, "stream %d (%d bytes)" % (i, len(r)))
        if res[i][3] < K:   # a uniform choice: the plain encoder's stream with that value
            assert res[i][2] == engine.encode([r], divans_b200.encode_options(cdf_model=int(blend), literal_pred_mode=2,
                                                                              literal_mixing_value=VALUES[res[i][3]], **okw))[0]
    flag = divans_b200.FLAG_CDF_BLEND if blend else 0
    assert engine.decode([x[2] for x in res], [len(r) + 64 for r in raws], flag) == [(0, r) for r in raws]
    if dcm != 0:
        assert any(x[3] == K for x in res), "no stream took a mixed record"


@pytest.mark.parametrize("call", ["host", "device"])
def test_cmds_match_oracle(engine, oracle, call):
    lists = C._lists(oracle)
    blobs = [cl.serialize() for _, cl in lists]
    okw = dict(window_size=22, dynamic_context_mixing=1)
    opts = divans_b200.encode_options(literal_pred_mode=0, **okw)
    res = (_host if call == "host" else _device)(engine, blobs, opts, True)
    for i, (name, cl) in enumerate(lists):
        _check(res[i], T.encode_cmds_mixmap(cl, 0, VALUES, **okw), name)
    replays = [oracle.decode(cl.encode(oracle.options(window_size=22)))[1] for _, cl in lists]
    assert engine.decode([x[2] for x in res], [len(r) + 64 for r in replays]) == [(0, r) for r in replays]


def test_waves_and_slot_succession(oracle):
    """a batch larger than the encoder slots (a context of 64) runs in waves; one decode slot then runs mixed, uniform and mixed
    streams in turn and decodes each exactly"""
    raws = _raws() * 8
    opts = divans_b200.encode_options(literal_pred_mode=2, window_size=10)
    eng = divans_b200.Engine(0, 64, 16)
    try:
        res = _host(eng, raws, opts, False)
        for i, r in enumerate(raws[:len(_raws())]):
            want = T.encode_mixmap(r, 2, VALUES, window_size=10)
            for j in range(i, len(raws), len(_raws())):
                _check(res[j], want, "stream %d" % j)
        mixed = [x[2] for x, r in zip(res, raws) if x[3] == K and len(r) > 1000]
        uni = [x[2] for x, r in zip(res, raws) if x[3] < K and len(r) > 1000]
        assert mixed and uni
        seq = [mixed[0], uni[0], mixed[1 % len(mixed)]]
        want = [oracle.decode(s, out_cap=1 << 16)[1] for s in seq]
        one = divans_b200.Engine(0, 1, 16)
        try:
            for s, w in zip(seq, want):
                assert one.decode([s], [len(w) + 64]) == [(0, w)]
                assert one.slot_header(0)[3] in (0, 1)
        finally:
            one.close()
    finally:
        eng.close()


def test_bad_values_are_refused(engine):
    buf, off, ln, out, ooff, ocap = C._host_layout([b"abc"])
    for vals, opts in (([], None), ([16], None), ([-1], None), (list(range(17)), None),
                       ([4], divans_b200.encode_options(literal_pred_mode=4))):
        with pytest.raises(divans_b200.DivansError):
            engine.encode_mixmap_batch_host(buf, off, ln, out, ooff, ocap, opts, vals if vals else np.zeros(0, np.int32))
