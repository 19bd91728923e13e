"""Literal speeds on the GPU (encode_speeds / encode_cmds_speeds): the uniform, halves and verify passes, the choice and the
streams, against the CPU oracle (oracle_tally: dvo_encode_speeds, dvo_encode_cmds_speeds)."""
import os

import numpy as np
import pytest

import divans_b200
import test_gpu_encode_auto as A
import regimes as R
import test_gpu_encode_cmds_auto as C
from oracle_tally import tally_py as T

pytestmark = pytest.mark.gpu

VALUES = divans_b200.DEFAULT_LITERAL_SPEEDS
K = len(VALUES)
MUD = (16, 8192)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _raws():
    """A._mixed() (text, UTF-8, records, bits, random, empty, 1 byte, lengths around 2^10) and text then records"""
    r = A._mixed()
    return r + [r[0][:1500] + A._records(1500, 4, 7)]


def _check(got, want, name):
    st, ln, out, ch, cost, halves = got
    rc, wout, wch, wcost, whalves = want
    assert (cost == wcost).all(), "%s: GPU cost %s, oracle %s" % (name, cost, wcost)
    assert (halves == whalves).all(), "%s: GPU halves %s, oracle %s" % (name, halves.tolist(), whalves.tolist())
    assert (ch == wch).all(), "%s: GPU chose %s, oracle %s" % (name, ch, wch)
    assert rc == st == 0 and out == wout, "%s: stream differs from the oracle's" % name


def _host(eng, blobs, opts, cmds, values=VALUES, caps=None):
    buf, off, ln, out, ooff, ocap = C._host_layout(blobs, caps)
    fn = eng.encode_cmds_speeds_batch_host if cmds else eng.encode_speeds_batch_host
    out_len, st, chosen, cost, halves = fn(buf, off, ln, out, ooff, ocap, opts, values)
    return [(int(st[i]), int(out_len[i]), out[int(ooff[i]):int(ooff[i] + out_len[i])].tobytes(), chosen[i], cost[i], halves[i])
            for i in range(len(blobs))]


def _device(eng, blobs, opts, cmds, values=VALUES):
    import torch
    n, k = len(blobs), len(values)
    buf, off, ln, out, ooff, ocap = C._host_layout(blobs)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    i64 = lambda a: dev(np.asarray(a, np.uint64).view(np.int64))
    d_in, d_off, d_len, d_out, d_ooff, d_ocap = dev(buf), i64(off), i64(ln), dev(out), i64(ooff), i64(ocap)
    d_olen, d_st = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d_ch = torch.zeros(n * 3, dtype=torch.int32, device="cuda")
    d_cost = torch.zeros(n * (k + 1), dtype=torch.int64, device="cuda")
    d_halves = torch.zeros(n * k * 2, dtype=torch.int64, device="cuda")
    outs = dict(d_chosen=d_ch.data_ptr(), d_cost=d_cost.data_ptr(), d_halves=d_halves.data_ptr(), opts=opts, values=values)
    if cmds:
        eng.encode_cmds_speeds_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()),
                                            max(C._replay_len(b) for b in blobs) + 1, d_out.data_ptr(), d_ooff.data_ptr(), d_ocap.data_ptr(),
                                            d_olen.data_ptr(), d_st.data_ptr(), **outs)
    else:
        eng.encode_speeds_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()), d_out.data_ptr(),
                                       d_ooff.data_ptr(), d_ocap.data_ptr(), d_olen.data_ptr(), d_st.data_ptr(), **outs)
    eng.synchronize()
    o, olen, st = d_out.cpu().numpy(), d_olen.cpu().numpy(), d_st.cpu().numpy()
    cost = d_cost.cpu().numpy().view(np.uint64).reshape(n, k + 1)
    halves = d_halves.cpu().numpy().view(np.uint64).reshape(n, k, 2)
    ch = d_ch.cpu().numpy().view(np.uint32).reshape(n, 3)
    return [(int(st[i]), int(olen[i]), o[int(ooff[i]):int(ooff[i] + olen[i])].tobytes(), ch[i], cost[i], halves[i]) for i in range(n)]


def _chosen_opts(base_kw, values, ch):
    a, b, c = (int(x) for x in ch)
    return divans_b200.encode_options(literal_adaptation=[values[a], values[a], values[b], values[c]], **base_kw)


def _golden_text(oracle):
    """alice29 and asyoulik from the golden streams (their raw SHA-256 is pinned in golden.json)"""
    out = []
    for name in ("alice29_literal_only.divans", "asyoulik_ir_mix2.divans"):
        rc, raw = oracle.decode(open(os.path.join(GOLDEN, name), "rb").read(), out_cap=1 << 20)[:2]
        assert rc == 0
        out.append(raw)
    return out


@pytest.mark.parametrize("blend,dcm", [(False, 0), (False, 1), (False, 2), (True, 0), (True, 1), (True, 2)])
@pytest.mark.parametrize("call", ["host", "device"])
def test_raw_matches_oracle(engine, oracle, oracle_blend, blend, dcm, call):
    raws = _raws()
    okw = dict(window_size=10, dynamic_context_mixing=dcm)
    base = dict(cdf_model=int(blend), literal_pred_mode=2, **okw)
    res = (_host if call == "host" else _device)(engine, raws, divans_b200.encode_options(**base), False)
    for i, r in enumerate(raws):
        _check(res[i], T.encode_speeds(r, 2, 4, VALUES, blend, **okw), "stream %d (%d bytes)" % (i, len(r)))
        assert res[i][2] == engine.encode([r], _chosen_opts(base, VALUES, res[i][3]))[0], "stream %d: contract" % i
    flag = divans_b200.FLAG_CDF_BLEND if blend else 0
    assert engine.decode([x[2] for x in res], [len(r) + 64 for r in raws], flag) == [(0, r) for r in raws]


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_every_mode(engine, oracle, mode):
    raws = _raws()
    okw = dict(window_size=12, dynamic_context_mixing=2)
    res = _host(engine, raws, divans_b200.encode_options(literal_pred_mode=mode, literal_mixing_value=5, **okw), False)
    for i, r in enumerate(raws):
        _check(res[i], T.encode_speeds(r, mode, 5, VALUES, **okw), "mode %d stream %d" % (mode, i))


@pytest.mark.parametrize("call", ["host", "device"])
@pytest.mark.parametrize("dcm", [1, 2])
def test_cmds_match_oracle(engine, oracle, call, dcm):
    lists = C._lists(oracle)
    blobs = [cl.serialize() for _, cl in lists]
    okw = dict(window_size=22, dynamic_context_mixing=dcm)
    opts = divans_b200.encode_options(literal_pred_mode=0, **okw)
    res = (_host if call == "host" else _device)(engine, blobs, opts, True)
    for i, (name, cl) in enumerate(lists):
        _check(res[i], T.encode_cmds_speeds(cl, VALUES, **okw), name)
        plain = C._plain_host(engine, [blobs[i]], _chosen_opts(dict(literal_pred_mode=0, **okw), VALUES, res[i][3]))
        assert plain[0][0] == 0 and plain[0][2] == res[i][2], "%s: contract" % name
    replays = [oracle.decode(cl.encode(oracle.options(window_size=22)))[1] for _, cl in lists]
    assert engine.decode([x[2] for x in res], [len(r) + 64 for r in replays]) == [(0, r) for r in replays]


def test_real_text_beats_mud(engine, oracle):
    """alice29 at dynamic mixing 2 gets strictly cheaper than under MUD alone, and decodes exactly"""
    texts = [t[:65536] for t in _golden_text(oracle)]
    okw = dict(window_size=22, dynamic_context_mixing=2)
    base = dict(literal_pred_mode=2, **okw)
    res = _host(engine, texts, divans_b200.encode_options(**base), False)
    mud = engine.encode(texts, divans_b200.encode_options(literal_adaptation=[MUD] * 4, **base))
    for i, t in enumerate(texts):
        _check(res[i], T.encode_speeds(t, 2, 4, VALUES, **okw), "text %d" % i)
    assert min(res[0][4][:K]) < res[0][4][0] or res[0][4][K] < res[0][4][0]
    assert len(res[0][2]) < len(mud[0])
    assert engine.decode([x[2] for x in res], [len(t) + 64 for t in texts]) == [(0, t) for t in texts]


def test_halves_match_binned_sums(engine, oracle):
    """the halves the fast loops tally equal the generic binned pass's sums: high = bins [0, 4096), low = bins [4096, 8192)"""
    text = _golden_text(oracle)[0][:16384]
    okw = dict(window_size=22, dynamic_context_mixing=2)
    res = _host(engine, [text], divans_b200.encode_options(literal_pred_mode=2, **okw), False)
    cs = int(res[0][3][0])
    for d in range(K):
        rc, cost, bins, nobin = T.tally_raw_bins(text, 2, 4, literal_adaptation=[VALUES[cs], VALUES[cs], VALUES[d], VALUES[d]], **okw)
        b = bins.astype(np.uint64)
        assert rc == 0 and int(res[0][5][d][0]) == int(b[4096:].sum()) and int(res[0][5][d][1]) == int(b[:4096].sum())


def test_status_2_and_waves(oracle):
    """a batch larger than the encoder slots (a context of 64) runs in waves; an output region too small gives status 2"""
    raws = _raws() * 8
    okw = dict(window_size=10, dynamic_context_mixing=2)
    opts = divans_b200.encode_options(literal_pred_mode=2, **okw)
    caps = [C._out_cap(r) for r in raws]
    caps[0] = 16
    eng = divans_b200.Engine(0, 64, 16)
    try:
        res = _host(eng, raws, opts, False, caps=caps)
        assert res[0][0] == 2
        for j in range(1, len(raws)):
            r = raws[j]
            _check(res[j], T.encode_speeds(r, 2, 4, VALUES, **okw), "stream %d" % j)
    finally:
        eng.close()


BAD = ([], [(1000, 16384)], [(-1, 1024)], [(16, 32767)], [(16384, 16384)], [(16, 8192)] * 17)


def test_bad_values_are_refused(engine, oracle):
    """every call refuses speeds that the f8 round trip changes, negative ones, (16384, 16384) (f8-exact, but it could wrap an
    i16 prior), and lists of 0 or 17 speeds, before any work: the device outputs stay untouched"""
    import torch
    good = R.command_list("lsb6", oracle).serialize()
    buf, off, ln, out, ooff, ocap = C._host_layout([good])
    d_buf = torch.from_numpy(buf).cuda()
    u64 = lambda a: torch.from_numpy(np.asarray(a, np.uint64).view(np.int64)).cuda()
    d_off, d_ln, d_ooff, d_ocap = u64(off), u64(ln), u64(ooff), u64(ocap)
    d_out = torch.zeros(out.size, dtype=torch.uint8, device="cuda")
    d_olen, d_st = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.full((1,), -7, dtype=torch.int32, device="cuda")
    dev = (1, d_buf.data_ptr(), d_off.data_ptr(), d_ln.data_ptr())
    tail = (d_out.data_ptr(), d_ooff.data_ptr(), d_ocap.data_ptr(), d_olen.data_ptr(), d_st.data_ptr())
    for vals in BAD:
        v = vals if vals else np.zeros((0, 2), np.int16)
        for call in (lambda: engine.encode_speeds_batch_host(buf, off, ln, out, ooff, ocap, None, v),
                     lambda: engine.encode_cmds_speeds_batch_host(buf, off, ln, out, ooff, ocap, None, v),
                     lambda: engine.encode_speeds_batch_device(*dev, len(good), *tail, values=v),
                     lambda: engine.encode_cmds_speeds_batch_device(*dev, len(good), C._replay_len(good) + 1, *tail, values=v)):
            with pytest.raises(divans_b200.DivansError):
                call()
    engine.synchronize()
    assert int(d_st[0]) == -7 and int(d_olen[0]) == 0


def _cmds_device(eng, blobs, opts, lens=None, max_blob_len=None, max_raw_len=None, misalign=None):
    """encode_cmds_speeds_batch_device with blobs at the given misalignment, declared lengths and bounds:
    [(status, out_len, bytes, chosen, cost, halves)]"""
    import torch
    n, k = len(blobs), K
    lens = [len(b) for b in blobs] if lens is None else list(lens)
    shift = [0] * n if misalign is None else list(misalign)
    offs, pos = [], 0
    for b, s in zip(blobs, shift):
        offs.append(pos + s)
        pos = (pos + s + len(b) + 16 + 255) & ~255
    inp = np.zeros(pos + 256, np.uint8)
    for b, o in zip(blobs, offs):
        inp[o:o + len(b)] = np.frombuffer(bytes(b), np.uint8)
    caps = [C._out_cap(b) for b in blobs]
    ooff = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    u64 = lambda a: torch.from_numpy(np.asarray(a, np.uint64).view(np.int64)).cuda()
    d_in, d_out = torch.from_numpy(inp).cuda(), torch.zeros(int(sum(caps)) + 16, dtype=torch.uint8, device="cuda")
    d_off, d_len, d_ooff, d_cap = u64(offs), u64(lens), u64(ooff), u64(caps)
    d_olen, d_st = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d_ch = torch.full((3 * n,), 99, dtype=torch.int32, device="cuda")
    d_cost, d_halves = torch.zeros(n * (k + 1), dtype=torch.int64, device="cuda"), torch.zeros(n * k * 2, dtype=torch.int64, device="cuda")
    mbl = max(lens) if max_blob_len is None else max_blob_len
    mrl = max(C._replay_len(b) for b in blobs) + 1 if max_raw_len is None else max_raw_len
    eng.encode_cmds_speeds_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), mbl, mrl, d_out.data_ptr(), d_ooff.data_ptr(),
                                        d_cap.data_ptr(), d_olen.data_ptr(), d_st.data_ptr(), d_chosen=d_ch.data_ptr(),
                                        d_cost=d_cost.data_ptr(), d_halves=d_halves.data_ptr(), opts=opts, values=VALUES)
    eng.synchronize()
    o, olen, st = d_out.cpu().numpy(), d_olen.cpu().numpy(), d_st.cpu().numpy()
    cost = d_cost.cpu().numpy().view(np.uint64).reshape(n, k + 1)
    halves = d_halves.cpu().numpy().view(np.uint64).reshape(n, k, 2)
    ch = d_ch.cpu().numpy().view(np.uint32).reshape(n, 3)
    return [(int(st[i]), int(olen[i]), o[int(ooff[i]):int(ooff[i]) + int(olen[i])].tobytes(), ch[i], cost[i], halves[i]) for i in range(n)]


def test_every_pass_failing(engine, oracle):
    """at dynamic mixing 2 (halves and verify passes run): a stream whose every pass fails -- replay beyond max_raw_len, a blob
    longer than max_blob_len, a misaligned blob -- reports chosen (0, 0, 0), UINT64_MAX costs and halves (skipped), status 2 or
    3, and its neighbours are the oracle's"""
    okw = dict(window_size=16, dynamic_context_mixing=2)
    opts = divans_b200.encode_options(literal_pred_mode=2, **okw)
    gcl = R.command_list("lsb6", oracle)
    good = gcl.serialize()
    want = T.encode_cmds_speeds(gcl, VALUES, **okw)
    assert (want[3] != T.TALLY_FAILED).all() and (want[4] != T.TALLY_FAILED).all()
    rl = C._replay_len(good)
    lz = oracle.Commands.lz77(R.text()[:rl + 5000], window=16).serialize()
    cases = [(2, _cmds_device(engine, [good, lz, good], opts, max_raw_len=rl)),
             (3, _cmds_device(engine, [good] * 3, opts, lens=[len(good), len(good) + 1, len(good)], max_blob_len=len(good)))]
    cases += [(3, _cmds_device(engine, [good] * 3, opts, misalign=[0, s, 0])) for s in (1, 2, 3)]
    for st, res in cases:
        _check(res[0], want, "neighbour before")
        _check(res[2], want, "neighbour after")
        f = res[1]
        assert f[0] == st and list(f[3]) == [0, 0, 0], (f[0], f[3])
        assert (f[4] == T.TALLY_FAILED).all() and (f[5] == T.TALLY_FAILED).all(), (f[4], f[5])
