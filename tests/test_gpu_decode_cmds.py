"""Decoding to command lists on the GPU (-m gpu): the recording decoders (the 16-lane decoder under either probability
model, dv2_kernels.cu) and the pack kernel (dv_kernels.cu), called through divans_b200_decode_cmds_batch_host / _device.  Every expected blob is the
oracle's: the command list dvo_decode_cmds recovers, serialised (oracle.decode_cmds(stream)[2].serialize())."""
import ctypes
import json
import os

import numpy as np
import pytest

import divans_b200
import mixval_regimes as M
import regimes as R
from irfuzz import random_ir

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _first_diff(a, b):
    return next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), min(len(a), len(b)))


def _same(got, ref, what):
    assert got == ref, "%s: len %d vs %d, first diff at %d" % (what, len(got), len(ref), _first_diff(got, ref))


def _oracle_blob(oracle, stream, cap, skip_crc=False, model_rev=0):
    rc, raw, cl = oracle.decode_cmds(stream, out_cap=cap, skip_crc=skip_crc, model_rev=model_rev)
    assert rc == 0
    return raw, cl.serialize()


def _check_batch(engine, oracle, streams, caps, flags=0, model_rev=0):
    res = engine.decode_cmds(streams, caps, flags)
    for i, ((st, raw, blob), s, cap) in enumerate(zip(res, streams, caps)):
        ref_raw, ref_blob = _oracle_blob(oracle, s, cap, skip_crc=bool(flags & divans_b200.FLAG_SKIP_CRC), model_rev=model_rev)
        assert st == 0, "stream %d: status %d" % (i, st)
        _same(raw, ref_raw, "stream %d bytes" % i)
        _same(blob, ref_blob, "stream %d blob" % i)
    return res


def test_golden_fixtures(engine, oracle, golden):
    streams = [open(e["path"], "rb").read() for e in golden]
    caps = [e["raw_len"] + 64 for e in golden]
    res = _check_batch(engine, oracle, streams, caps)
    assert engine.last_lanes() == 16
    for e, s, (_, _, blob) in zip(golden, streams, res):
        o = divans_b200.encode_options(**dict(dict(window_size=s[5]), **e["options"]))
        _same(engine.encode([blob], o, cmds=True)[0], s, "%s re-encoded" % e["name"])


def test_wasm_2018_stream(engine, oracle):
    meta = json.load(open(os.path.join(GOLD, "ref_wasm_example.json")))
    s = open(os.path.join(GOLD, "ref_wasm_example.divans"), "rb").read()
    (st, raw, blob), = _check_batch(engine, oracle, [s], [meta["plain_len"] + 64], divans_b200.FLAG_MODEL_WASM_2018,
                                    model_rev=oracle.MODEL_WASM_2018)
    assert raw.decode() == meta["plain_text"]
    # the options the reference's encoder wrote it with: no context map (mixing values 4), no mixing
    o = divans_b200.encode_options(window_size=s[5], use_context_map=0, dynamic_context_mixing=0, model_rev=divans_b200.MODEL_WASM_2018)
    got = engine.encode([blob], o, cmds=True)[0]
    assert len(got) == 113 and got == s


def test_regimes_and_reencode(engine, oracle):
    cases = [R.build(name, oracle) for name in R.GOOD]
    res = _check_batch(engine, oracle, [c.stream for c in cases], [c.cap for c in cases])
    for name, c, (_, _, blob) in zip(R.GOOD, cases, res):
        _same(engine.encode([blob], divans_b200.encode_options(**R.encode_options(name)), cmds=True)[0], c.stream, name)


def test_mixval_builders(engine, oracle):
    cases = [M.random_mix(oracle, 0), M.multi_pm(oracle, 0)] + [M.late_pm(oracle, v) for v in range(3)]
    cases += [M.chunk_at(oracle, at) for at in M.CHUNK_AT]
    _check_batch(engine, oracle, [c.stream for c in cases], [c.cap for c in cases])
    cl, stream, raw = M.wasm_2018(oracle, 0)
    (_, got, blob), = _check_batch(engine, oracle, [stream], [len(raw) + 64], divans_b200.FLAG_MODEL_WASM_2018,
                                   model_rev=oracle.MODEL_WASM_2018)
    assert got == raw


@pytest.mark.parametrize("n", [1, 3, 7, 33])
def test_mixed_warps_odd_batches(engine, oracle, n):
    # neighbours in a warp record different command kinds at different times
    names = R.GOOD
    cases = [R.build(names[(i * 5) % len(names)], oracle, variant=i % 3) for i in range(n)]
    _check_batch(engine, oracle, [c.stream for c in cases], [c.cap for c in cases])


def test_random_ir(engine, oracle):
    from divans_b200 import synth
    text = synth.text_corpus(1 << 18)
    streams, caps = [], []
    for seed in range(300):
        c = oracle.Commands.from_ir(random_ir(oracle, 7000 + seed, n_cmds=60 + seed % 90, window=16 + seed % 7, text=text))
        s = c.encode(oracle.options(window_size=c.window, dynamic_context_mixing=seed % 3, prior_depth=seed % 4))
        rc, raw = oracle.decode(s)
        assert rc == 0
        streams.append(s)
        caps.append(len(raw) + 64)
    _check_batch(engine, oracle, streams, caps)


def _blend_streams(oracle_blend, text):
    raws = [text[:n] for n in (1, 1000, 20000)]
    streams = [oracle_blend.encode_raw(r, oracle_blend.options(dynamic_context_mixing=k % 3)) for k, r in enumerate(raws)]
    for seed in range(6):
        c = oracle_blend.Commands.from_ir(random_ir(oracle_blend, 4100 + seed, n_cmds=100, window=16, text=text))
        streams.append(c.encode(oracle_blend.options(window_size=c.window, dynamic_context_mixing=seed % 3)))
    c = oracle_blend.Commands.lz77(text[:30000], window=16)
    streams.append(c.encode(oracle_blend.options(window_size=16)))
    caps = [len(oracle_blend.decode(s)[1]) + 64 for s in streams]
    return streams, caps


def test_blend_streams_and_transcode(engine, oracle, oracle_blend):
    from divans_b200 import synth
    text = synth.text_corpus(1 << 17)
    streams, caps = _blend_streams(oracle_blend, text)
    res = _check_batch(engine, oracle_blend, streams, caps, divans_b200.FLAG_CDF_BLEND)
    new = engine.transcode(streams, caps, flags=divans_b200.FLAG_CDF_BLEND)
    back = engine.decode(new, caps)
    for i, ((st, raw), (_, want, blob), s, n) in enumerate(zip(back, res, streams, new)):
        assert st == 0 and raw == want, i
        rc, _, cl = oracle_blend.decode_cmds(s, out_cap=caps[i])
        _same(n, _encode_frequentist(oracle, cl, oracle.options(window_size=s[5])), "transcoded stream %d" % i)


def _encode_frequentist(oracle, cl, opts):
    """the frequentist oracle's dvo_encode_cmds of a command list the blend oracle holds (both builds share the list's layout)"""
    cap = cl.c.n_lits * 2 + cl.c.n_cmds * 16 + (1 << 20)
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    lst = oracle.CmdList.from_address(ctypes.addressof(cl.c))
    assert oracle.lib().dvo_encode_cmds(ctypes.byref(lst), ctypes.byref(opts), ctypes.c_void_p(out.ctypes.data), cap, ctypes.byref(n)) == 0
    return out[: n.value].tobytes()


def test_transcode_to_dynamic_context_mixing_2(engine, oracle, golden):
    streams = [open(e["path"], "rb").read() for e in golden]
    caps = [e["raw_len"] + 64 for e in golden]
    o = divans_b200.encode_options(window_size=0, dynamic_context_mixing=2)
    new = engine.transcode(streams, caps, o)
    for s, n, (st, raw), cap in zip(streams, new, engine.decode(new, caps), caps):
        rc, want, cl = oracle.decode_cmds(s, out_cap=cap)
        assert st == 0 and raw == want
        _same(n, cl.encode(oracle.options(window_size=s[5], dynamic_context_mixing=2)), "transcode")


def _host_call(engine, streams, out_caps, blob_caps, flags=0, canary=0xA5):
    """decode_cmds_batch_host with a guard byte range around and between every region"""
    n = len(streams)
    in_len = np.array([len(s) for s in streams], np.uint64)
    in_off = np.zeros(n, np.uint64)
    if n > 1:
        in_off[1:] = np.cumsum(in_len + np.uint64(16))[:-1]
    inp = np.zeros(int((in_len + np.uint64(16)).sum()) + 16, np.uint8)
    for s, o in zip(streams, in_off):
        inp[int(o):int(o) + len(s)] = np.frombuffer(s, np.uint8)
    G = 64

    def regions(caps):
        caps = np.array(caps, np.uint64)
        off = np.zeros(n, np.uint64)
        off[:] = G + np.concatenate([[0], np.cumsum(caps + np.uint64(G))[:-1]]).astype(np.uint64)
        buf = np.full(int((caps + np.uint64(G)).sum()) + G, canary, np.uint8)
        return buf, off, caps

    out, out_off, out_cap = regions(out_caps)
    blobs, blob_off, blob_cap = regions(blob_caps)
    out_len, blob_len, status = engine.decode_cmds_batch_host(inp, in_off, in_len, out, out_off, out_cap, blobs, blob_off, blob_cap, flags)

    def guards_intact(buf, off, caps):
        mask = np.ones(buf.size, bool)
        for o, c in zip(off, caps):
            mask[int(o):int(o) + int(c)] = False
        return bool((buf[mask] == canary).all())

    assert guards_intact(out, out_off, out_cap) and guards_intact(blobs, blob_off, blob_cap), "a byte outside the regions changed"
    return out, out_off, out_len, blobs, blob_off, blob_len, status


def test_status_contract(engine, oracle):
    good = R.build("switches", oracle)
    trunc = [M.truncated(oracle, f) for f in (0.3, 0.9)]
    flips = [M.bitflip(oracle, s) for s in range(3)]
    bad = [R.build(name, oracle) for name in R.FAILING]
    streams = [good.stream] + [c.stream for c in trunc + flips + bad] + [good.stream[:len(good.stream) // 2]]
    caps = [good.cap] + [c.cap for c in trunc + flips + bad] + [good.cap]
    flags = divans_b200.FLAG_SKIP_CRC
    bcap = [1 << 20] * len(streams)
    out, out_off, out_len, blobs, blob_off, blob_len, status = _host_call(engine, streams, caps, bcap, flags)
    # the same statuses and lengths as a plain decode
    inb = np.frombuffer(b"".join(streams), np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in streams])[:-1]]).astype(np.uint64)
    pl_out = np.zeros(sum(caps) + 64, np.uint8)
    pl_off = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    pl_len, pl_status = engine.decode_batch_host(inb, offs, [len(s) for s in streams], pl_out, pl_off, caps, flags)
    assert list(status) == list(pl_status) and list(out_len) == list(pl_len)
    assert status[0] == 0 and (status[1:3] != 0).all() and status[-1] != 0
    for i in range(len(streams)):
        region = blobs[int(blob_off[i]):int(blob_off[i]) + bcap[i]]
        if status[i] != 0:
            assert blob_len[i] == 0 and not region.any(), i     # a failed stream's blob region holds zeros
        else:
            _, ref = _oracle_blob(oracle, streams[i], caps[i], skip_crc=True)
            assert region[:int(blob_len[i])].tobytes() == ref and not region[int(blob_len[i]):].any()
    # a good stream decoded after the failing ones on the same (single) slot
    eng1 = divans_b200.Engine(0, 2, 16)
    try:
        res = eng1.decode_cmds([streams[1], streams[-1], good.stream], [caps[1], caps[-1], good.cap], flags)
        assert res[0][0] != 0 and res[1][0] != 0 and res[2][0] == 0
        assert res[2][2] == _oracle_blob(oracle, good.stream, good.cap, skip_crc=True)[1]
    finally:
        eng1.close()


def test_output_and_blob_capacity(engine, oracle):
    c = R.build("short_literals", oracle)
    raw, ref = _oracle_blob(oracle, c.stream, c.cap)
    # output region too small: what a plain decode reports, no blob
    _, _, out_len, _, _, blob_len, status = _host_call(engine, [c.stream], [len(raw) - 1], [len(ref) + 100])
    assert status[0] == 2 and blob_len[0] == 0
    # blob region one byte short: status 2, the full output, the exact size; a retry with that size succeeds
    out, out_off, out_len, blobs, blob_off, blob_len, status = _host_call(engine, [c.stream, c.stream], [c.cap, c.cap], [len(ref) - 1, len(ref)])
    assert list(status) == [2, 0] and list(blob_len) == [len(ref), len(ref)]
    assert int(out_len[0]) == len(raw) and out[int(out_off[0]):int(out_off[0]) + len(raw)].tobytes() == raw
    assert not blobs[int(blob_off[0]):int(blob_off[0]) + len(ref) - 1].any()
    assert blobs[int(blob_off[1]):int(blob_off[1]) + len(ref)].tobytes() == ref
    # a region far too small for the prediction-mode record, and Engine.decode_cmds' retry
    _, _, _, _, _, blob_len, status = _host_call(engine, [c.stream], [c.cap], [100])
    assert status[0] == 2 and blob_len[0] == len(ref)


def _slots(eng):
    """the two slots of a one-block engine: total streams hosted, and the other header words of each slot (which of the two
    lane groups takes a stream is not fixed)"""
    h = [eng.slot_header(i) for i in range(2)]
    return sum(x[0] for x in h), sorted(tuple(x[1:]) for x in h)


def test_alternating_with_plain_decode(oracle):
    # one stream per call on two slots: bt256 (the full literal map: high-water mark), wide_speeds (untagged tables),
    # per_context_mix (a stale mixing mask), lsb6 after them
    cases = [R.build(name, oracle) for name in ("bt256", "wide_speeds", "per_context_mix", "lsb6", "no_predmode")]
    eng_a, eng_b = divans_b200.Engine(0, 2, 16), divans_b200.Engine(0, 2, 16)
    try:
        for c in cases:
            for eng in (eng_a, eng_b):
                (st, raw), = eng.decode([c.stream], [c.cap])
                assert st == 0 and raw == c.raw
            (st, raw, blob), = eng_a.decode_cmds([c.stream], [c.cap])
            assert st == 0 and raw == c.raw and blob == _oracle_blob(oracle, c.stream, c.cap)[1]
            eng_b.decode([c.stream], [c.cap])
            # the recording decoder leaves the slots as a plain decode of the same stream does
            assert _slots(eng_a) == _slots(eng_b)
    finally:
        eng_a.close()
        eng_b.close()


def test_device_entry_point(engine, oracle):
    torch = pytest.importorskip("torch")
    cases = [R.build(name, oracle) for name in ("switches", "bt256", "dcm2", "empty", "no_predmode")]
    streams, caps = [c.stream for c in cases], [c.cap for c in cases]
    host = engine.decode_cmds(streams, caps)
    n = len(streams)
    in_off = np.concatenate([[0], np.cumsum([len(s) for s in streams])[:-1]]).astype(np.uint64)
    out_off = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    bcap = [len(b) + 7 for _, _, b in host]
    blob_off = np.concatenate([[0], np.cumsum(bcap)[:-1]]).astype(np.uint64)
    dev = torch.device("cuda:0")
    t = lambda a, dt: torch.as_tensor(np.asarray(a).astype(dt).view(np.int64 if dt == np.uint64 else dt)).to(dev)
    d_in = torch.as_tensor(np.frombuffer(b"".join(streams), np.uint8).copy()).to(dev)
    d_out = torch.zeros(sum(caps), dtype=torch.uint8, device=dev)
    d_blobs = torch.zeros(sum(bcap), dtype=torch.uint8, device=dev)
    d_meta = [t(in_off, np.uint64), t([len(s) for s in streams], np.uint64), t(out_off, np.uint64), t(caps, np.uint64),
              t(blob_off, np.uint64), t(bcap, np.uint64)]
    d_out_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_blob_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_status = torch.full((n,), 3, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        engine.decode_cmds_batch_device(d_in.data_ptr(), d_meta[0].data_ptr(), d_meta[1].data_ptr(), d_out.data_ptr(), d_meta[2].data_ptr(),
                                        d_meta[3].data_ptr(), d_out_len.data_ptr(), d_blobs.data_ptr(), d_meta[4].data_ptr(),
                                        d_meta[5].data_ptr(), d_blob_len.data_ptr(), d_status.data_ptr(), n, sum(len(x) for x in streams),
                                        stream=s.cuda_stream)
    s.synchronize()
    out, blobs = d_out.cpu().numpy(), d_blobs.cpu().numpy()
    for i, (st, raw, blob) in enumerate(host):
        assert int(d_status[i]) == st == 0 and int(d_out_len[i]) == len(raw) and int(d_blob_len[i]) == len(blob)
        assert out[int(out_off[i]):int(out_off[i]) + len(raw)].tobytes() == raw
        assert blobs[int(blob_off[i]):int(blob_off[i]) + len(blob)].tobytes() == blob
