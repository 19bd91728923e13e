"""The device-resident command-list encoder (divans_b200_encode_cmds_batch_device) and the transcode that chains it to the
recording decoder (Engine.transcode_device).  The reference of every GPU check is the host call
divans_b200_encode_cmds_batch_host (itself tested against the oracle in test_gpu_encode.py) or the oracle: bytes, out_len and
status must be equal.  The first two tests need no GPU."""
import os
import re

import numpy as np
import pytest

import divans_b200
import mixval_regimes as M
import regimes as R
from irfuzz import random_ir, random_f8_speeds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
gpu = pytest.mark.gpu
CANARY = 0xA5
G = 64          # guard bytes around every output region


def test_prototype_in_header():
    h = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    m = re.search(r"DivansResult\s+divans_b200_encode_cmds_batch_device\(([^;]*)\);", h)
    assert m, "prototype missing"
    args = [a.strip() for a in " ".join(m.group(1).split()).split(",")]
    assert args == ["divans_b200_ctx *ctx", "size_t n", "const uint8_t *d_blobs", "const uint64_t *d_blob_off",
                    "const uint64_t *d_blob_len", "uint64_t max_blob_len", "uint64_t max_raw_len", "uint8_t *d_out",
                    "const uint64_t *d_out_off", "const uint64_t *d_out_cap", "uint64_t *d_out_len", "int32_t *d_status",
                    "const divans_b200_encode_options *opts", "void *cuda_stream"]


def test_symbol_listed():
    assert "divans_b200_encode_cmds_batch_device" in divans_b200.BATCH_SYMBOLS


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _hdr(b):
    return np.frombuffer(bytes(b[:32]).ljust(32, b"\0"), np.uint32)


def _replay_len(b):
    """bytes the encoder replays for a well-formed list (the host call's own sizing: 64 per dictionary word)"""
    h = _hdr(b)
    if len(b) < 32 or h[0] != 0x4C435644 or 32 + 20 * int(h[2]) > len(b):
        return 0
    r = np.frombuffer(bytes(b[32:32 + 20 * int(h[2])]), np.uint32).reshape(-1, 5)
    return int(r[r[:, 0] == 1, 2].sum() + r[r[:, 0] == 3, 2].sum() + 64 * (r[:, 0] == 2).sum())


def _out_cap(b):
    return (len(b) + len(b) // 2 + 70000 + 255) & ~255


def _host(eng, blobs, opts, caps=None):
    """encode_cmds_batch_host in one call: [(status, out_len, bytes)]"""
    caps = [(_out_cap(b)) for b in blobs] if caps is None else caps
    in_len = np.array([len(b) for b in blobs], np.uint64)
    in_off = np.concatenate([[0], np.cumsum((in_len + np.uint64(15)) & ~np.uint64(15))[:-1]]).astype(np.uint64)
    blob = np.zeros(int(in_off[-1] + in_len[-1]) + 16, np.uint8)
    for b, o in zip(blobs, in_off):
        blob[int(o):int(o) + len(b)] = np.frombuffer(bytes(b), np.uint8)
    out_off = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    out = np.zeros(int(sum(caps)) + 16, np.uint8)
    ln, st = eng.encode_batch_host(blob, in_off, in_len, out, out_off, np.array(caps, np.uint64), opts, cmds=True)
    return [(int(s), int(n), out[int(o):int(o) + int(n)].tobytes() if s == 0 else None) for s, n, o in zip(st, ln, out_off)]


def _device(eng, blobs, opts, caps=None, max_blob_len=None, max_raw_len=None, lens=None, misalign=None, stream=None, sync=True):
    """encode_cmds_batch_device with guard bytes around every output region: [(status, out_len, bytes)].  `lens` overrides
    the blob lengths passed, `misalign[i]` shifts blob i off its 4-byte boundary."""
    import torch
    n = len(blobs)
    caps = [_out_cap(b) for b in blobs] if caps is None else list(caps)
    lens = [len(b) for b in blobs] if lens is None else list(lens)
    shift = [0] * n if misalign is None else list(misalign)
    offs, pos = [], 0
    for b, s in zip(blobs, shift):
        offs.append(pos + s)
        pos = (pos + s + len(b) + 16 + 255) & ~255
    inp = np.zeros(pos + 256, np.uint8)
    for b, o in zip(blobs, offs):
        inp[o:o + len(b)] = np.frombuffer(bytes(b), np.uint8)
    out_off = [G + sum(c + G for c in caps[:i]) for i in range(n)]
    out = np.full(G + sum(c + G for c in caps), CANARY, np.uint8)
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.array(a, np.uint64).view(np.int64)).to(dev)
    d_in, d_out = torch.from_numpy(inp).to(dev), torch.from_numpy(out).to(dev)
    d_meta = [u64(offs), u64(lens), u64(out_off), u64(caps)]
    d_len = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
    d_st = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    mbl = max(lens, default=0) if max_blob_len is None else max_blob_len
    mrl = max([_replay_len(b) for b in blobs] + [1]) if max_raw_len is None else max_raw_len
    torch.cuda.current_stream().synchronize()      # (only the copies above: a call queued on the context stays queued)
    eng.encode_cmds_batch_device(n, d_in.data_ptr(), d_meta[0].data_ptr(), d_meta[1].data_ptr(), mbl, mrl, d_out.data_ptr(),
                                 d_meta[2].data_ptr(), d_meta[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), opts,
                                 None if stream is None else stream.cuda_stream)
    keep = (d_in, d_out, d_meta, d_len, d_st)

    def finish():
        if stream is not None:
            stream.synchronize()
        else:
            eng.synchronize()
        o = d_out.cpu().numpy()
        mask = np.ones(o.size, bool)
        for a, c in zip(out_off, caps):
            mask[a:a + c] = False
        assert (o[mask] == CANARY).all(), "a byte outside the output regions changed"
        st, ln = d_st.cpu().numpy()[:n], d_len.cpu().numpy()[:n].view(np.uint64)
        return [(int(s), int(l), o[a:a + int(l)].tobytes() if s == 0 else None) for s, l, a in zip(st, ln, out_off)]
    if sync:
        return finish()
    return finish, keep


def _same(eng, blobs, opts, what, **kw):
    h, d = _host(eng, blobs, opts, kw.get("caps")), _device(eng, blobs, opts, **kw)
    for i, (a, b) in enumerate(zip(d, h)):
        assert a[:2] == b[:2], "%s: stream %d: device (status, out_len) %s, host %s" % (what, i, a[:2], b[:2])
        assert a[2] == b[2], "%s: stream %d: bytes differ" % (what, i)
    return d


def _opts(**kw):
    return divans_b200.encode_options(**kw)


def _golden_blobs(engine, golden):
    streams = [open(e["path"], "rb").read() for e in golden]
    res = engine.decode_cmds(streams, [e["raw_len"] + 64 for e in golden])
    assert all(st == 0 for st, _, _ in res)
    return streams, [b for _, _, b in res]


# ---------------------------------------------------------------------------------------------------------------------
# 1. device equals host
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_golden_blobs(engine, golden):
    streams, blobs = _golden_blobs(engine, golden)
    for e, s, b in zip(golden, streams, blobs):
        o = _opts(**dict(dict(window_size=s[5]), **e["options"]))
        (st, _, got), = _same(engine, [b], o, e["name"])
        assert st == 0 and got == s, e["name"]      # its own options reproduce the stored stream
    # mixing 2, each stream in its own window: the host call, one stream at a time at that window
    d = _device(engine, blobs, _opts(window_size=0, dynamic_context_mixing=2))
    for e, s, b, got in zip(golden, streams, blobs, d):
        assert got == _host(engine, [b], _opts(window_size=s[5], dynamic_context_mixing=2))[0], e["name"]


@gpu
def test_regimes_mixval_and_random_ir(engine, oracle):
    blobs = [R.command_list(name, oracle).serialize() for name in R.GOOD]
    for name, b in zip(R.GOOD, blobs):
        _same(engine, [b], _opts(**R.encode_options(name)), name)
    cases = [M.random_mix(oracle, 0), M.multi_pm(oracle, 0)] + [M.late_pm(oracle, v) for v in range(3)]
    cases += [M.chunk_at(oracle, at) for at in M.CHUNK_AT]
    mv = [b for _, _, b in engine.decode_cmds([c.stream for c in cases], [c.cap for c in cases])]
    _same(engine, mv, _opts(window_size=16), "mixing-value builders")
    _same(engine, mv, _opts(window_size=16, dynamic_context_mixing=2), "mixing-value builders, mixing 2")
    text = R.text()
    ir = [oracle.Commands.from_ir(random_ir(oracle, 7000 + s, n_cmds=60 + s % 90, window=16, text=text)).serialize() for s in range(300)]
    for kw in (dict(window_size=16), dict(window_size=16, dynamic_context_mixing=2, prior_depth=1)):
        _same(engine, ir, _opts(**kw), "random IR %s" % kw)


@gpu
def test_wide_speeds_refused_like_the_host(engine, oracle):
    text = R.text()
    wins = [10, 14, 16, 22]
    cls = [oracle.Commands.from_ir(random_ir(oracle, 7000 + s, n_cmds=60, window=wins[s % 4], text=text, wide_speeds=True)).serialize()
           for s in range(48)]
    refused = 0
    for s in range(48):
        kw = dict(window_size=wins[s % 4], dynamic_context_mixing=s % 3)
        if s % 2:
            kw["literal_adaptation"] = random_f8_speeds(oracle, s)
        d = _same(engine, [cls[t] for t in range(s % 4, 48, 4)], _opts(**kw), "wide speeds %d" % s)
        refused += sum(x[0] == 3 for x in d)
    assert refused >= 3, refused


@gpu
def test_blend_and_wasm_2018(engine, oracle):
    blobs = [R.command_list(name, oracle).serialize() for name in ("lsb6", "dcm2", "switches", "short_literals")]
    _same(engine, blobs, _opts(window_size=16, cdf_model=divans_b200.CDF_BLEND), "blend")
    vec = open(os.path.join(GOLD, "ref_wasm_example.divans"), "rb").read()
    rc, _, cl = oracle.decode_cmds(vec, model_rev=oracle.MODEL_WASM_2018)
    assert rc == 0
    o = _opts(window_size=0, use_context_map=0, dynamic_context_mixing=0, model_rev=divans_b200.MODEL_WASM_2018)
    (st, n, got), = _device(engine, [cl.serialize()], o)
    assert st == 0 and n == 113 and got == vec


# ---------------------------------------------------------------------------------------------------------------------
# 2. per-stream window
# ---------------------------------------------------------------------------------------------------------------------
def _with_window(blob, w):
    b = bytearray(blob)
    b[20:24] = np.uint32(w).tobytes()
    return bytes(b)


@gpu
def test_per_stream_window(engine, oracle):
    text = R.text()
    wins = [10, 16, 22, 24, 30]          # 30: outside 10..24, clamped to 24
    blobs = []
    for k, w in enumerate(wins):
        c = oracle.Commands.lz77(text[k * 40000:k * 40000 + 30000], window=min(w, 24))
        blobs.append(_with_window(c.serialize(), w))
    d = _device(engine, blobs, _opts(window_size=0))
    for w, b, (st, _, got) in zip(wins, blobs, d):
        (hst, _, ref), = _host(engine, [b], _opts(window_size=min(w, 24)))
        assert st == 0 == hst and got == ref, w
        assert got[5] == min(w, 24)
    _same(engine, blobs[:2], _opts(window_size=18), "window 18")     # (lists of windows <= 18 copy within 18)


# ---------------------------------------------------------------------------------------------------------------------
# 3. contract
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_status_contract(engine, oracle):
    good = R.command_list("lsb6", oracle).serialize()
    (hst, need, ref), = _host(engine, [good], _opts(window_size=16))
    assert hst == 0
    o = _opts(window_size=16)
    # output region one byte short: status 2 and the size needed; exactly enough: the bytes
    d = _device(engine, [good, good], o, caps=[need - 1, need])
    assert d[0][:2] == (2, need) and d[1] == (0, need, ref)
    bad_magic = b"X" + good[1:]
    bad_version = good[:4] + np.uint32(2).tobytes() + good[8:]
    truncated = good[:31]
    h = _hdr(good)
    r = np.frombuffer(good[32:32 + 20 * int(h[2])], np.uint32).reshape(-1, 5)
    k = int(np.nonzero(r[:, 0] == 7)[0][0])
    pm_out = bytearray(good)
    pm_out[32 + 20 * k + 4:32 + 20 * k + 8] = np.uint32(h[3]).tobytes()
    rl = _replay_len(good)
    lz = oracle.Commands.lz77(R.text()[:rl + 5000], window=16).serialize()
    cases = [(bad_magic, 3), (bad_version, 3), (truncated, 3), (bytes(pm_out), 3)]
    for blob, want in cases:
        d = _device(engine, [good, blob, good], o)
        assert [x[0] for x in d] == [0, want, 0] and d[0][2] == d[2][2] == ref
        assert _host(engine, [blob], o)[0][0] == want
    # replay longer than max_raw_len: status 2, out_len 0
    d = _device(engine, [good, lz, good], o, max_raw_len=rl)
    assert d[1][:2] == (2, 0) and d[0][2] == d[2][2] == ref
    # blob longer than max_blob_len; misaligned blobs: status 3, neighbours unaffected
    d = _device(engine, [good, good, good], o, lens=[len(good), len(good) + 1, len(good)], max_blob_len=len(good))
    assert [x[0] for x in d] == [0, 3, 0] and d[0][2] == d[2][2] == ref
    for s in (1, 2, 3):
        d = _device(engine, [good, good, good], o, misalign=[0, s, 0])
        assert [x[0] for x in d] == [0, 3, 0] and d[0][2] == d[2][2] == ref, s
    assert _device(engine, [], o) == []


# ---------------------------------------------------------------------------------------------------------------------
# 4. the log bound is exact at both extremes
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_log_bound_exact(engine, oracle):
    """Blobs of exactly max_blob_len bytes at the two extremes of the derived command-log bound.  All PredictionMode records: three
    records with full 16384-entry literal and 1024-entry distance maps whose entries all take the escape path, and 8192 mixing
    values, each coded by its own command -- about 60400 of the 62000 entries the bound allows per record, so a cap one record
    short overflows.  All short records: copies with far, changing distances and long lengths, the commands that code the most
    symbols per 20-byte record."""
    esc = lambda n: [(i * 37) % 256 for i in range(n)]
    pm = R.pm_line("lsb6", lmap=esc(16384), dmap=esc(1024), mix=[(i * 7) % 9 for i in range(8192)])
    allpm = oracle.Commands.from_ir("window 16 0 0 0\n" + "\n".join([pm] * 3) + "\n").serialize()
    h = _hdr(allpm)
    assert (int(h[2]), int(h[3]), int(h[4])) == (3, 3, 0) and len(allpm) == 32 + 3 * (20 + divans_b200.PM_RECORD_BYTES)
    copies = ["insert 4 41424344", "copy 3000000 from 1 ctx 0"] + ["copy %d from %d ctx 0" % (60000 + i, 1000000 + (i * 7919) % 2000000)
                                                                  for i in range(400)]
    short = oracle.Commands.from_ir("window 22 0 0 0\n" + "\n".join(copies) + "\n").serialize()
    assert int(_hdr(short)[3]) == 0
    for name, blob, w in (("all PredictionMode records", allpm, 16), ("all short records", short, 22)):
        d = _same(engine, [blob], _opts(window_size=w), name, max_blob_len=len(blob))
        assert d[0][0] == 0, name


@gpu
def test_literal_records_re_reading_the_pool(engine, oracle):
    """ten literal records over the same 1000 pool bytes: the host call accepts the list, and so does the device call (its
    literal logs are sized from the replay window, not from the pool)"""
    one = oracle.Commands.from_ir("window 16 0 0 0\n" + R.pm_line("lsb6") + "\ninsert 1000 " + R.text()[:1000].hex() + "\n").serialize()
    h = _hdr(one).copy()
    assert (int(h[2]), int(h[4])) == (2, 1000)
    recs = np.frombuffer(one[32:72], np.uint32).reshape(2, 5)
    assert recs[1][0] == 3 and recs[1][1] == 0 and recs[1][2] == 1000
    h[2] = 11
    pm_and_pool = one[72:]
    blob = h.tobytes() + recs[0].tobytes() + recs[1].tobytes() * 10 + pm_and_pool
    (st, _, _), = _host(engine, [blob], _opts(window_size=16))
    assert st == 0
    _same(engine, [blob], _opts(window_size=16), "overlapping literals")
    assert _replay_len(blob) == 10000


# ---------------------------------------------------------------------------------------------------------------------
# 5. slots
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_more_streams_than_slots_and_alternating_with_decode(oracle):
    eng = divans_b200.Engine(0, 2, 16)
    try:
        blobs = [R.command_list(name, oracle).serialize() for name in ("lsb6", "switches", "short_literals", "bt256")] * 3
        _same(eng, blobs, _opts(window_size=16), "12 streams on one block")
        wide = [R.command_list("lsb6", oracle).serialize()] * 4
        o = _opts(window_size=16, literal_adaptation=[(16, 8192), (16, 8192), R.WIDE, R.WIDE])
        _same(eng, wide, o, "wide speeds")
        assert [eng.slot_header(i)[1] for i in range(2)] == [1, 1]     # the model pass left untagged 16-bit priors
        c = R.build("lsb6", oracle)
        res = eng.decode([c.stream] * 2, [c.cap] * 2)
        rc, ref = oracle.decode(c.stream, out_cap=c.cap)
        assert all(st == 0 and out == ref for st, out in res)
        assert [eng.slot_header(i)[1] for i in range(2)] == [0, 0]
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. asynchronous use
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_side_stream_with_a_queued_decode(engine, oracle):
    import torch
    c = R.build("lsb6", oracle)
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.array(a, np.uint64).view(np.int64)).to(dev)
    d_in = torch.from_numpy(np.frombuffer(c.stream * 4, np.uint8).copy()).to(dev)
    n = 4
    meta = [u64([len(c.stream) * i for i in range(n)]), u64([len(c.stream)] * n), u64([c.cap * i for i in range(n)]), u64([c.cap] * n)]
    d_out = torch.zeros(c.cap * n, dtype=torch.uint8, device=dev)
    d_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_st = torch.full((n,), 3, dtype=torch.int32, device=dev)
    blobs = [R.command_list(name, oracle).serialize() for name in ("switches", "dcm2")]
    host = _host(engine, blobs, _opts(window_size=16))
    torch.cuda.synchronize()
    engine.decode_batch_device(d_in.data_ptr(), meta[0].data_ptr(), meta[1].data_ptr(), d_out.data_ptr(), meta[2].data_ptr(),
                               meta[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), n, d_in.numel())
    side = torch.cuda.Stream()
    finish, _keep = _device(engine, blobs, _opts(window_size=16), stream=side, sync=False)
    got = finish()
    engine.synchronize()
    assert got == host
    rc, ref = oracle.decode(c.stream, out_cap=c.cap)
    out = d_out.cpu().numpy()
    for i in range(n):
        assert int(d_st[i]) == 0 and out[c.cap * i:c.cap * i + int(d_len[i])].tobytes() == ref


# ---------------------------------------------------------------------------------------------------------------------
# 7. transcode_device
# ---------------------------------------------------------------------------------------------------------------------
def _pack(streams):
    import torch
    in_len = np.array([len(s) for s in streams], np.uint64)
    in_off = np.concatenate([[0], np.cumsum((in_len + np.uint64(15)) & ~np.uint64(15))[:-1]]).astype(np.uint64)
    buf = np.zeros(int(in_off[-1] + in_len[-1]) + 16, np.uint8)
    for s, o in zip(streams, in_off):
        buf[int(o):int(o) + len(s)] = np.frombuffer(s, np.uint8)
    return torch.from_numpy(buf).to("cuda:0"), in_off, in_len


@gpu
def test_transcode_device_equals_transcode(engine, oracle, oracle_blend):
    from divans_b200 import synth
    blob, off, ln = synth.text_streams(64, 65536)
    raws = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]
    lit = [engine.encode(raws[:32])[k] for k in range(32)]
    lz = [oracle.Commands.lz77(r, window=16).encode(oracle.options(window_size=16)) for r in raws[32:]]
    streams, caps = lit + lz, [len(r) + 64 for r in raws]
    d_in, in_off, in_len = _pack(streams)
    for opts in (None, _opts(window_size=0, dynamic_context_mixing=2)):
        d_new, new_off, new_len, status = engine.transcode_device(d_in, in_off, in_len, caps, opts)
        assert engine.last_transcode_retried > 0     # LZ77 lists that do not fit the first guess run twice
        want = engine.transcode(streams, caps, opts)
        new = d_new.cpu().numpy()
        got = [new[int(o):int(o) + int(n)].tobytes() for o, n in zip(new_off, new_len)]
        assert list(status) == [0] * len(streams)
        assert got == want
        assert [r for _, r in engine.decode(got, caps)] == raws
    # blend to frequentist
    bl = [oracle_blend.encode_raw(r) for r in raws[:4]] + [oracle_blend.Commands.lz77(r, window=16).encode(oracle_blend.options(window_size=16))
                                                            for r in raws[4:8]]
    d_in, in_off, in_len = _pack(bl)
    d_new, new_off, new_len, status = engine.transcode_device(d_in, in_off, in_len, caps[:8], flags=divans_b200.FLAG_CDF_BLEND)
    new = d_new.cpu().numpy()
    got = [new[int(o):int(o) + int(n)].tobytes() for o, n in zip(new_off, new_len)]
    assert list(status) == [0] * 8 and got == engine.transcode(bl, caps[:8], flags=divans_b200.FLAG_CDF_BLEND)


@gpu
def test_transcode_device_failures(engine, oracle):
    c = R.build("lsb6", oracle)
    t = M.truncated(oracle, 0.3)
    f = R.build("corrupt_status3", oracle)
    streams = [c.stream, t.stream, c.stream, f.stream, c.stream]
    caps = [c.cap, t.cap, c.cap, f.cap, c.cap]
    d_in, in_off, in_len = _pack(streams)
    d_new, new_off, new_len, status = engine.transcode_device(d_in, in_off, in_len, caps, flags=divans_b200.FLAG_SKIP_CRC)
    plain = engine.decode(streams, caps, divans_b200.FLAG_SKIP_CRC)
    assert status[1] == plain[1][0] != 0 and status[3] == plain[3][0] != 0
    want = engine.transcode([c.stream], [c.cap])[0]
    new = d_new.cpu().numpy()
    for i in (0, 2, 4):
        assert status[i] == 0 and new[int(new_off[i]):int(new_off[i]) + int(new_len[i])].tobytes() == want
