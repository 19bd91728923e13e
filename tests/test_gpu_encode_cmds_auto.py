"""encode_cmds_auto on the GPU: command lists coded under the cheapest candidate literal model, whose PredictionMode record
replaces each of the list's own (or KEEP, the list as given).  The references are the oracle's tally and dvo_encode_cmds_auto,
and the plain command-list encoder on the blob with its records rewritten in numpy."""
import lzma
import os

import numpy as np
import pytest

import divans_b200
import mixval_regimes as M
import regimes as R
from divans_b200 import synth
from irfuzz import random_ir, random_f8_speeds
from oracle_tally import tally_py as T

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
KEEP = divans_b200.LITERAL_MODEL_KEEP
CANDS = [KEEP] + divans_b200.DEFAULT_LITERAL_MODELS
PMB = divans_b200.PM_RECORD_BYTES
CANARY = 0xA5
G = 64


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _hdr(b):
    return np.frombuffer(bytes(b[:32]).ljust(32, b"\0"), np.uint32)


def _raw_record(pm, mv):
    """the raw encoder's PredictionMode record of (pred_mode, mixing value) (include/divans_b200.h, DVCL)"""
    r = np.zeros(PMB, np.uint8)
    r[0], r[2], r[28], r[30] = pm, 1, 64, 4
    r[32:96] = np.arange(64)
    r[32 + 16384:32 + 16384 + 4] = np.arange(4)
    r[32 + 16384 + 1024:] = mv
    return r


def _rewrite(blob, cand):
    """the blob with every PredictionMode record replaced by cand's record (KEEP: the blob itself)"""
    if tuple(cand) == KEEP:
        return bytes(blob)
    h = _hdr(blob)
    b = np.frombuffer(bytes(blob), np.uint8).copy()
    at = 32 + 20 * int(h[2])
    for k in range(int(h[3])):
        b[at + k * PMB:at + (k + 1) * PMB] = _raw_record(*cand)
    return b.tobytes()


def _replay_len(b):
    h = _hdr(b)
    if len(b) < 32 or h[0] != 0x4C435644 or 32 + 20 * int(h[2]) > len(b):
        return 0
    r = np.frombuffer(bytes(b[32:32 + 20 * int(h[2])]), np.uint32).reshape(-1, 5)
    return int(r[r[:, 0] == 1, 2].sum() + r[r[:, 0] == 3, 2].sum() + 64 * (r[:, 0] == 2).sum())


def _out_cap(b):
    return (len(b) + len(b) // 2 + 70000 + 255) & ~255


def _host_layout(blobs, caps=None):
    caps = [_out_cap(b) for b in blobs] if caps is None else list(caps)
    in_len = np.array([len(b) for b in blobs], np.uint64)
    in_off = np.concatenate([[0], np.cumsum((in_len + np.uint64(15)) & ~np.uint64(15))[:-1]]).astype(np.uint64)
    buf = np.zeros(int(in_off[-1] + in_len[-1]) + 16, np.uint8)
    for b, o in zip(blobs, in_off):
        buf[int(o):int(o) + len(b)] = np.frombuffer(bytes(b), np.uint8)
    out_off = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    return buf, in_off, in_len, np.zeros(int(sum(caps)) + 16, np.uint8), out_off, np.array(caps, np.uint64)


def _auto_host(eng, blobs, opts, cands=CANDS, caps=None):
    """encode_cmds_auto_batch_host: ([(status, out_len, bytes)], chosen, cost)"""
    buf, off, ln, out, ooff, ocap = _host_layout(blobs, caps)
    out_len, st, chosen, cost = eng.encode_cmds_auto_batch_host(buf, off, ln, out, ooff, ocap, opts, cands)
    res = [(int(s), int(n), out[int(o):int(o) + int(n)].tobytes() if s == 0 else None) for s, n, o in zip(st, out_len, ooff)]
    return res, chosen, cost


def _plain_host(eng, blobs, opts, caps=None):
    buf, off, ln, out, ooff, ocap = _host_layout(blobs, caps)
    out_len, st = eng.encode_batch_host(buf, off, ln, out, ooff, ocap, opts, cmds=True)
    return [(int(s), int(n), out[int(o):int(o) + int(n)].tobytes() if s == 0 else None) for s, n, o in zip(st, out_len, ooff)]


def _auto_device(eng, blobs, opts, cands=CANDS, caps=None, max_blob_len=None, max_raw_len=None, lens=None, misalign=None, plain=False):
    """encode_cmds_auto_batch_device (plain: encode_cmds_batch_device) with guard bytes around every output region:
    ([(status, out_len, bytes)], chosen, cost)"""
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
    meta = [u64(offs), u64(lens), u64(out_off), u64(caps)]
    d_len = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
    d_st = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    d_ch = torch.full((max(n, 1),), 99, dtype=torch.int32, device=dev)
    d_cost = torch.zeros(max(n, 1) * len(cands), dtype=torch.int64, device=dev)
    mbl = max(lens, default=0) if max_blob_len is None else max_blob_len
    mrl = max([_replay_len(b) for b in blobs] + [1]) if max_raw_len is None else max_raw_len
    torch.cuda.current_stream().synchronize()
    args = (n, d_in.data_ptr(), meta[0].data_ptr(), meta[1].data_ptr(), mbl, mrl, d_out.data_ptr(), meta[2].data_ptr(), meta[3].data_ptr(),
            d_len.data_ptr(), d_st.data_ptr())
    if plain:
        eng.encode_cmds_batch_device(*args, opts)
    else:
        eng.encode_cmds_auto_batch_device(*args, d_ch.data_ptr(), d_cost.data_ptr(), opts, cands)
    eng.synchronize()
    o = d_out.cpu().numpy()
    mask = np.ones(o.size, bool)
    for a, c in zip(out_off, caps):
        mask[a:a + c] = False
    assert (o[mask] == CANARY).all(), "a byte outside the output regions changed"
    st, ln = d_st.cpu().numpy()[:n], d_len.cpu().numpy()[:n].view(np.uint64)
    res = [(int(s), int(l), o[a:a + int(l)].tobytes() if s == 0 else None) for s, l, a in zip(st, ln, out_off)]
    return res, d_ch.cpu().numpy()[:n].view(np.uint32), d_cost.cpu().numpy()[:n * len(cands)].view(np.uint64).reshape(n, len(cands))


def _records(n, width, seed):
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n].tobytes()


def _lists(oracle):
    """(name, oracle Commands) of every kind of input: lists decoded from the golden streams, the IR fixtures, LZ77 lists of
    text, UTF-8 text and 2/4/8-byte records, decoded literal-only streams, and random IR lists"""
    import json
    out = []
    for e in json.load(open(os.path.join(GOLD, "golden.json"))):
        rc, _, cl = oracle.decode_cmds(open(os.path.join(GOLD, e["name"] + ".divans"), "rb").read(), out_cap=e["raw_len"] + 64)
        assert rc == 0
        out.append((e["name"], cl))
    out.append(("asyoulik.ir", oracle.Commands.from_ir(lzma.decompress(open(os.path.join(GOLD, "asyoulik.ir.xz"), "rb").read()))))
    out.append(("ends_with_truncated_dictionary.ir", oracle.Commands.from_ir(open(os.path.join(GOLD, "ends_with_truncated_dictionary.ir"),
                                                                                 "rb").read())))
    blob, off, ln = synth.text_streams(3, 12000, seed=9)
    text = [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)]
    cyr = b"".join(chr(0x430 + (c % 26)).encode() if 97 <= c < 123 else bytes([c]) for c in text[1])[:12000]
    for name, data in (("text", text[0]), ("utf8", cyr), ("rec2", _records(12000, 2, 1)), ("rec4", _records(12000, 4, 2)),
                       ("rec8", _records(12000, 8, 3))):
        out.append(("lz77 " + name, oracle.Commands.lz77(data, window=16)))
    for name, data in (("text", text[2]), ("rec4", _records(9000, 4, 5))):
        rc, _, cl = oracle.decode_cmds(oracle.encode_raw(data, oracle.options(window_size=12)))
        assert rc == 0
        out.append(("literal-only " + name, cl))
    rt = R.text()
    for s in range(6):
        out.append(("random IR %d" % s, oracle.Commands.from_ir(random_ir(oracle, 9100 + s, n_cmds=60 + 17 * s, window=16, text=rt))))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. the cost matrix and the streams against the oracle and the rewritten blobs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("blend,dcm", [(False, 0), (False, 1), (False, 2), (True, 0), (True, 1), (True, 2)])
def test_cost_matrix_and_bytes(engine, oracle, oracle_blend, blend, dcm):
    lists = _lists(oracle)
    blobs = [cl.serialize() for _, cl in lists]
    okw = dict(window_size=22, dynamic_context_mixing=dcm)
    opts = divans_b200.encode_options(cdf_model=int(blend), **okw)
    res, chosen, cost = _auto_host(engine, blobs, opts)
    for i, ((name, cl), b) in enumerate(zip(lists, blobs)):
        rc, want, och, ocost = T.encode_cmds_auto(cl, CANDS, blend, **okw)
        assert (cost[i] == ocost).all(), "%s: GPU cost %s, oracle %s" % (name, cost[i], ocost)
        assert chosen[i] == och and rc == res[i][0] == 0, name
        assert res[i][2] == want, "%s: stream differs from the oracle's" % name
        assert res[i] == _plain_host(engine, [_rewrite(b, CANDS[och])], opts)[0], name
    # every output decodes to the list's replay
    replays = [oracle.decode(cl.encode(oracle.options(window_size=22)))[1] for _, cl in lists]
    dec = engine.decode([r[2] for r in res], [len(r) + 64 for r in replays], divans_b200.FLAG_CDF_BLEND if blend else 0)
    assert dec == [(0, r) for r in replays]
    assert len(set(chosen.tolist())) > 2, chosen     # the batch really picks different models


# ---------------------------------------------------------------------------------------------------------------------
# 2. identities
# ---------------------------------------------------------------------------------------------------------------------
def test_keep_alone_is_the_plain_call(engine, oracle):
    blobs = [R.command_list(name, oracle).serialize() for name in R.GOOD]
    for name, b in zip(R.GOOD, blobs):
        o = divans_b200.encode_options(**R.encode_options(name))
        res, chosen, cost = _auto_host(engine, [b], o, [KEEP])
        assert res == _plain_host(engine, [b], o) and chosen[0] == 0, name


def test_keep_wins_ties(engine, oracle):
    """a list generated with (2, 4): KEEP and (2, 4) cost the same whichever comes first, and the lower index wins"""
    cl = oracle.Commands.lz77(_records(20000, 4, 7), window=16, pred_mode=2, mixing_value=4)
    b = cl.serialize()
    o = divans_b200.encode_options(window_size=16)
    for cands in ([KEEP, (2, 4)], [(2, 4), KEEP]):
        res, chosen, cost = _auto_host(engine, [b], o, cands)
        assert cost[0][0] == cost[0][1] and chosen[0] == 0
        assert res[0] == _plain_host(engine, [b], o)[0]


def test_literal_only_transcode_is_encode_auto(engine):
    """streams the raw encoder stored with its default model, transcoded under DEFAULT_LITERAL_MODELS, are encode_auto of their
    input: the decoded list is the raw encoder's own list"""
    blob, off, ln = synth.text_streams(6, 20000, seed=31)
    raws = [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)] + [_records(20000, w, w) for w in (2, 4, 8)]
    for w in (10, 16):
        o = divans_b200.encode_options(window_size=w)
        stored = engine.encode(raws, o)
        new, chosen, cost = engine.transcode(stored, [len(r) + 64 for r in raws], divans_b200.encode_options(window_size=0),
                                             candidates=divans_b200.DEFAULT_LITERAL_MODELS)
        auto = engine.encode_auto(raws, o)
        assert new == [b for _, b, _ in auto] and list(chosen) == [c for _, _, c in auto], w


# ---------------------------------------------------------------------------------------------------------------------
# 3. contracts of the device call
# ---------------------------------------------------------------------------------------------------------------------
def test_device_equals_host(engine, oracle):
    lists = _lists(oracle)[-13:]
    blobs = [cl.serialize() for _, cl in lists]
    for kw in (dict(window_size=22), dict(window_size=22, dynamic_context_mixing=2, cdf_model=divans_b200.CDF_BLEND)):
        o = divans_b200.encode_options(**kw)
        h, hc, hk = _auto_host(engine, blobs, o)
        d, dc, dk = _auto_device(engine, blobs, o)
        assert d == h and (dc == hc).all() and (dk == hk).all(), kw
        # and each stream is the plain device call on the rewritten blob
        p, _, _ = _auto_device(engine, [_rewrite(b, CANDS[c]) for b, c in zip(blobs, dc)], o, plain=True)
        assert p == d


def test_window_zero_takes_each_header(engine, oracle):
    text = R.text()
    blobs = []
    for k, w in enumerate((10, 16, 22)):
        b = bytearray(oracle.Commands.lz77(text[k * 30000:k * 30000 + 20000], window=w).serialize())
        b[20:24] = np.uint32(w).tobytes()
        blobs.append(bytes(b))
    d, dc, _ = _auto_device(engine, blobs, divans_b200.encode_options(window_size=0))
    for w, b, c, x in zip((10, 16, 22), blobs, dc, d):
        h, hc, _ = _auto_host(engine, [b], divans_b200.encode_options(window_size=w))
        assert x == h[0] and c == hc[0] and x[2][5] == w


def test_more_pairs_than_slots_slot_reuse_and_v2_decode(oracle):
    """a one-warp context: 12 lists x 9 candidates run through its two slots; a plain encode before and a v2 decode after
    see no state of it"""
    eng = divans_b200.Engine(0, 2, 16)
    big = divans_b200.Engine(0, 0, 16)
    try:
        blobs = [R.command_list(name, oracle).serialize() for name in ("lsb6", "switches", "short_literals", "bt256")] * 3
        o = divans_b200.encode_options(window_size=16)
        eng.encode([b[::-1] for b in blobs[:2]], divans_b200.encode_options(literal_pred_mode=3, literal_mixing_value=9))
        ref = _auto_host(big, blobs, o)
        got = _auto_host(eng, blobs, o)
        assert got[0] == ref[0] and (got[1] == ref[1]).all() and (got[2] == ref[2]).all()
        assert _auto_device(eng, blobs, o)[0] == ref[0]
        c = R.build("lsb6", oracle)
        res = eng.decode([c.stream] * 2, [c.cap] * 2)
        rc, want = oracle.decode(c.stream, out_cap=c.cap)
        assert all(st == 0 and out == want for st, out in res)
        assert _auto_host(eng, blobs, o)[0] == ref[0]
    finally:
        eng.close()
        big.close()


def test_status_contract(engine, oracle):
    good = R.command_list("lsb6", oracle).serialize()
    o = divans_b200.encode_options(window_size=16)
    (ref,), (ch,), _ = _auto_host(engine, [good], o)
    assert ref[0] == 0
    need = ref[1]
    # output region one byte short: status 2 and the size the chosen stream needs
    d, dc, _ = _auto_device(engine, [good, good], o, caps=[need - 1, need])
    assert d[0][:2] == (2, need) and d[1] == ref and list(dc) == [ch, ch]
    h, hc, _ = _auto_host(engine, [good, good], o, caps=[need - 1, need])
    assert h == d and (hc == dc).all()
    # replay longer than max_raw_len: status 2, out_len 0; every pass failed
    rl = _replay_len(good)
    lz = oracle.Commands.lz77(R.text()[:rl + 5000], window=16).serialize()
    d, dc, dk = _auto_device(engine, [good, lz, good], o, max_raw_len=rl)
    assert d[1][:2] == (2, 0) and d[0] == d[2] == ref and (dk[1] == T.TALLY_FAILED).all() and dc[1] == 0
    # blob longer than max_blob_len; misaligned blobs: status 3 unread, every pass failed, neighbours unaffected
    d, dc, dk = _auto_device(engine, [good] * 3, o, lens=[len(good), len(good) + 1, len(good)], max_blob_len=len(good))
    assert [x[0] for x in d] == [0, 3, 0] and d[0] == d[2] == ref and (dk[1] == T.TALLY_FAILED).all()
    for s in (1, 2, 3):
        d, dc, dk = _auto_device(engine, [good] * 3, o, misalign=[0, s, 0])
        assert [x[0] for x in d] == [0, 3, 0] and d[0] == d[2] == ref and (dk[1] == T.TALLY_FAILED).all(), s
    assert _auto_device(engine, [], o)[0] == []


def test_wide_speeds_cost_the_maximum(engine, oracle):
    """lists whose stream-supplied speeds wrap under some options: the passes the encoder refuses cost UINT64_MAX, exactly where
    the oracle refuses them, and the stream is the plain call's on the rewritten list"""
    text = R.text()
    cls = [oracle.Commands.from_ir(random_ir(oracle, 7000 + s, n_cmds=60, window=16, text=text, wide_speeds=True)) for s in range(16)]
    blobs = [c.serialize() for c in cls]
    failed = 0
    for s in range(4):
        kw = dict(window_size=16, dynamic_context_mixing=s % 3, literal_adaptation=random_f8_speeds(oracle, 2 * s + 1))
        o = divans_b200.encode_options(**kw)
        d, dc, dk = _auto_device(engine, blobs, o)
        h, hc, hk = _auto_host(engine, blobs, o)
        assert d == h and (dc == hc).all() and (dk == hk).all()
        for i, c in enumerate(cls):
            rc, want, och, ocost = T.encode_cmds_auto(c, CANDS, **kw)
            assert (dk[i] == ocost).all() and dc[i] == och and d[i][2] == want, (s, i)
            assert d[i] == _plain_host(engine, [_rewrite(blobs[i], CANDS[dc[i]])], o)[0]
        failed += int((dk == T.TALLY_FAILED).sum())
    assert failed > 0


def test_refused_candidate_lists(engine, oracle):
    good = R.command_list("lsb6", oracle).serialize()
    buf, off, ln, out, ooff, ocap = _host_layout([good])
    for bad in ([], [(0, 4)] * 17, [(4, 4)], [(0, 16)], [(-1, 4)], [(0, -1)], [(-1, -2)]):
        with pytest.raises(divans_b200.DivansError):
            engine.encode_cmds_auto_batch_host(buf, off, ln, out, ooff, ocap, None, bad)
        with pytest.raises(divans_b200.DivansError):
            _auto_device(engine, [good], divans_b200.encode_options(window_size=16), cands=bad)
    # KEEP is a command-list candidate only
    raw = np.frombuffer(R.text()[:1000], np.uint8).copy()
    with pytest.raises(divans_b200.DivansError):
        engine.encode_auto_batch_host(raw, np.zeros(1, np.uint64), np.array([1000], np.uint64), np.zeros(80000, np.uint8),
                                      np.zeros(1, np.uint64), np.array([80000], np.uint64), None, [KEEP])
    assert engine.encode_cmds_auto([]) == []


def test_full_map_records_at_the_device_bound(engine, oracle):
    """a blob of exactly max_blob_len bytes at the extreme of the device call's bound for the list's own records (three
    PredictionMode records of full maps, each coded by its own command), coded under KEEP and under replaced records: each
    equals the plain device call on the rewritten blob.  (A replaced record codes fewer entries than these records; the
    extreme for replaced records is test_many_commands_re_reading_small_records.)"""
    esc = lambda n: [(i * 37) % 256 for i in range(n)]
    pm = R.pm_line("lsb6", lmap=esc(16384), dmap=esc(1024), mix=[(i * 7) % 9 for i in range(8192)])
    allpm = oracle.Commands.from_ir("window 16 0 0 0\n" + "\n".join([pm] * 3) + "\n").serialize()
    assert len(allpm) == 32 + 3 * (20 + PMB)
    o = divans_b200.encode_options(window_size=16)
    for cands in ([KEEP], [(0, 4)], [(3, 15)], CANDS):
        d, dc, _ = _auto_device(engine, [allpm], o, cands=cands, max_blob_len=len(allpm))
        p, _, _ = _auto_device(engine, [_rewrite(allpm, cands[dc[0]])], o, max_blob_len=len(allpm), plain=True)
        assert d[0][0] == 0 and d == p, cands


# ---------------------------------------------------------------------------------------------------------------------
# 4. transcode
# ---------------------------------------------------------------------------------------------------------------------
def _pack(streams):
    import torch
    in_len = np.array([len(s) for s in streams], np.uint64)
    in_off = np.concatenate([[0], np.cumsum((in_len + np.uint64(15)) & ~np.uint64(15))[:-1]]).astype(np.uint64)
    buf = np.zeros(int(in_off[-1] + in_len[-1]) + 16, np.uint8)
    for s, o in zip(streams, in_off):
        buf[int(o):int(o) + len(s)] = np.frombuffer(s, np.uint8)
    return torch.from_numpy(buf).to("cuda:0"), in_off, in_len


def test_transcode_device_equals_transcode(engine, oracle):
    blob, off, ln = synth.text_streams(16, 65536, seed=5)
    raws = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]
    raws[1::4] = [_records(65536, w, w) for w in (2, 4, 8, 4)]
    lit = engine.encode(raws[:8])
    lz = [oracle.Commands.lz77(r, window=16).encode(oracle.options(window_size=16)) for r in raws[8:]]
    streams, caps = lit + lz, [len(r) + 64 for r in raws]
    d_in, in_off, in_len = _pack(streams)
    # without candidates: today's outputs
    d_new, new_off, new_len, status = engine.transcode_device(d_in, in_off, in_len, caps)
    new = d_new.cpu().numpy()
    assert [new[int(o):int(o) + int(n)].tobytes() for o, n in zip(new_off, new_len)] == engine.transcode(streams, caps)
    for opts in (None, divans_b200.encode_options(window_size=0, dynamic_context_mixing=2)):
        d_new, new_off, new_len, status, chosen, cost = engine.transcode_device(d_in, in_off, in_len, caps, opts, candidates=CANDS)
        assert engine.last_transcode_retried > 0
        want, wch, wcost = engine.transcode(streams, caps, opts, candidates=CANDS)
        new = d_new.cpu().numpy()
        got = [new[int(o):int(o) + int(n)].tobytes() for o, n in zip(new_off, new_len)]
        assert list(status) == [0] * len(streams) and got == want
        assert (chosen == wch).all() and (cost == wcost).all()
        assert [r for _, r in engine.decode(got, caps)] == raws
        assert (chosen[1:8:4] > 0).all() and (chosen[9::4] > 0).all()      # the records pick a stride model, not the default
        assert sum(map(len, got)) < sum(map(len, streams))


def test_transcode_device_failures(engine, oracle):
    c = R.build("lsb6", oracle)
    t = M.truncated(oracle, 0.3)
    f = R.build("corrupt_status3", oracle)
    streams = [c.stream, t.stream, c.stream, f.stream, c.stream]
    caps = [c.cap, t.cap, c.cap, f.cap, c.cap]
    d_in, in_off, in_len = _pack(streams)
    d_new, new_off, new_len, status, chosen, cost = engine.transcode_device(d_in, in_off, in_len, caps, flags=divans_b200.FLAG_SKIP_CRC,
                                                                            candidates=CANDS)
    plain = engine.decode(streams, caps, divans_b200.FLAG_SKIP_CRC)
    assert status[1] == plain[1][0] != 0 and status[3] == plain[3][0] != 0
    assert (cost[1] == T.TALLY_FAILED).all() and (cost[3] == T.TALLY_FAILED).all()
    want, wch, wcost = engine.transcode([c.stream], [c.cap], candidates=CANDS)
    new = d_new.cpu().numpy()
    for i in (0, 2, 4):
        assert status[i] == 0 and new[int(new_off[i]):int(new_off[i]) + int(new_len[i])].tobytes() == want[0]
        assert chosen[i] == wch[0] and (cost[i] == wcost[0]).all()
    with pytest.raises(divans_b200.DivansError):
        engine.transcode(streams, caps, flags=divans_b200.FLAG_SKIP_CRC, candidates=CANDS)


def _re_reading_blob(m, p=7, pool=_records(400, 4, 11)):
    """m PredictionMode commands cycling over p minimal records (empty literal and distance maps), each followed by a literal
    command that re-reads the whole pool of 4-byte records"""
    cmds = []
    for k in range(m):
        cmds += [(7, k % p, 0, 0, 0), (3, 0, len(pool), 0, 0)]
    rec = np.zeros(PMB, np.uint8)
    rec[32 + 16384 + 1024:] = 4
    hdr = np.array([0x4C435644, 1, len(cmds), p, len(pool), 16, 0, 0], np.uint32)
    return hdr.tobytes() + np.array(cmds, np.uint32).tobytes() + rec.tobytes() * p + pool


def test_many_commands_re_reading_small_records(engine, oracle):
    """The command-log bound holds per record, and any number of commands may re-read one record.  A list whose commands
    re-read minimal records fits the logs as given but outgrows them once every command codes the raw record (64 literal-map
    and 4 distance-map entries more).  The cost pass counts those entries against the same capacity, so such a pair costs
    UINT64_MAX: the default candidates keep the list's records, and the stream is the plain call's."""
    o = divans_b200.encode_options(window_size=16)
    tight = None
    for m in range(40, 70):
        b = _re_reading_blob(m)
        keep = _plain_host(engine, [b], o)[0]
        if keep[0] == 0 and all(_plain_host(engine, [_rewrite(b, c)], o)[0][0] != 0 for c in divans_b200.DEFAULT_LITERAL_MODELS):
            tight = m
            break
    assert tight is not None, "no list between 40 and 69 commands fits as given but overflows under every replaced record"
    # a few commands fewer, every candidate fits, and a stride model is cheaper than the list's own records
    small = _re_reading_blob(tight - 6)
    res, chosen, cost = _auto_host(engine, [small], o)
    assert res[0][0] == 0 and chosen[0] != 0 and (cost[0] != T.TALLY_FAILED).all(), cost
    # at the limit: every replacing candidate would overflow, so KEEP is chosen and the stream is the list as given
    b = _re_reading_blob(tight)
    res, chosen, cost = _auto_host(engine, [b], o)
    assert chosen[0] == 0 and cost[0][0] != T.TALLY_FAILED and (cost[0][1:] == T.TALLY_FAILED).all(), cost
    assert res[0] == _plain_host(engine, [b], o)[0] and res[0][0] == 0
    # without KEEP every pass fails: chosen 0, and the stream fails as the plain call on that candidate's list does
    res, chosen, cost = _auto_host(engine, [b], o, divans_b200.DEFAULT_LITERAL_MODELS)
    assert chosen[0] == 0 and (cost[0] == T.TALLY_FAILED).all()
    assert res[0] == _plain_host(engine, [_rewrite(b, divans_b200.DEFAULT_LITERAL_MODELS[0])], o)[0] and res[0][0] != 0
    # the device call (its logs are sized from max_blob_len, at least the host's): the stream is the plain device call's on the
    # chosen candidate's list, and no candidate that fits is refused
    for blob in (small, b):
        d, dc, dk = _auto_device(engine, [blob], o)
        p, _, _ = _auto_device(engine, [_rewrite(blob, CANDS[dc[0]])], o, plain=True)
        assert d == p and d[0][0] == 0
