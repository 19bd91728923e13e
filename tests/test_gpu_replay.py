"""Replaying command lists to raw bytes on the GPU (divans_b200_replay_cmds_batch_host / _device, Engine.replay).  The reference of
every check is the CPU oracle: dvo_recode_blob (oracle_tally), itself pinned to the oracle's recode in test_replay_oracle.py,
or the raw bytes a list was made from.  Status, out_len and bytes must be equal; bytes around every output region must not
change.  The first two tests need no GPU."""
import hashlib
import json
import lzma
import os
import re

import numpy as np
import pytest

import divans_b200
from divans_b200 import synth

import dvcl
from dvcl import BT_L, COPY, DICT, LIT, PREDMODE, blob
from irfuzz import random_ir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
gpu = pytest.mark.gpu
CANARY = 0xA5
G = 64          # guard bytes around every output region


def test_prototypes_in_header():
    h = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    common = ["divans_b200_ctx *ctx", "size_t n"]
    for name, args in (("divans_b200_replay_cmds_batch_host",
                        ["const uint8_t *blobs", "const uint64_t *blob_off", "const uint64_t *blob_len", "uint8_t *out",
                         "const uint64_t *out_off", "const uint64_t *out_cap", "uint64_t *out_len", "int32_t *status",
                         "int32_t window_size"]),
                       ("divans_b200_replay_cmds_batch_device",
                        ["const uint8_t *d_blobs", "const uint64_t *d_blob_off", "const uint64_t *d_blob_len", "uint8_t *d_out",
                         "const uint64_t *d_out_off", "const uint64_t *d_out_cap", "uint64_t *d_out_len", "int32_t *d_status",
                         "int32_t window_size", "void *cuda_stream"])):
        m = re.search(r"DivansResult\s+%s\(([^;]*)\);" % name, h)
        assert m, name
        assert [a.strip() for a in " ".join(m.group(1).split()).split(",")] == common + args


def test_symbols_listed():
    assert {"divans_b200_replay_cmds_batch_host", "divans_b200_replay_cmds_batch_device"} <= set(divans_b200.BATCH_SYMBOLS)


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def T():
    from oracle_tally import tally_py
    tally_py.build()
    return tally_py


def _layout(caps):
    """output regions of caps[i] bytes with G guard bytes before, between and after them -> (out_off, total)"""
    off, pos = [], G
    for c in caps:
        off.append(pos)
        pos += int(c) + G
    return off, pos


def _check_regions(o, out_off, caps):
    mask = np.ones(o.size, bool)
    for a, c in zip(out_off, caps):
        mask[a:a + int(c)] = False
    assert (o[mask] == CANARY).all(), "a byte outside the output regions changed"


def _host(eng, blobs, caps, window=0, shift=None, alias=False):
    """replay_cmds_batch_host: [(status, out_len, region bytes)].  `shift[i]` puts blob i at an offset that is not 4-byte
    aligned; `alias`: every list is blobs[0] at one offset."""
    n = len(blobs)
    shift = [0] * n if shift is None else shift
    offs, pos = [], 0
    for b, s in zip(blobs, shift):
        offs.append(pos + s)
        pos = (pos + s + len(b) + 15) & ~15
    inp = np.zeros(pos + 16, np.uint8)
    for b, o in zip(blobs, offs):
        inp[o:o + len(b)] = np.frombuffer(bytes(b), np.uint8)
    if alias:
        offs = [offs[0]] * n
    out_off, total = _layout(caps)
    out = np.full(total, CANARY, np.uint8)
    ln, st = eng.replay_cmds_batch_host(inp, offs, [len(b) for b in blobs], out, out_off, caps, window)
    _check_regions(out, out_off, caps)
    return [(int(s), int(l), out[a:a + int(c)].tobytes()) for s, l, a, c in zip(st, ln, out_off, caps)]


def _device(eng, blobs, caps, window=0, misalign=None, lens=None, stream=None):
    """replay_cmds_batch_device with guard bytes around every output region: [(status, out_len, region bytes)]"""
    import torch
    n = len(blobs)
    shift = [0] * n if misalign is None else misalign
    lens = [len(b) for b in blobs] if lens is None else lens
    offs, pos = [], 0
    for b, s in zip(blobs, shift):
        offs.append(pos + s)
        pos = (pos + s + len(b) + 16 + 255) & ~255
    inp = np.zeros(pos + 256, np.uint8)
    for b, o in zip(blobs, offs):
        inp[o:o + len(b)] = np.frombuffer(bytes(b), np.uint8)
    out_off, total = _layout(caps)
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.array(a, np.uint64).reshape(-1).view(np.int64)).to(dev)
    d_in = torch.from_numpy(inp).to(dev)
    d_out = torch.full((total,), CANARY, dtype=torch.uint8, device=dev)
    d_meta = [u64(offs), u64(lens), u64(out_off), u64(caps)]
    d_len = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
    d_st = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    torch.cuda.current_stream().synchronize()
    eng.replay_cmds_batch_device(n, d_in.data_ptr(), d_meta[0].data_ptr(), d_meta[1].data_ptr(), d_out.data_ptr(), d_meta[2].data_ptr(),
                                 d_meta[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), window, None if stream is None else stream.cuda_stream)
    if stream is not None:
        stream.synchronize()
    else:
        eng.synchronize()
    o = d_out.cpu().numpy()
    _check_regions(o, out_off, caps)
    st, ln = d_st.cpu().numpy()[:n], d_len.cpu().numpy()[:n].view(np.uint64)
    return [(int(s), int(l), o[a:a + int(c)].tobytes()) for s, l, a, c in zip(st, ln, out_off, caps)]


def _expect(T, blobs, caps, window=0):
    return [T.recode_blob(b, window, int(c)) for b, c in zip(blobs, caps)]


def _agree(got, want, what, host):
    """got: [(status, out_len, region)], want: dvo_recode_blob's [(rc, out_len, bytes)]"""
    for i, ((s, n, region), (rc, n_ref, ref)) in enumerate(zip(got, want)):
        assert (s, n) == (rc, n_ref), "%s: list %d: (status, out_len) %s, oracle %s" % (what, i, (s, n), (rc, n_ref))
        k = min(n, len(region))
        assert region[:k] == ref[:k], "%s: list %d: bytes differ" % (what, i)
        if host:   # host regions are written whole: zeros past what the list produced
            assert region[k:] == bytes(len(region) - k), "%s: list %d: host region not zero past out_len" % (what, i)


def _both(eng, T, blobs, caps=None, window=0, what=""):
    """host and device calls against the oracle (and so against each other)"""
    caps = [T.recode_blob(b, window, 0)[1] for b in blobs] if caps is None else list(caps)
    caps = [min(int(c), 1 << 26) for c in caps]
    want = _expect(T, blobs, caps, window)
    h, d = _host(eng, blobs, caps, window), _device(eng, blobs, caps, window)
    _agree(h, want, what + " (host)", True)
    _agree(d, want, what + " (device)", False)
    assert [x[:2] for x in h] == [x[:2] for x in d]
    return h


def _records(n, width, seed):
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n].tobytes()


def _ir_fixtures():
    """(blob, window, raw sha256) of the two stored IR fixtures through divans_b200.ir_to_cmds, with the window the oracle's
    fixture test replays them with (c.window or 22)"""
    raw = open(os.path.join(GOLD, "ends_with_truncated_dictionary"), "rb").read()
    b1, w1 = divans_b200.ir_to_cmds(open(os.path.join(GOLD, "ends_with_truncated_dictionary.ir"), "rb").read())
    b2, w2 = divans_b200.ir_to_cmds(lzma.decompress(open(os.path.join(GOLD, "asyoulik.ir.xz"), "rb").read()))
    e = [g for g in json.load(open(os.path.join(GOLD, "golden.json"))) if g["name"] == "asyoulik_ir_mix2"][0]
    return [(b1, w1 or 22, hashlib.sha256(raw).hexdigest()), (b2, w2 or 22, e["raw_sha256"])]


def _edge_list(w, seed, T):
    """a list at window w with what random IR rarely reaches: a copy at distance (1 << w) - 1 reaching before position 0,
    copies of distance < 32 that overlap their own output, a dictionary word under every transform, and (w <= 16) a copy of
    distance (1 << w) - 1 after more than a ring of output"""
    rng = np.random.default_rng(seed)
    pool = bytes(rng.integers(0, 256, 3000).astype(np.uint8))
    ring = 1 << w
    cmds = [(PREDMODE, 0, 0, 0, 0), (COPY, ring - 1, 40, 0, 0), (LIT, 0, 1000, 0, 0), (COPY, ring - 1, 300, 0, 0)]
    for d in range(1, 32):
        cmds += [(LIT, int(rng.integers(0, 2900)), int(rng.integers(1, 40)), 0, 0), (COPY, d, int(rng.integers(1, 200)), 0, 0)]
    buf = np.zeros(64, np.uint8)
    from oracle import oracle_py as O
    for t in range(121):
        while True:
            ws = int(rng.integers(4, 25))
            bits = [0, 0, 0, 0, 10, 10, 11, 11, 10, 10, 10, 10, 10, 9, 9, 8, 7, 7, 8, 7, 7, 6, 6, 5, 5][ws]
            wid = int(rng.integers(0, 1 << bits))
            n = O.lib().dvo_dict_word(ws, wid, t, buf.ctypes.data)
            if n > 0:
                break
        cmds.append((DICT, wid, ws, t, n if t % 2 else 0))
    if w <= 16:
        cmds += [(LIT, 0, 3000, 0, 0)] * (ring // 3000 + 1) + [(COPY, ring - 1, 500, 0, 0), (COPY, 7, ring, 0, 0)]
    cmds.append((COPY, 1, 33, 0, 0))
    return blob(cmds, pool, n_pms=1, window=w)


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_golden_ir_fixtures(engine, T):
    for b, w, sha in _ir_fixtures():
        n = T.recode_blob(b, w, 0)[1]
        for res in (_host(engine, [b], [n], w), _device(engine, [b], [n], w)):
            (st, ln, out), = res
            assert st == 0 and ln == n and hashlib.sha256(out).hexdigest() == sha
        (st, out), = engine.replay([b], w)
        assert st == 0 and hashlib.sha256(out).hexdigest() == sha


@gpu
@pytest.mark.parametrize("window", [10, 14, 16, 22, 24])
def test_random_ir(engine, oracle, T, window):
    text = synth.text_corpus(1 << 18)
    blobs = [oracle.Commands.from_ir(random_ir(oracle, 900 + 17 * window + s, n_cmds=160, window=window, text=text)).serialize()
             for s in range(10)]
    blobs += [_edge_list(window, window, T)]
    _both(engine, T, blobs, window=0, what="random IR, header window %d" % window)
    _both(engine, T, blobs, window=window, what="random IR, window %d" % window)
    # the replay of a random IR list is the oracle's recode of it
    c = oracle.Commands.from_ir(random_ir(oracle, 4242 + window, n_cmds=160, window=window, text=text))
    rc, ref = c.recode(window)
    assert rc == 0 and engine.replay([c.serialize()]) == [(0, ref)]


@gpu
def test_lz77_lists(engine):
    blob_, off, ln = synth.text_streams(3, 40000, seed=5)
    text = [blob_[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)]
    cyr = b"".join(chr(0x430 + (c % 26)).encode() if 97 <= c < 123 else bytes([c]) for c in text[1])[:40000]
    raws = [text[0], cyr, _records(30000, 2, 1), _records(30000, 4, 2), _records(30000, 8, 3), text[2][:1], b""]
    packed, roff, rlen = divans_b200._pack(raws)
    bl, boff, blen = divans_b200.lz77_cmds_batch(packed, roff, rlen, window=16)
    blobs = [bl[int(o):int(o) + int(l)].tobytes() for o, l in zip(boff, blen)]
    assert engine.replay(blobs) == [(0, r) for r in raws]
    caps = [len(r) for r in raws]
    for res in (_host(engine, blobs, caps), _device(engine, blobs, caps)):
        assert [(s, n, o) for s, n, o in res] == [(0, len(r), r) for r in raws]


def _golden_streams():
    gold = json.load(open(os.path.join(GOLD, "golden.json")))
    return [open(os.path.join(GOLD, e["name"] + ".divans"), "rb").read() for e in gold], [e["raw_len"] for e in gold]


@gpu
def test_decoded_streams_host(engine):
    streams, lens = _golden_streams()
    blob_, off, ln = synth.text_streams(24, 65536, seed=3)
    raws = [blob_[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)]
    streams += engine.encode(raws)
    lens += [len(r) for r in raws]
    dec = engine.decode_cmds(streams, [n + 64 for n in lens])
    assert all(st == 0 for st, _, _ in dec)
    assert engine.replay([b for _, _, b in dec]) == [(0, raw) for _, raw, _ in dec]


@gpu
def test_decoded_streams_device(engine):
    """decode_cmds_batch_device, then the replay of its blobs where the decoder left them in HBM, against the decoded bytes"""
    import torch
    streams, lens = _golden_streams()
    blob_, off, ln = synth.text_streams(40, 65536, seed=4)
    raws = [blob_[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)]
    streams += engine.encode(raws)
    lens += [len(r) for r in raws]
    n = len(streams)
    packed, in_off, in_len = divans_b200._pack(streams)
    out_cap = np.array([x + 64 for x in lens], np.uint64)
    host = engine.decode_cmds(streams, out_cap)   # (the IR streams' lists outgrow first_blob_cap: take each list's size)
    blob_cap = np.array([len(b) for _, _, b in host], np.uint64)
    (out_off, out_total), (blob_off, blobs_total), (rep_off, rep_total) = (divans_b200._regions(out_cap), divans_b200._regions(blob_cap),
                                                                           divans_b200._regions(out_cap))
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev)
    d_in = torch.from_numpy(packed).to(dev)
    M = [u64(a) for a in (in_off, in_len, out_off, out_cap, blob_off, blob_cap, rep_off)]
    d_out = torch.zeros(out_total, dtype=torch.uint8, device=dev)
    d_blobs = torch.zeros(blobs_total, dtype=torch.uint8, device=dev)
    d_rep = torch.zeros(rep_total, dtype=torch.uint8, device=dev)
    d_res = torch.zeros(4 * n, dtype=torch.int64, device=dev)     # out_len | blob_len | replay out_len | both statuses
    d_st = d_res[3 * n:].view(torch.int32)
    torch.cuda.current_stream().synchronize()
    engine.decode_cmds_batch_device(d_in.data_ptr(), M[0].data_ptr(), M[1].data_ptr(), d_out.data_ptr(), M[2].data_ptr(), M[3].data_ptr(),
                                    d_res.data_ptr(), d_blobs.data_ptr(), M[4].data_ptr(), M[5].data_ptr(), d_res[n:].data_ptr(),
                                    d_st[:n].data_ptr(), n, int(in_len.sum()))
    engine.replay_cmds_batch_device(n, d_blobs.data_ptr(), M[4].data_ptr(), d_res[n:].data_ptr(), d_rep.data_ptr(), M[6].data_ptr(),
                                    M[3].data_ptr(), d_res[2 * n:].data_ptr(), d_st[n:].data_ptr())
    engine.synchronize()
    r = d_res.cpu().numpy()
    st = r[3 * n:].view(np.int32)
    assert (st == 0).all()
    assert (r[:n] == r[2 * n:3 * n]).all() and list(r[:n]) == lens
    o, rep = d_out.cpu().numpy(), d_rep.cpu().numpy()
    for i in range(n):
        a, b = int(out_off[i]), int(rep_off[i])
        assert rep[b:b + lens[i]].tobytes() == o[a:a + lens[i]].tobytes() == host[i][1], "stream %d" % i


@gpu
def test_status_2(engine, oracle, T):
    text = synth.text_corpus(1 << 17)
    blobs = [oracle.Commands.from_ir(random_ir(oracle, 55 + s, n_cmds=120, window=16, text=text)).serialize() for s in range(6)]
    blobs += [b for b, _, _ in _ir_fixtures()[:1]]
    lens = [T.recode_blob(b, 16, 0)[1] for b in blobs]
    assert min(lens) > 1
    for caps in ([0] * len(blobs), [n - 1 for n in lens], [n // 3 for n in lens]):
        res = _both(engine, T, blobs, caps, 16, "caps %s" % caps[:3])
        assert all(s == 2 and ln == n for (s, ln, _), n in zip(res, lens))


@gpu
def test_hostile_blobs(engine, oracle, T):
    cases = dvcl.refusal_cases()
    blobs = [b for _, b, _, _ in cases]
    for w in sorted({w for _, _, w, _ in cases}):
        idx = [i for i, c in enumerate(cases) if c[2] == w]
        res = _both(engine, T, [blobs[i] for i in idx], [64] * len(idx), w, "refusal rules, window %d" % w)
        for k, i in enumerate(idx):
            assert res[k][:2] == (3, cases[i][3]), cases[i][0]
    # misaligned device blobs: refused before any byte is read
    good = blob([(LIT, 0, 3, 0, 0)], b"abc")
    res = _device(engine, [good] * 4, [16] * 4, misalign=[0, 1, 2, 3])
    assert [r[:2] for r in res] == [(0, 3), (3, 0), (3, 0), (3, 0)]
    # the host call takes any offset: its blobs are re-based
    assert [r[:2] for r in _host(engine, [good] * 4, [16] * 4, shift=[0, 1, 2, 3])] == [(0, 3)] * 4
    # pool offsets and copy lengths near 2^32: refused, or (64-bit positions) walked without moving bytes
    lits = b"abcdefgh"
    near = [blob([(LIT, 0, 3, 0, 0), (LIT, 0xFFFFFFF8, 0x10, 0, 0)], lits),
            blob([(LIT, 0, 3, 0, 0), (LIT, 4, 0xFFFFFFFE, 0, 0)], lits),
            blob([(LIT, 0, 3, 0, 0), (COPY, 1, 0xFFFFFFF0, 0, 0)], lits),
            blob([(LIT, 0, 3, 0, 0), (COPY, 1, 0xFFFFFFFF, 0, 0), (COPY, 2, 0xFFFFFFFF, 0, 0), (LIT, 0, 8, 0, 0)], lits),
            blob([(LIT, 0, 3, 0, 0), (COPY, 1, 0xFFFFFFFF, 0, 0), (COPY, 0, 1, 0, 0)], lits)]
    res = _both(engine, T, near, [100] * len(near), 0, "near 2^32")
    assert [r[:2] for r in res] == [(3, 3), (3, 3), (2, 3 + 0xFFFFFFF0), (2, 3 + 2 * 0xFFFFFFFF + 8), (3, 3 + 0xFFFFFFFF)]
    # truncation at every 4-byte boundary, and seeded bit flips in the header and the records
    small = blob([(LIT, 0, 30, 0, 0), (COPY, 7, 50, 0, 0), (DICT, 9, 8, 30, 0), (BT_L, 1, 0, 0, 0), (LIT, 30, 33, 0, 0)],
                 bytes(range(100, 163)), window=12)
    cuts = [small[:k] for k in range(0, len(small) + 1, 4)]
    _both(engine, T, cuts, [256] * len(cuts), 0, "truncated")
    rng = np.random.default_rng(1234)
    base = blob([(PREDMODE, 0, 0, 0, 0), (LIT, 0, 40, 0, 0), (COPY, 3, 20, 0, 0), (DICT, 5, 6, 7, 0), (COPY, 40, 100, 0, 0),
                 (LIT, 10, 20, 0, 0), (DICT, 100, 10, 50, 0)], bytes(range(40)), n_pms=1, window=10)
    n_rec = 32 + 20 * 7
    muts = []
    for k in range(400):
        m = bytearray(base)
        for _ in range(int(rng.integers(1, 4))):
            bit = int(rng.integers(0, 8 * (32 if k % 2 else n_rec)))
            m[bit >> 3] ^= 1 << (bit & 7)
        muts.append(bytes(m))
    _both(engine, T, muts, [300] * len(muts), 0, "bit flips")


@gpu
def test_batch_behaviour(engine, oracle, T):
    import torch
    # n == 0
    assert engine.replay([]) == []
    ln, st = engine.replay_cmds_batch_host(np.zeros(1, np.uint8), [], [], np.zeros(1, np.uint8), [], [])
    assert ln.size == 0 and st.size == 0
    engine.replay_cmds_batch_device(0, 0, 0, 0, 0, 0, 0, 0, 0)
    # aliased inputs: one list replayed n times from one offset
    b = oracle.Commands.from_ir(random_ir(oracle, 5, n_cmds=80, window=14)).serialize()
    n = T.recode_blob(b, 0, 0)[1]
    want = T.recode_blob(b, 0, n)
    assert _host(engine, [b] * 5, [n] * 5, alias=True) == [want] * 5
    # more lists than resident warps, one launch: 20 000 small lists, each a literal and a copy of its own
    rng = np.random.default_rng(9)
    many = [blob([(LIT, 0, 1 + i % 7, 0, 0), (COPY, 1 + i % 5, i % 13, 0, 0)], bytes(rng.integers(0, 256, 8).astype(np.uint8)),
                 window=10) for i in range(20000)]
    caps = [1 + i % 7 + i % 13 for i in range(20000)]
    want = _expect(T, many, caps)
    before = engine.launch_count
    _agree(_device(engine, many, caps), want, "20000 lists (device)", False)
    assert engine.launch_count == before + 1
    _agree(_host(engine, many, caps), want, "20000 lists (host)", True)
    assert engine.launch_count == before + 2
    # a fresh context, on a CUDA stream of its own
    eng = divans_b200.Engine(0, 0, 16)
    try:
        s = torch.cuda.Stream()
        blobs = [oracle.Commands.from_ir(random_ir(oracle, 60 + k, n_cmds=60, window=16)).serialize() for k in range(8)]
        caps = [T.recode_blob(x, 0, 0)[1] for x in blobs]
        _agree(_device(eng, blobs, caps, stream=s), _expect(T, blobs, caps), "fresh context, own stream", False)
        assert eng.launch_count == 1
        assert eng.last_kernel_ms() > 0
    finally:
        eng.close()


@gpu
def test_launch_count(engine, oracle):
    b = oracle.Commands.from_ir(random_ir(oracle, 8, n_cmds=40, window=16)).serialize()
    before = engine.launch_count
    _host(engine, [b, b], [10, 10**5])
    assert engine.launch_count == before + 1
    _device(engine, [b, b], [10, 10**5])
    assert engine.launch_count == before + 2
    engine.replay([b, b])                 # a length pass and an exact pass
    assert engine.launch_count == before + 4


def _replay_len(b):
    """the encoder host call's replay bound of a well-formed list: 64 bytes per dictionary word"""
    h = np.frombuffer(bytes(b[:32]), np.uint32)
    r = np.frombuffer(bytes(b[32:32 + 20 * int(h[2])]), np.uint32).reshape(-1, 5)
    return int(r[r[:, 0] == 1, 2].sum() + r[r[:, 0] == 3, 2].sum() + 64 * (r[:, 0] == 2).sum())


@gpu
def test_device_sizing_of_the_encoder(engine, oracle, T):
    """max_raw_len of encode_cmds_batch_device from a device length pass: lists with dictionary words, where the host-side
    bound overstates the length, encode with exactly the longest measured length, and decode to the replayed bytes"""
    import torch
    text = synth.text_corpus(1 << 18)
    groups = [([oracle.Commands.from_ir(random_ir(oracle, 3100 + s, n_cmds=200, window=16, text=text)).serialize() for s in range(12)], 0),
              ([b for b, _, _ in _ir_fixtures()], 22)]
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev)
    for blobs, w in groups:
        n = len(blobs)
        packed, off, ln = divans_b200._pack(blobs)
        d_blobs, d_off, d_len = torch.from_numpy(packed).to(dev), u64(off), u64(ln)
        d_zero = u64(np.zeros(n, np.uint64))
        d_res = torch.zeros(2 * n, dtype=torch.int64, device=dev)
        torch.cuda.current_stream().synchronize()
        engine.replay_cmds_batch_device(n, d_blobs.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), d_blobs.data_ptr(), d_zero.data_ptr(),
                                        d_zero.data_ptr(), d_res.data_ptr(), d_res[n:].data_ptr(), w)
        engine.synchronize()
        r = d_res.cpu().numpy()
        assert (r[n:].view(np.int32)[:n] != 3).all()
        lens = r[:n].view(np.uint64)
        max_raw = int(lens.max())
        assert any(_replay_len(b) > x for b, x in zip(blobs, lens))   # lists whose length the host-side bound overstates
        assert list(lens) == [T.recode_blob(b, w, 0)[1] for b in blobs]
        out_cap = divans_b200._encoded_cap(ln)
        out_off, total = divans_b200._regions(out_cap)
        d_out = torch.zeros(total, dtype=torch.uint8, device=dev)
        d_o, d_c = u64(out_off), u64(out_cap)
        d_enc = torch.zeros(2 * n, dtype=torch.int64, device=dev)
        engine.encode_cmds_batch_device(n, d_blobs.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()), max_raw, d_out.data_ptr(),
                                        d_o.data_ptr(), d_c.data_ptr(), d_enc.data_ptr(), d_enc[n:].data_ptr(),
                                        divans_b200.encode_options(window_size=w))
        engine.synchronize()
        e = d_enc.cpu().numpy()
        assert (e[n:].view(np.int32)[:n] == 0).all()
        o = d_out.cpu().numpy()
        streams = [o[int(a):int(a) + int(k)].tobytes() for a, k in zip(out_off, e[:n])]
        rep = engine.replay(blobs, w)
        assert engine.decode(streams, [int(x) + 64 for x in lens]) == rep


@gpu
def test_copy_longer_than_one_chunk(engine):
    """A copy of more than 2^31 bytes into a region that holds it: the kernel hands replay_copy chunks of at most 2^31 bytes, the
    first one from before position 0 (distance 5 after 3 bytes), the next rebased at its source.  The output is periodic:
    byte j is P[(j + 2) mod 5] with P = 00 00 'a' 'b' 'c'.  Checked on the device, slice by slice."""
    import torch
    L = (1 << 31) + 80
    b = blob([(LIT, 0, 3, 0, 0), (COPY, 5, L - 3, 0, 0)], b"abc", window=10)
    dev = torch.device("cuda:0")
    torch.cuda.empty_cache()
    d_in = torch.from_numpy(np.frombuffer(b, np.uint8).copy()).to(dev)
    d_out = torch.full((L + 2 * G,), CANARY, dtype=torch.uint8, device=dev)
    d_meta = torch.from_numpy(np.array([0, len(b), G, L], np.uint64).view(np.int64)).to(dev)
    d_len = torch.zeros(1, dtype=torch.int64, device=dev)
    d_st = torch.full((1,), -1, dtype=torch.int32, device=dev)
    torch.cuda.current_stream().synchronize()
    before = engine.launch_count
    engine.replay_cmds_batch_device(1, d_in.data_ptr(), d_meta[0:].data_ptr(), d_meta[1:].data_ptr(), d_out.data_ptr(),
                                    d_meta[2:].data_ptr(), d_meta[3:].data_ptr(), d_len.data_ptr(), d_st.data_ptr())
    engine.synchronize()
    assert engine.launch_count == before + 1
    assert (int(d_st.item()), int(d_len.item())) == (0, L)
    assert bool((d_out[:G] == CANARY).all()) and bool((d_out[G + L:] == CANARY).all())
    S = 1 << 26
    pat = torch.tensor([0, 0, ord("a"), ord("b"), ord("c")], dtype=torch.uint8, device=dev).repeat(S // 5 + 2)
    for s in range(0, L, S):
        k = min(S, L - s)
        o = (s + 2) % 5
        assert torch.equal(d_out[G + s:G + s + k], pat[o:o + k]), "bytes differ in [%d, %d)" % (s, s + k)
    del d_out
    torch.cuda.empty_cache()
    # Engine.replay measures before it allocates: a 4 GiB run is refused above its bound, not allocated
    huge = blob([(LIT, 0, 3, 0, 0), (COPY, 1, 0xFFFFFFFF, 0, 0)], b"abc", window=10)
    with pytest.raises(divans_b200.DivansError, match="max_bytes"):
        engine.replay([huge])
