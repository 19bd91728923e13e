"""GPU tests (-m gpu) of the blend model at every regime, framing edge, record chain, block composition and slot succession the
default model is tested at (tests/test_gpu_slot_state.py, test_gpu_parity.py, test_gpu_encode.py, test_gpu_decode_cmds.py).

The blend decoder is the v2 decoder body instantiated with BLEND (dv2_kernels.cu): every literal nibble goes through the
generic path, the literal priors live in lazily initialised slabs, a block holds two warps (four 16-lane groups), and the slot
is reset in full.  Every status, every output byte, every recorded command list and every encoded stream is compared with
the blend oracle (oracle/oracle_blend.py); the regimes and edges are the ones of tests/regimes.py built with that oracle
(BLEND_EDGES for the payload edges, whose lengths differ under the blend model)."""
import ctypes
import itertools

import numpy as np
import pytest

import divans_b200
import dvcl
import regimes as R

pytestmark = pytest.mark.gpu

BLEND = divans_b200.FLAG_CDF_BLEND
ONE_BLOCK = (0, 4, 8)      # Engine(0, 4, 8): one blend block of four slots; the 8-lane layout runs one warp on the same four


@pytest.fixture(scope="module")
def bcases(oracle_blend):
    return {n: R.build(n, oracle_blend) for n in R.ALL}


@pytest.fixture(scope="module")
def bedges(oracle_blend):
    res = {}
    for n in R.EDGE_NAMES:
        _cl, raw, stream = R.edge(n, oracle_blend)
        res[n] = R.Case(stream, raw, 0, 0, len(raw) + 64)
    return res


@pytest.fixture
def block():
    eng = divans_b200.Engine(*ONE_BLOCK)
    yield eng
    eng.close()


def _first_diff(a, b):
    return next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), min(len(a), len(b)))


_REF = {}


def _ref(oracle, c, skip_crc):
    """(status, bytes) of the oracle's decode of case `c` (memoised: the composition tests send each case many times)"""
    key = (R.is_blend(oracle), c.stream, c.cap, skip_crc)
    if key not in _REF:
        _REF[key] = oracle.decode(c.stream, out_cap=c.cap, skip_crc=skip_crc)
    return _REF[key]


def _check(eng, oracle, cases, what=""):
    """one launch of `cases` under `oracle`'s model; every status equals the oracle's (and the case's), every output its bytes"""
    flags = BLEND if R.is_blend(oracle) else 0
    for c in cases:
        flags |= c.flags
    res = eng.decode([c.stream for c in cases], [c.cap for c in cases], flags)
    for i, ((st, out), c) in enumerate(zip(res, cases)):
        rc, ref = _ref(oracle, c, bool(flags & divans_b200.FLAG_SKIP_CRC))
        assert rc == c.status, (what, i)
        assert st == rc, "%s: stream %d: status %d, oracle %d" % (what, i, st, rc)
        if rc == 0:
            assert out == ref, "%s: stream %d: first diff at %d" % (what, i, _first_diff(out, ref))
    return res


# ---------------------------------------------------------------------------------------------------------------------
# decode: every regime and edge, on every engine
# ---------------------------------------------------------------------------------------------------------------------
def test_regimes_and_edges_on_every_engine(engine, oracle_blend, bcases, bedges):
    """One batch of every regime and every blend edge on the session engine, an 8-lane context and an automatic-lanes context:
    the blend model has the 16-lane layout only, whatever the context's lane choice."""
    cases = [bcases[n] for n in R.ALL] + [bedges[n] for n in R.EDGE_NAMES]
    eng8, auto = divans_b200.Engine(0, 0, 8), divans_b200.Engine(0, 0, 0)
    try:
        for what, eng in (("session", engine), ("8 lanes", eng8), ("auto", auto)):
            _check(eng, oracle_blend, cases, what)
            assert eng.last_lanes() == 16, what
            # each edge alone, CRC checked: the batch above skips the CRC for the corrupted regimes
            _check(eng, oracle_blend, [bedges[n] for n in R.EDGE_NAMES] + [bcases[n] for n in R.GOOD], what + ", CRC")
    finally:
        eng8.close()
        auto.close()


# ---------------------------------------------------------------------------------------------------------------------
# record chains
# ---------------------------------------------------------------------------------------------------------------------
def test_remuxed_blend_edges_on_every_layout(engine, oracle_blend, bedges):
    """every blend edge under every record layout (one-byte records only where the payloads are short), next to the stream as
    the mux wrote it"""
    cases = []
    for name in R.EDGE_NAMES:
        c = bedges[name]
        lens = tuple(len(p) for p in oracle_blend.demux(c.stream))
        cases.append(c)
        for k, lay in enumerate(R.LAYOUTS):
            if lay == "one_byte" and sum(lens) > 40000:
                continue
            s2 = R.mux_records(oracle_blend, c.stream, R.layout(lay, lens, seed=k))
            cases.append(R.Case(s2, c.raw, 0, 0, c.cap))
    assert len(cases) >= 3 * len(R.EDGE_NAMES)
    _check(engine, oracle_blend, cases, "re-muxed")


def test_hostile_blend_record_chains_match_the_oracle(engine, oracle_blend, bedges):
    """truncation inside a three-byte record header and inside a one-byte-code record, a code k > 3, a header byte 2..15:
    statuses and accepted outputs equal the blend oracle's"""
    c = bedges["both_over"]
    lens = tuple(len(p) for p in oracle_blend.demux(c.stream))
    plan = R.layout("codes", lens, seed=1)
    starts = R.record_starts(plan)
    good = R.mux_records(oracle_blend, c.stream, plan)
    body = good[:len(good) - 11]
    three = [i for i, (_c, _n, k) in enumerate(plan) if k is None]
    coded = [i for i, (_c, _n, k) in enumerate(plan) if k is not None]
    streams = []
    for i in three[:3]:
        streams += [good[:starts[i] - 2], good[:starts[i] - 1]]
    for i in coded[:3]:
        streams.append(good[:starts[i] + plan[i][1] // 2])
    for i, kk in zip(coded[:3], (4, 9, 15)):
        b = bytearray(body); b[starts[i] - 1] = plan[i][0] | (kk << 4)
        streams.append(R.close(oracle_blend, bytes(b)))
    for i, v in zip(three[:4], (2, 7, 12, 15)):
        b = bytearray(body); b[starts[i] - 3] = (v & ~1) | plan[i][0]
        if b[starts[i] - 3] < 2:
            b[starts[i] - 3] += 2
        streams.append(R.close(oracle_blend, bytes(b)))
    streams = [c.stream, good] + streams + [c.stream]
    ref = [oracle_blend.decode(s, out_cap=c.cap) for s in streams]
    assert [r[0] for r in ref].count(0) >= 6 and {r[0] for r in ref} >= {0, 1, 3}, [r[0] for r in ref]
    res = engine.decode(streams, [c.cap] * len(streams), BLEND)
    for i, ((st, out), (rc, rb)) in enumerate(zip(res, ref)):
        assert st == rc, "stream %d: status %d, oracle %d" % (i, st, rc)
        if rc == 0:
            assert out == rb == c.raw, i


# ---------------------------------------------------------------------------------------------------------------------
# block composition: four groups in two warps
# ---------------------------------------------------------------------------------------------------------------------
def test_every_pair_of_regimes_in_one_block(block, oracle_blend, bcases):
    """[a, b, a, b] on one block of four slots: each warp's two groups take a and b (groups 2 and 3 are the second warp's)"""
    for a, b in itertools.combinations_with_replacement(R.ALL, 2):
        _check(block, oracle_blend, [bcases[a], bcases[b], bcases[a], bcases[b]], "%s + %s" % (a, b))
    assert block.last_lanes() == 16


def test_seeded_quads_of_regimes_in_one_block(block, oracle_blend, bcases):
    rng = np.random.default_rng(2025)
    for _ in range(80):
        pick = [R.ALL[int(k)] for k in rng.integers(0, len(R.ALL), 4)]
        _check(block, oracle_blend, [bcases[n] for n in pick], " + ".join(pick))


# ---------------------------------------------------------------------------------------------------------------------
# slot succession: one launch per step, each of the four slots takes one stream
# ---------------------------------------------------------------------------------------------------------------------
def _headers(eng):
    return [eng.slot_header(i) for i in range(4)]


def _step(eng, oracle, c, what):
    """one launch in which every slot decodes `c`; returns the slot headers after it.  A blend launch leaves header word 0
    (the default model's generation counter) alone and sets word 1 (the next default stream must wipe the tables)."""
    before = _headers(eng) if eng.launch_count else [[0] * 4] * 4
    _check(eng, oracle, [c] * 4, what)
    after = _headers(eng)
    if R.is_blend(oracle):
        assert [h[0] for h in after] == [h[0] for h in before], (what, before, after)
        assert [h[1] for h in after] == [1] * 4, (what, after)
    else:
        assert [h[0] - b[0] for h, b in zip(after, before)] == [1] * 4, (what, before, after)
    return after


def test_blend_after_blend(block, oracle_blend, bcases):
    """the full-map stream, then the stream without PredictionMode (a zero map); per-context mixing values, then mixing value 0
    everywhere; each failing regime, then plain and mixing streams"""
    h = _step(block, oracle_blend, bcases["bt256"], "bt256")
    assert [x[2] for x in h] == [16384] * 4
    h = _step(block, oracle_blend, bcases["no_predmode"], "no_predmode after bt256")
    assert [x[2] for x in h] == [0] * 4
    h = _step(block, oracle_blend, bcases["per_context_mix"], "per_context_mix")
    assert [x[3] for x in h] == [1] * 4
    h = _step(block, oracle_blend, bcases["no_predmode"], "no_predmode after per_context_mix")
    assert [x[3] for x in h] == [0] * 4
    for f in R.FAILING:
        for n in (f, "lsb6", "dcm2"):
            _step(block, oracle_blend, bcases[n], "%s after %s" % (n, f))


def test_default_after_blend(block, oracle, oracle_blend, bcases):
    """a blend stream leaves the map high-water mark and the stale-mixing flag for the default model's lazy reset"""
    h = _step(block, oracle_blend, bcases["bt256"], "blend bt256")
    assert [x[2] for x in h] == [16384] * 4
    h = _step(block, oracle, R.build("no_predmode", oracle), "default no_predmode after blend bt256")
    assert [x[2] for x in h] == [0] * 4 and [x[1] for x in h] == [0] * 4
    h = _step(block, oracle_blend, bcases["per_context_mix"], "blend per_context_mix")
    assert [x[3] for x in h] == [1] * 4
    h = _step(block, oracle, R.build("no_predmode", oracle, 1), "default no_predmode after blend per_context_mix")
    assert [x[3] for x in h] == [0] * 4
    _step(block, oracle, R.build("lsb6", oracle), "default lsb6")


def test_blend_after_default(block, oracle, oracle_blend, bcases):
    """default streams with untagged priors (wide speeds), the full map, and mixing priors, each followed by blend streams"""
    h = _step(block, oracle, R.build("wide_midstream", oracle), "default wide_midstream")
    assert [x[1] for x in h] == [1] * 4
    for n in ("lsb6", "bt256"):
        _step(block, oracle_blend, bcases[n], "blend %s after default wide_midstream" % n)
    h = _step(block, oracle, R.build("bt256", oracle), "default bt256")
    assert [x[2] for x in h] == [16384] * 4 and [x[1] for x in h] == [0] * 4
    for n in ("no_predmode", "switches"):
        _step(block, oracle_blend, bcases[n], "blend %s after default bt256" % n)
    _step(block, oracle, R.build("dcm2", oracle), "default dcm2")
    for n in ("dcm2", "per_context_mix", "no_predmode"):
        _step(block, oracle_blend, bcases[n], "blend %s after default dcm2" % n)


# ---------------------------------------------------------------------------------------------------------------------
# the recording decoder
# ---------------------------------------------------------------------------------------------------------------------
def _blob(oracle_blend, c):
    rc, raw, cl = oracle_blend.decode_cmds(c.stream, out_cap=c.cap)
    assert rc == 0
    return raw, cl.serialize()


def test_recording_decoder(engine, oracle_blend, bcases, bedges):
    """decode_cmds of every good regime and every blend edge records the blend oracle's command list; the failing regimes
    report the oracle's status and record nothing"""
    cases = [bcases[n] for n in R.GOOD] + [bedges[n] for n in R.EDGE_NAMES]
    names = R.GOOD + R.EDGE_NAMES
    res = engine.decode_cmds([c.stream for c in cases], [c.cap for c in cases], BLEND)
    for name, c, (st, raw, blob) in zip(names, cases, res):
        ref_raw, ref_blob = _blob(oracle_blend, c)
        assert st == 0 and raw == ref_raw == c.raw, name
        assert blob == ref_blob, "%s: blob len %d vs %d, first diff at %d" % (name, len(blob), len(ref_blob), _first_diff(blob, ref_blob))
    # failing regimes between good ones, through the host call itself (blob_len is visible there)
    mix = [bcases["lsb6"]] + [bcases[n] for n in R.FAILING] + [bcases["switches"]]
    blob, in_off, in_len = divans_b200._pack([c.stream for c in mix])
    out_cap = np.array([c.cap for c in mix], np.uint64)
    blob_cap = divans_b200.first_blob_cap(out_cap)
    for i, c in enumerate(mix):
        if c.status == 0:       # exactly the blob's size (switches has three PredictionMode records: more than the first guess)
            blob_cap[i] = len(_blob(oracle_blend, c)[1])
    out_off, out_total = divans_b200._regions(out_cap)
    blob_off, blobs_total = divans_b200._regions(blob_cap)
    out, blobs = np.zeros(out_total, np.uint8), np.zeros(blobs_total, np.uint8)
    out_len, blob_len, status = engine.decode_cmds_batch_host(blob, in_off, in_len, out, out_off, out_cap, blobs, blob_off, blob_cap,
                                                              BLEND | divans_b200.FLAG_SKIP_CRC)
    for i, c in enumerate(mix):
        rc, _ = _ref(oracle_blend, c, True)
        assert status[i] == rc == c.status, (i, status[i], rc)
        if rc != 0:
            assert blob_len[i] == 0, i
        else:
            got = blobs[int(blob_off[i]):int(blob_off[i] + blob_len[i])].tobytes()
            assert got == _blob(oracle_blend, c)[1], i


def test_recording_decoder_device_entry_point(engine, oracle_blend, bcases, bedges):
    import torch
    cases = [bcases[n] for n in ("switches", "bt256", "per_context_mix", "dcm2", "empty", "no_predmode", "chunk_restart")]
    cases += [bedges[n] for n in ("lit69632", "cmd4096", "nib65537", "both_over")]
    streams, caps = [c.stream for c in cases], [c.cap for c in cases]
    want = [_blob(oracle_blend, c) for c in cases]
    n = len(cases)
    in_blob, in_off, in_len = divans_b200._pack(streams)
    out_off, out_total = divans_b200._regions(caps)
    bcap = [len(b) + 7 for _, b in want]
    blob_off, blob_total = divans_b200._regions(bcap)
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev)
    d_in = torch.from_numpy(in_blob).to(dev)
    d_out = torch.zeros(out_total, dtype=torch.uint8, device=dev)
    d_blobs = torch.zeros(blob_total, dtype=torch.uint8, device=dev)
    d_meta = [u64(in_off), u64(in_len), u64(out_off), u64(caps), u64(blob_off), u64(bcap)]
    d_out_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_blob_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_status = torch.full((n,), 3, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    engine.decode_cmds_batch_device(d_in.data_ptr(), d_meta[0].data_ptr(), d_meta[1].data_ptr(), d_out.data_ptr(), d_meta[2].data_ptr(),
                                    d_meta[3].data_ptr(), d_out_len.data_ptr(), d_blobs.data_ptr(), d_meta[4].data_ptr(),
                                    d_meta[5].data_ptr(), d_blob_len.data_ptr(), d_status.data_ptr(), n, int(in_blob.size), BLEND)
    engine.synchronize()
    out, blobs = d_out.cpu().numpy(), d_blobs.cpu().numpy()
    st, ol, bl = d_status.cpu().numpy(), d_out_len.cpu().numpy(), d_blob_len.cpu().numpy()
    for i, (raw, ref) in enumerate(want):
        assert st[i] == 0 and ol[i] == len(raw) and bl[i] == len(ref), i
        assert out[int(out_off[i]):int(out_off[i]) + len(raw)].tobytes() == raw, i
        assert blobs[int(blob_off[i]):int(blob_off[i]) + len(ref)].tobytes() == ref, i


# ---------------------------------------------------------------------------------------------------------------------
# the encoder
# ---------------------------------------------------------------------------------------------------------------------
def _opts(**kw):
    return divans_b200.encode_options(cdf_model=divans_b200.CDF_BLEND, **kw)


def _encode_host(eng, items, opts, cmds):
    """one encode_batch_host launch (cmds: encode_cmds_batch_host) over `items`: [(status, bytes or None)]"""
    blob, in_off, in_len = divans_b200._pack(items)
    cap = divans_b200._encoded_cap(in_len)
    out_off, total = divans_b200._regions(cap)
    out = np.zeros(total, np.uint8)
    ln, st = eng.encode_batch_host(blob, in_off, in_len, out, out_off, cap, opts, cmds)
    return [(int(s), out[int(o):int(o) + int(n)].tobytes() if s == 0 else None) for s, o, n in zip(st, out_off, ln)]


def _encode_device(eng, items, opts, cmds, max_raw_len=0):
    """the same through encode_batch_device / encode_cmds_batch_device, inputs and outputs in HBM"""
    import torch
    blob, in_off, in_len = divans_b200._pack(items)
    cap = divans_b200._encoded_cap(in_len)
    out_off, total = divans_b200._regions(cap)
    n = len(items)
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev)
    d_in, d_out = torch.from_numpy(blob).to(dev), torch.zeros(total, dtype=torch.uint8, device=dev)
    d_meta = [u64(in_off), u64(in_len), u64(out_off), u64(cap)]
    d_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_st = torch.full((n,), -1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    if cmds:
        eng.encode_cmds_batch_device(n, d_in.data_ptr(), d_meta[0].data_ptr(), d_meta[1].data_ptr(), int(in_len.max()), max_raw_len,
                                     d_out.data_ptr(), d_meta[2].data_ptr(), d_meta[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), opts)
    else:
        eng.encode_batch_device(n, d_in.data_ptr(), d_meta[0].data_ptr(), d_meta[1].data_ptr(), int(in_len.max()), d_out.data_ptr(),
                                d_meta[2].data_ptr(), d_meta[3].data_ptr(), d_len.data_ptr(), d_st.data_ptr(), opts)
    eng.synchronize()
    o, st, ln = d_out.cpu().numpy(), d_st.cpu().numpy(), d_len.cpu().numpy()
    return [(int(s), o[int(a):int(a) + int(l)].tobytes() if s == 0 else None) for s, a, l in zip(st, out_off, ln)]


def _compare(got, want, names, what):
    for name, (st, out), (ws, wb) in zip(names, got, want):
        assert st == ws, "%s: %s: status %d, oracle %d" % (what, name, st, ws)
        if ws == 0:
            assert out == wb, "%s: %s: len %d vs %d, first diff at %d" % (what, name, len(out), len(wb), _first_diff(out, wb))


def test_encoder_regimes_and_edges(engine, oracle_blend):
    """every good regime's command list and every blend edge, through the host and device entry points, byte for byte the
    blend oracle's stream: command lists for the regimes and the LZ77 edges, raw mode for the random-byte edges"""
    jobs = {}       # (options, raw mode) -> [(name, input, raw length, oracle stream)]
    for name in R.GOOD:
        cl = R.command_list(name, oracle_blend)
        kw = R.encode_options(name)
        jobs.setdefault((tuple(sorted(kw.items())), False), []).append(
            (name, cl.serialize(), len(R.build(name, oracle_blend).raw), cl.encode(oracle_blend.options(**kw))))
    for name in R.EDGE_NAMES:
        cl, raw, stream = R.edge(name, oracle_blend)
        rawmode = R.BLEND_EDGES[name][0] == "rnd"
        kw = R.edge_options(name, oracle_blend)
        jobs.setdefault((tuple(sorted(kw.items())), rawmode), []).append((name, raw if rawmode else cl.serialize(), len(raw), stream))
    assert len(jobs) >= 4
    for (key, rawmode), items in jobs.items():
        names = [x[0] for x in items]
        want = [(0, x[3]) for x in items]
        o = _opts(**dict(key))
        _compare(_encode_host(engine, [x[1] for x in items], o, not rawmode), want, names, "host %s" % (key,))
        _compare(_encode_device(engine, [x[1] for x in items], o, not rawmode, max(x[2] for x in items) + 64), want, names,
                 "device %s" % (key,))


def test_encoder_slot_succession(oracle_blend):
    """Engine(0, 2, 16): the encoder runs one 64-thread block, 4 slots, and `[A] * 4 + [X] * 4 + ...` gives every slot A, then
    X.  The good regimes, one launch per option set on the same engine, alternate with a list whose literal ends past the pool
    and a list that overflows the command log; good streams equal the blend oracle's bytes, the others fail with status 3.
    (The blend model has no adaptation speeds: the wide-speed list the default model refuses is a good list here.)"""
    groups = {}
    for name in R.GOOD:
        groups.setdefault(tuple(sorted(R.encode_options(name).items())), []).append(name)
    pm_only = oracle_blend.Commands.from_ir("window 16 0 0 0\n" + R.pm_line("lsb6", lmap=[1 + (i * 37 + i // 64 * 11) % 255 for i in range(16384)],
                                                                            mix=[(i * 7) % 9 for i in range(8192)]) + "\n")
    per_pm = oracle_blend.decode(pm_only.encode(oracle_blend.options(window_size=16)), stats=True)[2]["cmd_nibbles"]
    eng = divans_b200.Engine(0, 2, 16)
    try:
        for key, names in groups.items():
            kw = dict(key)
            good = [R.command_list(n, oracle_blend).serialize() for n in names]
            want_good = [R.command_list(n, oracle_blend).encode(oracle_blend.options(**kw)) for n in names]
            cap = max(32 * int(np.frombuffer(b[:32], np.uint32)[2]) + 62000 * int(np.frombuffer(b[:32], np.uint32)[3]) + 64 for b in good)
            bad = [dvcl.literal_outside_pool(good[[i for i, n in enumerate(names) if n != "empty"][0]]),
                   dvcl.pm_flood(pm_only.serialize(), cap // per_pm + 2)]
            seq, want = [], []
            for i, (b, w) in enumerate(zip(good, want_good)):
                seq += [b] * 4 + [bad[i % 2]] * 4
                want += [(0, w)] * 4 + [(3, None)] * 4
            if len(names) < 2:
                seq += [bad[1]] * 4 + good[:1] * 4
                want += [(3, None)] * 4 + [(0, want_good[0])] * 4
            got = _encode_host(eng, seq, _opts(**kw), True)
            _compare(got, want, ["%d" % i for i in range(len(seq))], "group %s" % names)
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# corpus: the golden command lists under the blend model, and the 2018 model revision
# ---------------------------------------------------------------------------------------------------------------------
def _blend_encode_of(oracle_blend, cl, kw):
    """the blend oracle's dvo_encode_cmds of a command list the default oracle holds (both builds share the list's layout)"""
    cap = cl.c.n_lits * 2 + cl.c.n_cmds * 16 + (1 << 20)
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    lst = oracle_blend.CmdList.from_address(ctypes.addressof(cl.c))
    o = oracle_blend.options(**kw)
    assert oracle_blend.lib().dvo_encode_cmds(ctypes.byref(lst), ctypes.byref(o), ctypes.c_void_p(out.ctypes.data), cap, ctypes.byref(n)) == 0
    return out[:n.value].tobytes()


def test_golden_command_lists_under_blend(engine, oracle, oracle_blend, golden):
    """each golden stream's command list, re-encoded by the blend oracle under the golden options: the GPU decodes it, records
    the blend oracle's list, and encodes that list back to the same bytes"""
    streams, raws, opts = [], [], []
    for e in golden:
        s = open(e["path"], "rb").read()
        rc, raw, cl = oracle.decode_cmds(s, out_cap=e["raw_len"] + 64)
        assert rc == 0
        kw = dict(dict(window_size=s[5]), **e["options"])
        bs = _blend_encode_of(oracle_blend, cl, kw)
        rc, back = oracle_blend.decode(bs, out_cap=len(raw) + 64)
        assert rc == 0 and back == raw, e["name"]
        streams.append(bs); raws.append(raw); opts.append(kw)
    caps = [len(r) + 64 for r in raws]
    for (st, out), r, e in zip(engine.decode(streams, caps, BLEND), raws, golden):
        assert st == 0 and out == r, e["name"]
    rec = engine.decode_cmds(streams, caps, BLEND)
    for (st, raw, blob), s, r, kw, e in zip(rec, streams, raws, opts, golden):
        rc, ref_raw, cl = oracle_blend.decode_cmds(s, out_cap=len(r) + 64)
        assert st == 0 and raw == r and blob == cl.serialize(), e["name"]
        (gst, got), = _encode_host(engine, [blob], _opts(**kw), True)
        assert gst == 0 and got == s, "%s: first diff at %d" % (e["name"], _first_diff(got, s))


def test_wasm_2018_revision_under_blend(engine, oracle_blend):
    """the 2018 model revision (FLAG_MODEL_WASM_2018) together with the blend model: decode, record and encode"""
    wasm = oracle_blend.MODEL_WASM_2018
    flags = BLEND | divans_b200.FLAG_MODEL_WASM_2018
    names = ["lsb6", "dcm2", "per_context_mix", "switches", "short_literals"]
    streams, raws, kws = [], [], []
    for name in names:
        kw = dict(R.encode_options(name), model_rev=wasm)
        s = R.command_list(name, oracle_blend).encode(oracle_blend.options(**kw))
        rc, raw, _cl = oracle_blend.decode_cmds(s, out_cap=len(R.build(name, oracle_blend).raw) + 64, model_rev=wasm)
        assert rc == 0 and raw == R.build(name, oracle_blend).raw, name
        streams.append(s); raws.append(raw); kws.append(kw)
    assert all(s != R.build(n, oracle_blend).stream for s, n in zip(streams, names))    # the revision changes the coding
    caps = [len(r) + 64 for r in raws]
    for name, (st, out), r in zip(names, engine.decode(streams, caps, flags), raws):
        assert st == 0 and out == r, name
    for name, (st, raw, blob), s, r, kw in zip(names, engine.decode_cmds(streams, caps, flags), streams, raws, kws):
        cl = oracle_blend.decode_cmds(s, out_cap=len(r) + 64, model_rev=wasm)[2]
        assert st == 0 and raw == r and blob == cl.serialize(), name
        (gst, got), = _encode_host(engine, [blob], _opts(**dict(kw, model_rev=divans_b200.MODEL_WASM_2018)), True)
        assert gst == 0 and got == s, name
