"""GPU encoder parity (-m gpu): the CUDA encoder (model pass + reverse rANS pass + mux/CRC pass), called through the
C ABI, must produce byte-identical .divans streams to the CPU oracle's encoder on the same commands and options."""
import io

import numpy as np
import pytest

import dvcl
from irfuzz import random_ir

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def text():
    from divans_b200 import synth
    return synth.text_corpus(1 << 20)


def _first_diff(a, b):
    return next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), min(len(a), len(b)))


def _check(got, ref, what):
    assert len(got) == len(ref) and got == ref, "%s: len %d vs %d, first diff at %d" % (what, len(got), len(ref), _first_diff(got, ref))


OPTION_SETS = [
    dict(),
    dict(window_size=10),
    dict(window_size=16, dynamic_context_mixing=1),
    dict(dynamic_context_mixing=2),
    dict(dynamic_context_mixing=3, prior_depth=2),
    dict(force_stride=0),
    dict(force_stride=3, use_context_map=1),
    dict(use_context_map=0, dynamic_context_mixing=2),
    dict(literal_adaptation=[(2, 1024), (16, 8192), (128, 16384), (1, 128)]),
    dict(dynamic_context_mixing=2, literal_adaptation=[(32, 4096), (4, 1024), (64, 16384), (512, 16384)]),
]


@pytest.mark.parametrize("kw", OPTION_SETS, ids=lambda d: ",".join("%s=%s" % (k, v if not isinstance(v, list) else "set") for k, v in d.items()) or "default")
def test_raw_encode_matches_oracle(engine, oracle, text, kw):
    import divans_b200
    rng = np.random.default_rng(5)
    raws = [text[:n] for n in [0, 1, 2, 15, 16, 17, 1023, 1024, 1025, 4097, 40000]]
    raws.append(rng.integers(0, 256, 3000).astype(np.uint8).tobytes())
    raws.append(bytes(7000))
    got = engine.encode(raws, divans_b200.encode_options(**kw))
    for i, r in enumerate(raws):
        _check(got[i], oracle.encode_raw(r, oracle.options(**kw)), "raw stream %d (len %d) opts %s" % (i, len(r), kw))


def test_raw_encode_chunk_restart_and_big_records(engine, oracle, text):
    # > 65536 literal nibbles (rANS chunk restart, ans.rs:57,138) and coder payloads > 65536 B (fixed-size mux records)
    rng = np.random.default_rng(9)
    raws = [text[:65535], text[:65536], text[:65537], text[:200000], rng.integers(0, 256, 150000).astype(np.uint8).tobytes(),
            text[:32768] + rng.integers(0, 256, 140000).astype(np.uint8).tobytes()]
    got = engine.encode(raws)
    for i, r in enumerate(raws):
        _check(got[i], oracle.encode_raw(r), "stream %d" % i)


@pytest.mark.parametrize("pm", [0, 1, 2, 3])
def test_raw_encode_prediction_modes(engine, oracle, text, pm):
    import divans_b200
    for mv in range(9):
        r = text[5000 * mv: 5000 * mv + 4000]
        out, off, ln = oracle.encode_batch(np.frombuffer(r, np.uint8), [0], [len(r)], oracle.options(), 1, False, pm, mv)
        got = engine.encode([r], divans_b200.encode_options(literal_pred_mode=pm, literal_mixing_value=mv))
        _check(got[0], out[: int(ln[0])].tobytes(), "pm %d mixing %d" % (pm, mv))


def test_command_lists_lz77(engine, oracle, text):
    import divans_b200
    for win, pm, mv, kw in [(16, 2, 4, {}), (10, 0, 4, dict(window_size=10)), (16, 3, 1, dict(dynamic_context_mixing=2)),
                            (16, 1, 6, dict(force_stride=2))]:
        cls = [oracle.Commands.lz77(text[o:o + n], win, pm, mv) for o, n in [(0, 100), (500, 5000), (9000, 70000), (100000, 30000)]]
        kw = dict(kw); kw.setdefault("window_size", win)
        got = engine.encode([c.serialize() for c in cls], divans_b200.encode_options(**kw), cmds=True)
        for i, c in enumerate(cls):
            _check(got[i], c.encode(oracle.options(**kw)), "lz77 list %d win %d" % (i, win))


def test_command_lists_random_ir(engine, oracle, text):
    import divans_b200
    cls, refs = [], []
    for seed in range(24):
        c = oracle.Commands.from_ir(random_ir(oracle, seed, n_cmds=150, window=16, text=text))
        cls.append(c)
    for kw in [dict(window_size=16), dict(window_size=16, dynamic_context_mixing=2, prior_depth=1), dict(window_size=16, force_stride=5)]:
        got = engine.encode([c.serialize() for c in cls], divans_b200.encode_options(**kw), cmds=True)
        for i, c in enumerate(cls):
            _check(got[i], c.encode(oracle.options(**kw)), "random IR seed %d opts %s" % (i, kw))


def test_reference_held_stream_is_reproduced_by_the_gpu_encoder(engine, oracle):
    """Commands of the reference-held stream (wasm/wasm.html:98-107) -> GPU encoder under model revision WASM_2018 ->
    the reference encoder's own 113 bytes; under today's revision -> the oracle's bytes for today's model."""
    import os
    import divans_b200
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    vec = open(os.path.join(d, "ref_wasm_example.divans"), "rb").read()
    rc, plain, cmds = oracle.decode_cmds(vec, model_rev=oracle.MODEL_WASM_2018)
    assert rc == 0
    blob = cmds.serialize()
    kw = dict(window_size=22, use_context_map=0, dynamic_context_mixing=0)
    got = engine.encode([blob, blob], divans_b200.encode_options(model_rev=divans_b200.MODEL_WASM_2018, **kw), cmds=True)
    assert got[0] == vec and got[1] == vec
    now = engine.encode([blob], divans_b200.encode_options(**kw), cmds=True)[0]
    _check(now, cmds.encode(oracle.options(**kw)), "2018 commands under today's model")


def test_bad_command_list_is_rejected_not_crashing(engine):
    blob = np.zeros(64, np.uint8)
    out = np.zeros(1 << 16, np.uint8)
    ln, st = engine.encode_batch_host(blob, [0], [64], out, [0], [1 << 16], None, cmds=True)
    assert st[0] != 0


def test_output_capacity_too_small(engine, oracle, text):
    r = text[:5000]
    ref = oracle.encode_raw(r)
    out = np.zeros(1 << 16, np.uint8)
    blob = np.frombuffer(r, np.uint8)
    ln, st = engine.encode_batch_host(blob, [0], [len(r)], out, [0], [len(ref) - 1])
    assert st[0] == 2 and int(ln[0]) == len(ref)      # NEEDS_MORE_OUTPUT + the size that would have been needed
    ln, st = engine.encode_batch_host(blob, [0], [len(r)], out, [0], [len(ref)])
    assert st[0] == 0 and out[: len(ref)].tobytes() == ref


def test_reference_ffi_compressor_writer(engine, oracle, text):
    import divans_b200
    r = text[:100000]
    sink = io.BytesIO()
    w = divans_b200.DivansCompressorWriter(sink)
    for o in range(0, len(r), 7777):
        w.write(r[o:o + 7777])
    w.close()
    stream = sink.getvalue()
    rc, back = oracle.decode(stream, out_cap=len(r) + 64)
    assert rc == 0 and back == r
    (st, out), = engine.decode([stream], [len(r) + 64])
    assert st == 0 and out == r


def test_full_size_encode_decode_round_trip(engine, oracle):
    # BASELINE config 4 shape: 4096 x 64 KiB through the GPU encoder, back through the GPU decoder
    import divans_b200
    from divans_b200 import synth
    n, size = 4096, 65536
    corpus = synth.text_corpus(n * size // 4)
    raws = [corpus[(i * size) % (len(corpus) - size): (i * size) % (len(corpus) - size) + size] for i in range(n)]
    streams = engine.encode(raws, divans_b200.encode_options(window_size=16))
    for i in [0, 1, n // 2, n - 1]:
        _check(streams[i], oracle.encode_raw(raws[i], oracle.options(window_size=16)), "stream %d" % i)
    res = engine.decode(streams, [size + 64] * n)
    assert all(st == 0 for st, _ in res)
    assert all(out == raws[i] for i, (_, out) in enumerate(res))


def test_ir_text_end_to_end(engine, oracle, text):
    # reference IR text -> product parser (C ABI) -> GPU encoder == oracle encoder; GPU decode == oracle replay of the IR
    import divans_b200
    irs = [random_ir(oracle, 100 + seed, n_cmds=120, window=16, text=text) for seed in range(8)]
    blobs = [divans_b200.ir_to_cmds(ir)[0] for ir in irs]
    got = engine.encode(blobs, divans_b200.encode_options(window_size=16, dynamic_context_mixing=1), cmds=True)
    raws = []
    for i, ir in enumerate(irs):
        c = oracle.Commands.from_ir(ir)
        _check(got[i], c.encode(oracle.options(window_size=16, dynamic_context_mixing=1)), "IR %d" % i)
        rc, raw = c.recode(16)
        assert rc == 0
        raws.append(raw)
    res = engine.decode(got, [len(r) + 64 for r in raws])
    assert all(st == 0 and out == r for (st, out), r in zip(res, raws))


def test_corrupted_command_lists_never_hang(engine, oracle, text):
    # hostile DVCL blobs (random words overwritten in the header / command records): a status per stream, no fault
    rng = np.random.default_rng(5)
    blobs = [np.frombuffer(oracle.Commands.from_ir(random_ir(oracle, 300 + s, n_cmds=100, window=16, text=text)).serialize(), np.uint8) for s in range(10)]
    for _ in range(6):
        bad = []
        for b in blobs:
            w = b.copy().view(np.uint32) if b.size % 4 == 0 else np.concatenate([b, np.zeros(4 - b.size % 4, np.uint8)]).view(np.uint32)
            w = w.copy()
            n_cmds = int(w[2])
            for _m in range(int(rng.integers(1, 5))):
                i = int(rng.integers(2, 8 + 5 * n_cmds))
                w[i] = rng.integers(0, 1 << 32, dtype=np.uint64).astype(np.uint32) if rng.random() < 0.5 else np.uint32(rng.integers(0, 70000))
            bad.append(w.view(np.uint8))
        in_len = np.array([x.size for x in bad], np.uint64)
        in_off = np.zeros(len(bad), np.uint64)
        in_off[1:] = np.cumsum((in_len + np.uint64(15)) & ~np.uint64(15))[:-1]
        blob = np.zeros(int(in_off[-1] + in_len[-1]) + 16, np.uint8)
        for x, o in zip(bad, in_off):
            blob[int(o):int(o) + x.size] = x
        cap = np.full(len(bad), 1 << 20, np.uint64)
        out_off = np.arange(len(bad), dtype=np.uint64) * np.uint64(1 << 20)
        out = np.zeros(len(bad) << 20, np.uint8)
        try:
            ln, st = engine.encode_batch_host(blob, in_off, in_len, out, out_off, cap, None, cmds=True)
            assert all(int(x) in (0, 1, 2, 3) for x in st)
        except Exception as e:      # the host marshaller may refuse a batch whose header asks for absurd sizes
            assert "too large" in str(e) or "encode_batch_host" in str(e)
    good = engine.encode([blobs[0].tobytes()], None, cmds=True)
    assert len(good[0]) > 24


# ---------------------------------------------------------------------------------------------------------------------
# wide speeds: the encoder refuses exactly the streams the oracle refuses
# ---------------------------------------------------------------------------------------------------------------------
def _encode_host(eng, items, opts, cmds):
    """one encode_batch_host launch over `items` (raw byte strings or DVCL blobs): [(status, bytes)]"""
    bufs = [np.frombuffer(x, np.uint8) if len(x) else np.zeros(0, np.uint8) for x in items]
    in_len = np.array([b.size for b in bufs], np.uint64)
    pad = (in_len + np.uint64(15)) & ~np.uint64(15)
    in_off = np.concatenate([[0], np.cumsum(pad)[:-1]]).astype(np.uint64)
    blob = np.zeros(int(pad.sum()) + 16, np.uint8)
    for b, o in zip(bufs, in_off):
        blob[int(o):int(o) + b.size] = b
    cap = (in_len * np.uint64(2) + np.uint64(70000 + 255)) & ~np.uint64(255)
    out_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
    out = np.zeros(int(cap.sum()), np.uint8)
    ln, st = eng.encode_batch_host(blob, in_off, in_len, out, out_off, cap, opts, cmds)
    return [(int(s), out[int(o):int(o) + int(n)].tobytes() if s == 0 else None) for s, o, n in zip(st, out_off, ln)]


def _oracle_cmds(cl, oracle, kw):
    """(status, stream) of the oracle encoder: 3 where it refuses a symbol of frequency <= 0"""
    try:
        return 0, cl.encode(oracle.options(**kw))
    except ValueError:
        return 3, None


def _oracle_raw(oracle, raws, kw, pred_mode, mixing_value):
    """(status, stream) per raw input of the oracle's raw-mode encoder with a literal prediction mode and mixing value"""
    return oracle.encode_raw_list(raws, oracle.options(**kw), pred_mode, mixing_value)


def _compare(got, ref, what):
    for i, ((st, out), (rs, rb)) in enumerate(zip(got, ref)):
        assert st == rs, "%s: stream %d: status %d, oracle %d" % (what, i, st, rs)
        if rs == 0:
            _check(out, rb, "%s: stream %d" % (what, i))


def test_wide_speed_command_lists_refused_like_the_oracle(engine, oracle, text):
    """The wide-speed IR lists of the decoder's f8 fuzz test (speeds over the whole f8 range: i16 counters wrap), 96 seeds.
    Each seed's option set encodes, in one batch, every list of its window, so streams the oracle refuses (a coded
    frequency <= 0) share warps with streams it accepts.  Statuses equal the oracle's; accepted streams are byte-equal."""
    import divans_b200
    import irfuzz
    wins = [10, 14, 16, 22]
    cls = [oracle.Commands.from_ir(irfuzz.random_ir(oracle, 7000 + s, n_cmds=60, window=wins[s % 4], text=text, wide_speeds=True))
           for s in range(96)]
    refused = accepted = mixed = 0
    for s in range(96):
        adapt = irfuzz.random_f8_speeds(oracle, s) if s % 2 else None
        kw = dict(window_size=wins[s % 4], dynamic_context_mixing=s % 3)
        if adapt is not None:
            kw["literal_adaptation"] = adapt
        batch = [cls[t] for t in range(s % 4, 96, 4)]
        ref = [_oracle_cmds(c, oracle, kw) for c in batch]
        got = _encode_host(engine, [c.serialize() for c in batch], divans_b200.encode_options(**kw), True)
        _compare(got, ref, "option set %d" % s)
        n3 = sum(r[0] == 3 for r in ref)
        refused += n3; accepted += len(ref) - n3; mixed += 0 < n3 < len(ref)
    assert refused >= 50 and accepted >= 500 and mixed >= 10, (refused, accepted, mixed)


def test_wide_speed_raw_encodes_refused_like_the_oracle(engine, oracle, text):
    """Raw mode with literal_adaptation over the whole f8 range, every literal prediction mode, dynamic context mixing
    0..2: eight texts per option set in one batch."""
    import divans_b200
    import irfuzz
    refused = accepted = 0
    for k in range(48):
        pm, dcm = k % 4, (k // 4) % 3
        adapt = irfuzz.random_f8_speeds(oracle, 100 + k)
        raws = [text[(8 * k + j) * 2500:(8 * k + j) * 2500 + 1000 + 500 * j] for j in range(8)]
        kw = dict(dynamic_context_mixing=dcm, literal_adaptation=adapt)
        ref = _oracle_raw(oracle, raws, kw, pm, 4)
        got = _encode_host(engine, raws, divans_b200.encode_options(literal_pred_mode=pm, literal_mixing_value=4, **kw), False)
        _compare(got, ref, "pm %d dcm %d speeds %s" % (pm, dcm, adapt))
        n3 = sum(r[0] == 3 for r in ref)
        refused += n3; accepted += len(ref) - n3
    assert refused >= 20 and accepted >= 200, (refused, accepted)


# ---------------------------------------------------------------------------------------------------------------------
# slot succession: one block of 4 encoder slots, good regimes between refused and hostile lists
# ---------------------------------------------------------------------------------------------------------------------
def test_encoder_slot_succession(oracle):
    """Engine(0, 2, 16): the encoder runs one 64-thread block, 4 slots.  `[A] * 4 + [X] * 4 + [B] * 4 ...` gives every slot
    A, then X, then B.  The GOOD regimes, grouped by option set (one launch per group, consecutive launches on the same
    engine), alternate with a wide-speed list the oracle refuses, a list with a literal outside the pool and a list that
    overflows the command log.  Good streams equal the oracle's bytes; the others fail with status 3."""
    import divans_b200
    import irfuzz
    import regimes as R
    groups = {}
    for name in R.GOOD:
        groups.setdefault(tuple(sorted(R.encode_options(name).items())), []).append(name)
    assert len(groups) >= 3
    pm_only = oracle.Commands.from_ir("window 16 0 0 0\n" + R.pm_line("lsb6", lmap=[1 + (i * 37 + i // 64 * 11) % 255 for i in range(16384)],
                                                                      mix=[(i * 7) % 9 for i in range(8192)]) + "\n")
    per_pm = oracle.decode(pm_only.encode(oracle.options(window_size=16)), stats=True)[2]["cmd_nibbles"]
    eng = divans_b200.Engine(0, 2, 16)
    try:
        for key, names in groups.items():
            kw = dict(key)
            refused = None
            for seed in range(400):
                c = oracle.Commands.from_ir(irfuzz.random_ir(oracle, 9000 + seed, n_cmds=60, window=kw["window_size"], text=R.text(), wide_speeds=True))
                if _oracle_cmds(c, oracle, kw)[0] == 3:
                    refused = c.serialize()
                    break
            assert refused is not None, kw
            good = [R.command_list(n, oracle).serialize() for n in names]
            cap = max(32 * int(np.frombuffer(b[:32], np.uint32)[2]) + 62000 * int(np.frombuffer(b[:32], np.uint32)[3]) + 64 for b in good + [refused])
            flood = dvcl.pm_flood(pm_only.serialize(), cap // per_pm + 2)
            bad = [refused, dvcl.literal_outside_pool(good[[i for i, n in enumerate(names) if n != "empty"][0]]), flood]
            seq, want = [], []
            for i, (n, b) in enumerate(zip(names, good)):
                seq += [b] * 4; want += [(0, R.build(n, oracle).stream)] * 4
                seq += [bad[i % 3]] * 4; want += [(3, None)] * 4
            if len(names) < 3:      # every kind of failure in every group
                for j in range(len(names), 3):
                    seq += [bad[j]] * 4 + good[:1] * 4; want += [(3, None)] * 4 + [(0, R.build(names[0], oracle).stream)] * 4
            got = _encode_host(eng, seq, divans_b200.encode_options(**kw), True)
            _compare(got, want, "group %s" % names)
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# framing and chunk edges
# ---------------------------------------------------------------------------------------------------------------------
def test_framing_edges_encode_like_the_oracle_and_decode(engine, engine16, oracle):
    """Literal payloads of exactly 4096, 16384, 65536, 65536 + 4096, 65536 + 16384 and 131072 bytes, command payloads of
    4096 and 16384 bytes, 65535 / 65536 / 65537 command nibbles, both payloads over 131073 bytes: the GPU encoder equals
    the oracle (raw mode for the random-byte edges, command lists for the LZ77 ones), and every decode layout returns the
    input."""
    import divans_b200
    import regimes as R
    streams, raws = [], []
    for name in R.EDGE_NAMES:
        cl, raw, ref = R.edge(name, oracle)
        kw = R.edge_options(name)
        if R.EDGES[name][0] == "rnd":
            got = engine.encode([raw], divans_b200.encode_options(**kw))[0]
        else:
            got = engine.encode([cl.serialize()], divans_b200.encode_options(**kw), cmds=True)[0]
        _check(got, ref, name)
        streams.append(ref); raws.append(raw)
    for eng in (engine, engine16):
        res = eng.decode(streams, [len(r) + 64 for r in raws])
        for name, (st, out), r in zip(R.EDGE_NAMES, res, raws):
            assert st == 0 and out == r, (name, eng.last_lanes())


def test_remuxed_streams_decode_on_every_layout(engine, engine16, oracle):
    """The same payloads under other record chains (1-byte records, random sizes and coder order, one-byte codes, all
    literal records first, record starts at every offset mod 16), mixed into one batch with the streams as the mux
    wrote them: the oracle and every GPU decode layout return the original bytes."""
    import regimes as R
    streams, raws = [], []
    for name in ("lit16384", "lit131072", "cmd4096", "nib65537", "both_over"):
        _cl, raw, stream = R.edge(name, oracle)
        lens = tuple(len(p) for p in oracle.demux(stream))
        streams.append(stream); raws.append(raw)
        for k, lay in enumerate(R.LAYOUTS):
            if lay == "one_byte" and sum(lens) > 40000:
                continue
            s2 = R.mux_records(oracle, stream, R.layout(lay, lens, seed=k))
            rc, out = oracle.decode(s2, out_cap=len(raw) + 64)
            assert rc == 0 and out == raw, (name, lay)
            streams.append(s2); raws.append(raw)
    for eng in (engine, engine16):
        res = eng.decode(streams, [len(r) + 64 for r in raws])
        for i, ((st, out), r) in enumerate(zip(res, raws)):
            assert st == 0 and out == r, (i, eng.last_lanes())


def test_hostile_record_chains_match_the_oracle(engine, engine16, oracle):
    """Record-chain damage: truncation inside a three-byte record header, truncation inside a one-byte-code record, a code
    k > 3, and a header byte 2..15 (the low bit picks the coder, mux.rs; valid once the CRC is recomputed).  Every status
    equals the oracle's, and so does every output the oracle accepts."""
    import regimes as R
    _cl, raw, stream = R.edge("both_over", oracle)
    lens = tuple(len(p) for p in oracle.demux(stream))
    plan = R.layout("codes", lens, seed=1)
    starts = R.record_starts(plan)
    good = R.mux_records(oracle, stream, plan)
    body = good[:len(good) - 11]
    three = [i for i, (_c, _n, k) in enumerate(plan) if k is None]
    coded = [i for i, (_c, _n, k) in enumerate(plan) if k is not None]
    cases = []
    for i in three[:3]:
        cases += [good[:starts[i] - 2], good[:starts[i] - 1]]                 # inside a three-byte header
    for i in coded[:3]:
        cases.append(good[:starts[i] + plan[i][1] // 2])                      # inside a one-byte-code record
    for i, kk in zip(coded[:3], (4, 9, 15)):
        b = bytearray(body); b[starts[i] - 1] = plan[i][0] | (kk << 4)        # code k > 3
        cases.append(R.close(oracle, bytes(b)))
    for i, v in zip(three[:4], (2, 7, 12, 15)):
        b = bytearray(body); b[starts[i] - 3] = (v & ~1) | plan[i][0]         # header byte 2..15, same coder
        if b[starts[i] - 3] < 2:
            b[starts[i] - 3] += 2
        cases.append(R.close(oracle, bytes(b)))
    streams = [stream, good] + cases + [stream]
    cap = len(raw) + 64
    ref = [oracle.decode(s, out_cap=cap) for s in streams]
    assert [r[0] for r in ref].count(0) >= 6 and {r[0] for r in ref} >= {0, 1, 3}, [r[0] for r in ref]
    for eng in (engine, engine16):
        res = eng.decode(streams, [cap] * len(streams))
        for i, ((st, out), (rc, rb)) in enumerate(zip(res, ref)):
            assert st == rc, "stream %d: status %d, oracle %d (lanes %d)" % (i, st, rc, eng.last_lanes())
            if rc == 0:
                assert out == rb == raw, i
