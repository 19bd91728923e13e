"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle on the same inputs.
Bit-exact bar (integer/byte path)."""
import hashlib
import io
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _decode_and_compare(engine, oracle, streams, raws=None, flags=0, layout=""):
    caps = [(len(r) if r is not None else 1 << 20) + 64 for r in (raws or [None] * len(streams))]
    res = engine.decode(streams, caps, flags)
    for i, (st, out) in enumerate(res):
        rc, ref = oracle.decode(streams[i], out_cap=caps[i])
        assert rc == 0, "oracle failed on stream %d" % i
        assert st == 0, "%s: gpu status %d on stream %d" % (layout, st, i)
        assert out == ref, "%s: stream %d: first diff at %d" % (
            layout, i, next((k for k in range(min(len(out), len(ref))) if out[k] != ref[k]), -1))
        if raws and raws[i] is not None:
            assert out == raws[i]


@pytest.fixture
def decode_engines(engine, engine16, engine32):
    """every decode layout, as (name, engine): the v2 engine with two (16 lanes) and four (8 lanes) streams per warp, and the
    round-1 kernel with one warp per stream (32 lanes)"""
    return [("16 lanes", engine), ("8 lanes", engine16), ("32 lanes", engine32)]


@pytest.fixture(scope="module")
def text():
    from divans_b200 import synth
    return synth.text_corpus(1 << 20)


def test_golden_fixtures(engine, oracle, golden):
    streams = [open(e["path"], "rb").read() for e in golden]
    res = engine.decode(streams, [e["raw_len"] + 64 for e in golden])
    for e, (st, out) in zip(golden, res):
        assert st == 0 and len(out) == e["raw_len"], e["name"]
        assert hashlib.sha256(out).hexdigest() == e["raw_sha256"], e["name"]   # == the reference's raw testdata file


def test_golden_fixtures_other_lane_layouts(engine16, engine32, oracle, golden):
    # 16 lanes per stream (two streams per warp) and 32 (one warp owns one stream: the upper half-warp mirrors the lower)
    streams = [open(e["path"], "rb").read() for e in golden]
    for eng in (engine16, engine32):
        res = eng.decode(streams, [e["raw_len"] + 64 for e in golden])
        for e, (st, out) in zip(golden, res):
            assert st == 0 and hashlib.sha256(out).hexdigest() == e["raw_sha256"], e["name"]


def test_reference_held_stream(engine, engine16, engine32, oracle):
    """The one compressed stream the reference tree holds (wasm/wasm.html:98-107, written by the reference's Rust encoder):
    both lane layouts decode it bit-exactly under its model revision (include/divans_b200.h), CRC checked on the GPU; under
    today's model revision it is rejected exactly like the oracle rejects it."""
    import json
    import divans_b200
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    vec = open(os.path.join(d, "ref_wasm_example.divans"), "rb").read()
    meta = json.load(open(os.path.join(d, "ref_wasm_example.json")))
    want = meta["plain_text"].encode("ascii")
    assert want == b"It snowed, rained, and hailed the same morning.\n" * 7
    for eng in (engine, engine16, engine32):
        # a batch that mixes the 2018 stream with copies of itself exercises both groups of a warp
        res = eng.decode([vec] * 5, [len(want) + 64] * 5, divans_b200.FLAG_MODEL_WASM_2018)
        for st, out in res:
            assert st == 0 and out == want
        st, out = eng.decode([vec], [len(want) + 64])[0]
        rc, ref = oracle.decode(vec, out_cap=len(want) + 64)
        assert rc == oracle.NEEDS_MORE_INPUT and st == rc
    rc, ref, _ = oracle.decode_cmds(vec, model_rev=oracle.MODEL_WASM_2018)
    assert rc == 0 and ref == want


def test_edge_lengths_literal_only(decode_engines, oracle, text):
    raws = [text[:n] for n in [0, 1, 2, 7, 8, 9, 14, 15, 16, 17, 255, 4097, 32767, 32768, 32769, 70001]] + [bytes(range(256)) * 5]
    for win in [10, 22]:
        streams = [oracle.encode_raw(r, oracle.options(window_size=win)) for r in raws]
        for layout, eng in decode_engines:
            _decode_and_compare(eng, oracle, streams, raws, layout=layout)


@pytest.mark.parametrize("pm", [0, 1, 2, 3])
def test_prediction_modes_and_mixing_values(decode_engines, oracle, text, pm):
    raws, streams = [], []
    for mv in range(9):
        r = text[7000 * mv: 7000 * mv + 5000]
        blob = np.frombuffer(r, np.uint8)
        out, off, ln = oracle.encode_batch(blob, [0], [len(r)], oracle.options(), 1, False, pm, mv)
        raws.append(r)
        streams.append(out[: int(ln[0])].tobytes())
    for layout, eng in decode_engines:
        _decode_and_compare(eng, oracle, streams, raws, layout=layout)


@pytest.mark.parametrize("mixing", [1, 2, 3])
def test_dynamic_context_mixing(decode_engines, oracle, text, mixing):
    raws, streams = [], []
    for mv in [0, 1, 2, 3, 4, 6]:
        r = text[3000 * mv: 3000 * mv + 9000]
        blob = np.frombuffer(r, np.uint8)
        out, off, ln = oracle.encode_batch(blob, [0], [len(r)], oracle.options(dynamic_context_mixing=mixing), 1, False, 2, mv)
        raws.append(r)
        streams.append(out[: int(ln[0])].tobytes())
    for layout, eng in decode_engines:
        _decode_and_compare(eng, oracle, streams, raws, layout=layout)


def test_lz77_copies_and_window_wrap(decode_engines, oracle, text):
    rng = np.random.default_rng(9)
    base = rng.integers(97, 105, 3000).astype(np.uint8).tobytes()
    raws = [text[:20000], text[3000:70000], text[:300] * 50, base * 30, b"a" * 5000, b"ab" * 4000]
    for win in [10, 12, 16, 22]:
        streams = [oracle.Commands.lz77(r, window=win).encode(oracle.options(window_size=win, dynamic_context_mixing=2 if win == 12 else 0))
                   for r in raws]
        for layout, eng in decode_engines:
            _decode_and_compare(eng, oracle, streams, raws, layout=layout)


def test_random_ir_fuzz(decode_engines, oracle, text):
    import irfuzz
    streams = []
    for seed in range(40):
        ir = irfuzz.random_ir(oracle, seed, n_cmds=150, window=[10, 14, 16, 22][seed % 4], text=text)
        c = oracle.Commands.from_ir(ir)
        o = oracle.options(window_size=c.window, dynamic_context_mixing=seed % 3, use_context_map=0 if seed % 7 == 3 else 1,
                           force_stride=9 if seed % 5 else 3, prior_depth=seed % 4)
        streams.append(c.encode(o))
    for layout, eng in decode_engines:
        _decode_and_compare(eng, oracle, streams, layout=layout)


def test_random_ir_fuzz_one_warp_per_stream(engine32, oracle, text):
    import irfuzz
    streams = []
    for seed in range(100, 112):
        c = oracle.Commands.from_ir(irfuzz.random_ir(oracle, seed, n_cmds=100, window=16, text=text))
        streams.append(c.encode(oracle.options(window_size=16, dynamic_context_mixing=seed % 3)))
    _decode_and_compare(engine32, oracle, streams)


def test_random_ir_fuzz_full_f8_speed_range(engine, engine16, engine32, oracle, text):
    """Speeds are carried by the stream: the literal fast loops (32-bit adaptive arithmetic) must hand over to the generic
    core (i16 wrap + the reference's literal LUT divide) whenever a counter could wrap.  GPU and oracle must agree on
    status and on every output byte, whether or not the stream decodes back to its input."""
    import irfuzz
    streams = []
    for seed in range(48):
        win = [10, 14, 16, 22][seed % 4]
        c = oracle.Commands.from_ir(irfuzz.random_ir(oracle, 7000 + seed, n_cmds=60, window=win, text=text, wide_speeds=True))
        adapt = irfuzz.random_f8_speeds(oracle, seed) if seed % 2 else None
        try:
            streams.append(c.encode(oracle.options(window_size=win, dynamic_context_mixing=seed % 3, literal_adaptation=adapt)))
        except ValueError:
            pass   # a wrapped counter gave a coded symbol frequency <= 0: the reference encoder divides by it and panics
    caps = [1 << 18] * len(streams)
    for eng in (engine, engine16, engine32):
        res = eng.decode(streams, caps, 1)   # FLAG_SKIP_CRC: payloads are well-formed, only the model misbehaves
        for i, (st, out) in enumerate(res):
            rc, ref = oracle.decode(streams[i], out_cap=caps[i], skip_crc=True)
            assert st == rc, (i, st, rc)
            if rc == 0:
                assert out == ref, i


def test_chunk_restart_every_65536_symbols(decode_engines, oracle):
    # > 65536 literal nibbles and > 65536 command nibbles per coder (ans.rs:236,138)
    rng = np.random.default_rng(4)
    raw = rng.integers(0, 256, 150000).astype(np.uint8).tobytes()       # 300k literal nibbles, incompressible
    s1 = oracle.encode_raw(raw)
    rep = (b"abcdefgh" * 3 + b"xyz") * 40000                                # > 65536 command nibbles from many short copies
    s2 = oracle.Commands.lz77(rep[:600000], window=16).encode(oracle.options(window_size=16))
    for layout, eng in decode_engines:
        _decode_and_compare(eng, oracle, [s1, s2], [raw, rep[:600000]], layout=layout)


def test_status_codes(decode_engines, oracle, text):
    raw = text[:30000]
    enc = oracle.encode_raw(raw)
    cut = [enc[:5], enc[:16], enc[:40], enc[: len(enc) - 9], enc[: len(enc) - 1]]
    bad_magic = b"\x00" + enc[1:]
    bad_window = enc[:5] + b"\x09" + enc[6:]
    flipped = bytearray(enc); flipped[len(enc) // 2] ^= 0x40
    bad_tail = enc[:-1] + b"!"
    wrong_crc = enc[:-8] + b"\x00\x00\x00\x00" + enc[-4:]
    for layout, eng in decode_engines:
        res = eng.decode(cut, [len(raw) + 64] * len(cut))
        assert all(st == 1 for st, _ in res), (layout, [st for st, _ in res])                # NEEDS_MORE_INPUT
        res = eng.decode([bad_magic, bad_window, bytes(flipped), bad_tail, enc], [len(raw) + 64] * 5)
        assert [st for st, _ in res] == [3, 3, 3, 3, 0], layout
        # skip_crc: trailer CRC bytes ignored, "ans~" still required (codec/decoder.rs:204-210)
        res = eng.decode([wrong_crc, bad_tail], [len(raw) + 64] * 2, flags=1)
        assert res[0][0] == 0 and res[0][1] == raw and res[1][0] == 3, layout
        # output capacity too small
        res = eng.decode([enc], [100])
        assert res[0][0] == 2, layout
        # a failing stream must not poison its batch
        res = eng.decode([enc, bytes(flipped), enc], [len(raw) + 64] * 3)
        assert [st for st, _ in res] == [0, 3, 0] and res[0][1] == raw and res[2][1] == raw, layout


def test_reference_ffi_streaming_reader(oracle, golden):
    # BASELINE config 1: alice29 through DivansDecompressorReader / divans_decode with the buffer sizes the reference's
    # integration tests use (src/bin/integration_test.rs:270-272: 65536 / 15 / 1)
    import divans_b200
    e = [g for g in golden if g["name"] == "alice29_literal_only"][0]
    enc = open(e["path"], "rb").read()
    for name in ["alice29_literal_only", "alice29_priors_mix2"]:
        e = [g for g in golden if g["name"] == name][0]
        enc = open(e["path"], "rb").read()
        for bs in [65536, 4096, 15, 1]:
            rd = divans_b200.DivansDecompressorReader(io.BytesIO(enc), bs, False, True)
            out = bytearray()
            chunk = bytearray(bs if bs > 1 else 1)
            while True:
                n = rd.readinto(chunk)
                if not n:
                    break
                out += chunk[:n]
            rd.close()
            assert hashlib.sha256(bytes(out)).hexdigest() == e["raw_sha256"], (name, bs)
    # truncated input -> UnexpectedEof, corrupt -> InvalidData (src/reader.rs:96-98,279-281)
    rd = divans_b200.DivansDecompressorReader(io.BytesIO(enc[:-3]), 4096)
    with pytest.raises(EOFError):
        rd.readinto(bytearray(1 << 20))
    bad = bytearray(enc); bad[100] ^= 1
    rd = divans_b200.DivansDecompressorReader(io.BytesIO(bytes(bad)), 4096)
    with pytest.raises(ValueError):
        rd.readinto(bytearray(1 << 20))


def test_full_size_batch_roundtrip_property(engine, oracle):
    # BASELINE config 2 size: 4096 independent 64 KiB streams; size-independent property = encode -> decode identity,
    # plus a sample of streams checked byte for byte against the oracle's decode
    from divans_b200 import synth
    n = 4096
    blob, off, ln = synth.text_streams(n, 65536)
    enc, eoff, elen = oracle.encode_batch(blob, off, ln, oracle.options(), os.cpu_count() or 4)
    out = np.zeros(blob.size + 256, np.uint8)
    out_len, status = engine.decode_batch_host(enc, eoff, elen, out, off, ln)
    assert (status == 0).all() and (out_len == 65536).all()
    assert (out[: blob.size] == blob).all()
    pick = [0, 1, 17, 2047, 4095]
    for i in pick:
        rc, ref = oracle.decode(enc[int(eoff[i]): int(eoff[i] + elen[i])].tobytes(), out_cap=65600)
        assert rc == 0 and ref == out[int(off[i]): int(off[i]) + 65536].tobytes()


@pytest.mark.parametrize("p", [0.5, 0.9, 0.99])
def test_entropy_sweep_one_mib_streams(engine, oracle, p):
    # BASELINE configs[4] shape at reduced count: 1 MiB Bernoulli(p) streams (16 chunk restarts per coder, ans.rs:57,138)
    import divans_b200
    from divans_b200 import synth
    blob, off, ln = synth.bernoulli_streams(6, 1 << 20, p, seed=int(p * 100))
    raws = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]
    streams = engine.encode(raws, divans_b200.encode_options())
    assert streams[0] == oracle.encode_raw(raws[0]) and streams[5] == oracle.encode_raw(raws[5])
    res = engine.decode(streams, [len(r) + 64 for r in raws])
    assert all(st == 0 and out == r for (st, out), r in zip(res, raws))
    rc, ref = oracle.decode(streams[3], out_cap=(1 << 20) + 64)
    assert rc == 0 and ref == raws[3]


def test_corrupted_streams_without_crc_never_hang(decode_engines, oracle, text):
    # hostile input: records / payload bytes corrupted, CRC check skipped (reference: skip_crc) -> every stream comes back
    # with the oracle's DivansResult code and, where that is 0, the oracle's bytes (codec/decoder.rs:204-210 relaxes only the
    # checksum).  A payload that runs dry inside the literal fast loop (which shifts in the word after the payload) and in the
    # generic coder (which shifts in zero) must both report 1.  out_len of a failed stream is not defined by
    # include/divans_b200.h and is not compared.  Afterwards the uncorrupted bases decode exactly on the same engine: the
    # hostile batches left no state behind in the slots.
    rng = np.random.default_rng(77)
    import irfuzz
    base = [oracle.Commands.from_ir(irfuzz.random_ir(oracle, seed, n_cmds=150, window=16, text=text)).encode(
        oracle.options(window_size=16, dynamic_context_mixing=seed % 3)) for seed in range(12)]
    base += [oracle.encode_raw(text[k * 9000: k * 9000 + 20000], oracle.options(window_size=10 + k)) for k in range(6)]
    rounds = []
    for _ in range(8):
        streams = []
        for s in base:
            b = bytearray(s)
            for _m in range(int(rng.integers(1, 6))):
                pos = int(rng.integers(16, len(b) - 8))
                if rng.random() < 0.5:
                    b[pos] ^= 1 << int(rng.integers(0, 8))
                else:
                    ln = min(int(rng.integers(1, 64)), len(b) - 8 - pos)
                    b[pos:pos + ln] = rng.integers(0, 256, ln).astype(np.uint8).tobytes()
            streams.append(bytes(b))
        rounds.append([(s, oracle.decode(s, out_cap=1 << 20, skip_crc=True)) for s in streams])
    for layout, engine in decode_engines:
        for rnd in rounds:
            res = engine.decode([s for s, _ in rnd], [1 << 20] * len(rnd), flags=1)
            for i, ((st, out), (_, (rc, ref))) in enumerate(zip(res, rnd)):
                assert st == rc, (layout, i, st, rc)
                if rc == 0:
                    assert out == ref, (layout, i)
        _decode_and_compare(engine, oracle, base, layout=layout)
        (st, out), = engine.decode([base[-1]], [1 << 20])
        assert st == 0 and out == text[5 * 9000: 5 * 9000 + 20000], layout


def test_pipelined_host_api_matches_blocking_call(engine, oracle, text):
    # divans_b200_decode_batch_host_async / _wait: several batches back to back, two in flight, different contents per batch
    import torch
    batches = []
    for b in range(5):
        raws = [text[(b * 37 + i) * 1000: (b * 37 + i) * 1000 + 3000 + 997 * i] for i in range(24)]
        streams = [oracle.encode_raw(r, oracle.options(window_size=12 + (i % 6))) for i, r in enumerate(raws)]
        in_len = np.array([len(s) for s in streams], np.uint64)
        in_off = np.zeros(len(streams), np.uint64)
        in_off[1:] = np.cumsum((in_len + np.uint64(15)) & ~np.uint64(15))[:-1]
        blob = torch.zeros(int(in_off[-1] + in_len[-1]) + 16, dtype=torch.uint8).pin_memory()
        for s, o in zip(streams, in_off):
            blob.numpy()[int(o):int(o) + len(s)] = np.frombuffer(s, np.uint8)
        cap = np.array([len(r) for r in raws], np.uint64)
        out_off = np.zeros(len(raws), np.uint64)
        out_off[1:] = np.cumsum((cap + np.uint64(63)) & ~np.uint64(63))[:-1]
        out = torch.zeros(int(out_off[-1] + cap[-1]) + 64, dtype=torch.uint8).pin_memory()
        batches.append((raws, blob, in_off, in_len, out, out_off, cap))
    pend = []
    for raws, blob, in_off, in_len, out, out_off, cap in batches:
        pend.append(engine.decode_batch_host_async(blob.numpy(), in_off, in_len, out.numpy(), out_off, cap))
        if len(pend) == 2:
            pend.pop(0).wait()
    results = [p.wait() for p in pend]
    assert len(results) >= 1
    for raws, blob, in_off, in_len, out, out_off, cap in batches:
        o = out.numpy()
        for r, oo in zip(raws, out_off):
            assert o[int(oo):int(oo) + len(r)].tobytes() == r
    # and the out_len / status arrays of the last batch
    ol, st = results[-1]
    assert (st == 0).all() and (ol == batches[-1][6]).all()


def test_host_api_writes_only_declared_regions_and_accepts_aliased_inputs(engine, oracle, text):
    """(1) nothing outside out[out_off[i] .. +out_cap[i]) is written, by the blocking and by the pipelined call (guard bytes
    between and around the regions survive); (2) input regions may alias: the same stream decoded n times."""
    import torch
    raws = [text[i * 5000: i * 5000 + 2000 + 700 * i] for i in range(12)]
    streams = [oracle.encode_raw(r, oracle.options(window_size=16)) for r in raws]
    in_len = np.array([len(s) for s in streams], np.uint64)
    in_off = np.zeros(len(streams), np.uint64)
    in_off[1:] = np.cumsum(in_len)[:-1]
    blob = np.frombuffer(b"".join(streams), np.uint8).copy()
    cap = np.array([len(r) + (0 if i % 3 else 40) for i, r in enumerate(raws)], np.uint64)    # some regions exactly full
    gap = np.array([0 if i % 4 == 1 else 100 + 13 * i for i in range(len(raws))], np.uint64)  # some regions exactly adjacent
    out_off = np.zeros(len(raws), np.uint64)
    out_off[0] = 77
    for i in range(1, len(raws)):
        out_off[i] = out_off[i - 1] + cap[i - 1] + gap[i]
    total = int(out_off[-1] + cap[-1]) + 333
    covered = np.zeros(total, bool)
    for o, c in zip(out_off, cap):
        covered[int(o):int(o + c)] = True
    for mode in ("blocking", "pipelined"):
        out = torch.full((total,), 0xA5, dtype=torch.uint8).pin_memory().numpy()
        if mode == "blocking":
            ol, st = engine.decode_batch_host(blob, in_off, in_len, out, out_off, cap)
        else:
            ol, st = engine.decode_batch_host_async(blob, in_off, in_len, out, out_off, cap).wait()
        assert (st == 0).all() and (ol == np.array([len(r) for r in raws], np.uint64)).all()
        for r, o in zip(raws, out_off):
            assert out[int(o):int(o) + len(r)].tobytes() == r
        assert (out[~covered] == 0xA5).all(), mode
    # aliased inputs: every descriptor points at the same bytes
    n = 300
    s0 = np.frombuffer(streams[5], np.uint8).copy()
    caps = np.full(n, len(raws[5]), np.uint64)
    offs = np.arange(n, dtype=np.uint64) * np.uint64(len(raws[5]))
    out = np.zeros(n * len(raws[5]), np.uint8)
    ol, st = engine.decode_batch_host(s0, np.zeros(n, np.uint64), np.full(n, s0.size, np.uint64), out, offs, caps)
    assert (st == 0).all() and out.tobytes() == raws[5] * n


def test_pipelined_call_survives_dropped_handles_and_empty_batches(oracle, text):
    """A caller that drops the pending handle without wait(): the engine keeps the buffers alive and retires the batch itself
    (next call on the lane, or close()).  An empty batch returns the no-op ticket."""
    import gc
    import divans_b200
    eng = divans_b200.Engine(0, 64, 16)
    raws = [text[i * 3000: i * 3000 + 4000] for i in range(8)]
    streams = [oracle.encode_raw(r) for r in raws]
    for rep in range(5):
        h = eng.decode(streams, [len(r) for r in raws])          # warm
        blob = np.frombuffer(b"".join(streams), np.uint8).copy()
        in_len = np.array([len(s) for s in streams], np.uint64)
        in_off = np.concatenate([[0], np.cumsum(in_len)[:-1]]).astype(np.uint64)
        cap = np.array([len(r) for r in raws], np.uint64)
        out_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
        out = np.zeros(int(cap.sum()), np.uint8)
        eng.decode_batch_host_async(blob, in_off, in_len, out, out_off, cap)   # handle dropped on the floor
        del blob, out
        gc.collect()
    e = eng.decode_batch_host_async(np.zeros(1, np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(1, np.uint8),
                                    np.zeros(0, np.uint64), np.zeros(0, np.uint64))
    ol, st = e.wait()
    assert len(ol) == 0 and len(st) == 0
    res = eng.decode(streams, [len(r) for r in raws])
    assert all(st == 0 and o == r for (st, o), r in zip(res, raws))
    eng.close()
