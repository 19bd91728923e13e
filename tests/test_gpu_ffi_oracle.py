"""-m gpu: the reference's FFI surface (divans_new_compressor, divans_set_option, divans_encode, divans_encode_flush,
divans_decode) against the oracle.

 * Option table: every selector 1..20 at and around the edges of its values.  ref_set_option restates the reference's
   OptionStage (src/ffi/compressor.rs:63-166, defaults src/interface.rs:462-484) on the options the encoder sees; the FFI must
   accept or refuse as it does (or as the header's departures say), and an accepted sequence must give byte for byte the
   oracle's stream under the mapped options, which Engine.encode gives too and the oracle decodes back to the input.
 * Order: the first literal-adaptation option sets all four speeds, later ones their own slot.
 * Streaming: splits, zero-length calls, calls entered at a non-zero *input_offset, 1/7/15/65536-byte output windows, calls
   after the end, refusals at the byte that makes a stream invalid, trailing bytes left unconsumed.
 * Output growth up to DIVANS_B200_MAX_OUTPUT, and host threads driving their own states next to a batch Engine.
Drivers: tests/ffi_streams.py."""
import hashlib
import itertools
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np
import pytest

import ffi_streams as F

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

QUALITY, WINDOW, LGBLOCK, MIXING, BROTLI_CMD, BROTLI_BITSTREAM, CONTEXT_MAP, ADAPT_CM_HIGH, STRIDE, STRIDE_DETECTION, \
    PRIOR_DEPTH, ADAPT_STRIDE_HIGH, ADAPT_CM_LOW, ADAPT_STRIDE_LOW, BYTE_SCORE, SPEED_DETECTION, BITMASK_DETECTION, Q9_5, \
    CONTEXT_MODE, IR_OPTIMIZER = range(1, 21)   # src/ffi/interface.rs:18-37

# Speed::ENCODER_DEFAULT_PALETTE, src/probability/interface.rs:303-320: (inc, lim)
PALETTE = [(0, 1024), (2, 1024), (1, 128), (1, 16384), (2, 2048), (4, 1024), (8, 8192), (16, 48), (16, 8192), (32, 4096),
           (64, 16384), (128, 256), (128, 16384), (512, 16384), (1664, 16384)]
# the slot of DivansCompressorOptions::literal_adaptation each selector writes once the speeds are set
ADAPT_SLOT = {ADAPT_STRIDE_LOW: 0, ADAPT_STRIDE_HIGH: 1, ADAPT_CM_LOW: 2, ADAPT_CM_HIGH: 3}
# command-selection knobs: stored by the reference for the brotli crate, no effect on the entropy half
KNOBS = (QUALITY, LGBLOCK, STRIDE_DETECTION, BYTE_SCORE, SPEED_DETECTION, BITMASK_DETECTION, Q9_5, IR_OPTIMIZER)

# DivansCompressorOptions::default() as the encoder sees it: window 22, dynamic context mixing 1, prior depth None (0), context
# map on, stride UseBrotliRec (from the command: 9), speeds None, and the literal-only record's mode LSB6 (0)
DEFAULTS = dict(window_size=22, dynamic_context_mixing=1, prior_depth=0, use_context_map=1, force_stride=9,
                literal_adaptation=None, literal_pred_mode=0)


def ref_set_option(o, sel, value):
    """(reference accepts, options after the call, departs) of the reference's set_option on the encoder-visible options `o`.  A
    refused value leaves the options as they were.  `departs`: the reference accepts the value but cannot code it, and the
    library refuses it (include/divans_b200.h, section 1)."""
    o = dict(o)
    u8 = value & 0xff
    if sel in KNOBS:
        return True, o, False
    if sel == WINDOW:     # Some(value as i32), clamped to 10..24 by the compressor (src/divans_compressor.rs:90)
        i32 = value - (1 << 32) if value >= 1 << 31 else value
        o["window_size"] = min(24, max(10, i32))
        return True, o, False
    if sel == MIXING:                  # `value as u8`; encoding asserts it fits 3 bits (codec/context_map.rs:192)
        o["dynamic_context_mixing"] = u8
        return True, o, u8 > 7
    if sel == PRIOR_DEPTH:             # `value as u8`, coded as a nibble
        o["prior_depth"] = u8
        return True, o, u8 > 15
    if sel == CONTEXT_MODE:            # LiteralPredictionModeNibble(value as u8)
        o["literal_pred_mode"] = u8
        return True, o, u8 > 3
    if sel == BROTLI_CMD:
        return value <= 2, o, False
    if sel == BROTLI_BITSTREAM:
        return value == 1, o, False
    if sel == CONTEXT_MAP:
        if value > 1:
            return False, o, False
        o["use_context_map"] = value
        return True, o, False
    if sel == STRIDE:
        if value > 8:
            return False, o, False
        o["force_stride"] = value
        return True, o, False
    if sel in ADAPT_SLOT:
        if value >= len(PALETTE):
            return False, o, False
        if o["literal_adaptation"] is None:
            o["literal_adaptation"] = [PALETTE[value]] * 4
        else:
            la = list(o["literal_adaptation"])
            la[ADAPT_SLOT[sel]] = PALETTE[value]
            o["literal_adaptation"] = la
        return True, o, False
    return False, o, False


def ref_options(seq):
    """the library's expected (results of set_option, mapped options) for a sequence of (selector, value)"""
    o, rcs = dict(DEFAULTS), []
    for sel, val in seq:
        ok, new, departs = ref_set_option(o, sel, val)
        if ok and not departs:
            o = new
        rcs.append(F.SUCCESS if ok and not departs else F.FAILURE)
    return rcs, o


# ---- the table: every selector at and around its edges ----
U32 = (1 << 32) - 1
CASES = [(sel, v) for sel in (ADAPT_CM_HIGH, ADAPT_STRIDE_HIGH, ADAPT_CM_LOW, ADAPT_STRIDE_LOW) for v in list(range(15)) + [15, U32]]
CASES += [(STRIDE, v) for v in list(range(10)) + [U32]]
CASES += [(WINDOW, v) for v in (0, 9, 10, 11, 16, 22, 23, 24, 25, 1 << 31, U32)]
CASES += [(MIXING, v) for v in (0, 1, 2, 3, 7, 8, 15, 16, 255, 256, 258)]
CASES += [(PRIOR_DEPTH, v) for v in (0, 1, 2, 3, 15, 16, 255, 256, 257)]
CASES += [(CONTEXT_MAP, v) for v in (0, 1, 2)]
CASES += [(BROTLI_CMD, v) for v in (0, 1, 2, 3)] + [(BROTLI_BITSTREAM, v) for v in (0, 1, 2)]
CASES += [(CONTEXT_MODE, v) for v in (0, 1, 2, 3, 4, 15, 16, 255, 256, 259)]
CASES += [(sel, v) for sel in KNOBS for v in (0, 1, U32)]
CASES += [(sel, 0) for sel in (0, 21, 255)]


def _inputs():
    rng = np.random.default_rng(7)
    words = b"the quick brown fox jumps over a lazy dog. Mary had a little lamb, its fleece was white as snow. ".split(b" ")
    text = b" ".join(words[int(i)] for i in rng.integers(0, len(words), 1200))[:5000]
    rnd = rng.integers(0, 256, 3000).astype(np.uint8).tobytes()
    # > 65536 literal nibbles: the literal coder flushes a rANS chunk and the mux writes several records
    long = (text * 8)[:24000] + rng.integers(0, 256, 16000).astype(np.uint8).tobytes()
    return [b"", b"A", text, rnd, long]


INPUTS = _inputs()


@pytest.fixture(scope="module")
def lib():
    import divans_b200
    return divans_b200.load_library()


def _engine_kw(o):
    kw = dict(o)
    if kw["literal_adaptation"] is None:
        del kw["literal_adaptation"]
    return kw


def _oracle_streams(oracle, raws, o):
    """(status, stream) per raw input: the oracle's literal-only encode under the mapped options, mixing value 4"""
    kw = {k: v for k, v in o.items() if k != "literal_pred_mode"}
    return oracle.encode_raw_list(raws, oracle.options(**kw), o["literal_pred_mode"], 4)


def _engine_streams(engine, raws, o):
    import divans_b200
    blob = np.frombuffer(b"".join(raws) or b"\0", np.uint8)
    in_len = np.array([len(r) for r in raws], np.uint64)
    in_off = np.concatenate([[0], np.cumsum(in_len)[:-1]]).astype(np.uint64)
    cap = in_len * np.uint64(2) + np.uint64(70000)
    out_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
    out = np.zeros(int(cap.sum()), np.uint8)
    ln, st = engine.encode_batch_host(blob, in_off, in_len, out, out_off, cap, divans_b200.encode_options(**_engine_kw(o)))
    return [(int(s), out[int(a):int(a) + int(n)].tobytes() if s == 0 else None) for s, a, n in zip(st, out_off, ln)]


def _check_sequence(engine, oracle, seq, raws):
    """seq through the FFI, per input: set_option results as the reference's (or the documented departures), and the stream
    equal to the oracle's and Engine.encode's under the mapped options, decoding back to the input"""
    want_rcs, o = ref_options(seq)
    ref = _oracle_streams(oracle, raws, o)
    eng = _engine_streams(engine, raws, o)
    for i, raw in enumerate(raws):
        rcs, frc, got = F.compress(seq, raw)
        assert rcs == want_rcs, "set_option results %s, reference %s (%s)" % (rcs, want_rcs, seq)
        rs, rb = ref[i]
        assert eng[i] == ref[i], "input %d: Engine.encode under %s differs from the oracle (status %d / %d)" % (i, o, eng[i][0], rs)
        if rs != 0:
            assert frc == F.FAILURE, "input %d: the oracle refuses %s (status %d), the FFI flush gave %d" % (i, o, rs, frc)
            continue
        assert frc == F.SUCCESS and got == rb, "input %d: FFI stream under %s differs from the oracle (%s vs %d bytes)" % (
            i, seq, None if got is None else len(got), len(rb))
        rc, back = oracle.decode(got, out_cap=len(raw) + 64)
        assert rc == 0 and back == raw, "input %d: the oracle does not decode the stream of %s back (rc %d)" % (i, seq, rc)
    return o


@pytest.mark.parametrize("sel,value", CASES, ids=["sel%d-%d" % c for c in CASES])
def test_option_table_matches_the_reference(engine, oracle, sel, value):
    _check_sequence(engine, oracle, [(sel, value)], INPUTS)


ORDERS = [list(zip(p, (3, 6, 9, 12))) for p in itertools.permutations((ADAPT_STRIDE_LOW, ADAPT_STRIDE_HIGH, ADAPT_CM_LOW, ADAPT_CM_HIGH))]
SEQUENCES = ORDERS + [
    [(ADAPT_CM_HIGH, 3), (ADAPT_CM_HIGH, 9)],                                   # the same selector twice
    [(ADAPT_CM_LOW, 8), (ADAPT_CM_LOW, 8), (ADAPT_STRIDE_LOW, 2)],
    [(ADAPT_STRIDE_LOW, 99), (ADAPT_CM_HIGH, 4)],                               # a refused first speed sets nothing
    [(WINDOW, 16), (MIXING, 2), (ADAPT_STRIDE_HIGH, 5), (PRIOR_DEPTH, 2), (ADAPT_CM_LOW, 7)],   # speeds between other options
    [(ADAPT_STRIDE_HIGH, 5), (ADAPT_CM_LOW, 7), (WINDOW, 16), (MIXING, 2), (PRIOR_DEPTH, 2)],
    [(MIXING, 2), (CONTEXT_MODE, 2), (ADAPT_CM_HIGH, 11), (ADAPT_CM_LOW, 1), (STRIDE, 1), (WINDOW, 23)],
    [(MIXING, 2), (MIXING, 0), (CONTEXT_MAP, 0), (CONTEXT_MAP, 1), (CONTEXT_MODE, 3), (CONTEXT_MODE, 7), (WINDOW, 30), (WINDOW, 12)],
    [(QUALITY, 5), (BROTLI_CMD, 0), (Q9_5, 1), (IR_OPTIMIZER, 1), (BITMASK_DETECTION, 0), (ADAPT_CM_HIGH, 2)],
]


@pytest.mark.parametrize("seq", SEQUENCES, ids=["seq%d" % i for i in range(len(SEQUENCES))])
def test_option_order_matches_the_reference(engine, oracle, seq):
    _check_sequence(engine, oracle, seq, INPUTS[2:4])


def test_refused_literal_context_modes_and_raw_records(engine, lib):
    """The FFI refuses a context mode whose low byte is above 3 (the reference's brotli path would take it as SIGN); the raw
    encoders that build their record from opts refuse literal_pred_mode outside 0..3 before any work, as mixmap does."""
    import divans_b200
    for v in (4, 15, 16, 255, 260, U32):
        rcs, frc, got = F.compress([(CONTEXT_MODE, v)], INPUTS[2])
        assert rcs == [F.FAILURE] and frc == F.SUCCESS
        assert got == F.compress([], INPUTS[2])[2], "a refused context mode changed the options"
    import torch
    blob = np.frombuffer(INPUTS[2], np.uint8)
    out = np.zeros(1 << 16, np.uint8)
    d_in = torch.from_numpy(blob.copy()).to("cuda:0")
    d_out = torch.zeros(out.size, dtype=torch.uint8, device="cuda:0")
    d_meta = torch.tensor([0, blob.size, 0, out.size], dtype=torch.int64, device="cuda:0")   # in_off, in_len, out_off, out_cap
    d_len = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    d_status = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    for pm in (-1, 4, 255, 256):
        o = divans_b200.encode_options(literal_pred_mode=pm)
        with pytest.raises(divans_b200.DivansError, match="literal_pred_mode %d is outside 0..3" % pm):
            engine.encode_batch_host(blob, [0], [blob.size], out, [0], [out.size], o)
        # the device call gets real regions: if the refusal ever came after the launch, the stream would be coded (status 3, or
        # mode 256 as LSB6) and the checks below would say so
        d_status.fill_(-1)
        d_len.zero_()
        with pytest.raises(divans_b200.DivansError, match="literal_pred_mode"):
            engine.encode_batch_device(1, d_in.data_ptr(), d_meta[0:1].data_ptr(), d_meta[1:2].data_ptr(), blob.size, d_out.data_ptr(),
                                       d_meta[2:3].data_ptr(), d_meta[3:4].data_ptr(), d_len.data_ptr(), d_status.data_ptr(), o)
        engine.synchronize()
        assert int(d_status[0]) == -1 and int(d_len[0]) == 0, "the device encode ran for mode %d" % pm
        with pytest.raises(divans_b200.DivansError, match="literal_pred_mode"):
            engine.encode_speeds_batch_host(blob, [0], [blob.size], out, [0], [out.size], o)
    o = divans_b200.encode_options(literal_pred_mode=3)
    ln, st = engine.encode_batch_host(blob, [0], [blob.size], out, [0], [out.size], o)
    assert st[0] == 0
    engine.encode_batch_device(1, d_in.data_ptr(), d_meta[0:1].data_ptr(), d_meta[1:2].data_ptr(), blob.size, d_out.data_ptr(),
                               d_meta[2:3].data_ptr(), d_meta[3:4].data_ptr(), d_len.data_ptr(), d_status.data_ptr(), o)
    engine.synchronize()
    assert int(d_status[0]) == 0 and int(d_len[0]) == int(ln[0])
    assert d_out[:int(ln[0])].cpu().numpy().tobytes() == out[:int(ln[0])].tobytes()


def test_blend_deployment_option_table(oracle_blend):
    """DIVANS_B200_FFI_CDF=blend (read once per process: a child process) against the blend oracle, on a reduced table"""
    seqs = [[], [(ADAPT_CM_HIGH, 3)], [(WINDOW, 16)], [(MIXING, 2)], [(MIXING, 0)], [(CONTEXT_MODE, 2)], [(CONTEXT_MAP, 0)],
            [(STRIDE, 3)], [(PRIOR_DEPTH, 2)], [(ADAPT_STRIDE_HIGH, 5), (ADAPT_CM_LOW, 9)], [(MIXING, 16)]]
    raws = INPUTS[1:4]
    with tempfile.TemporaryDirectory() as d:
        job = os.path.join(d, "job.json")
        json.dump(dict(seqs=seqs, raws=[r.hex() for r in raws]), open(job, "w"))
        code = ("import json, sys\nsys.path[:0] = [%r, %r]\nimport ffi_streams as F\n"
                "j = json.load(open(%r))\n"
                "res = [[list(F.compress(s, bytes.fromhex(r))) for r in j['raws']] for s in j['seqs']]\n"
                "json.dump([[[a, b, c.hex() if c is not None else None] for a, b, c in row] for row in res], open(%r, 'w'))\n"
                ) % (ROOT, HERE, job, os.path.join(d, "out.json"))
        subprocess.run([sys.executable, "-c", code], check=True, env=dict(os.environ, DIVANS_B200_FFI_CDF="blend"), timeout=300)
        res = json.load(open(os.path.join(d, "out.json")))
    for seq, row in zip(seqs, res):
        want_rcs, o = ref_options([tuple(x) for x in seq])
        ref = _oracle_streams(oracle_blend, raws, o)
        for raw, (rcs, frc, got), (rs, rb) in zip(raws, row, ref):
            assert rcs == want_rcs, (seq, rcs, want_rcs)
            assert rs == 0 and frc == F.SUCCESS and bytes.fromhex(got) == rb, "blend: %s on %d bytes differs from the blend oracle" % (seq, len(raw))
            rc, back = oracle_blend.decode(rb, out_cap=len(raw) + 64)
            assert rc == 0 and back == raw


# ---- encoder streaming ----
def test_encoder_streaming_contract(oracle, lib):
    import ctypes
    raw = INPUTS[4][:20000]
    seq = [(MIXING, 2), (WINDOW, 18)]
    _, o = ref_options(seq)
    ref = _oracle_streams(oracle, [raw], o)[0][1]
    for cuts in ([], [0], [0, 0, 5, 5, 100, 100], [1, 2, 3, len(raw) - 1, len(raw)], list(range(0, len(raw), 4097))):
        for win in (1, 15, 65536):
            if win == 1 and len(cuts) > 2:
                continue   # (1-byte windows once per split kind is enough: they only exercise the output cursor)
            rcs, frc, got = F.compress(seq, raw, cuts, win)
            assert rcs == [0, 0] and frc == F.SUCCESS and got == ref, "cuts %s window %d" % (cuts[:6], win)
    st = lib.divans_new_compressor()
    try:
        buf = np.frombuffer(raw, np.uint8)
        p = ctypes.c_void_p(buf.ctypes.data)
        assert lib.divans_set_option(st, WINDOW, 18) == F.SUCCESS
        off, oo = ctypes.c_size_t(0), ctypes.c_size_t(0)
        assert lib.divans_encode(st, p, 0, ctypes.byref(off), None, 0, ctypes.byref(oo)) == F.NEEDS_MORE_INPUT
        # the first divans_encode, even of nothing, leaves the OptionStage
        assert lib.divans_set_option(st, MIXING, 2) == F.FAILURE
        assert lib.divans_set_option(st, 200, 0) == F.FAILURE
        assert lib.divans_encode(st, p, len(raw), ctypes.byref(off), None, 0, ctypes.byref(oo)) == F.NEEDS_MORE_INPUT
        assert off.value == len(raw)
        win = np.zeros(1 << 17, np.uint8)
        oo = ctypes.c_size_t(0)
        assert lib.divans_encode_flush(st, ctypes.c_void_p(win.ctypes.data), win.size, ctypes.byref(oo)) == F.SUCCESS
        assert win[:oo.value].tobytes() == F.compress([(WINDOW, 18)], raw)[2]
        n = oo.value
        assert lib.divans_encode_flush(st, ctypes.c_void_p(win.ctypes.data), win.size, ctypes.byref(oo)) == F.SUCCESS
        assert oo.value == n, "a flush after SUCCESS wrote more"
        off = ctypes.c_size_t(0)
        assert lib.divans_encode(st, p, len(raw), ctypes.byref(off), None, 0, ctypes.byref(oo)) == F.FAILURE
        assert lib.divans_set_option(st, WINDOW, 20) == F.FAILURE
    finally:
        lib.divans_free_compressor(st)
    # a flush with no divans_encode also ends the OptionStage
    st = lib.divans_new_compressor()
    try:
        oo = ctypes.c_size_t(0)
        assert lib.divans_encode_flush(st, ctypes.c_void_p(win.ctypes.data), win.size, ctypes.byref(oo)) == F.SUCCESS
        assert win[:oo.value].tobytes() == _oracle_streams(oracle, [b""], dict(DEFAULTS))[0][1]
        assert lib.divans_set_option(st, WINDOW, 20) == F.FAILURE
    finally:
        lib.divans_free_compressor(st)


# ---- decoder streaming ----
def test_decoder_every_split_through_small_windows(oracle):
    for raw in (b"", b"A", INPUTS[2][:60]):
        s = oracle.encode_raw(raw)
        rc, ref = oracle.decode(s, out_cap=len(raw) + 64)
        assert rc == 0 and ref == raw
        for k in range(len(s) + 1):
            for win in (1, 7):
                rc, out, used, _ = F.decompress(s, [k], win)
                assert rc == F.SUCCESS and out == ref and used == len(s), "split at %d of %d, window %d: rc %d" % (k, len(s), win, rc)


def test_decoder_stops_at_the_trailer_and_ends_in_success(oracle, lib):
    import ctypes
    import divans_b200
    raw = INPUTS[2]
    s = oracle.encode_raw(raw)
    for tail in (b"\0", b"garbage" * 9, s):
        rc, out, used, _ = F.decompress(s + tail)
        assert rc == F.SUCCESS and out == raw and used == len(s), "trailing %d bytes: consumed %d of %d" % (len(tail), used, len(s))
    st = lib.divans_new_decompressor_with_custom_alloc(divans_b200.CAllocator(None, None, None), 0, 1)
    try:
        rc, out, used, _ = F.decompress(s, [len(s) // 2], 4096, state=st)
        assert rc == F.SUCCESS and out == raw
        more = np.frombuffer(b"more input", np.uint8)
        win = np.zeros(64, np.uint8)
        for _ in range(2):   # after SUCCESS: SUCCESS, nothing taken, nothing written
            off, oo = ctypes.c_size_t(0), ctypes.c_size_t(0)
            rc = lib.divans_decode(st, ctypes.c_void_p(more.ctypes.data), more.size, ctypes.byref(off), ctypes.c_void_p(win.ctypes.data),
                                   win.size, ctypes.byref(oo))
            assert rc == F.SUCCESS and off.value == 0 and oo.value == 0
    finally:
        lib.divans_free_decompressor(st)


def _bad_streams(s):
    """(name, stream, index of the byte whose arrival makes it invalid) -- s is the stream of an empty input"""
    assert s[-11:-8] == b"\xff\xfe\xff" and s[16] < 0x40, "the stream's layout changed"
    n = len(s)
    cases = [("magic%d" % i, s[:i] + bytes([s[i] ^ 0x10]) + s[i + 1:], 15) for i in range(4)]
    cases += [("window%d" % w, s[:5] + bytes([w]) + s[6:], 15) for w in (0, 9, 25, 255)]
    cases += [("record%x" % h, s[:16] + bytes([h]) + s[17:], 16) for h in (0x40, 0x80, 0xfe)]
    cases += [("eof1", s[:n - 10] + b"\0" + s[n - 9:], n - 9), ("eof2", s[:n - 9] + b"\0" + s[n - 8:], n - 9)]
    return cases


def test_decoder_refuses_at_the_offending_byte_and_stays_failed(oracle, lib):
    import divans_b200
    s = oracle.encode_raw(b"")
    for name, bad, at in _bad_streams(s):
        assert oracle.decode(bad)[0] == oracle.FAILURE, name
        st = lib.divans_new_decompressor_with_custom_alloc(divans_b200.CAllocator(None, None, None), 0, 1)
        try:
            rc, out, used, k = F.decompress(bad, list(range(1, len(bad))), 7, state=st)   # one byte per call
            assert rc == F.FAILURE and k == at and out == b"", "%s: result %d at byte %d, expected FAILURE at %d" % (name, rc, k, at)
            rc, out, used, k = F.decompress(s, state=st)   # a failed state stays failed, even on a good stream
            assert rc == F.FAILURE and out == b"" and k == 0, name
        finally:
            lib.divans_free_decompressor(st)
        # the whole stream in one call: the same verdict
        assert F.decompress(bad)[0] == F.FAILURE, name


def test_reader_truncated_and_corrupt_streams(oracle):
    import io
    import divans_b200
    raw = INPUTS[3]
    s = oracle.encode_raw(raw)

    def read_all(data, **kw):
        rd = divans_b200.DivansDecompressorReader(io.BytesIO(data), 1000, **kw)
        try:
            return rd.read()
        finally:
            rd.close()
    for k in (0, 5, 15, 16, 17, len(s) // 2, len(s) - 11, len(s) - 9, len(s) - 1):
        assert oracle.decode(s[:k])[0] == oracle.NEEDS_MORE_INPUT
        with pytest.raises(EOFError):
            read_all(s[:k])
    for pos in (len(s) - 8, len(s) - 5):
        bad = s[:pos] + bytes([s[pos] ^ 4]) + s[pos + 1:]
        assert oracle.decode(bad)[0] == oracle.FAILURE
        with pytest.raises(ValueError):
            read_all(bad)
        rc, ref = oracle.decode(bad, skip_crc=True)
        assert rc == 0 and ref == raw
        assert read_all(bad, skip_crc=True) == ref
    bad = s[:-3] + b"x" + s[-2:]   # the "ans~" magic is checked with skip_crc too
    assert oracle.decode(bad, skip_crc=True)[0] == oracle.FAILURE
    with pytest.raises(ValueError):
        read_all(bad, skip_crc=True)


# ---- output growth ----
GROW_CHILD = """
import hashlib, json, sys
sys.path[:0] = [%r, %r]
import ctypes, divans_b200, ffi_streams as F
L = divans_b200.load_library()
data = open(%r, 'rb').read()
st = L.divans_new_decompressor()
rc, out, used, _ = F.decompress(data, [], 1 << 22, state=st)
again = F.decompress(data, [], 1 << 22, state=st)[0]
L.divans_free_decompressor(st)
print(json.dumps(dict(rc=rc, n=len(out), sha=hashlib.sha256(out).hexdigest(), used=used, again=again)))
"""


def test_output_growth_up_to_the_limit(oracle, tmp_path):
    """A 100 MiB stream of a few hundred bytes: the first guess (8 x its size + 64 KiB) is regrown 4x at a time, to the
    oracle's output at the default limit and at a limit of exactly its length; one byte less fails and stays failed."""
    seed = bytes(range(64))
    ir = "window 22 0 0 0\ninsert 64 %s\n" % seed.hex() + "copy %d from 64 ctx 0\n" % (1 << 23) * 12 + "insert 3 414243\n"
    stream = oracle.Commands.from_ir(ir).encode(oracle.options(window_size=22))
    L = 64 + 12 * (1 << 23) + 3
    rc, ref = oracle.decode(stream, out_cap=L + 64)
    assert rc == 0 and len(ref) == L
    first = 8 * len(stream) + 65536
    assert L > first * 4 ** 4, "the stream must need several regrowths"
    path = tmp_path / "bomb.divans"
    path.write_bytes(stream)
    sha = hashlib.sha256(ref).hexdigest()
    del ref
    for limit in (None, L, L - 1):
        env = dict(os.environ)
        env.pop("DIVANS_B200_MAX_OUTPUT", None)
        if limit is not None:
            env["DIVANS_B200_MAX_OUTPUT"] = str(limit)
        p = subprocess.run([sys.executable, "-c", GROW_CHILD % (ROOT, HERE, str(path))], env=env, capture_output=True, text=True, timeout=300)
        assert p.returncode == 0, "limit %s: child exited %d: %s" % (limit, p.returncode, p.stderr[-2000:])
        assert "terminate called" not in p.stderr and "exception" not in p.stderr.lower(), p.stderr[-2000:]
        r = json.loads(p.stdout.strip().splitlines()[-1])
        if limit == L - 1:
            assert r["rc"] == F.FAILURE and r["n"] == 0 and r["again"] == F.FAILURE, (limit, r)
        else:
            assert r["rc"] == F.SUCCESS and r["n"] == L and r["sha"] == sha and r["used"] == len(stream), (limit, r)
            assert r["again"] == F.SUCCESS


# ---- threads ----
def test_host_threads_with_their_own_states_and_an_engine(oracle):
    """16 host threads, each with its own compressor or decompressor state, and one thread batch-encoding and decoding on its own
    Engine, all at once: every result equals its single-threaded, oracle-checked one."""
    import divans_b200
    rng = np.random.default_rng(11)
    text = INPUTS[2] * 8
    raws = [text[int(a):int(a) + n] + rng.integers(0, 256, n // 7).astype(np.uint8).tobytes()
            for a, n in zip(rng.integers(0, 1000, 8), (100, 900, 4000, 9000, 17000, 25000, 31000, 38000))]
    seqs = [[], [(WINDOW, 16)], [(MIXING, 2)], [(ADAPT_CM_HIGH, 5)], [(CONTEXT_MODE, 2)], [(STRIDE, 1)], [(MIXING, 0)],
            [(PRIOR_DEPTH, 2), (MIXING, 2)]]
    streams = [oracle.encode_raw(r, oracle.options(window_size=w, dynamic_context_mixing=m))
               for r, w, m in zip(raws, (16, 18, 20, 22, 24, 16, 18, 20), (0, 1, 2, 1, 0, 2, 1, 2))]
    jobs = [("enc", i, lambda i=i: F.compress(seqs[i], raws[i], list(range(0, len(raws[i]), 997 + 500 * i)), 15 + 4000 * i)[2])
            for i in range(8)]
    jobs += [("dec", i, lambda i=i: F.decompress(streams[i], list(range(0, len(streams[i]), 13 + 700 * i)), 7 + 3000 * i)[1])
             for i in range(8)]
    single = {}
    for kind, i, fn in jobs:
        single[(kind, i)] = fn()
        if kind == "enc":
            _, o = ref_options(seqs[i])
            assert single[(kind, i)] == _oracle_streams(oracle, [raws[i]], o)[0][1], "enc %d" % i
        else:
            assert single[(kind, i)] == raws[i], "dec %d" % i
    eng = divans_b200.Engine(0, 0, 16)
    threads = []
    try:
        eng_ref = (eng.encode(raws), eng.decode(streams, [len(r) + 64 for r in raws]))
        assert eng_ref[0] == [oracle.encode_raw(r) for r in raws] and all(st == 0 and o == r for (st, o), r in zip(eng_ref[1], raws))
        results, errors = {}, []
        start = threading.Barrier(len(jobs) + 1)

        def run(key, fn, reps=3):
            try:
                start.wait(timeout=60)
                results[key] = [fn() for _ in range(reps)]
            except Exception as e:   # reported below, after every thread has been joined
                errors.append((key, repr(e)))
        # daemon threads: a hung worker fails the test without keeping the process alive
        threads = [threading.Thread(target=run, args=((kind, i), fn), daemon=True) for kind, i, fn in jobs]
        threads.append(threading.Thread(target=run, args=(("engine", 0), lambda: (eng.encode(raws), eng.decode(streams, [len(r) + 64 for r in raws]))),
                                        daemon=True))
        for t in threads:
            t.start()
        deadline = time.monotonic() + 240
        for t in threads:
            t.join(timeout=max(0.0, deadline - time.monotonic()))
        alive = [t for t in threads if t.is_alive()]
        assert not alive, "%d threads still running after 240 s" % len(alive)
        assert not errors, errors
        for kind, i, _ in jobs:
            assert results[(kind, i)] == [single[(kind, i)]] * 3, "%s %d differs under threads" % (kind, i)
        assert results[("engine", 0)] == [eng_ref] * 3
    finally:
        if not any(t.is_alive() for t in threads):   # (a thread still inside the engine keeps it)
            eng.close()
