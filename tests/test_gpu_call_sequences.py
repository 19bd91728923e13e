"""GPU tests (-m gpu) of every entry point in sequences on one shared context (DESIGN.md section 3, "Slot state of the v2
decoder, and the tests that pin it").  A context keeps state from call to call: the arena slots' headers, scratch that
calls of different kinds lay out in their own ways and grow, one `ev_busy` event that orders launch sets across CUDA streams, and two pipelined host
lanes.  The kinds of call are in tests/call_catalogue.py, each with its oracle result and what it may do to a slot header.

* ordered pairs of kinds on the one-warp engines of tests/test_gpu_slot_state.py: every pair whose second call is a
  default-model decode, and a seeded half of the rest (about 560 of the 961 pairs per layout; they take 64 s and 112 s on an
  H100, so the full product would take about 5 minutes); every result and every slot header after each call checked;
* eight seeded sequences of 60 calls on an eight-slot context, across three CUDA streams, batch sizes changing by up to 16x,
  the arena reallocated once, pipelined host decodes in flight and waited on out of order; results read at the end;
* two contexts, each driven by a thread of its own, next to a third thread on the reference FFI's shared context."""
import itertools
import threading

import numpy as np
import pytest

import call_catalogue as C

pytestmark = pytest.mark.gpu

LAYOUTS = {"16lanes_2slots": (2, 16), "8lanes_4slots": (4, 8)}
V2_DECODES = ["dec", "dec_dev", "dec_wasm", "dec_cmds", "dec_cmds_dev"]


@pytest.fixture(scope="module")
def cat(oracle, oracle_blend, golden):
    kinds = C.catalogue(oracle, oracle_blend, golden)
    for k in kinds.values():
        k.unit_expect   # the oracle's results, computed once
    return kinds


def _result(r):
    if callable(r):
        import torch
        torch.cuda.synchronize()
        return r()
    return r


def _first_diff(got, want):
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            fields = [j for j, (a, b) in enumerate(zip(g, w)) if a != b] if isinstance(g, tuple) and isinstance(w, tuple) else None
            return "item %d differs in fields %s: status %s, want %s" % (i, fields, g[0] if isinstance(g, tuple) else g,
                                                                       w[0] if isinstance(w, tuple) else w)
    return "lengths %d, %d" % (len(got), len(want))


def _assert_result(kind, rep, got, what):
    want = kind.expect(rep)
    assert got == want, "%s: %s: %s" % (what, kind.name, _first_diff(got, want))


def headers(eng):
    """every slot's header, for as many slots as the arena holds"""
    import divans_b200
    out = []
    while True:
        try:
            out.append(eng.slot_header(len(out)))
        except divans_b200.DivansError:
            return out


def test_fresh_context_gives_the_expectation(cat):
    """Each kind on a context of its own equals its oracle result: otherwise the catalogue is wrong, not a sequence."""
    import divans_b200
    failed = []
    for name, k in cat.items():
        eng = divans_b200.Engine(0, 2, 16)
        try:
            _assert_result(k, 2, _result(k.run(eng, 2)), "fresh")
            C.check_headers(k, 2, [], headers(eng), 2, 16, "fresh " + name)
        except AssertionError as e:
            failed.append(str(e).split("\n")[0])
        finally:
            eng.close()
    assert not failed, failed


def _pairs(names):
    rng = np.random.default_rng(1234)
    out = []
    for a, b in itertools.product(names, repeat=2):
        if b in V2_DECODES or rng.random() < 0.5:
            out.append((a, b))
    return out


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_every_ordered_pair(cat, layout):
    """A, then B, on one one-warp context: every slot runs A's inputs, then B's.  B's result is its oracle result and every
    slot header matches the model after each call."""
    import divans_b200
    g, lanes = LAYOUTS[layout]
    eng = divans_b200.Engine(0, g, lanes)
    try:
        h = headers(eng)
        for a, b in _pairs(list(cat)):
            for k in (cat[a], cat[b]):
                what = "%s then %s (%s)" % (a, b, k.name)
                _assert_result(k, g, _result(k.run(eng, g)), what)
                h2 = headers(eng)
                C.check_headers(k, g, h, h2, g, lanes, what)
                h = h2
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# seeded sequences across CUDA streams and scratch sizes
# ---------------------------------------------------------------------------------------------------------------------
def _async_decode(eng, kind, rep):
    """decode_batch_host_async of `rep` copies of kind's unit: (pending handle, function of its (out_len, status) -> result)"""
    import divans_b200
    cases = C._rep(kind.unit, rep)
    blob, off, ln = divans_b200._pack([c.stream for c in cases])
    cap = np.array([c.cap for c in cases], np.uint64)
    ooff, total = divans_b200._regions(cap)
    out = np.zeros(total, np.uint8)
    p = eng.decode_batch_host_async(blob, off, ln, out, ooff, cap, C.R.SKIP_CRC)
    return p, lambda r: C._norm_dec(r[1], [out[int(o):int(o + n)].tobytes() for o, n in zip(ooff, r[0])])


def run_sequence(eng, cat, seed, n_calls=60, check_arena=True):
    """n_calls calls drawn from the catalogue on `eng`: device calls on the context's stream or one of two torch streams with
    no host synchronisation between them, blocking host calls, and pipelined host decodes.  Returns [(what, kind, rep,
    result or reader)], read after the sequence."""
    import torch
    rng = np.random.default_rng(seed)
    streams = [None, torch.cuda.Stream(), torch.cuda.Stream()]
    names = list(cat)
    done, pending = [], []
    if check_arena:
        # a two-stream decode sizes the arena at two slots; the first encoder call needs eight: ensure_arena reallocates,
        # and every generation counter restarts at zero
        k = cat["dec_wasm"]
        done.append(("seed %d call 0" % seed, k, 1, k.run(eng, 1)))
        h = headers(eng)
        assert len(h) == 2 and sum(x[0] for x in h) == 2, h
        k = cat["enc_raw"]
        done.append(("seed %d call 1" % seed, k, 2, k.run(eng, 2)))
        h = headers(eng)
        assert len(h) == 8 and all(x[0] == 0 for x in h), h
    for i in range(len(done), n_calls):
        what = "seed %d call %d" % (seed, i)
        rep = int(rng.choice([1, 2, 4, 8, 16], p=[0.3, 0.3, 0.2, 0.1, 0.1]))
        if rng.random() < 0.12:
            k = cat["dec"]
            if len(pending) == 2:          # two tickets in flight: retire one of them, the newer one half of the time
                j = int(rng.integers(0, 2))
                p, conv, w = pending.pop(j)
                done.append(w + (conv(p.wait()),))
            p, conv = _async_decode(eng, k, rep)
            pending.append((p, conv, (what + " (async)", k, rep)))
            continue
        k = cat[names[int(rng.integers(0, len(names)))]]
        s = streams[int(rng.integers(0, 3))] if k.device else None
        done.append((what + " (%s)" % ("own stream" if s is None else "torch stream"), k, rep, k.run(eng, rep, s)))
    for p, conv, w in reversed(pending):
        done.append(w + (conv(p.wait()),))
    torch.cuda.synchronize()
    eng.synchronize()
    return done


def check_sequence(done):
    for what, k, rep, r in done:
        _assert_result(k, rep, r() if callable(r) else r, what)


@pytest.mark.parametrize("seed", range(8))
def test_seeded_sequence(cat, seed):
    import divans_b200
    eng = divans_b200.Engine(0, 8, 0)
    try:
        check_sequence(run_sequence(eng, cat, 100 + seed))
    finally:
        eng.close()


def test_two_contexts_and_the_ffi_context_at_once(cat, oracle):
    """Two Engines on one device, each driven by its own thread, and a third thread on the shared context behind the reference
    FFI (DivansCompressorWriter / DivansDecompressorReader): nothing is shared, so every result is its own oracle result."""
    import io
    import divans_b200
    for k in cat.values():      # upload every device kind's inputs before the threads start
        if k.device and k.name not in ("choose_dev", "choose_pick_dev"):
            for rep in (1, 2, 4, 8, 16):
                k.dev_inputs(rep)
    errors, results = [], {}

    def engine_thread(seed):
        try:
            eng = divans_b200.Engine(0, 8, 0)
            try:
                results[seed] = run_sequence(eng, cat, seed, n_calls=30, check_arena=False)
                check_sequence(results[seed])
            finally:
                eng.close()
        except BaseException as e:   # noqa: BLE001 (re-raised in the main thread)
            errors.append((seed, e))

    def ffi_thread():
        try:
            for i, r in enumerate(C.raws(6, 3000, 200)):
                buf = io.BytesIO()
                w = divans_b200.DivansCompressorWriter(buf)
                w.write(r)
                w.close()
                rc, ref = oracle.decode(buf.getvalue(), out_cap=len(r) + 64)
                assert rc == 0 and ref == r, "FFI stream %d" % i
                got = divans_b200.DivansDecompressorReader(io.BytesIO(oracle.encode_raw(r)), buffer_size=997).read()
                assert got == r, "FFI decode %d" % i
        except BaseException as e:   # noqa: BLE001
            errors.append(("ffi", e))

    ts = [threading.Thread(target=engine_thread, args=(s,)) for s in (300, 301)] + [threading.Thread(target=ffi_thread)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise errors[0][1]
