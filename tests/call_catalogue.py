"""The catalogue of call kinds that tests/test_gpu_call_sequences.py runs in sequences on one shared context.

A kind is a small, fixed batch through one entry point.  Its *unit* is a list of inputs; a batch of the kind repeats every
input ``rep`` times in a row (``[a] * rep + [b] * rep + ...``), so on a one-warp engine with ``rep`` slots every slot runs
every input once, in order, and a larger ``rep`` grows the context's scratch.  ``expect(rep)`` is the kind's full result for
such a batch, computed once from the CPU oracle (oracle/, oracle_tally/) with the helpers the per-feature test files use.

``run(eng, rep, stream)`` issues the call: host kinds call the blocking host entry point and return their result; device
kinds enqueue the device entry point on ``stream`` (a torch.cuda.Stream, or None for the context's own stream) with output
tensors of their own, and return a function that reads the result, to be called after the device has finished.

``phases`` model what a kind may do to the slot headers (DESIGN.md section 3, "Slot state of the v2 decoder, and the tests that pin it"), one
entry per launch set that touches the arena, in order: (engine, inputs per unit, word 1, words 2 and 3) with engine one of
``v2`` (a default-model decode, plain or recording: it advances word 0 by one per stream it starts and clears word 1 after
wiping), ``rec`` (the recording decoder: as v2, on the 16-lane layout), ``blend`` (the blend decoder: reset_slot, word 1 set)
and ``enc`` (the encoder's model walk and cost passes: reset_slot per stream).  Word 1 is 1 (the phase must leave it set),
0 (cleared), None (may set it) or "keep".  Words 2 and 3 are the set of (high-water mark, stale flag) pairs a used slot may end
with, or None where the inputs differ in them.  Kinds with no phase leave every header word alone."""
import functools
import json
import os

import numpy as np

import regimes as R
import bill_corpora as B
import irfuzz

HERE = os.path.dirname(os.path.abspath(__file__))

RAW_HDR = {(64, 1)}        # a raw-mode stream's record: the 64-entry identity literal map and 8192 mixing values
NOPM_HDR = {(0, 0)}        # no PredictionMode command; a literal before one zeroes the mask

# the decode unit: no_predmode first (it reads the literal map and the mixing mask an earlier call left), the failing streams
# between good ones, and two raw-mode streams last, so that every slot ends in the same header state
DEC_UNIT = [("no_predmode", 0), ("bt256", 0), ("corrupt_status1", 0), ("wide_midstream", 0), ("per_context_mix", 0), ("dcm2", 0),
            ("wide_speeds", 0), ("mix2_flat", 0), ("out_cap_small", 0), ("corrupt_status3", 0), ("msb6", 0), ("lsb6", 1)]
LIST_UNIT = ["bt256", "no_predmode", "switches", "per_context_mix"]   # window-16 command lists; bt256: a 16384-byte literal map
WIDE_OPTS = dict(literal_adaptation=[(16, 8192), (16, 8192), R.WIDE, R.WIDE])   # context-map speeds outside speed_is_small


def text(n, seed):
    return B.text(n, seed=seed)


def raws(k, base, seed=0):
    return [text(base + 300 * i, seed + i) for i in range(k)]


def _rep(items, rep):
    return [x for x in items for _ in range(rep)]


def _u64(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev)


class Kind:
    def __init__(self, name, unit, expect_unit, run, phases=(), device=False, gens=0):
        self.name, self._unit, self._expect_unit, self._run = name, unit, expect_unit, run
        self.phases, self.device, self._gens = list(phases), device, gens
        self._dev = {}

    @functools.cached_property
    def unit(self):
        return self._unit()

    @functools.cached_property
    def unit_expect(self):
        return self._expect_unit(self.unit)

    def expect(self, rep):
        return _rep(self.unit_expect, rep)

    @property
    def gens(self):
        """streams per unit the default-model decoder starts (word 0 advances by one for each)"""
        return self._gens(self.unit) if callable(self._gens) else self._gens

    def run(self, eng, rep, stream=None):
        """host kinds: the result; device kinds: a function that returns the result once the device has finished"""
        return self._run(self, eng, rep, stream)

    def dev_inputs(self, rep, dev="cuda:0"):
        """the batch's inputs packed and uploaded once (device kinds upload nothing inside a sequence)"""
        key = (rep, dev)
        if key not in self._dev:
            import divans_b200
            items = _rep(self.unit_inputs(), rep)
            blob, off, ln = divans_b200._pack(items)
            import torch
            self._dev[key] = dict(blob=torch.from_numpy(blob).to(dev), off=_u64(off, dev), len=_u64(ln, dev), n=len(items),
                                  max=int(ln.max()), total=int(ln.sum()), host_len=ln)
        return self._dev[key]

    def unit_inputs(self):
        return [u if isinstance(u, bytes) else u[0] for u in self.unit]


# ---------------------------------------------------------------------------------------------------------------------
# device plumbing: outputs allocated per call on the call's stream, read at the end
# ---------------------------------------------------------------------------------------------------------------------
class _On:
    """``with _On(stream):`` allocations and copies go to ``stream``; for the context's own stream (None) they go to the
    current stream, which is then drained so that the library's stream finds them written"""
    def __init__(self, stream):
        self.s = stream

    def __enter__(self):
        import torch
        self.ctx = torch.cuda.stream(self.s) if self.s is not None else None
        if self.ctx:
            self.ctx.__enter__()
        return self.s.cuda_stream if self.s is not None else None

    def __exit__(self, *a):
        import torch
        if self.ctx:
            self.ctx.__exit__(*a)
        else:
            torch.cuda.current_stream().synchronize()


def _zeros(n, dtype=None):
    import torch
    return torch.zeros(max(int(n), 1), dtype=dtype or torch.uint8, device="cuda:0")


# ---------------------------------------------------------------------------------------------------------------------
# decodes
# ---------------------------------------------------------------------------------------------------------------------
def _dec_unit(oracle):
    return [R.build(n, oracle, v) for n, v in DEC_UNIT]


def _dec_expect(oracle, flags):
    def f(unit):
        out = []
        for c in unit:
            rc, ref = oracle.decode(c.stream, out_cap=c.cap, skip_crc=bool(flags & R.SKIP_CRC))
            out.append((rc, ref if rc == 0 else None))
        return out
    return f


def _norm_dec(status, outs):
    return [(int(s), o if s == 0 else None) for s, o in zip(status, outs)]


def _run_dec_host(flags):
    def f(kind, eng, rep, stream):
        cases = _rep(kind.unit, rep)
        res = eng.decode([c.stream for c in cases], [c.cap for c in cases], flags)
        return _norm_dec([s for s, _ in res], [o for _, o in res])
    return f


def _run_dec_dev(flags):
    def f(kind, eng, rep, stream):
        import divans_b200
        d = kind.dev_inputs(rep)
        caps = np.array([c.cap for c in _rep(kind.unit, rep)], np.uint64)
        off, total = divans_b200._regions(caps)
        if "ocap" not in d:
            d["ooff"], d["ocap"] = _u64(off, "cuda:0"), _u64(caps, "cuda:0")
        with _On(stream) as s:
            out, res = _zeros(total), _zeros(2 * d["n"], _i64())
            eng.decode_batch_device(d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), out.data_ptr(), d["ooff"].data_ptr(),
                                    d["ocap"].data_ptr(), res.data_ptr(), res[d["n"]:].data_ptr(), d["n"], d["total"], flags, s)

        def read():
            r = res.cpu().numpy()
            ln, st = r[:d["n"]].view(np.uint64), r[d["n"]:].view(np.int32)[:d["n"]]
            h = out.cpu().numpy()
            return _norm_dec(st, [h[int(o):int(o + n)].tobytes() for o, n in zip(off, ln)])
        return read
    return f


def _i64():
    import torch
    return torch.int64


def _wasm_unit():
    d = os.path.join(HERE, "golden")
    vec = open(os.path.join(d, "ref_wasm_example.divans"), "rb").read()
    want = json.load(open(os.path.join(d, "ref_wasm_example.json")))["plain_text"].encode("ascii")
    return [R.Case(vec, want, 0, 0, len(want) + 64)] * 2


def _blend_unit(oracle_blend):
    return [R.Case(oracle_blend.encode_raw(r, oracle_blend.options(dynamic_context_mixing=m)), r, 0, 0, len(r) + 64)
            for r, m in zip(raws(2, 2500, 60), (0, 2))]


# ---- decoding to command lists ----
def _cmds_unit(oracle, golden):
    tr = [e for e in golden if e["name"] == "truncated_dictionary"][0]
    trs = open(tr["path"], "rb").read()
    several = R.from_ir(oracle, [R.pm_line("lsb6", mix=4), R.insert(text(1500, 70)), R.pm_line("msb6", mix=5),
                                 R.insert(text(1200, 71)), R.pm_line("utf8", mix=8), R.insert(text(900, 72))])
    lsb = R.build("lsb6", oracle, 2)
    return [R.Case(trs, None, 0, 0, tr["raw_len"] + 64), R.Case(several, None, 0, 0, 1500 + 1200 + 900 + 64),
            R.build("bt256", oracle, 1), lsb]


def _cmds_expect(oracle):
    def f(unit):
        out = []
        for c in unit:
            rc, raw, cl = oracle.decode_cmds(c.stream, out_cap=c.cap)
            out.append((rc, raw, cl.serialize()) if rc == 0 else (rc, None, None))
        return out
    return f


def _run_dec_cmds_host(kind, eng, rep, stream):
    cases = _rep(kind.unit, rep)
    return [(s, r, b) if s == 0 else (s, None, None) for s, r, b in eng.decode_cmds([c.stream for c in cases], [c.cap for c in cases])]


def _run_dec_cmds_dev(kind, eng, rep, stream):
    import divans_b200
    d = kind.dev_inputs(rep)
    caps = np.array([c.cap for c in _rep(kind.unit, rep)], np.uint64)
    bcap = divans_b200.first_blob_cap(caps) + np.uint64(4 * divans_b200.PM_RECORD_BYTES)   # room for every record of the unit
    (off, total), (boff, btotal) = divans_b200._regions(caps), divans_b200._regions(bcap)
    if "meta" not in d:
        d["meta"] = _u64(np.concatenate([off, caps, boff, bcap]), "cuda:0")
    n, M = d["n"], d["meta"]
    with _On(stream) as s:
        out, blobs, res = _zeros(total), _zeros(btotal), _zeros(3 * n, _i64())
        eng.decode_cmds_batch_device(d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), out.data_ptr(), M.data_ptr(),
                                     M[n:].data_ptr(), res.data_ptr(), blobs.data_ptr(), M[2 * n:].data_ptr(), M[3 * n:].data_ptr(),
                                     res[n:].data_ptr(), res[2 * n:].data_ptr(), n, d["total"], 0, s)

    def read():
        r = res.cpu().numpy()
        ln, bl, st = r[:n].view(np.uint64), r[n:2 * n].view(np.uint64), r[2 * n:].view(np.int32)[:n]
        h, hb = out.cpu().numpy(), blobs.cpu().numpy()
        return [(int(x), h[int(o):int(o + a)].tobytes(), hb[int(bo):int(bo + b)].tobytes()) if x == 0 else (int(x), None, None)
                for x, o, a, bo, b in zip(st, off, ln, boff, bl)]
    return read


def _decoded_twice(n):
    """gens of a host call through Engine.decode_cmds: n streams, and once more each one whose list outgrows first_blob_cap"""
    def f(unit):
        import divans_b200
        from oracle import oracle_py as O
        return n + sum(len(O.decode_cmds(c.stream, out_cap=c.cap)[2].serialize()) > int(divans_b200.first_blob_cap(c.cap)) for c in unit)
    return f


def _transcode_expect(oracle, T, cands):
    def f(unit):
        out = []
        for c in unit:
            rc, _, cl = oracle.decode_cmds(c.stream, out_cap=c.cap)
            assert rc == 0
            erc, s, ch, cost = T.encode_cmds_auto(cl, cands, window_size=cl.window)
            out.append((erc, s, ch, tuple(int(x) for x in cost)))
        return out
    return f


def _run_transcode(cands):
    def f(kind, eng, rep, stream):
        cases = _rep(kind.unit, rep)
        res, chosen, cost = eng.transcode([c.stream for c in cases], [c.cap for c in cases], None, 0, cands)
        return [(0, s, int(ch), tuple(int(x) for x in co)) for s, ch, co in zip(res, chosen, cost)]
    return f


# ---------------------------------------------------------------------------------------------------------------------
# encoders
# ---------------------------------------------------------------------------------------------------------------------
def _enc_expect(fn):
    return lambda unit: [fn(u) for u in unit]


def _run_enc_host(okw, cmds=False):
    def f(kind, eng, rep, stream):
        import divans_b200
        st, outs = eng._encode_lists(_rep(kind.unit_inputs(), rep), divans_b200.encode_options(**okw), cmds)
        return [(int(s), o) for s, o in zip(st, outs)]
    return f


def _run_enc_dev(okw, cmds=False, max_raw=0):
    def f(kind, eng, rep, stream):
        import divans_b200
        d = kind.dev_inputs(rep)
        cap = divans_b200._encoded_cap(d["host_len"])
        off, total = divans_b200._regions(cap)
        if "ecap" not in d:
            d["eoff"], d["ecap"] = _u64(off, "cuda:0"), _u64(cap, "cuda:0")
        n, o = d["n"], divans_b200.encode_options(**okw)
        with _On(stream) as s:
            out, res = _zeros(total), _zeros(2 * n, _i64())
            args = (d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr())
            tail = (out.data_ptr(), d["eoff"].data_ptr(), d["ecap"].data_ptr(), res.data_ptr(), res[n:].data_ptr())
            if cmds:
                eng.encode_cmds_batch_device(n, *args, d["max"], max_raw, *tail, o, s)
            else:
                eng.encode_batch_device(n, *args, d["max"], *tail, o, s)
        return lambda: _read_enc(out, res, off, n)
    return f


def _read_enc(out, res, off, n, extra=None):
    r, h = res.cpu().numpy(), out.cpu().numpy()
    ln, st = r[:n].view(np.uint64), r[n:2 * n].view(np.int32)[:n]
    return [(int(x), h[int(o):int(o + a)].tobytes() if x == 0 else None) for x, o, a in zip(st, off, ln)]


def _lists(oracle, names):
    return [R.command_list(nm, oracle).serialize() for nm in names]


def _list_expect(oracle, okw):
    def f(unit):
        out = []
        for b in unit:
            cl = __import__("oracle_tally.tally_py", fromlist=["x"]).from_blob(oracle, b)
            try:
                out.append((0, cl.encode(oracle.options(**okw))))
            except Exception:
                out.append((3, None))
        return out
    return f


# ---------------------------------------------------------------------------------------------------------------------
# cost selections
# ---------------------------------------------------------------------------------------------------------------------
def _run_auto_host(okw):
    def f(kind, eng, rep, stream):
        import divans_b200
        st, outs, ch, cost = eng._encode_lists(_rep(kind.unit_inputs(), rep), divans_b200.encode_options(**okw), False, eng._auto_host, None)
        return [(int(s), o, int(c), tuple(int(x) for x in co)) for s, o, c, co in zip(st, outs, ch, cost)]
    return f


def _run_auto_dev(okw):
    def f(kind, eng, rep, stream):
        import divans_b200
        d = kind.dev_inputs(rep)
        cap = divans_b200._encoded_cap(d["host_len"])
        off, total = divans_b200._regions(cap)
        if "ecap" not in d:
            d["eoff"], d["ecap"] = _u64(off, "cuda:0"), _u64(cap, "cuda:0")
        n, k = d["n"], len(divans_b200.DEFAULT_LITERAL_MODELS)
        with _On(stream) as s:
            out, res = _zeros(total), _zeros((3 + k) * n, _i64())
            eng.encode_auto_batch_device(n, d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), d["max"], out.data_ptr(),
                                         d["eoff"].data_ptr(), d["ecap"].data_ptr(), res.data_ptr(), res[n:].data_ptr(),
                                         res[2 * n:].data_ptr(), res[3 * n:].data_ptr(), divans_b200.encode_options(**okw), None, s)

        def read():
            base = _read_enc(out, res, off, n)
            r = res.cpu().numpy()
            ch, cost = r[2 * n:3 * n].view(np.uint32)[:n], r[3 * n:].view(np.uint64).reshape(n, k)
            return [(s_, o, int(c), tuple(int(x) for x in co)) for (s_, o), c, co in zip(base, ch, cost)]
        return read
    return f


def _auto_expect(T, okw):
    import divans_b200
    def f(unit):
        out = []
        for r in unit:
            rc, s, ch, cost = T.encode_auto(r, divans_b200.DEFAULT_LITERAL_MODELS, **okw)
            out.append((rc, s, ch, tuple(int(x) for x in cost)))
        return out
    return f


def _run_mixmap_host(okw):
    def f(kind, eng, rep, stream):
        import divans_b200
        st, outs, ch, mix, cost, _ = eng._encode_lists(_rep(kind.unit_inputs(), rep), divans_b200.encode_options(**okw), False,
                                                       eng._mixmap_host, None, False)
        return [(int(s), o, int(c), m.tobytes(), tuple(int(x) for x in co)) for s, o, c, m, co in zip(st, outs, ch, mix, cost)]
    return f


def _run_mixmap_dev(okw):
    def f(kind, eng, rep, stream):
        import divans_b200
        import torch
        d = kind.dev_inputs(rep)
        cap = divans_b200._encoded_cap(d["host_len"])
        off, total = divans_b200._regions(cap)
        if "ecap" not in d:
            d["eoff"], d["ecap"] = _u64(off, "cuda:0"), _u64(cap, "cuda:0")
        n, k, E = d["n"], len(divans_b200.DEFAULT_MIXING_VALUES), divans_b200.MIX_ENTRIES
        with _On(stream) as s:
            out, res = _zeros(total), _zeros((3 + k + 1) * n, _i64())
            mixing, bins = _zeros(n * E), _zeros(n * k * E, torch.int64)
            eng.encode_mixmap_batch_device(n, d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), d["max"], out.data_ptr(),
                                           d["eoff"].data_ptr(), d["ecap"].data_ptr(), res.data_ptr(), res[n:].data_ptr(),
                                           res[2 * n:].data_ptr(), mixing.data_ptr(), res[3 * n:].data_ptr(), bins.data_ptr(),
                                           divans_b200.encode_options(**okw), None, s)

        def read():
            base = _read_enc(out, res, off, n)
            r = res.cpu().numpy()
            ch, cost = r[2 * n:3 * n].view(np.uint32)[:n], r[3 * n:].view(np.uint64).reshape(n, k + 1)
            mx, bn = mixing.cpu().numpy().reshape(n, E), bins.cpu().numpy().view(np.uint64).reshape(n, k, E)
            return [(s_, o, int(c), m.tobytes(), tuple(int(x) for x in co), int(b.sum(dtype=np.uint64)))
                    for (s_, o), c, m, co, b in zip(base, ch, mx, cost, bn)]
        return read
    return f


def _mixmap_expect(T, okw, bins=False):
    import divans_b200
    def f(unit):
        out = []
        for r in unit:
            rc, s, ch, mixing, cost, b = T.encode_mixmap(r, 0, divans_b200.DEFAULT_MIXING_VALUES, **okw)
            e = (rc, s, ch, np.asarray(mixing, np.uint8).tobytes(), tuple(int(x) for x in cost))
            out.append(e + (int(np.asarray(b, np.uint64).sum(dtype=np.uint64)),) if bins else e)
        return out
    return f


def _run_speeds_host(kind, eng, rep, stream):
    import divans_b200
    st, outs, ch, cost, halves = eng._encode_lists(_rep(kind.unit_inputs(), rep), divans_b200.encode_options(), False, eng._speeds_host, None)
    return [(int(s), o, tuple(int(x) for x in c), tuple(int(x) for x in co), tuple(int(x) for x in h.reshape(-1)))
            for s, o, c, co, h in zip(st, outs, ch, cost, halves)]


def _run_speeds_dev(kind, eng, rep, stream):
    import divans_b200
    d = kind.dev_inputs(rep)
    cap = divans_b200._encoded_cap(d["host_len"])
    off, total = divans_b200._regions(cap)
    if "ecap" not in d:
        d["eoff"], d["ecap"] = _u64(off, "cuda:0"), _u64(cap, "cuda:0")
    n, k = d["n"], len(divans_b200.DEFAULT_LITERAL_SPEEDS)
    with _On(stream) as s:
        out, res = _zeros(total), _zeros(2 * n + 2 * n + (k + 1) * n + 2 * k * n, _i64())
        at = lambda i: res[i:].data_ptr()
        eng.encode_speeds_batch_device(n, d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), d["max"], out.data_ptr(),
                                       d["eoff"].data_ptr(), d["ecap"].data_ptr(), at(0), at(n), at(2 * n), at(4 * n),
                                       at((5 + k) * n), None, None, s)

    def read():
        base = _read_enc(out, res, off, n)
        r = res.cpu().numpy()
        ch = r[2 * n:4 * n].view(np.uint32)[:3 * n].reshape(n, 3)
        cost = r[4 * n:(5 + k) * n].view(np.uint64).reshape(n, k + 1)
        hv = r[(5 + k) * n:].view(np.uint64).reshape(n, 2 * k)
        return [(s_, o, tuple(int(x) for x in c), tuple(int(x) for x in co), tuple(int(x) for x in h))
                for (s_, o), c, co, h in zip(base, ch, cost, hv)]
    return read


def _speeds_expect(T):
    import divans_b200
    def f(unit):
        out = []
        for r in unit:
            rc, s, ch, cost, halves = T.encode_speeds(r, 0, 4, divans_b200.DEFAULT_LITERAL_SPEEDS)
            out.append((rc, s, tuple(int(x) for x in ch), tuple(int(x) for x in cost), tuple(int(x) for x in np.asarray(halves).reshape(-1))))
        return out
    return f


# ---- choosing among command lists ----
def _choose_unit(oracle, T):
    import divans_b200
    out = []
    for i in range(4):
        r = text(2200 + 500 * i, 80 + i)
        ls = [T.lz77_parse(oracle, r, mm, lz).serialize() for mm, lz in divans_b200.DEFAULT_LZ77_PARSES]
        if i == 1:
            ls[0] = B.refused_blob(oracle)          # one list that every encoder refuses: another parse is chosen
        if i == 3:
            ls = [B.refused_blob(oracle)] * len(ls)   # every list refused: the stream fails
        out.append((ls, len(r)))
    return out


def _choose_expect(oracle, T, with_out):
    def f(unit):
        out = []
        for ls, _ in unit:
            rc, s, ch, cost = T.encode_cmds_choose([T.from_blob(oracle, b) for b in ls], window_size=16)
            c = tuple(int(x) for x in cost)
            out.append((rc, s, ch, c) if with_out else (ch, c))
        return out
    return f


def _run_choose(with_out):
    def f(kind, eng, rep, stream):
        import divans_b200
        unit = _rep(kind.unit, rep)
        n, k = len(unit), len(unit[0][0])
        key = ("choose", rep)
        if key not in kind._dev:
            blobs = [unit[i][0][c] for c in range(k) for i in range(n)]   # candidate-major
            blob, off, ln = divans_b200._pack(blobs)
            import torch
            kind._dev[key] = dict(blob=torch.from_numpy(blob).to("cuda:0"), off=_u64(off, "cuda:0"), len=_u64(ln, "cuda:0"),
                                  max=int(ln.max()), raw=max(r for _, r in unit))
        d = kind._dev[key]
        cap = divans_b200._encoded_cap(np.full(n, d["max"], np.uint64))
        off, total = divans_b200._regions(cap)
        if "meta" not in d:
            d["meta"] = _u64(np.concatenate([off, cap]), "cuda:0")
        meta, o = d["meta"], divans_b200.encode_options(window_size=16)
        with _On(stream) as s:
            out, res = _zeros(total), _zeros((3 + k) * n, _i64())
            outs = (out.data_ptr(), meta.data_ptr(), meta[n:].data_ptr(), res.data_ptr(), res[n:].data_ptr()) if with_out else (None,) * 5
            eng.encode_cmds_choose_batch_device(n, k, d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), d["max"], d["raw"],
                                                *outs, res[2 * n:].data_ptr(), res[3 * n:].data_ptr(), o, s)

        def read():
            r = res.cpu().numpy()
            ch, cost = r[2 * n:3 * n].view(np.uint32)[:n], r[3 * n:].view(np.uint64).reshape(n, k)
            sel = [(int(c), tuple(int(x) for x in co)) for c, co in zip(ch, cost)]
            if not with_out:
                return sel
            return [(s_, o_) + x for (s_, o_), x in zip(_read_enc(out, res, off, n), sel)]
        return read
    return f


# ---- billing ----
def _bill_norm(bill, status):
    return [(int(s), np.asarray(b, np.uint64).tobytes()) for b, s in zip(bill, status)]


def _run_bill_host(okw):
    def f(kind, eng, rep, stream):
        import divans_b200
        return _bill_norm(*eng.bill(_rep(kind.unit_inputs(), rep), divans_b200.encode_options(**okw)))
    return f


def _bill_expect(T, okw, cmds=False, oracle=None):
    def f(unit):
        out = []
        for u in unit:
            rc, _, rows = T.bill_cmds(T.from_blob(oracle, u[0]), **okw) if cmds else T.bill_raw(u, 0, 4, **okw)
            out.append((rc, np.asarray(rows, np.uint64).tobytes()))
        return out
    return f


def _run_bill_cmds_dev(okw):
    def f(kind, eng, rep, stream):
        import divans_b200
        import torch
        d = kind.dev_inputs(rep)
        n, S = d["n"], len(divans_b200.BILL_STATES)
        with _On(stream) as s:
            bill, st = _zeros(n * S * 2, torch.int64), _zeros(n, torch.int32)
            eng.bill_device(n, d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), d["max"], bill.data_ptr(), st.data_ptr(),
                            divans_b200.encode_options(**okw), True, max(r for _, r in kind.unit), s)
        return lambda: _bill_norm(bill.cpu().numpy().view(np.uint64).reshape(n, S, 2), st.cpu().numpy()[:n])
    return f


# ---- LZ77 generation and replay ----
def _lz77_expect(window, parse):
    """the library's host generator (divans_b200.lz77_cmds_batch), which tests/test_lz77_*_oracle.py compare with the oracle"""
    def f(unit):
        import divans_b200
        bl, bo, bn = divans_b200.lz77_cmds_batch(*divans_b200._pack(unit), window=window, parse=parse)
        return [(0, bl[int(o):int(o + n)].tobytes()) for o, n in zip(bo, bn)]
    return f


def _run_lz77_dev(window, parse):
    def f(kind, eng, rep, stream):
        import divans_b200
        d = kind.dev_inputs(rep)
        cap = divans_b200.lz77_blob_cap(d["host_len"])
        off, total = divans_b200._regions(cap)
        if "bcap" not in d:
            d["boff"], d["bcap"] = _u64(off, "cuda:0"), _u64(cap, "cuda:0")
        n = d["n"]
        with _On(stream) as s:
            blobs, res = _zeros(total), _zeros(2 * n, _i64())
            eng.lz77_cmds_batch_device(n, d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), d["max"], window, 2, 4,
                                       blobs.data_ptr(), d["boff"].data_ptr(), d["bcap"].data_ptr(), res.data_ptr(), res[n:].data_ptr(),
                                       s, parse=parse)

        def read():
            r, h = res.cpu().numpy(), blobs.cpu().numpy()
            ln, st = r[:n].view(np.uint64), r[n:].view(np.int32)[:n]
            return [(int(x), h[int(o):int(o + a)].tobytes()) for x, o, a in zip(st, off, ln)]
        return read
    return f


def _replay_unit(oracle):
    out = []
    import divans_b200
    rs = raws(4, 1800, 90)
    bl, bo, bn = divans_b200.lz77_cmds_batch(*divans_b200._pack(rs), window=16)
    for r, o, n in zip(rs, bo, bn):
        out.append((bl[int(o):int(o + n)].tobytes(), r))
    bad = bytearray(out[0][0])
    bad[0] ^= 1                       # bad magic: the list is refused
    out.insert(2, (bytes(bad), None))
    return out


def _replay_expect(unit):
    return [(0, r) if r is not None else (3, None) for _, r in unit]


def _run_replay_host(kind, eng, rep, stream):
    return [(s, o) if s == 0 else (s, None) for s, o in eng.replay(_rep(kind.unit_inputs(), rep))]


def _run_replay_dev(kind, eng, rep, stream):
    import divans_b200
    d = kind.dev_inputs(rep)
    unit = _rep(kind.unit, rep)
    cap = np.array([len(r) if r is not None else 64 for _, r in unit], np.uint64)
    off, total = divans_b200._regions(cap)
    if "rcap" not in d:
        d["roff"], d["rcap"] = _u64(off, "cuda:0"), _u64(cap, "cuda:0")
    n = d["n"]
    with _On(stream) as s:
        out, res = _zeros(total), _zeros(2 * n, _i64())
        eng.replay_cmds_batch_device(n, d["blob"].data_ptr(), d["off"].data_ptr(), d["len"].data_ptr(), out.data_ptr(), d["roff"].data_ptr(),
                                     d["rcap"].data_ptr(), res.data_ptr(), res[n:].data_ptr(), 0, s)

    def read():
        r, h = res.cpu().numpy(), out.cpu().numpy()
        ln, st = r[:n].view(np.uint64), r[n:].view(np.int32)[:n]
        return [(int(x), h[int(o):int(o + a)].tobytes() if x == 0 else None) for x, o, a in zip(st, off, ln)]
    return read


# ---------------------------------------------------------------------------------------------------------------------
# the catalogue
# ---------------------------------------------------------------------------------------------------------------------
def catalogue(oracle, oracle_blend, golden):
    """{name: Kind}, in a fixed order"""
    import divans_b200
    from oracle_tally import tally_py as T
    F = divans_b200
    SK = R.SKIP_CRC
    f8 = irfuzz.random_f8_speeds(oracle, 4)   # three of the four outside speed_is_small
    keep_cands = [F.LITERAL_MODEL_KEEP] + F.DEFAULT_LITERAL_MODELS
    enc_raws = lambda: raws(4, 2500, 20)
    list_unit = lambda: _lists(oracle, LIST_UNIT) + [B.refused_blob(oracle)]
    pairs = lambda: [(b, r) for b, r in ((T.lz77_parse(oracle, text(2000 + 400 * i, 100 + i), 6, 1).serialize(), 2000 + 400 * i)
                                         for i in range(4))]
    ks = [
        Kind("dec", lambda: _dec_unit(oracle), _dec_expect(oracle, SK), _run_dec_host(SK), [("v2", len(DEC_UNIT), 0, RAW_HDR)], gens=len(DEC_UNIT)),
        Kind("dec_dev", lambda: _dec_unit(oracle), _dec_expect(oracle, SK), _run_dec_dev(SK), [("v2", len(DEC_UNIT), 0, RAW_HDR)], True,
             gens=len(DEC_UNIT)),
        Kind("dec_wasm", _wasm_unit, lambda u: [(0, c.raw) for c in u], _run_dec_host(F.FLAG_MODEL_WASM_2018), [("v2", 2, 0, None)], gens=2),
        Kind("dec_blend", lambda: _blend_unit(oracle_blend), lambda u: [(0, c.raw) for c in u], _run_dec_host(F.FLAG_CDF_BLEND),
             [("blend", 2, 1, RAW_HDR)]),
        Kind("dec_cmds", lambda: _cmds_unit(oracle, golden), _cmds_expect(oracle), _run_dec_cmds_host, [("rec", 4, 0, RAW_HDR)],
             gens=_decoded_twice(4)),
        Kind("dec_cmds_dev", lambda: _cmds_unit(oracle, golden), _cmds_expect(oracle), _run_dec_cmds_dev, [("rec", 4, 0, RAW_HDR)], True,
             gens=4),
        Kind("transcode", lambda: _cmds_unit(oracle, golden)[1:], _transcode_expect(oracle, T, keep_cands), _run_transcode(keep_cands),
             [("rec", 3, 0, RAW_HDR), ("enc", 3 * (1 + len(keep_cands)), "keep", None)], gens=_decoded_twice(3)),
        Kind("enc_raw", enc_raws, _enc_expect(lambda r: (0, oracle.encode_raw(r))), _run_enc_host({}), [("enc", 4, "keep", RAW_HDR)]),
        Kind("enc_raw_dev", enc_raws, _enc_expect(lambda r: (0, oracle.encode_raw(r))), _run_enc_dev({}), [("enc", 4, "keep", RAW_HDR)], True),
        Kind("enc_wide", enc_raws, _enc_expect(lambda r: (0, oracle.encode_raw(r, oracle.options(**WIDE_OPTS)))), _run_enc_host(WIDE_OPTS),
             [("enc", 4, 1, RAW_HDR)]),
        Kind("enc_f8", enc_raws, _enc_expect(lambda r: (0, oracle.encode_raw(r, oracle.options(literal_adaptation=f8)))),
             _run_enc_host(dict(literal_adaptation=f8)), [("enc", 4, None, RAW_HDR)]),
        Kind("enc_dcm2", enc_raws, _enc_expect(lambda r: (0, oracle.encode_raw(r, oracle.options(dynamic_context_mixing=2)))),
             _run_enc_host(dict(dynamic_context_mixing=2)), [("enc", 4, "keep", RAW_HDR)]),
        Kind("enc_blend", enc_raws, _enc_expect(lambda r: (0, oracle_blend.encode_raw(r, oracle_blend.options()))),
             _run_enc_host(dict(cdf_model=F.CDF_BLEND)), [("enc", 4, 1, RAW_HDR)]),
        Kind("enc_cmds", list_unit, _list_expect(oracle, dict(window_size=16)), _run_enc_host(dict(window_size=16), True),
             [("enc", 5, "keep", None)]),
        Kind("enc_cmds_dev", list_unit, _list_expect(oracle, dict(window_size=16)),
             _run_enc_dev(dict(window_size=16), True, max_raw=1 << 16), [("enc", 5, "keep", None)], True),
        Kind("enc_nopm", lambda: [R.command_list("no_predmode", oracle, v).serialize() for v in (0, 1)],
             _list_expect(oracle, dict(window_size=16)), _run_enc_host(dict(window_size=16), True), [("enc", 2, "keep", NOPM_HDR)]),
        Kind("auto", enc_raws, _auto_expect(T, WIDE_OPTS), _run_auto_host(WIDE_OPTS), [("enc", 4 * 9, 1, RAW_HDR)]),
        Kind("auto_dev", enc_raws, _auto_expect(T, {}), _run_auto_dev({}), [("enc", 4 * 9, "keep", RAW_HDR)], True),
        Kind("mixmap", enc_raws, _mixmap_expect(T, WIDE_OPTS), _run_mixmap_host(WIDE_OPTS), [("enc", 4 * 8, 1, None)]),
        Kind("mixmap_dev", enc_raws, _mixmap_expect(T, {}, bins=True), _run_mixmap_dev({}), [("enc", 4 * 8, "keep", None)], True),
        Kind("speeds", enc_raws, _speeds_expect(T), _run_speeds_host, [("enc", 4 * 8, "keep", RAW_HDR)]),
        Kind("speeds_dev", enc_raws, _speeds_expect(T), _run_speeds_dev, [("enc", 4 * 8, "keep", RAW_HDR)], True),
        Kind("choose_dev", lambda: _choose_unit(oracle, T), _choose_expect(oracle, T, True), _run_choose(True), [("enc", 4 * 5, "keep", None)],
             True),
        Kind("choose_pick_dev", lambda: _choose_unit(oracle, T), _choose_expect(oracle, T, False), _run_choose(False),
             [("enc", 4 * 4, "keep", None)], True),
        Kind("bill", enc_raws, _bill_expect(T, WIDE_OPTS), _run_bill_host(WIDE_OPTS), [("enc", 4, 1, RAW_HDR)]),
        Kind("bill_cmds_dev", pairs, _bill_expect(T, dict(window_size=16), True, oracle), _run_bill_cmds_dev(dict(window_size=16)),
             [("enc", 4, "keep", RAW_HDR)], True),
        Kind("lz77_dev", lambda: raws(4, 2000, 110), _lz77_expect(10, None), _run_lz77_dev(10, None), device=True),
        Kind("lz77_dict_dev", lambda: [R.text()[i * 4000:i * 4000 + 3000] for i in range(4)], _lz77_expect(24, (7, 2, 4)),
             _run_lz77_dev(24, (7, 2, 4)), device=True),
        Kind("lz77_words_dev", lambda: [R.text()[20000 + i * 4000:20000 + i * 4000 + 3000] for i in range(4)],
             _lz77_expect(16, (10, 2, 4, 1)), _run_lz77_dev(16, (10, 2, 4, 1)), device=True),
        Kind("replay", lambda: _replay_unit(oracle), _replay_expect, _run_replay_host),
        Kind("replay_dev", lambda: _replay_unit(oracle), _replay_expect, _run_replay_dev, device=True),
    ]
    return {k.name: k for k in ks}


# ---------------------------------------------------------------------------------------------------------------------
# the header model
# ---------------------------------------------------------------------------------------------------------------------
ENCODE_GROUPS_PER_BLOCK = 4   # dv_capi.cu: the encoder's model pass and the blend decoder run whole blocks of four 16-lane groups


def slots_used(engine_kind, max_resident, lanes, n):
    """the arena slots a launch set of n streams (or pairs) uses on an engine of ``max_resident`` slots, one warp per block
    (``lanes`` 16: two slots per warp, 8: four), as dv_capi.cu sizes it"""
    if engine_kind in ("v2", "rec"):
        gpb = 4 if (lanes == 8 and engine_kind == "v2") else 2   # lanes 0 (by batch size): 16 on an H100
        cap = max(max_resident, gpb)
        return -(-min(n, cap) // gpb) * gpb
    g = ENCODE_GROUPS_PER_BLOCK
    cap = max(max_resident, g) if engine_kind == "blend" else max_resident
    return -(-min(n, cap) // g) * g


def check_headers(kind, rep, before, after, max_resident, lanes, what=""):
    """Compare every slot's header after one call of ``kind`` (rep copies of its unit) with the model.  ``before`` and
    ``after``: the headers of every slot of the arena before and after the call.  A phase that needs more slots than the arena
    holds makes ensure_arena reallocate it: every word of every slot starts again at zero, also what earlier phases of the
    same call wrote (transcode on a two-slot arena: the recording decoder, then the encoder's four slots)."""
    arena = len(before)
    if arena < len(after):
        before = before + [[0, 0, 0, 0]] * (len(after) - arena)
    assert len(after) == len(before), (what, len(before), len(after))
    g0 = sum(h[0] for h in before)           # the model's sum of word 0 over the slots
    w0 = [b[0] for b in before]              # per slot: the least word 0
    w1 = [("eq", b[1]) for b in before]      # per slot: ("eq", v) or ("ge", v)
    w23 = [{tuple(b[2:])} for b in before]   # per slot: the allowed (word 2, word 3), None = any
    for eng_kind, n_unit, p1, p23 in kind.phases:
        used = slots_used(eng_kind, max_resident, lanes, n_unit * rep)
        assert used <= len(after), (what, eng_kind, used, len(after))
        if used > arena:                     # ensure_arena reallocates here: every word of every slot starts again at 0
            arena, g0 = used, 0
            w0, w1, w23 = [0] * len(after), [("eq", 0)] * len(after), [{(0, 0)}] * len(after)
        if eng_kind in ("v2", "rec"):
            g0 += kind.gens * rep
        for i in range(used):
            if p1 in (0, 1):
                w1[i] = ("eq", p1)
            elif p1 is None:
                w1[i] = ("ge", w1[i][1])
            w23[i] = None if p23 is None else set(p23)
    assert sum(h[0] for h in after) == g0, "%s: word 0 sums to %d, the model says %d (before %s)" % (
        what, sum(h[0] for h in after), g0, [b[0] for b in before])
    v2 = any(p[0] in ("v2", "rec") for p in kind.phases)
    for i, (h, b) in enumerate(zip(after, w0)):
        assert h[0] >= b if v2 else h[0] == b, "%s: slot %d: word 0 %d -> %d" % (what, i, b, h[0])
        op, v = w1[i]
        assert (h[1] == v) if op == "eq" else (v <= h[1] <= 1), "%s: slot %d: word 1 is %d, the model says %s %d (before %s)" % (
            what, i, h[1], op, v, b)
        assert w23[i] is None or tuple(h[2:]) in w23[i], "%s: slot %d: words 2, 3 are %s, the model allows %s (before %s)" % (
            what, i, h[2:], w23[i], b)
