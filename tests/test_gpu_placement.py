"""GPU tests (-m gpu) of WHERE the batch calls write: every decode and encode entry point with its regions at every byte
alignment, packed edge to edge, one byte short, and past 2^32 (tests/placement.py), each stream against the CPU oracle.

Every region of a call lives in one allocation filled with CANARY.  Per stream the status, the length and the bytes are the
oracle's; past the length a region holds what the header promises for that call (host decode calls: zeros; every other call:
the canary, nothing is written there); every byte outside every region is still the canary, and every input is unchanged.  The
decode tests assert the lane layout each call ran on."""
import numpy as np
import pytest

import divans_b200
import placement as P
import regimes as R
import test_gpu_encode_auto as A
import test_gpu_lz77_device as LZ
import test_gpu_replay as RP
from oracle_tally import tally_py as T

pytestmark = pytest.mark.gpu

CANARY = P.CANARY
SKIP = divans_b200.FLAG_SKIP_CRC
BLEND = divans_b200.FLAG_CDF_BLEND
DEVICE_LAYOUTS = P.LAYOUTS + ["high"]


# The contexts of this file are its own, 64 slots each, and closed when the file is done (as in test_gpu_mixing_values.py).
@pytest.fixture(scope="module")
def ctx():
    import torch
    e = {"16": divans_b200.Engine(0, 64, 16), "8": divans_b200.Engine(0, 64, 8), "auto": divans_b200.Engine(0, 64, 0)}
    yield e
    for x in e.values():
        x.close()
    _HIGH.clear()
    torch.cuda.empty_cache()


_HIGH = []   # the one allocation of HIGH_BYTES the high layout's calls share (filled with the canary again by each call)


def _high_allocation():
    """HIGH_BYTES in HBM when the GPU has them free, else pinned host memory, which the kernels address the same way (unified
    addressing): in a whole session the session's contexts can hold all but a few hundred MiB of the GPU"""
    import torch
    if not _HIGH:
        try:
            _HIGH.append(torch.empty(P.HIGH_BYTES, dtype=torch.uint8, device="cuda"))
        except torch.OutOfMemoryError:
            _HIGH.append(torch.empty(P.HIGH_BYTES, dtype=torch.uint8, pin_memory=True))
    return _HIGH[0]


# ---------------------------------------------------------------------------------------------------------------------
# one allocation per call
# ---------------------------------------------------------------------------------------------------------------------
def _u64(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.uint64).reshape(-1)).view(np.int64)).cuda()


class _Dev:
    """the allocation of a device call: the plan's window on the GPU, CANARY but for the inputs.  The call's base pointers are
    the allocation plus `shift` = (inputs, outputs, blobs) bytes, and its offsets the plan's minus them: every region sits at the
    address the plan says, but no offset's residue is its address's (a kernel that took an alignment from an offset would err).
    Lists the device calls read as u32 need a multiple of 4 for the input shift."""

    def __init__(self, plan, inputs, shift=(1, 5, 6)):
        import torch
        self.plan = plan
        win = torch.from_numpy(P.host_buffer(plan, inputs))
        if plan.lo:
            self.t = _high_allocation()
            self.t.fill_(CANARY)
        else:
            self.t = torch.empty(plan.total, dtype=torch.uint8, device="cuda")
        self.t[plan.lo:plan.total].copy_(win)
        si, so, sb = shift
        self.pin, self.pout, self.pblob = (self.t.data_ptr() + s for s in shift)
        self.d = [_u64(a) for a in (plan.in_off - np.uint64(si), plan.in_len, plan.out_off - np.uint64(so), plan.out_cap,
                                    plan.blob_off - np.uint64(sb), plan.blob_cap)]
        n = len(plan.in_off)
        self.d_len = torch.full((n,), -1, dtype=torch.int64, device="cuda")
        self.d_len2 = torch.full((n,), -1, dtype=torch.int64, device="cuda")
        self.d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()

    def p(self, k):
        return self.d[k].data_ptr()

    def fetch(self):
        """(window as numpy, out_len, blob_len, status) once the call is done; checks the bytes below the window where they are"""
        import torch
        torch.cuda.synchronize()
        lo = self.plan.lo
        if lo:
            c64 = int(np.frombuffer(bytes([CANARY]) * 8, np.int64)[0])
            for a in range(0, lo - lo % 8, 1 << 30):
                part = self.t[a:min(a + (1 << 30), lo - lo % 8)].view(torch.int64)
                assert bool((part == c64).all()), "a byte below the high regions changed (an offset narrowed to 32 bits?)"
        return (self.t[lo:self.plan.total].cpu().numpy().copy(), self.d_len.cpu().numpy().view(np.uint64), self.d_len2.cpu().numpy().view(np.uint64),
                self.d_st.cpu().numpy())


def _outside(buf, plan, inputs):
    """every byte outside every region is the canary and every input is unchanged"""
    bad = np.flatnonzero((buf != CANARY) & ~P.region_mask(plan))
    assert bad.size == 0, "%s: %d bytes outside the regions changed, the first at offset %d" % (plan.layout, bad.size, bad[0] + plan.lo)
    for i, (o, x) in enumerate(zip(plan.in_off, inputs)):
        _same(_reg(buf, plan, o, len(x)), bytes(x), "%s: input %d" % (plan.layout, i))


def _reg(buf, plan, off, n):
    return buf[int(off) - plan.lo:int(off) - plan.lo + int(n)].tobytes()


def _tail(region, n, host, what):
    """past the length: zeros (host decode calls write the region whole) or the canary (nothing written)"""
    want = 0 if host else CANARY
    _same(region[n:], bytes([want]) * (len(region) - n), "%s: region past the length (want %s)" % (what, "zeros" if host else "the canary"))


def _same(got, want, what):
    """bytes equality, reported without pytest's diff of the two (which takes minutes on kilobytes)"""
    if got != want:
        n = min(len(got), len(want))
        d = np.flatnonzero(np.frombuffer(got[:n], np.uint8) != np.frombuffer(want[:n], np.uint8))
        raise AssertionError("%s: %d bytes, want %d, first difference at %d" % (what, len(got), len(want), d[0] if d.size else n))


# ---------------------------------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------------------------------
def _lz77_streams(oracle):
    """copies and (golden fixtures) dictionary words"""
    t = R.text()
    return [oracle.Commands.lz77(t[o:o + n], window=16).encode(oracle.options(window_size=16)) for o, n in ((3001, 9000), (77, 2500))]


@pytest.fixture(scope="module")
def dec(oracle, golden):
    """every decode stream: the GOOD and FAILING regimes (lit_quirk_w10 twice: literals within 8 bytes of position 0 and of a
    ring wrap at window 10), LZ77 streams and the golden fixtures of at most 64 KiB; with caps (the free layouts') and exact
    output lengths (the oracle's out_len with a region large enough)"""
    cases = [R.build(n, oracle) for n in R.GOOD + R.FAILING] + [R.build("lit_quirk_w10", oracle, 1)]
    streams = [c.stream for c in cases] + _lz77_streams(oracle)
    caps = [c.cap for c in cases] + [9064, 2564]
    for e in golden:
        if e["raw_len"] <= 1 << 16:
            streams.append(open(e["path"], "rb").read())
            caps.append(e["raw_len"] + 64)
    exact = [ln for _, ln, _ in _oracle_decode(oracle, streams, [max(c, 1 << 17) for c in caps])]
    return streams, caps, exact


def _oracle_decode(O, streams, caps, skip_crc=True):
    """[(status, out_len, bytes)] of the oracle's batch decode at its own placement"""
    blob = np.frombuffer(b"".join(streams), np.uint8)
    ln = np.array([len(s) for s in streams], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    cap = np.array(caps, np.uint64)
    ooff = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
    out, out_len, status = O.decode_batch(blob, off, ln, ooff, cap, skip_crc=skip_crc)
    return [(int(s), int(n), out[int(o):int(o) + min(int(n), int(c))].tobytes()) for s, n, o, c in zip(status, out_len, ooff, cap)]


def _check_out(region, st, ln, want, host, w):
    """one output region against the oracle's (status, out_len, bytes).  A stream that fails reports the oracle's status, and
    out_len the bytes it wrote into the region (the oracle counts differently there: the whole literal that ran dry is not
    counted, and a region too small by up to 16 bytes counts the bytes that did not fit), so its bytes are not compared"""
    ws, wn, wb = want
    if ws != 0:
        assert st == ws and ln <= len(region), "%s: (status, out_len) %s, oracle status %d" % (w, (st, ln), ws)
    else:
        assert (st, ln) == (0, wn), "%s: (status, out_len) %s, oracle %s" % (w, (st, ln), (ws, wn))
        _same(region[:ln], wb, "%s: bytes against the oracle's" % w)
    _tail(region, ln, host, w)


def _check_decode(O, streams, plan, buf, out_len, status, host, what):
    want = _oracle_decode(O, streams, plan.out_cap)
    for i, x in enumerate(want):
        region = _reg(buf, plan, plan.out_off[i], plan.out_cap[i])
        _check_out(region, int(status[i]), int(out_len[i]), x, host, "%s: %s stream %d" % (what, plan.layout, i))
    if plan.layout == "tight_minus_one":
        assert sum(s == 2 for s, _, _ in want) > len(want) // 2
    _outside(buf, plan, streams)


# ---------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------
def _decode_host(eng, plan, streams, flags, pending=False):
    buf = P.host_buffer(plan, streams)
    args = (buf, plan.in_off, plan.in_len, buf, plan.out_off, plan.out_cap, flags)
    if pending:
        return buf, eng.decode_batch_host_async(*args)
    return (buf,) + eng.decode_batch_host(*args)


def _decode_device(eng, plan, streams, flags):
    d = _Dev(plan, streams)
    eng.decode_batch_device(d.pin, d.p(0), d.p(1), d.pout, d.p(2), d.p(3), d.d_len.data_ptr(), d.d_st.data_ptr(), len(streams),
                            int(plan.in_len.sum()), flags)
    buf, ln, _, st = d.fetch()
    return buf, ln, st


LANES = {"host": ("16", 16), "dev16": ("16", 16), "dev8": ("8", 8), "dev_auto": ("auto", 16)}


@pytest.mark.parametrize("call", list(LANES))
@pytest.mark.parametrize("layout", DEVICE_LAYOUTS)
def test_decode(ctx, oracle, dec, layout, call):
    """decode_batch_host and decode_batch_device on the 16-lane, 8-lane and batch-size-chosen layouts (an 80 GB H100 with 64
    slots picks 16 lanes).  Flags SKIP_CRC: the corrupt regimes need it, and it changes no good stream's output."""
    if layout == "high" and call == "host":
        pytest.skip("the high layout is for device calls")
    streams, caps, exact = dec
    key, lanes = LANES[call]
    eng = ctx[key]
    plan = P.place(layout, [len(s) for s in streams], exact, caps)
    if call == "host":
        buf, ln, st = _decode_host(eng, plan, streams, SKIP)
    else:
        buf, ln, st = _decode_device(eng, plan, streams, SKIP)
    assert eng.last_lanes() == lanes
    _check_decode(oracle, streams, plan, buf, ln, st, call == "host", call)


@pytest.mark.parametrize("layout", P.LAYOUTS)
def test_decode_host_async(ctx, oracle, dec, layout):
    """two pipelined batches in flight, the second at the next layout of the list"""
    streams, caps, exact = dec
    other = P.LAYOUTS[(P.LAYOUTS.index(layout) + 1) % len(P.LAYOUTS)]
    plans = [P.place(x, [len(s) for s in streams], exact, caps) for x in (layout, other)]
    eng = ctx["16"]
    runs = [_decode_host(eng, p, streams, SKIP, pending=True) for p in plans]
    for p, (buf, h) in zip(plans, runs):
        ln, st = h.wait()
        _check_decode(oracle, streams, p, buf, ln, st, True, "async")
    assert eng.last_lanes() == 16


@pytest.fixture(scope="module")
def blend_streams(oracle_blend):
    t = R.text()
    raws = [t[5000 + 3000 * k:5000 + 3000 * k + n] for k, n in enumerate((1, 9, 700, 2500, 4097))]
    out = [T.encode_raw_model(r, k % 4, 4, True, window_size=16, dynamic_context_mixing=k % 3)[1] for k, r in enumerate(raws)]
    return out + [oracle_blend.Commands.lz77(t[:6000], window=16).encode(oracle_blend.options(window_size=16))], raws


@pytest.mark.parametrize("call", ["host", "dev16"])
@pytest.mark.parametrize("layout", DEVICE_LAYOUTS)
def test_decode_blend(ctx, oracle_blend, blend_streams, layout, call):
    """blend streams run on the generic per-nibble path, 16 lanes whatever the context's layout"""
    if layout == "high" and call == "host":
        pytest.skip("the high layout is for device calls")
    streams, raws = blend_streams
    exact = [len(r) for r in raws] + [6000]
    plan = P.place(layout, [len(s) for s in streams], exact)
    eng = ctx["8"]
    buf, ln, st = (_decode_host if call == "host" else _decode_device)(eng, plan, streams, BLEND)
    assert eng.last_lanes() == 16
    _check_decode(oracle_blend, streams, plan, buf, ln, st, call == "host", "blend " + call)


# ---------------------------------------------------------------------------------------------------------------------
# decode to command lists
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cmds_set(ctx, oracle, dec):
    """streams that decode (GOOD, LZ77, golden), their oracle blobs, and the blobs decode_cmds gives at aligned placement"""
    streams, caps, exact = dec
    keep = [i for i, s in enumerate(streams) if _oracle_decode(oracle, [s], [caps[i]])[0][0] == 0]
    streams, caps, exact = [streams[i] for i in keep], [caps[i] for i in keep], [exact[i] for i in keep]
    blobs = [oracle.decode_cmds(s, out_cap=c)[2].serialize() for s, c in zip(streams, caps)]
    aligned = ctx["16"].decode_cmds(streams, caps)
    assert [b for _, _, b in aligned] == blobs
    return streams, caps, exact, blobs


@pytest.mark.parametrize("call", ["host", "device"])
@pytest.mark.parametrize("layout", DEVICE_LAYOUTS)
def test_decode_cmds(ctx, oracle, cmds_set, layout, call):
    """output and blob regions at independent residues.  tight_minus_one: odd streams' output regions are one byte short (the
    plain decode's status 2, blob_len 0), even streams' blob regions (status 2, blob_len the exact size, no record left)"""
    if layout == "high" and call == "host":
        pytest.skip("the high layout is for device calls")
    streams, caps, exact, blobs = cmds_set
    eng = ctx["16"]
    plan = P.place(layout, [len(s) for s in streams], exact, caps, blob_exact=[len(b) for b in blobs],
                   blob_caps=[len(b) + P.SLACK[i % 5] for i, b in enumerate(blobs)])
    host = call == "host"
    if host:
        buf = P.host_buffer(plan, streams)
        ln, bl, st = eng.decode_cmds_batch_host(buf, plan.in_off, plan.in_len, buf, plan.out_off, plan.out_cap, buf, plan.blob_off,
                                                plan.blob_cap)
    else:
        d = _Dev(plan, streams)
        eng.decode_cmds_batch_device(d.pin, d.p(0), d.p(1), d.pout, d.p(2), d.p(3), d.d_len.data_ptr(), d.pblob, d.p(4), d.p(5),
                                     d.d_len2.data_ptr(), d.d_st.data_ptr(), len(streams), int(plan.in_len.sum()))
        buf, ln, bl, st = d.fetch()
    assert eng.last_lanes() == 16
    want = _oracle_decode(oracle, streams, plan.out_cap)
    for i, ((ws, wn, wb), blob) in enumerate(zip(want, blobs)):
        w = "%s %s stream %d" % (call, layout, i)
        out = _reg(buf, plan, plan.out_off[i], plan.out_cap[i])
        region = _reg(buf, plan, plan.blob_off[i], plan.blob_cap[i])
        short = ws == 0 and len(blob) > len(region)   # a good decode whose blob region is too small: status 2, decoded to its end
        _check_out(out, 0 if short else int(st[i]), int(ln[i]), (ws, wn, wb), host, w)
        if ws != 0:
            assert int(bl[i]) == 0, w
        elif len(blob) > len(region):
            assert (int(st[i]), int(ln[i]), int(bl[i])) == (2, wn, len(blob)), "%s: blob region too small" % w
        else:
            assert (int(st[i]), int(ln[i]), int(bl[i])) == (0, wn, len(blob)), w
            _same(region[:len(blob)], blob, "%s: blob" % w)
            if host:
                _tail(region, len(blob), True, w + " blob")
            else:   # the device call zeroes where the decoder staged the prediction-mode records, at the region's end
                assert set(region[len(blob):]) <= {0, CANARY}, "%s: bytes past blob_len are neither the canary nor zero" % w
            continue
        # a failed stream, or a blob region too small: the host call's region holds zeros; the device call leaves no record
        # (every byte zero or the canary)
        if host:
            _same(region, bytes(len(region)), "%s: blob region (want zeros)" % w)
        else:
            assert set(region) <= {0, CANARY}, "%s: a partial record was left in the blob region" % w
    if layout == "tight_minus_one":
        assert sum(int(s) == 2 and int(b) > 0 for s, b in zip(st, bl)) >= 5 and sum(int(s) == 2 and int(b) == 0 for s, b in zip(st, bl)) >= 5
    _outside(buf, plan, streams)


# ---------------------------------------------------------------------------------------------------------------------
# encode
# ---------------------------------------------------------------------------------------------------------------------
# (dynamic context mixing, blend model, literal context mode) of the encodes at each layout
OPTIONS = [(0, False, 0), (1, False, 2), (2, False, 3), (2, True, 1)]


def _enc_kw(dcm):
    return dict(window_size=16, dynamic_context_mixing=dcm)


def _check_encode(plan, buf, out_len, status, want, inputs, what):
    """want: the oracle's streams.  Every encoder writes only the stream: the canary survives past out_len, and a stream that
    does not fit (status 2, out_len the size it needs) writes nothing"""
    for i, w in enumerate(want):
        s = "%s %s stream %d" % (what, plan.layout, i)
        region = _reg(buf, plan, plan.out_off[i], plan.out_cap[i])
        if len(w) > int(plan.out_cap[i]):
            assert (int(status[i]), int(out_len[i])) == (2, len(w)), "%s: (status, out_len) %s, want (2, %d)" % (s, (int(status[i]), int(out_len[i])), len(w))
            _tail(region, 0, False, s)
            continue
        assert (int(status[i]), int(out_len[i])) == (0, len(w)), "%s: (status, out_len) %s, want (0, %d)" % (s, (int(status[i]), int(out_len[i])), len(w))
        _same(region[:len(w)], w, "%s: stream against the oracle's" % s)
        _tail(region, len(w), False, s)
    if plan.layout == "tight_minus_one":
        assert (np.asarray(status) == 2).all()
    _outside(buf, plan, inputs)


def _raw_device(eng, plan, raws, opts, fn="encode_batch_device", extra=None):
    d = _Dev(plan, raws)
    args = (len(raws), d.pin, d.p(0), d.p(1), max(1, int(plan.in_len.max())), d.pout, d.p(2), d.p(3), d.d_len.data_ptr(), d.d_st.data_ptr())
    if extra is None:
        getattr(eng, fn)(*args, opts)
    else:
        getattr(eng, fn)(*args, opts=opts, **extra)
    buf, ln, _, st = d.fetch()
    return buf, ln, st


@pytest.mark.parametrize("call", ["host", "device"])
@pytest.mark.parametrize("layout", DEVICE_LAYOUTS)
def test_encode_raw(ctx, layout, call):
    """encode_batch_host / _device: raw inputs at every input residue, outputs at every output residue; dynamic context mixing
    0, 1, 2 and the blend model"""
    if layout == "high" and call == "host":
        pytest.skip("the high layout is for device calls")
    raws = A._mixed()
    eng = ctx["16"]
    for dcm, blend, mode in OPTIONS:
        want = [T.encode_raw_model(r, mode, 4, blend, **_enc_kw(dcm))[1] for r in raws]
        plan = P.place(layout, [len(r) for r in raws], [len(w) for w in want])
        opts = divans_b200.encode_options(cdf_model=int(blend), literal_pred_mode=mode, **_enc_kw(dcm))
        if call == "host":
            buf = P.host_buffer(plan, raws)
            ln, st = eng.encode_batch_host(buf, plan.in_off, plan.in_len, buf, plan.out_off, plan.out_cap, opts)
        else:
            buf, ln, st = _raw_device(eng, plan, raws, opts)
        _check_encode(plan, buf, ln, st, want, raws, "%s dcm %d blend %d" % (call, dcm, blend))


@pytest.fixture(scope="module")
def lists(oracle):
    """command lists: every GOOD regime's but the two with wide speeds (which may wrap a prior at dynamic mixing 2, and test the
    decoder's tables), and LZ77 lists of text (copies); as oracle Commands and DVCL blobs"""
    lz = [oracle.Commands.lz77(R.text()[o:o + n], window=16) for o, n in ((3001, 9000), (77, 2500))]
    cls = [R.command_list(n, oracle) for n in R.GOOD if not n.startswith("wide")] + lz
    blobs = [c.serialize() for c in cls]
    # (the oracle's LZ77 lists leave the header's window 0: give them the window they were made for, so that replay takes it)
    blobs[-len(lz):] = [b[:20] + (16).to_bytes(4, "little") + b[24:] for b in blobs[-len(lz):]]
    return cls, blobs


BAD_BLOB = 1   # the device call's list at an offset that is not 4-byte aligned


@pytest.mark.parametrize("call", ["host", "device"])
@pytest.mark.parametrize("layout", DEVICE_LAYOUTS)
def test_encode_cmds(ctx, oracle, lists, layout, call):
    """encode_cmds_batch_host with blobs at any byte; encode_cmds_batch_device with blobs at residues 0, 4, 8, 12 mod 16,
    except list BAD_BLOB at residue 2: status 3, unread, while its warp-mates match the oracle"""
    if layout == "high" and call == "host":
        pytest.skip("the high layout is for device calls")
    cls, blobs = lists
    eng = ctx["16"]
    res = P.IN_RESIDUES if call == "host" else [0, 2] + [4, 8, 12, 0] * 8   # (BAD_BLOB alone at residue 2)
    max_raw = max(len(c.recode(16)[1]) for c in cls)
    for dcm, _, _ in OPTIONS[:3]:
        want = [c.encode(oracle.options(**_enc_kw(dcm))) for c in cls]
        plan = P.place(layout, [len(b) for b in blobs], [len(w) for w in want], in_residues=res)
        opts = divans_b200.encode_options(**_enc_kw(dcm))
        if call == "host":
            buf = P.host_buffer(plan, blobs)
            ln, st = eng.encode_batch_host(buf, plan.in_off, plan.in_len, buf, plan.out_off, plan.out_cap, opts, cmds=True)
        else:
            assert int(plan.in_off[BAD_BLOB]) % 4 == 2
            d = _Dev(plan, blobs, (4, 5, 0))
            eng.encode_cmds_batch_device(len(blobs), d.pin, d.p(0), d.p(1), max(len(b) for b in blobs), max_raw, d.pout, d.p(2), d.p(3),
                                         d.d_len.data_ptr(), d.d_st.data_ptr(), opts)
            buf, ln, _, st = d.fetch()
            assert (int(st[BAD_BLOB]), int(ln[BAD_BLOB])) == (3, 0), "the misaligned list was not refused"
            _tail(_reg(buf, plan, plan.out_off[BAD_BLOB], plan.out_cap[BAD_BLOB]), 0, False, "misaligned list")
            keep = [i for i in range(len(blobs)) if i != BAD_BLOB]
            sub = plan._replace(out_off=plan.out_off[keep], out_cap=plan.out_cap[keep])
            _check_encode(sub, buf, ln[keep], st[keep], [want[i] for i in keep], [], "%s dcm %d" % (call, dcm))
            _outside(buf, plan, blobs)
            continue
        _check_encode(plan, buf, ln, st, want, blobs, "%s dcm %d" % (call, dcm))


# ---------------------------------------------------------------------------------------------------------------------
# encode_auto, encode_mixmap, encode_speeds: their final encode shares the mux pass
# ---------------------------------------------------------------------------------------------------------------------
SEL_KW = dict(window_size=16, dynamic_context_mixing=2)


def _sel_want(kind, raws):
    """the oracle's (stream, chosen, cost) of each raw input under the default candidates"""
    out = []
    for r in raws:
        if kind == "auto":
            rc, s, ch, cost = T.encode_auto(r, divans_b200.DEFAULT_LITERAL_MODELS, **SEL_KW)
        elif kind == "mixmap":
            rc, s, ch, _, cost, _ = T.encode_mixmap(r, 0, divans_b200.DEFAULT_MIXING_VALUES, **SEL_KW)
        else:
            rc, s, ch, cost, _ = T.encode_speeds(r, 0, 4, divans_b200.DEFAULT_LITERAL_SPEEDS, **SEL_KW)
        assert rc == 0
        out.append((s, np.atleast_1d(np.asarray(ch, np.uint32)), np.asarray(cost, np.uint64)))
    return out


@pytest.mark.parametrize("call", ["host", "device"])
@pytest.mark.parametrize("layout", ["mixed", "adjacent"])
@pytest.mark.parametrize("kind", ["auto", "mixmap", "speeds"])
def test_selecting_encoders(ctx, kind, layout, call):
    """bytes, chosen and cost equal the oracle's, so the placement changes none of them"""
    import torch
    raws = A._mixed()
    n = len(raws)
    want = _sel_want(kind, raws)
    plan = P.place(layout, [len(r) for r in raws], [len(w[0]) for w in want])
    opts = divans_b200.encode_options(literal_pred_mode=0, **SEL_KW)
    k = {"auto": len(divans_b200.DEFAULT_LITERAL_MODELS), "mixmap": len(divans_b200.DEFAULT_MIXING_VALUES) + 1,
         "speeds": len(divans_b200.DEFAULT_LITERAL_SPEEDS) + 1}[kind]
    eng = ctx["16"]
    if call == "host":
        buf = P.host_buffer(plan, raws)
        fn = {"auto": eng.encode_auto_batch_host, "mixmap": eng.encode_mixmap_batch_host, "speeds": eng.encode_speeds_batch_host}[kind]
        r = fn(buf, plan.in_off, plan.in_len, buf, plan.out_off, plan.out_cap, opts)
        ln, st, chosen = r[0], r[1], r[2]
        cost = r[4] if kind == "mixmap" else r[3]
    else:
        d_ch = torch.zeros(3 * n, dtype=torch.int32, device="cuda")
        d_cost = torch.zeros(n * k, dtype=torch.int64, device="cuda")
        extra = dict(d_chosen=d_ch.data_ptr(), d_cost=d_cost.data_ptr())
        buf, ln, st = _raw_device(eng, plan, raws, opts, "encode_%s_batch_device" % kind, extra)
        chosen = d_ch.cpu().numpy().view(np.uint32)[:n * (3 if kind == "speeds" else 1)].reshape(n, -1)
        cost = d_cost.cpu().numpy().view(np.uint64).reshape(n, k)
    for i, (s, ch, c) in enumerate(want):
        assert (np.atleast_1d(chosen[i]) == ch).all() and (cost[i] == c).all(), "%s %s %s stream %d: chosen / cost differ" % (kind, call, layout, i)
    _check_encode(plan, buf, ln, st, [w[0] for w in want], raws, "%s %s" % (kind, call))


# ---------------------------------------------------------------------------------------------------------------------
# replay and the LZ77 generator: regions edge to edge, in reverse order, and past 2^32 (their misaligned inputs are tested in
# test_gpu_replay.py and test_gpu_lz77_device.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("call", ["host", "device"])
@pytest.mark.parametrize("layout", ["adjacent", "reversed", "high"])
def test_replay(ctx, lists, layout, call):
    if layout == "high" and call == "host":
        pytest.skip("the high layout is for device calls")
    _, blobs = lists
    want = RP._expect(T, blobs, [T.recode_blob(b)[1] for b in blobs])
    plan = P.place(layout, [len(b) for b in blobs], [n for _, n, _ in want], in_residues=[0, 4, 8, 12])
    eng = ctx["16"]
    if call == "host":
        buf = P.host_buffer(plan, blobs)
        ln, st = eng.replay_cmds_batch_host(buf, plan.in_off, plan.in_len, buf, plan.out_off, plan.out_cap)
    else:
        d = _Dev(plan, blobs, (4, 5, 0))
        eng.replay_cmds_batch_device(len(blobs), d.pin, d.p(0), d.p(1), d.pout, d.p(2), d.p(3), d.d_len.data_ptr(), d.d_st.data_ptr())
        buf, ln, _, st = d.fetch()
    got = [(int(s), int(n), _reg(buf, plan, o, c)) for s, n, o, c in zip(st, ln, plan.out_off, plan.out_cap)]
    RP._agree(got, want, "%s %s" % (call, layout), call == "host")
    _outside(buf, plan, blobs)


@pytest.mark.parametrize("layout", ["adjacent", "reversed", "high"])
def test_lz77_device(ctx, layout):
    """blob regions 4-byte aligned, as the generator requires: the contiguous layouts round each exact size up to 4"""
    raws = A._mixed()
    want = LZ._host(raws)
    plan = P.place(layout, [len(r) for r in raws], [0] * len(raws), [0] * len(raws), blob_exact=[len(w) for w in want], blob_align=4)
    assert (plan.blob_off % np.uint64(4) == 0).all()
    d = _Dev(plan, raws, (1, 5, 4))
    ctx["16"].lz77_cmds_batch_device(len(raws), d.pin, d.p(0), d.p(1), max(len(r) for r in raws), 16, 2, 4, d.pblob, d.p(4), d.p(5),
                                     d.d_len2.data_ptr(), d.d_st.data_ptr())
    buf, _, bl, st = d.fetch()
    for i, w in enumerate(want):
        region = _reg(buf, plan, plan.blob_off[i], plan.blob_cap[i])
        assert (int(st[i]), int(bl[i])) == (0, len(w)), "stream %d: (status, blob_len) %s" % (i, (int(st[i]), int(bl[i])))
        _same(region[:len(w)], w, "stream %d: blob against the host generator's" % i)
        _tail(region, len(w), False, "stream %d" % i)
    _outside(buf, plan, raws)
