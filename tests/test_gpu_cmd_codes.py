"""GPU tests (-m gpu) of the command coder against the CPU oracle, byte for byte and status for status: the command-code
catalogue (tests/cmd_codes.py) decoded on every lane layout, by the recording decoder and the blend decoder, and encoded by
every command-list encoder; the forged decoder-only streams; records no stream can carry, at their limits and fuzzed; one-warp
pairings and slot succession over the streams that reach the last CTYPE / DPRIOR slabs and the largest maps."""
import numpy as np
import pytest

import divans_b200
import cmd_codes as K
import dvcl as D
import test_gpu_encode_cmds_auto as C
import test_gpu_encode_mixmap as X
from oracle_tally import tally_py as T

pytestmark = pytest.mark.gpu

BLEND = divans_b200.FLAG_CDF_BLEND


# The contexts of this file are its own, with few slots, and closed when the file is done: a context's arena and scratch only
# grow and stay allocated until it closes (DESIGN.md), and batches larger than the slots reuse slots.
@pytest.fixture(scope="module")
def small():
    eng = divans_b200.Engine(0, 8, 16)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def small8():
    eng = divans_b200.Engine(0, 8, 8)
    yield eng
    eng.close()


def _window(blob):
    return int(np.frombuffer(blob[20:24], np.uint32)[0])


def _records(blob):
    h = np.frombuffer(bytes(blob[:32]), np.uint32)
    return np.frombuffer(bytes(blob[32:32 + 20 * int(h[2])]), np.uint32).reshape(-1, 5)


@pytest.fixture(scope="module")
def catalogue(oracle):
    """[(name, blob, stream, replay)]: each list, its oracle encoding and its replay"""
    out = []
    for name, blob in K.lists():
        rc, stream, _ = T.encode_forged(T.from_blob(oracle, blob), window_size=_window(blob))
        assert rc == 0
        rc_r, n, replay = T.recode_blob(blob)
        assert rc_r == 0
        out.append((name, blob, stream, replay))
    return out


@pytest.fixture(scope="module")
def forged(oracle):
    return K.forged(T, oracle)


def _stop_len(oracle, stream, cap):
    """the output length before the first command that does not fit in `cap` bytes: the oracle's decoded records, summed"""
    _, _, dec = oracle.decode_cmds(stream, out_cap=cap)
    n = 0
    for t, a, b, c, d in _records(dec.serialize()):
        k = int(b) if t in (D.COPY, D.LIT) else int(d) if t == D.DICT else 0
        if n + k > cap:
            break
        n += k
    return n


def _same(got, want, oracle, stream, cap):
    """(status, bytes) of a GPU decoder against the oracle's.  At status 2 the oracle also writes the part of the command that
    does not fit; the GPU stops before that command, so its out_len is the length of the commands before it"""
    if want[0] != 2:
        return got == want
    return got[0] == 2 and got[1] == want[1][:_stop_len(oracle, stream, cap)]


def _decode_all(eng, items, flags=0):
    """items: [(name, stream, status, output)] of status 0; one launch, then the same batch reversed"""
    for batch in (items, items[::-1]):
        res = eng.decode([s for _, s, _, _ in batch], [len(o) + (1 << 16) for _, _, _, o in batch], flags)
        for (name, _, st, want), (got_st, got) in zip(batch, res):
            assert (got_st, got) == (st, want), "%s: status %d (oracle %d), %s" % (name, got_st, st, "bytes differ" if got_st == st else "")


# ---------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes", ["16", "8", "auto"])
def test_decode_catalogue(catalogue, small, small8, lanes):
    eng = {"16": small, "8": small8}.get(lanes) or divans_b200.Engine(0, 8, 0)
    try:
        _decode_all(eng, [(n, s, 0, r) for n, _, s, r in catalogue])
    finally:
        if lanes == "auto":
            eng.close()


def test_recording_decoder(catalogue, oracle, small):
    """the recording decoder's blob of each stream holds the oracle's decoded list, and replays to the stream's bytes"""
    res = small.decode_cmds([s for _, _, s, _ in catalogue], [len(r) + 64 for _, _, _, r in catalogue])
    for (name, blob, stream, replay), (st, out, got) in zip(catalogue, res):
        assert st == 0 and out == replay, name
        rc, _, dec = oracle.decode_cmds(stream, out_cap=len(replay) + 64)
        assert rc == 0
        assert (_records(got) == _records(dec.serialize())).all(), name
        assert T.recode_blob(got)[2] == replay, name


def test_huge_count_status_2(oracle, small, small8):
    stream = open(K.HUGE_COUNT_STREAM, "rb").read()
    want = oracle.decode(stream, out_cap=1 << 16)
    assert want[0] == 2 and _stop_len(oracle, stream, 1 << 16) == 10
    for eng in (small, small8):
        assert _same(eng.decode([stream], [1 << 16])[0], want, oracle, stream, 1 << 16)


def test_gpu_replay(catalogue, small):
    """the replay kernel (replay_cmds_*) on every catalogue list equals the oracle's replay of the blob: status, exact length
    and bytes; the 2^31 - 1 copy at status 2 with its exact length and its first 64 KiB"""
    res = small.replay([b for _, b, _, _ in catalogue])
    for (name, blob, _, replay), (st, out) in zip(catalogue, res):
        assert (st, out) == (0, replay), name
    huge = K.huge_count()
    blob, off, ln = divans_b200._pack([huge])
    out = np.zeros(1 << 16, np.uint8)
    n, st = small.replay_cmds_batch_host(blob, off, ln, out, np.zeros(1, np.uint64), np.array([1 << 16], np.uint64))
    rc, want_n, want = T.recode_blob(huge, cap=1 << 16)
    assert (int(st[0]), int(n[0]), out.tobytes()) == (rc, want_n, want) and rc == 2


@pytest.mark.parametrize("lanes", ["16", "8", "auto", "rec"])
def test_forged_streams(forged, oracle, small, small8, lanes):
    """every forged stream: the oracle's status and out_len, and its output up to out_len, on each layout and on the recording
    decoder"""
    streams = [s for _, s, _, _, _ in forged]
    if lanes == "rec":
        res = [(st, out) for st, out, _ in small.decode_cmds(streams, [1 << 20] * len(forged))]
    else:
        eng = {"16": small, "8": small8}.get(lanes) or divans_b200.Engine(0, 8, 0)
    try:
        if lanes != "rec":
            res = eng.decode(streams, [1 << 20] * len(forged))
        for (name, stream, st, want, _), got in zip(forged, res):
            assert _same(got, (st, want), oracle, stream, 1 << 20), "%s: status %d (oracle %d)" % (name, got[0], st)
    finally:
        if lanes == "auto":
            eng.close()


@pytest.mark.parametrize("layout", [(2, 16), (4, 8)])
def test_one_warp_mates(catalogue, layout):
    """one warp: each command-heavy stream next to the literal-heavy one, in both orders"""
    g, lanes = layout
    eng = divans_b200.Engine(0, g, lanes)
    try:
        by = {n: (n, s, 0, r) for n, _, s, r in catalogue}
        lit = by["lit_lengths"]
        for name in ("distances", "dictionary", "block_switches", "extents", "context_maps", "cmd_types"):
            for pair in ([by[name], lit], [lit, by[name]]):
                batch = pair * (g // 2)
                res = eng.decode([s for _, s, _, _ in batch], [len(r) + 64 for _, _, _, r in batch])
                for (n, _, _, r), (st, out) in zip(batch, res):
                    assert st == 0 and out == r, "%s + %s: %s" % (pair[0][0], pair[1][0], n)
        assert eng.last_lanes() == lanes
    finally:
        eng.close()


def test_slot_succession(catalogue):
    """two slots: the streams that touch CTYPE / DPRIOR slabs up to 255 and the 16384 / 1024-entry maps, then streams that
    read those slabs and maps fresh -- each slot handed on several times"""
    by = {n: (n, s, 0, r) for n, _, s, r in catalogue}
    order = ["extents", "cmd_types", "copy_lengths_per_dtype", "end_after_copy_dict", "context_maps", "distances",
             "block_switches", "end_after_lit_bt", "dictionary", "copy_counts"]
    eng = divans_b200.Engine(0, 2, 16)
    try:
        _decode_all(eng, [by[n] for n in order])
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# encode
# ---------------------------------------------------------------------------------------------------------------------
# the lists of many output bytes (copies of up to 2^26 bytes, literals of up to 2^20) run at dynamic mixing 0 only: their
# PredictionMode records are what dynamic mixing changes, and every other list has the same records
LARGE = ("copy_counts", "lit_lengths")


@pytest.mark.parametrize("dcm", [0, 1, 2])
def test_encode_catalogue(catalogue, oracle, small, dcm):
    """encode_cmds host and device, and encode_cmds_auto with KEEP alone, equal the oracle's bytes"""
    for name, blob, stream, _ in catalogue:
        if dcm and name in LARGE:
            continue
        w = _window(blob)
        if dcm == 0:
            want = stream
        else:
            rc, want, _ = T.encode_forged(T.from_blob(oracle, blob), window_size=w, dynamic_context_mixing=dcm)
            assert rc == 0
        o = divans_b200.encode_options(window_size=w, dynamic_context_mixing=dcm)
        assert C._plain_host(small, [blob], o)[0][2] == want, name
        assert C._auto_device(small, [blob], o, plain=True)[0][0][2] == want, name
        auto, chosen, _ = C._auto_host(small, [blob], o, [C.KEEP])
        assert auto[0][2] == want and int(chosen[0]) == 0, name


def test_blend_catalogue(catalogue, oracle_blend, small):
    """the blend model: the GPU encoder equals the blend oracle, and the blend decoder decodes the stream"""
    for name, blob, _, replay in catalogue:
        w = _window(blob)
        rc, want, _ = T.encode_forged(T.from_blob(oracle_blend, blob), blend=True, window_size=w)
        assert rc == 0
        got = C._plain_host(small, [blob], divans_b200.encode_options(window_size=w, cdf_model=1))[0]
        assert got[2] == want, name
        assert small.decode([want], [len(replay) + 64], BLEND) == [(0, replay)], name


# ---------------------------------------------------------------------------------------------------------------------
# records no stream can carry
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["limits", "fuzz"])
def test_unrepresentable_records(oracle, small, kind):
    """status 0 only for a stream that the GPU and the oracle decode to the list's replay, and the oracle encoder's status
    and bytes; status 3 for every record no stream can carry -- on encode_cmds (host, device), encode_cmds_auto with KEEP
    and encode_cmds_mixmap"""
    # (the 2^30-byte literals of D.long_literal_cases are left out: the host calls refuse their sizes as a whole)
    cases = D.limit_cases() if kind == "limits" else D.fuzzed_cmd_blobs()
    blobs = [b for _, b, _ in cases]
    o = divans_b200.encode_options(window_size=16)
    host = C._plain_host(small, blobs, o)
    dev, _, _ = C._auto_device(small, blobs, o, plain=True)
    auto, _, cost = C._auto_host(small, blobs, o, [C.KEEP])
    mm = X._host(small, blobs, divans_b200.encode_options(window_size=16, literal_pred_mode=0), True)
    good = []
    for (name, blob, carried), h, d, a, c, m in zip(cases, host, dev, auto, cost, mm):
        cl = T.from_blob(oracle, blob)
        rc, want, _ = T.encode_forged(cl, window_size=16) if cl is not None else (3, b"", 0)
        assert h[0] == rc and (rc != 0 or h[2] == want), "%s: host status %d, oracle %d" % (name, h[0], rc)
        assert d[0] == rc and (rc != 0 or d[2] == want), "%s: device status %d, oracle %d" % (name, d[0], rc)
        assert a[0] == rc and (rc != 0 or a[2] == want), "%s: auto KEEP status %d, oracle %d" % (name, a[0], rc)
        assert (c[0] == T.TALLY_FAILED) == (rc == 3), name
        assert m[0] in (0, 3) and (rc == 0 or m[0] == 3), "%s: mixmap status %d" % (name, m[0])
        if carried is False:
            assert rc == 3, name
        if rc == 0:
            rc_r, n, replay = T.recode_blob(blob)
            assert rc_r == 0, name
            good.append((name, want, replay))
    if good:
        res = small.decode([s for _, s, _ in good], [len(r) + 64 for _, _, r in good])
        for (name, s, replay), (st, out) in zip(good, res):
            assert oracle.decode(s, out_cap=len(replay) + 64) == (0, replay), name
            assert (st, out) == (0, replay), name
