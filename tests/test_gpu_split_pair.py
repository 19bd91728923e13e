"""The 16-lane plain literal loop advances the two rANS states of a byte on separate halves of the group: lanes 0-7 keep state
`a` (high nibbles), lanes 8-15 keep `b` (low nibbles), and one set of instructions steps both (rans_split16, dv2_core.cuh).
These tests check one byte of it against the oracle's two sequential steps and the reference's refill order (`a` before
`b`), at every offset of some walk states, and whole streams through both 16-lane plain loops against the oracle (-m gpu)."""
import ctypes
import os

import numpy as np
import pytest

import regimes as R
from test_gpu_arith import HIGH_WORDS, step_states  # noqa: F401  (step_states: fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_LIB = os.path.join(ROOT, "divans_b200", "lib", "libdivans_b200_split_probe.so")


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE_LIB), "%s is missing: build() makes it (make -C divans_b200/csrc)" % PROBE_LIB
    L = ctypes.CDLL(PROBE_LIB)
    L.dvp_split_byte.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 13
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _split_byte(probe, c):
    n = len(c["a"])
    o = dict(h=np.zeros(n, np.int32), l=np.zeros(n, np.int32), a=np.zeros(n, np.uint64), b=np.zeros(n, np.uint64),
             wi=np.zeros(n, np.uint32), under=np.zeros(n, np.uint32))
    args = [np.ascontiguousarray(c[k], t) for k, t in (("cdf_h", np.int16), ("cdf_l", np.int16), ("a", np.uint64), ("b", np.uint64),
                                                       ("words", np.uint32), ("wi", np.uint32), ("wmax", np.uint32))]
    assert probe.dvp_split_byte(n, *[_p(x) for x in args], *[_p(o[k]) for k in ("h", "l", "a", "b", "wi", "under")]) == 0
    return o


def _expected(oracle, c, spd_h, spd_l):
    """the oracle's step of `a` on the high prior and of `b` on the low one, then the eager refills in payload order: each
    state below 2^31 takes the next word, the cursor saturating at wmax; the coder underflowed when it ends at wmax"""
    rh = oracle.cdf_steps(c["cdf_h"], np.stack([spd_h, spd_h], 1), state=c["a"])   # (the context-map speed is unused)
    rl = oracle.cdf_steps(c["cdf_l"], np.stack([spd_l, spd_l], 1), state=c["b"])
    n = len(c["a"])
    a, b = rh["state"].astype(np.uint64), rl["state"].astype(np.uint64)
    wi = c["wi"].astype(np.int64).copy()
    wmax = c["wmax"].astype(np.int64)
    rows = np.arange(n)
    needs = []
    for x in (a, b):
        need = x < np.uint64(1 << 31)
        w = c["words"][rows, wi].astype(np.uint64)
        x[need] = (x[need] << np.uint64(32)) | w[need]
        wi = np.where(need, np.minimum(wi + 1, wmax), wi)
        needs.append(need)
    want = dict(h=rh["sym"], l=rl["sym"], a=a, b=b, wi=wi.astype(np.uint32), under=(wi >= wmax).astype(np.uint32))
    return want, needs[0], needs[1]


def _cases(rng, cdf, spd, n_full=16, n_rand=4096, offsets=64):
    """pairs of walk states (high prior, low prior); the first `n_full` pairs sweep every offset of `a`, the next `n_full`
    every offset of `b` (offset 0 included: the t = -1 of a corrupted payload), the rest take random offsets.  High state
    words from HIGH_WORDS and random, so that `a` only, `b` only, both and neither refill; cursors that start anywhere up
    to wmax and payloads that end before the first word, between the two words, right after the second, or later"""
    n = len(cdf)
    full = np.arange(32768)
    ih = np.concatenate([np.repeat(rng.integers(0, n, 2 * n_full), 32768), np.repeat(rng.integers(0, n, n_rand), offsets)])
    il = rng.integers(0, n, ih.size)
    m = ih.size
    oa, ob = rng.integers(0, 32768, m), rng.integers(0, 32768, m)
    oa[:n_full * 32768] = np.tile(full, n_full)
    ob[n_full * 32768:2 * n_full * 32768] = np.tile(full, n_full)
    hw = np.array(HIGH_WORDS + [int(x) for x in rng.integers(1, 1 << 48, 60)], np.uint64)
    a = (hw[rng.integers(0, hw.size, m)] << np.uint64(15)) | oa.astype(np.uint64)
    b = (hw[rng.integers(0, hw.size, m)] << np.uint64(15)) | ob.astype(np.uint64)
    wi = rng.integers(0, 4, m)
    wmax = np.minimum(wi + rng.choice([0, 1, 2, 3, 7], m), 7)
    words = rng.integers(0, 1 << 32, (m, 8), dtype=np.uint64).astype(np.uint32)
    return dict(cdf_h=cdf[ih], cdf_l=cdf[il], a=a, b=b, words=words, wi=wi.astype(np.uint32), wmax=wmax.astype(np.uint32)), spd[ih], spd[il]


def test_split_byte_equals_two_oracle_steps_and_refills(probe, oracle, step_states):  # noqa: F811
    cdf, spd, _ = step_states["small"]
    c, sh, sl = _cases(np.random.default_rng(71), cdf, spd)
    got, (want, na, nb) = _split_byte(probe, c), _expected(oracle, c, sh, sl)
    bad = np.zeros(len(c["a"]), bool)
    for k in ("h", "l", "a", "b", "wi", "under"):
        bad |= got[k] != want[k]
    cover = {
        "a only": int((na & ~nb).sum()), "b only": int((~na & nb).sum()), "both": int((na & nb).sum()),
        "underflow": int(want["under"].sum()), "offset 0 of a": int(((c["a"] & np.uint64(0x7FFF)) == 0).sum()),
        "offset 0 of b": int(((c["b"] & np.uint64(0x7FFF)) == 0).sum()),
        "sym 0 / 15 high": (int((want["h"] == 0).sum()), int((want["h"] == 15).sum())),
        "sym 0 / 15 low": (int((want["l"] == 0).sum()), int((want["l"] == 15).sum())),
    }
    print("split byte: %d cases, %d mismatches, %s" % (len(bad), int(bad.sum()), cover))
    for k, v in cover.items():
        assert (min(v) if isinstance(v, tuple) else v) > 0, k
    i = np.nonzero(bad)[0][:4]
    assert not bad.any(), [{k: (int(np.asarray(got[k])[j]), int(np.asarray(want[k])[j])) for k in got} for j in i]


def test_split_refill_at_the_payload_end(probe, oracle, step_states):  # noqa: F811
    """every refill combination against every payload end near the cursor: no word left, one word (the payload ends between
    the two words), exactly two, plenty; and a cursor already at wmax"""
    cdf, spd, _ = step_states["small"]
    rng = np.random.default_rng(72)
    idx = rng.integers(0, len(cdf), 256)
    rows = []
    for hwa in (1, 1 << 47):                      # 1: the state refills, 1 << 47: it does not
        for hwb in (1, 1 << 47):
            for wi in range(4):
                for left in (0, 1, 2, 7):
                    rows.append((hwa, hwb, wi, min(wi + 1 + left, 7) if left < 7 else 7))
                rows.append((hwa, hwb, wi, wi))  # cursor already saturated
    rows = np.array(rows, np.uint64)
    r = np.repeat(rows, idx.size, axis=0)
    k = np.tile(idx, len(rows))
    off = rng.integers(0, 32768, (len(r), 2)).astype(np.uint64)
    c = dict(cdf_h=cdf[k], cdf_l=cdf[np.roll(k, 1)], a=(r[:, 0] << np.uint64(15)) | off[:, 0], b=(r[:, 1] << np.uint64(15)) | off[:, 1],
             words=rng.integers(0, 1 << 32, (len(r), 8), dtype=np.uint64).astype(np.uint32),
             wi=r[:, 2].astype(np.uint32), wmax=r[:, 3].astype(np.uint32))
    got, (want, _na, _nb) = _split_byte(probe, c), _expected(oracle, c, spd[k], spd[np.roll(k, 1)])
    bad = np.zeros(len(r), bool)
    for key in ("h", "l", "a", "b", "wi", "under"):
        bad |= got[key] != want[key]
    print("split refill: %d cases, %d underflows, %d mismatches" % (len(r), int(want["under"].sum()), int(bad.sum())))
    assert 0 < want["under"].sum() < len(r)
    i = np.nonzero(bad)[0][:4]
    assert not bad.any(), [dict(row=r[j].tolist(), **{key: (int(got[key][j]), int(want[key][j])) for key in got}) for j in i]


@pytest.fixture(scope="module")
def engine16l():
    import divans_b200
    eng = divans_b200.Engine(0, 0, 16)
    yield eng
    eng.close()


@pytest.mark.parametrize("mode", ["lsb6", "msb6", "utf8", "sign"])
def test_split_loop_streams_cross_a_chunk_restart(oracle, engine16l, mode):
    """literal-only streams of more than 32768 bytes (65536 nibbles: the coder's chunk restarts inside the fast loop) and odd
    lengths, three per batch so that the second warp carries a dummy group; LSB6 / MSB6 take the T2S loop, UTF8 / SIGN the
    global-T2 one.  Bit-exact against the oracle."""
    from divans_b200 import synth
    rng = np.random.default_rng(73 + ["lsb6", "msb6", "utf8", "sign"].index(mode))
    corpus = synth.text_corpus(1 << 20)
    raws = []
    for n in (40001, 65535 + 2 * int(rng.integers(0, 2000)), 33333):
        o = int(rng.integers(0, len(corpus) - n))
        raws.append(corpus[o:o + n])
    streams = [R._raw_mode(oracle, r, ["lsb6", "msb6", "utf8", "sign"].index(mode), 4) for r in raws]
    for s, r in zip(streams, raws):
        rc, out = oracle.decode(s, out_cap=len(r) + 64)
        assert rc == 0 and out == r
    res = engine16l.decode(streams, [len(r) + 64 for r in raws])
    for i, ((st, out), r) in enumerate(zip(res, raws)):
        assert st == 0 and out == r, "stream %d (%d bytes): GPU output differs from the oracle" % (i, len(r))
