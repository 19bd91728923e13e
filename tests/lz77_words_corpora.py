"""Inputs and helpers shared by the tests of dictionary words under every transform in the LZ77 parse (include/divans_b200.h,
"dictionary words under every transform in the LZ77 parse"): transformed words as the decoder writes them (the oracle's
dvo_dict_word), buffers built from them, and a check of every Dictionary record of a list."""
import functools

import numpy as np

import lz77_dict_corpora as C


@functools.lru_cache(maxsize=None)
def tables():
    """lz77_dict_corpora.tables(), read once"""
    return C.tables()


TYPES = sorted({typ for _, typ, _ in tables()[3]})   # the transform types the tables use (0..20 but 19)


@functools.lru_cache(maxsize=None)
def transformed(size, wid, t):
    """the bytes the decoder writes for Dictionary(wid, size, t)"""
    from oracle import oracle_py
    buf = np.zeros(64, np.uint8)
    n = int(oracle_py.lib().dvo_dict_word(size, wid, t, buf.ctypes.data))
    assert n >= 0
    return buf[:n].tobytes()


def core_len(size, t):
    """the bytes of a word of `size` that transform t keeps"""
    typ = tables()[3][t][1]
    return size - (typ if typ <= 9 else typ - 11 if typ >= 12 else 0)


def forms_buffer(n_words=300, seed=1, types=None):
    """dictionary words under random transforms (of the given types, default all) whose core keeps 4 or more bytes, mostly
    back to back, now and then with a byte between them that no transform writes"""
    rng = np.random.default_rng(seed)
    size_bits, _, _, tr = tables()
    ts = [t for t in range(121) if types is None or tr[t][1] in types]
    out = bytearray()
    while n_words:
        size, t = int(rng.integers(4, 25)), ts[int(rng.integers(0, len(ts)))]
        if core_len(size, t) < 4:
            continue
        out += transformed(size, int(rng.integers(0, 1 << size_bits[size])), t)
        if rng.random() < 0.3:
            out += b"\x01"
        n_words -= 1
    return bytes(out)


def forms_at_end(seed=2):
    """short streams that end at, one byte short of, and one byte after a transformed word, for every transform"""
    rng = np.random.default_rng(seed)
    size_bits = tables()[0]
    raws = []
    for t in range(121):
        size = 4 + (t * 7) % 21
        if core_len(size, t) < 4:
            size = 24
        w = transformed(size, int(rng.integers(0, 1 << size_bits[size])), t)
        head = bytes(rng.integers(128, 256, t % 5, dtype=np.uint8))
        raws += [head + w, head + w[:-1], head + w + b"\x02"]
    return raws


def short_cores(seed=4):
    """words under the transforms that leave them fewer than 4 bytes (omit-first or omit-last), alone and between bytes that no
    transform writes"""
    rng = np.random.default_rng(seed)
    size_bits = tables()[0]
    raws = []
    for t in range(121):
        for size in range(4, 13):
            if core_len(size, t) < 4:
                w = transformed(size, int(rng.integers(0, 1 << size_bits[size])), t)
                raws += [w, b"\xff" + w + b"\xfe"]
    return raws


def records_of(blob):
    return C.records_of(blob)


def check_words(blob, raw):
    """every Dictionary record of the DVCL `blob` of `raw`: a word of size 4..24 with an id in range, a transform 0..120 whose
    core keeps 4 or more bytes, d == |w|, and w at the record's position of `raw`.  Returns the records' (size, transform)."""
    size_bits = tables()[0]
    h = np.frombuffer(blob[:32], np.uint32)
    pos, got = 0, []
    for t, a, b, c, d in records_of(blob):
        if t in (1, 3):
            pos += int(b)
        elif t == 2:
            assert 4 <= b <= 24 and a < (1 << size_bits[b]) and c < 121 and core_len(int(b), int(c)) >= 4, (a, b, c, d)
            w = transformed(int(b), int(a), int(c))
            assert d == len(w) and raw[pos:pos + len(w)] == w, (a, b, c, d, pos)
            pos += len(w)
            got.append((int(b), int(c)))
    assert pos == len(raw) and int(h[4]) == len(raw)
    return got
