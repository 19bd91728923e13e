"""Inputs and helpers shared by the tests of dictionary words in the LZ77 parse (include/divans_b200.h, "dictionary words in the
LZ77 parse"): the RFC 7932 dictionary and transform set read from brotli_tables.bin, and buffers built from its words."""
import os
import struct

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLES = os.path.join(ROOT, "divans_b200", "csrc", "brotli_tables.bin")


def tables():
    """(size_bits [32], offsets [32], dictionary bytes, transforms [(prefix, type, suffix)] of all 121)"""
    b = open(TABLES, "rb").read()
    size_bits = list(b[24:56])
    offsets = struct.unpack("<32I", b[56:184])
    tr = b[2232:2232 + 363]
    psmap = struct.unpack("<64H", b[2616:2744])
    ps = b[2744:3000]

    def s(i):
        o = psmap[i]
        return ps[o + 1:o + 1 + ps[o]]
    return size_bits, offsets, b[3000:], [(s(tr[3 * t]), tr[3 * t + 1], s(tr[3 * t + 2])) for t in range(121)]


def transform_set():
    """the transform ids with an empty prefix and the identity type, and their suffixes"""
    _, _, _, tr = tables()
    return [(t, sfx) for t, (pre, typ, sfx) in enumerate(tr) if pre == b"" and typ == 0]


def word(size, wid):
    size_bits, offsets, d, _ = tables()
    assert 4 <= size <= 24 and wid < (1 << size_bits[size])
    return d[offsets[size] + wid * size:offsets[size] + (wid + 1) * size]


def word_buffer(n_words=300, seed=1):
    """dictionary words of every size joined by the transform set's suffixes (and now and then a byte that is no suffix)"""
    rng = np.random.default_rng(seed)
    size_bits = tables()[0]
    sfx = [s for _, s in transform_set()]
    out = bytearray()
    for _ in range(n_words):
        size = int(rng.integers(4, 25))
        out += word(size, int(rng.integers(0, 1 << size_bits[size])))
        out += sfx[int(rng.integers(0, len(sfx)))] if rng.random() < 0.9 else b"\x01"
    return bytes(out)


def words_at_end(seed=2):
    """short streams that end inside, at, or one byte after a transformed word"""
    rng = np.random.default_rng(seed)
    size_bits = tables()[0]
    sfx = [s for _, s in transform_set()]
    raws = []
    for k in range(24):
        size = 4 + k % 21
        w = word(size, int(rng.integers(0, 1 << size_bits[size]))) + sfx[k % len(sfx)]
        head = bytes(rng.integers(128, 256, k % 7, dtype=np.uint8))
        raws += [head + w, head + w[:-1], head + w + b"\x02", w]
    return raws


def words_cut_short(seed=3):
    """words with their last byte changed or dropped, alone and before other bytes"""
    rng = np.random.default_rng(seed)
    size_bits = tables()[0]
    raws = []
    for size in range(4, 25):
        w = word(size, int(rng.integers(0, 1 << size_bits[size])))
        raws += [w[:-1], w[:-1] + b"\x03\x04\x05", w[:-1] + bytes([w[-1] ^ 0x80]) + b"xyz"]
    return raws


def records_of(blob):
    h = np.frombuffer(blob[:32], np.uint32)
    return np.frombuffer(blob[32:32 + 20 * int(h[2])], np.uint32).reshape(-1, 5)


def check_words(blob, raw):
    """every Dictionary record of the DVCL `blob` of `raw`: a word of size 4..24 with an id in range, a transform of the set,
    d == |w|, and w at the record's position of `raw`.  Returns the number of such records."""
    size_bits = tables()[0]
    sfx = dict(transform_set())
    h = np.frombuffer(blob[:32], np.uint32)
    pos, n = 0, 0
    for t, a, b, c, d in records_of(blob):
        if t == 3:
            pos += int(b)
        elif t == 1:
            pos += int(b)
        elif t == 2:
            assert 4 <= b <= 24 and a < (1 << size_bits[b]) and c in sfx, (a, b, c, d)
            w = word(int(b), int(a)) + sfx[int(c)]
            assert d == len(w) and raw[pos:pos + len(w)] == w, (a, b, c, d, pos)
            pos += len(w)
            n += 1
    assert pos == len(raw) and int(h[4]) == len(raw)
    return n
