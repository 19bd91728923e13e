"""Hand-built DVCL command-list blobs (include/divans_b200.h): builders (`blob`, and `Lst` for whole lists), one blob per refusal
rule of divans_b200_replay_cmds_batch_* together with the status and out_len the rule gives, blobs the encoders refuse, and
record fields at and around each limit of what a stream can carry (`limit_cases`, `long_literal_cases`, `fuzzed_cmd_blobs`)."""
import functools

import numpy as np

MAGIC = 0x4C435644
PM_RECORD_BYTES = 32 + 16384 + 1024 + 8192
COPY, DICT, LIT, BT_L, BT_C, BT_D, PREDMODE = 1, 2, 3, 4, 5, 6, 7


def blob(cmds, lits=b"", n_pms=0, window=16, magic=MAGIC, version=1, n_cmds=None, n_pms_hdr=None, n_lits=None):
    """header + records (type, a, b, c, d) + n_pms zeroed PredictionMode records + literal pool.  The n_*= arguments override
    the counts the header states."""
    h = np.array([magic, version, len(cmds) if n_cmds is None else n_cmds, n_pms if n_pms_hdr is None else n_pms_hdr,
                  len(lits) if n_lits is None else n_lits, window, 0, 0], np.uint32)
    recs = np.array(cmds, np.uint32).reshape(-1, 5) if len(cmds) else np.zeros((0, 5), np.uint32)
    return h.tobytes() + recs.tobytes() + bytes(PM_RECORD_BYTES * n_pms) + bytes(lits)


def refusal_cases():
    """[(name, blob, window_size, out_len)]: each blob is refused (status 3) with that out_len.  Record-level refusals follow a
    3-byte literal, so out_len shows that the bytes before the refused command count and nothing after them does."""
    pre = [(LIT, 0, 3, 0, 0)]
    lits = b"abcdefgh"
    good = blob(pre, lits)
    cases = [
        ("short blob", good[:31], 0, 0),
        ("empty blob", b"", 0, 0),
        ("bad magic", blob(pre, lits, magic=MAGIC ^ 1), 0, 0),
        ("bad version", blob(pre, lits, version=2), 0, 0),
        ("pool past the blob", blob(pre, lits, n_lits=9), 0, 0),
        ("records past the blob", blob(pre, lits, n_cmds=2), 0, 0),
        ("records past the blob (64-bit)", blob(pre, lits, n_cmds=0xFFFFFFFF), 0, 0),
        ("predmode records past the blob (64-bit)", blob(pre, lits, n_pms_hdr=0xFFFFFFFF), 0, 0),
        ("pool size past the blob (64-bit)", blob(pre, lits, n_lits=0xFFFFFFFF), 0, 0),
        ("type 0", blob(pre + [(0, 0, 0, 0, 0)], lits), 0, 3),
        ("type 8", blob(pre + [(8, 0, 0, 0, 0)], lits), 0, 3),
        ("type 0xffffffff", blob(pre + [(0xFFFFFFFF, 0, 0, 0, 0)], lits), 0, 3),
        ("literal past the pool", blob(pre + [(LIT, 5, 4, 0, 0)], lits), 0, 3),
        ("literal past the pool (64-bit)", blob(pre + [(LIT, 0xFFFFFFFF, 2, 0, 0)], lits), 0, 3),
        ("literal length past the pool (64-bit)", blob(pre + [(LIT, 2, 0xFFFFFFFF, 0, 0)], lits), 0, 3),
        ("copy distance 0", blob(pre + [(COPY, 0, 5, 0, 0)], lits), 0, 3),
        ("copy distance = ring (header window)", blob(pre + [(COPY, 1 << 16, 5, 0, 0)], lits, window=16), 0, 3),
        ("copy distance = ring (window override)", blob(pre + [(COPY, 1 << 12, 5, 0, 0)], lits, window=16), 12, 3),
        ("copy distance = ring (header window 0 clamps to 10)", blob(pre + [(COPY, 1 << 10, 5, 0, 0)], lits, window=0), 0, 3),
        ("copy distance = ring (window 30 clamps to 24)", blob(pre + [(COPY, 1 << 24, 5, 0, 0)], lits, window=30), 0, 3),
        ("dictionary word size 3", blob(pre + [(DICT, 0, 3, 0, 0)], lits), 0, 3),
        ("dictionary word size 25", blob(pre + [(DICT, 0, 25, 0, 0)], lits), 0, 3),
        ("dictionary transform 121", blob(pre + [(DICT, 0, 4, 121, 0)], lits), 0, 3),
        ("dictionary word past the dictionary", blob(pre + [(DICT, 1 << 20, 4, 0, 0)], lits), 0, 3),
        ("dictionary word id near 2^32", blob(pre + [(DICT, 0xFFFFFFFF, 24, 0, 0)], lits), 0, 3),
        ("dictionary length differs from d", blob(pre + [(DICT, 0, 4, 0, 5)], lits), 0, 3),
    ]
    return cases


def literal_outside_pool(b):
    """the first literal command of DVCL blob `b` made to end past the literal pool"""
    w = np.frombuffer(b, np.uint8).copy()
    h = w[:32].view(np.uint32)
    for c in range(int(h[2])):
        r = w[32 + 20 * c: 52 + 20 * c].view(np.uint32)
        if r[0] == LIT:
            r[1] = h[4] - min(int(r[2]), int(h[4])) + 1
            return w.tobytes()
    raise AssertionError("no literal")


def pm_flood(pm_blob, k):
    """k PredictionMode commands that all point at the one record of `pm_blob` (a list holding a single PredictionMode):
    more command nibbles than the header's sizes allow for, i.e. a command-log overflow"""
    h = np.frombuffer(pm_blob[:32], np.uint32)
    assert int(h[2]) == 1 and int(h[3]) == 1
    rec = pm_blob[52:]
    hdr = np.array([h[0], 1, k, 1, 0, h[5], 0, 0], np.uint32).tobytes()
    return hdr + np.tile(np.array([PREDMODE, 0, 0, 0, 0], np.uint32), k).tobytes() + rec[:len(rec) - int(h[4])]


BITS = [0, 0, 0, 0, 10, 10, 11, 11, 10, 10, 10, 10, 10, 9, 9, 8, 7, 7, 8, 7, 7, 6, 6, 5, 5]   # dictionary id bits per word size


def pm_record(pred_mode=0, lit_map=None, dist_map=None, mixing=4):
    """one PredictionMode record: the maps (lengths = their sizes) and one uniform mixing value"""
    r = np.zeros(PM_RECORD_BYTES, np.uint8)
    r[0] = pred_mode
    lm = np.zeros(0, np.uint8) if lit_map is None else np.asarray(lit_map, np.uint8)
    dm = np.zeros(0, np.uint8) if dist_map is None else np.asarray(dist_map, np.uint8)
    r[28:30] = np.frombuffer(np.uint16(lm.size).tobytes(), np.uint8)
    r[30:32] = np.frombuffer(np.uint16(dm.size).tobytes(), np.uint8)
    r[32:32 + lm.size] = lm
    r[32 + 16384:32 + 16384 + dm.size] = dm
    r[32 + 16384 + 1024:] = mixing
    return r.tobytes()


class Lst:
    """a command list under construction; `out` tracks the bytes it produces, so copies can stay inside what exists"""

    def __init__(self, window=16, pms=None):
        self.cmds, self.lits, self.window, self.out = [], bytearray(), window, 0
        self.pms = [pm_record(lit_map=np.arange(64) & 7, dist_map=np.arange(4))] if pms is None else pms
        self.cmds.append((PREDMODE, 0, 0, 0, 0))

    def lit(self, data, he=0):
        self.cmds.append((LIT, len(self.lits), len(data), he, 0))
        self.lits += data
        self.out += len(data)
        return self

    def text(self, n, seed=0):
        rng = np.random.default_rng(seed + n)
        return self.lit(bytes(rng.choice(list(b"etaoin shrdlu"), n).astype(np.uint8)))

    def copy(self, n, d):
        self.cmds.append((COPY, d, n, 0, 0))
        self.out += n
        return self

    def dict(self, size, wid, tr, n):
        self.cmds.append((DICT, wid, size, tr, n))
        self.out += n
        return self

    def bt(self, which, t, stride=0):
        self.cmds.append((BT_L + which, t, stride if which == 0 else 0, 0, 0))
        return self

    def pm(self, k=0):
        """a PredictionMode command with a record of its own (a copy of record k): the encoders size their command logs by
        the blob, so a list does not point many commands at one record"""
        self.pms.append(self.pms[k])
        self.cmds.append((PREDMODE, len(self.pms) - 1, 0, 0, 0))
        return self

    def blob(self):
        h = np.array([MAGIC, 1, len(self.cmds), len(self.pms), len(self.lits), self.window, 0, 0], np.uint32)
        return h.tobytes() + np.array(self.cmds, np.uint32).tobytes() + b"".join(self.pms) + bytes(self.lits)


@functools.lru_cache(None)
def dict_len(size, wid, tr):
    """the length of dictionary word (size, wid) under transform tr, from the oracle's dictionary; <= 0: no word"""
    from oracle import oracle_py
    buf = np.zeros(64, np.uint8)
    return int(oracle_py.lib().dvo_dict_word(size, wid, tr, buf.ctypes.data))


def limit_cases():
    """[(name, blob, carried)]: record fields at values around each limit of the DVCL rule (include/divans_b200.h).  carried:
    a stream can carry the record (the encode succeeds, or fails where the decoder would); else it must be refused"""
    def one(rec, lits=0):
        L = Lst(window=16).text(3000)
        if lits:
            L.lits += bytes(lits)
        L.cmds.append(rec)
        L.text(5)
        return L.blob()

    def first(rec):   # the record before any other: refused before the stream's first nibble
        L = Lst(window=16)
        L.cmds.insert(0, rec)
        return L.text(5).blob()

    out = []
    for t in (0, 8, 14, 15, 16, 17, 31, 255, 0xFFFFFFFF):
        out.append(("type %d" % t, one((t, 0, 0, 0, 0)), False))
        out.append(("type %d first" % t, first((t, 0, 0, 0, 0)), False))
    for rec in ((COPY, 0, 4, 0, 0), (LIT, 0, 0, 0, 0), (DICT, 0, 3, 0, 0), (DICT, 0, 4, 256, 0), (BT_C, 256, 0, 0, 0), (BT_L, 1, 16, 0, 0)):
        out.append(("%s first" % (rec,), first(rec), False))
    for d in (1, 2999, (1 << 30) - 1):
        out.append(("copy distance %d" % d, one((COPY, d, 4, 0, 0)), d < 1 << 16))
    for d in (0, 1 << 30, (1 << 31) + 5, 0xFFFFFFFF):
        out.append(("copy distance %d" % d, one((COPY, d, 4, 0, 0)), False))
    out.append(("literal length 0", one((LIT, 0, 0, 0, 0), 1 << 16), False))
    out.append(("literal length 0 high-entropy", one((LIT, 0, 0, 1, 0), 1 << 16), False))
    for size in (0, 3, 25, 35, 260, 0xFFFFFFFF):
        out.append(("dict size %d" % size, one((DICT, 0, size, 0, 0)), False))
    for size in (4, 13, 24):
        bits = BITS[size]
        top = 1 << (-(-bits // 4) * 4)
        out.append(("dict size %d id %d" % (size, (1 << bits) - 1), one((DICT, (1 << bits) - 1, size, 0, 0)), True))
        out.append(("dict size %d id %d" % (size, top - 1), one((DICT, top - 1, size, 0, 0)), True))   # past the dictionary: carried
        out.append(("dict size %d id %d" % (size, top), one((DICT, top, size, 0, 0)), False))
    for tr in (120, 121, 255):
        out.append(("dict transform %d" % tr, one((DICT, 0, 4, tr, 0)), True))
    for tr in (256, 257, 376, 0xFFFFFFFF):
        out.append(("dict transform %d" % tr, one((DICT, 0, 4, tr, 0)), False))
    for w in range(3):
        for t in (0, 13, 255):
            out.append(("block switch %d type %d" % (w, t), one((BT_L + w, t, 0, 0, 0)), True))
        for t in (256, 257, 0xFFFFFFFF):
            out.append(("block switch %d type %d" % (w, t), one((BT_L + w, t, 0, 0, 0)), False))
    for s in (0, 8, 9, 15):
        out.append(("stride %d" % s, one((BT_L, 1, s, 0, 0)), True))
    for s in (16, 17, 255, 0xFFFFFFFF):
        out.append(("stride %d" % s, one((BT_L, 1, s, 0, 0)), False))
    out.append(("predmode record past the list", one((PREDMODE, 1, 0, 0, 0)), False))
    return out


def long_literal_cases():
    """literal lengths at the limit: 2^30 + 14 is carried (and refused for want of pool), 2^30 + 15 is not"""
    out = []
    for n, carried in (((1 << 30) + 14, True), ((1 << 30) + 15, False), (0xFFFFFFFF, False)):
        L = Lst(window=16).text(10)
        L.cmds.append((LIT, 0, n, 0, 0))
        out.append(("literal length %d" % n, L.blob(), carried))
    return out


def fuzzed_cmd_blobs(n=64, seed=91):
    """[(name, blob, None)]: random words written into command-record fields of short lists, as pm fuzzes do for PredictionMode
    records (never a dictionary record's d, which no nibble codes and the replay checks)"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = Lst(window=16).text(500, i)
        for _ in range(12):
            r = rng.integers(0, 5)
            [lambda: L.copy(int(rng.integers(1, 40)), int(rng.integers(1, 400))), lambda: L.text(int(rng.integers(1, 30)), i),
             lambda: L.dict(4, int(rng.integers(0, 1024)), 0, 4),   # (every size-4 word is 4 bytes long under transform 0)
             lambda: L.bt(int(rng.integers(0, 3)), int(rng.integers(0, 4)), int(rng.integers(0, 9))), lambda: L.pm(0)][r]()
        recs = np.array(L.cmds, np.uint32)
        for _ in range(int(rng.integers(1, 4))):
            j = int(rng.integers(1, len(recs)))
            f = int(rng.integers(0, 4))
            v = [int(rng.integers(0, 16)), int(rng.integers(0, 300)), 1 << int(rng.integers(0, 32)), int(rng.integers(0, 1 << 32))][int(rng.integers(0, 4))]
            if recs[j, 0] == DICT and f == 3:
                f = 2
            if recs[j, 0] in (COPY, LIT) and f == 2:
                v &= 255   # lengths the host calls' output sizing accepts
            recs[j, f] = v
        L.cmds = [tuple(int(x) for x in r) for r in recs]
        out.append(("fuzz %d" % i, L.blob(), None))
    return out
