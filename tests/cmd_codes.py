"""A deterministic catalogue of DVCL command lists (include/divans_b200.h) that drives the command coder -- the copy, dictionary,
block-switch, literal-length and context-map nibbles of `transition` (divans_b200/csrc/dv_engine_kernel.cuh) -- through the
codes and prior indices random IR rarely reaches, and a set of forged streams that carry codes no encoder writes.

Each catalogue entry is named for what it reaches.  `lists()` gives (name, blob); every blob is a valid list the oracle encodes
with status 0.  `forged(T, oracle)` gives (name, stream, status, output): the oracle's encoding of a short list with some
command nibbles replaced (oracle_tally.encode_forged), each a CRC-valid stream, and the oracle decoder's verdict on it."""
import functools
import os

import numpy as np

import dvcl as D

from dvcl import BITS, Lst, dict_len as _dict_len, pm_record   # noqa: F401  (the builders live in dvcl.py)

PMB = D.PM_RECORD_BYTES


def mnemonic_of(lru, d):
    """the distance mnemonic the encoder codes for distance d (distance_mnemonic_code, codec/interface.rs:469-477), 15: none"""
    for i in range(15):
        if i < 4:
            v, ok = lru[i], True
        else:
            us = i >> 2
            v = (lru[(i & 2) >> 1] + (-us if i & 1 else us))
            ok = v > 0
        if ok and v == d:
            return i
    return 15


def obs_distance(lru, d):
    if d == lru[1]:
        return [d, lru[0], lru[2], lru[3]]
    if d == lru[2]:
        return [d, lru[0], lru[1], lru[3]]
    if d != lru[0]:
        return [d, lru[0], lru[1], lru[2]]
    return lru


# ---------------------------------------------------------------------------------------------------------------------
# the catalogue
# ---------------------------------------------------------------------------------------------------------------------
def lit_lengths():
    """literal lengths 1..16 (15 and 16: the SizeBegNib 0/1 path that keeps last_llen), both ends of every SizeBegNib 2..14 and
    of SizeLastNib 0..5, every mantissa nibble (lengths 31..46), the high-entropy flag; each followed by a copy of each length class, so CountSmall's index sees every
    last_llen bucket under every last-two-commands state"""
    L = Lst(window=22)
    lens = list(range(1, 17)) + [15 + v for k in range(2, 21) for v in (1 << (k - 1), (1 << k) - 1)] + list(range(31, 47))
    for i, n in enumerate(lens):
        L.text(n, i)
        L.copy([1, 3, 5, 15, 17][i % 5], 1 + i % 7)
    for i, n in enumerate([1, 14, 15, 16, 40, 300]):
        L.cmds.append((D.LIT, 0, n, 1, 0))   # high-entropy flag
        L.out += n
        L.copy(2, 1)
    return L


def copy_counts():
    """counts 0..14, both ends of every bit length 4..26 (CountBegNib 0..14, CountLastNib 0..7), each first-mantissa index
    (last_clen % 4) + 1"""
    L = Lst(window=16).text(64)
    counts = list(range(0, 15)) + [v for k in range(4, 27) for v in (1 << (k - 1), (1 << k) - 1)] + list(range(16, 32)) + \
        [(1 << 12) + 257 * i for i in range(16)]
    for i, n in enumerate(counts):
        L.copy(n, 1 + i % 50)
        if i % 3 == 0:
            L.text(1 + i % 20, i)
    return L


def distances():
    """every mnemonic 0..14 (lru values far apart, so each target has one code), the lru[1] - 3 shortcut, distance 1, codes whose
    value would be <= 0 (small lru values), the four obs_distance rules, and both ends of every bit length 2..24 at window 24 --
    distances that reach before the first byte included (they read zeros)"""
    L = Lst(window=24).text(3000)
    lru = [4, 11, 15, 16]
    seen = set()

    def cp(d, n=4):
        nonlocal lru
        seen.add(mnemonic_of(lru, d))
        L.copy(n, d)
        lru = obs_distance(lru, d)

    for d in (1, 2, 3, 2, 1, 1, 3):   # small lru values: codes 5, 7, 9, 11, 13 would be <= 0
        cp(d)
    for d in (1000, 2000, 3000, 4000, 3, 2):   # distances 3 and 2 coded explicitly: DistanceBegNib 1
        cp(d)
    for i in range(15):
        cp(1000)
        cp(2000)   # lru = [2000, 1000, ...]
        us = i >> 2
        target = lru[i] if i < 4 else lru[(i & 2) >> 1] + (-us if i & 1 else us)
        assert mnemonic_of(lru, target) == i, (i, lru, target)
        cp(target)
    cp(1500); cp(2500); cp(2500 - 0)        # repeat of lru0: no change
    cp(1500)                                  # lru1: swap
    cp(2000); cp(1500); cp(2500)              # lru2
    cp(1203); cp(1000); cp(1200 - 3 + 3)      # new values
    cp(lru[1] - 3)                            # the DistanceBegNib 15 shortcut (copy.rs:199-201)
    cp(1)
    for k in range(2, 25):
        for d in (1 << (k - 1), (1 << k) - 1):
            cp(d, 1 + k % 6)
    assert seen >= set(range(16)), sorted(set(range(16)) - seen)
    return L


def copy_lengths_per_dtype():
    """a 1024-entry distance map whose values cover 0..255, switched through dtype 0..255; under each, copies of length
    0, 1, 2, 3, 4 and 5 (distance-map index min(max(len, 2) - 2, 3)), an explicit and a mnemonic distance"""
    dm = (np.arange(1024) * 37 + (np.arange(1024) >> 8)) & 255
    assert set(dm.tolist()) == set(range(256))
    L = Lst(window=16, pms=[pm_record(lit_map=np.arange(64) & 7, dist_map=dm)]).text(400)
    for t in list(range(256)) + list(range(255, -1, -17)):
        L.bt(2, t)
        for n in (0, 1, 2, 3, 4, 5):
            L.copy(n, 7 + (t * 13 + n) % 300)
        L.copy(5, 1)
    return L


def dictionary():
    """every word size 4..24 x every transform 0..120, word id 0 and the largest id of the size, under distance priors up to
    255 (dtype switches over a 1024-entry map)"""
    dm = ((np.arange(1024) >> 2) + 64 * (np.arange(1024) & 3)) & 255   # dtype t, size >= 5: distance prior t + 192
    L = Lst(window=16, pms=[pm_record(lit_map=np.arange(64) & 7, dist_map=dm)]).text(20)
    k = 0
    for size in range(4, 25):
        for tr in range(121):
            for wid in (0, (1 << BITS[size]) - 1):
                n = _dict_len(size, wid, tr)
                if n <= 0:
                    continue
                L.bt(2, k & 255)
                L.dict(size, wid, tr, n)
                k += 1
    return L


def block_switches():
    """for L, C and D: every mnemonic 0..15 -- types 0..255 ascending (mnemonic 1, max + 1), mnemonic 1 at max_seen 255 (wraps
    to 0), then 255..0 descending through the two-nibble path and the types 0..12 of mnemonics 2..14, and lru[1] (mnemonic 0);
    literal strides 0..15 from the record"""
    L = Lst(window=16, pms=[pm_record(lit_map=np.arange(16384) & 31, dist_map=np.arange(1024) & 255)]).text(50)
    for which in range(3):
        seq = list(range(256)) + [0] + list(range(255, -1, -1)) + [7, 9, 7, 9, 3, 3]
        for i, t in enumerate(seq):
            L.bt(which, t, stride=i % 16)
            if i % 16 == 0:
                L.text(2, i)
                L.copy(3, 1 + i % 9)
    return L


def extents():
    """ctype 0..255 with a literal, a copy and a dictionary word under each; literal block types 0..255 over a 16384-entry literal
    map with values 0..255, a literal under each"""
    lm = (np.arange(16384) * 7 + (np.arange(16384) >> 6)) & 255
    L = Lst(window=16, pms=[pm_record(lit_map=lm, dist_map=np.arange(1024) & 255)]).text(40)
    for t in range(256):
        L.bt(1, t)
        L.text(3, t).copy(4, 1 + t % 30).dict(5 + t % 20, t % 31, t % 121, _dict_len(5 + t % 20, t % 31, t % 121))
    for t in list(range(256)) + [255, 0, 128]:
        L.bt(0, t, stride=t % 9)
        L.text(2 + t % 5, t)
    return L


def context_maps():
    """context-map mnemonics 0..15: a literal map of exactly 16384 entries and a distance map of exactly 1024, values that
    climb 0..255 (mnemonic 13, max + 1), wrap at max 255 (13 to 0), hit each of the 13 LRU places and escape to two nibbles"""
    rng = np.random.default_rng(5)
    lm = np.concatenate([np.arange(256), [0, 0, 1], rng.integers(0, 256, 16384 - 259)]).astype(np.uint8)
    lm[300:400] = np.tile(np.arange(13) * 5, 8)[:100]   # LRU hits at every place
    dm = np.concatenate([np.arange(256), [0], rng.integers(0, 256, 1024 - 257)]).astype(np.uint8)
    pms = [pm_record(p, lm, dm) for p in range(4)] + [pm_record(0, lm[:100], dm[:10])]
    L = Lst(window=16, pms=pms)
    for k in range(5):
        L.cmds.append((D.PREDMODE, k, 0, 0, 0))
        for t in (0, 3, 200, 255):
            L.bt(0, t, stride=t % 9).text(30, k * 7 + t).copy(4, 1 + t % 20)
    return L


KINDS = {"bt": lambda L: L.bt(1, 2), "copy": lambda L: L.copy(3, 1), "lit": lambda L: L.text(2), "dict": lambda L: L.dict(4, 0, 0, _dict_len(4, 0, 0))}
NEXT = {1: lambda L: L.copy(2, 2), 2: lambda L: L.dict(5, 1, 1, _dict_len(5, 1, 1)), 3: lambda L: L.text(1),
        4: lambda L: L.bt(0, 1), 5: lambda L: L.bt(1, 0), 6: lambda L: L.bt(2, 1), 7: lambda L: L.pm(0)}


def cmd_types():
    """every (last_4_states >> 4, type) pair of the command-type prior: each pair of command kinds, then each type 1..7; and
    every CountSmall index: each kind before a copy under last_llen 3 and 9"""
    L = Lst(window=16).text(8)
    for ln in (3, 9):
        for a in KINDS:
            L.text(ln)
            KINDS[a](L)
            L.copy(2, 2)
    for a in KINDS:
        for b in KINDS:
            for t in NEXT:
                KINDS[a](L); KINDS[b](L); NEXT[t](L)
    return L


def end_after(a, b):
    """end of stream after the kinds a, b"""
    L = Lst(window=16).text(8)
    KINDS[a](L); KINDS[b](L)
    return L


BUILDERS = {"lit_lengths": lit_lengths, "copy_counts": copy_counts, "distances": distances, "copy_lengths_per_dtype": copy_lengths_per_dtype,
            "dictionary": dictionary, "block_switches": block_switches, "extents": extents, "context_maps": context_maps,
            "cmd_types": cmd_types}
for _a in KINDS:
    for _b in KINDS:
        BUILDERS["end_after_%s_%s" % (_a, _b)] = functools.partial(end_after, _a, _b)


@functools.lru_cache(None)
def blob_of(name):
    return BUILDERS[name]().blob()


def lists():
    return [(n, blob_of(n)) for n in BUILDERS]


def huge_count():
    """a copy of 2^31 - 1 bytes (CountBegNib 15, CountLastNib 12): decoded with a small out_cap, status 2"""
    return Lst(window=16).text(10).copy((1 << 31) - 1, 3).blob()


# the oracle's encoding of huge_count() (its encoder replays the 2 GiB copy, which takes seconds): tests/golden, checked
# against a fresh encoding by the CPU tests
HUGE_COUNT_STREAM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cmd_codes_huge_count.divans")


# ---------------------------------------------------------------------------------------------------------------------
# forged streams
# ---------------------------------------------------------------------------------------------------------------------
def _prefix(blob, j):
    """blob with only its first j records"""
    b = bytearray(blob)
    h = np.frombuffer(bytes(b[:32]), np.uint32).copy()
    n = int(h[2])
    h[2] = j
    return h.tobytes() + bytes(b[32:32 + 20 * j]) + bytes(b[32 + 20 * n:])


def nibble_at(T, oracle, blob, j):
    """the index of record j's command-type nibble in the oracle's encoding of blob"""
    rc, _, n = T.encode_forged(T.from_blob(oracle, _prefix(blob, j)), window_size=BASE_WINDOW)
    assert rc == 0
    return n - 1


def _with(blob, j, rec):
    b = bytearray(blob)
    b[32 + 20 * j:52 + 20 * j] = np.array(rec, np.uint32).tobytes()
    return bytes(b)


BASE_WINDOW = 22


def _base():
    """the list the forged streams are made from; record j below is the j-th command"""
    L = Lst(window=BASE_WINDOW).text(600)                  # 1
    L.copy(1 << 18, 7)                                     # 2: CountSmall 15, CountBegNib 15, CountLastNib 0
    L.dict(19, 1, 0, _dict_len(19, 1, 0))                  # 3: DC_SizeBegNib 15, DC_SizeLastNib 0, 2 index nibbles
    L.text(20000)                                          # 4
    L.copy(6, 1 << 14)                                     # 5: DistanceBegNib 14, DistanceLastNib 0
    L.bt(0, 1, 2)                                          # 6: mnemonic 0, then the stride
    L.text(30)                                             # 7
    L.copy(5, (1 << BASE_WINDOW) - 1)                      # 8: lru[0] = ring - 1
    L.copy(5, 3)                                           # 9: mnemonics 4 and 8 reach the ring
    L.copy(4, 1)                                           # 10
    L.copy(4, 2)                                           # 11: lru = [2, 1, 3, ring - 1]
    L.copy(4, 5)                                           # 12: mnemonics 7, 9, 11, 13 are <= 0; lru[1] - 3 < 0
    L.dict(4, 5, 0, _dict_len(4, 5, 0))                    # 13: 12 index bits for 10: ids 1024.. are past the dictionary
    return L.blob()


def _maps_base():
    """a PredictionMode record whose maps are all zeros (one mnemonic nibble per entry) of exactly 16384 and 1024 entries"""
    L = Lst(window=BASE_WINDOW, pms=[pm_record(lit_map=np.zeros(16384), dist_map=np.zeros(1024))])
    return L.text(40).copy(4, 1).blob()


# the first map mnemonic of record 0 (after the type, mode, mixing and depth nibbles and 16 speed nibbles)
MAP0 = 20


def forged_cases():
    """(name, base, record j, [(offset from record j's type nibble, value)], the oracle's status) over BASES"""
    out = []
    for v in [0] + list(range(8, 15)):
        out.append(("cmd nibble %d" % v, "base", 2, [(0, v)], 3))   # CommandCodeOutOfBounds after the 600-byte literal
    out.append(("cmd nibble 15", "base", 2, [(0, 15)], 0))          # end of stream after the first literal
    # CountLastNib 14 / 15: 8 / 9 mantissa nibbles, the first at shift 28 / 32 (32 is taken mod 32: the low nibble)
    for last, mants in ((14, ([0] * 8, [0] * 7 + [9], [0] * 6 + [1, 9])),
                        (15, ([0] * 9, [3] + [0] * 7 + [5], [0] * 8 + [9], [15] + [0] * 8, [0, 1] + [0] * 7))):
        for mant in mants:
            st = 2 if mant[:2] == [0, 1] else 0   # 2 | 1 << 28 bytes: past the 1 MiB of output
            out.append(("CountLastNib %d mantissa %s" % (last, "".join("%x" % m for m in mant)), "base", 2,
                        [(3, last)] + [(4 + i, m) for i, m in enumerate(mant)], st))
    for m in (0, 3, 6, 7):   # long form of counts 8..15: CountSmall 15, CountBegNib 0, one mantissa nibble
        out.append(("long-form count %d" % (8 + m), "base", 2, [(2, 0), (3, m)], 0))
    # record 9 (lru = [ring - 1, 2^14, 7, 4]): 4, 8 and 12 reach ring .. ring + 2; record 12 (lru = [2, 1, 3, ring - 1]): 7, 9, 11,
    # 13 give 0 or less (CopyDistanceMnemonicCodeBad); every other code is a valid distance
    for mn in range(4, 15):
        out.append(("distance mnemonic %d near the ring" % mn, "base", 9, [(2, mn)], 3 if mn in (4, 8, 12) else 0))
        out.append(("distance mnemonic %d near 0" % mn, "base", 12, [(2, mn)], 3 if mn in (7, 9, 11, 13) else 0))
    out.append(("DistanceBegNib 15 with lru[1] < 3", "base", 12, [(2, 15), (3, 15)], 3))
    for last in range(10, 16):   # 25..30-bit distances: past the ring
        out.append(("DistanceLastNib %d" % last, "base", 5, [(4, last)], 3))
    for last in range(6, 16):    # word sizes 25..34: DictWordSizeTooLarge
        out.append(("dict SizeLastNib %d" % last, "base", 3, [(2, last)], 3))
    for hi in range(8, 16):      # transforms 128..: DictTransformIndexUndefined
        out.append(("dict transform hi %d" % hi, "base", 3, [(5, hi)], 3))
    out.append(("dict transform 121", "base", 3, [(5, 7), (6, 9)], 3))
    # size-4 ids 1024..4095: past the size's 1024 words, the word is read from the next sizes' words while it stays inside the
    # dictionary (the reference's bound is the whole dictionary), so these decode
    for hi in (4, 8, 15):
        out.append(("dict word id %d.. past the size's words" % (hi << 8), "base", 13, [(2, hi)], 0))
    for st in range(9, 16):
        out.append(("literal stride %d" % st, "base", 6, [(2, st)], 0))
    # a literal of 2^29 + 15 bytes and more (SizeLastNib 15): past the 1 MiB of output
    out.append(("literal SizeLastNib 15", "base", 4, [(3, 15)], 2))
    # one more map entry where the map has ended at exactly 16384 / 1024 entries: IndexBeyondContextMapSize
    out.append(("literal map index 16384", "maps", 0, [(MAP0 + 16384, 0)], 3))
    out.append(("distance map index 1024", "maps", 0, [(MAP0 + 16385 + 1024, 0)], 3))
    for p in range(4, 16):       # PredictionModeOutOfBounds, at the end of the record
        out.append(("pred_mode %d" % p, "base", 0, [(1, p)], 3))
    return out


BASES = {"base": lambda: _base(), "maps": lambda: _maps_base()}


def forged(T, oracle):
    """[(name, stream, oracle status, oracle output, stated status)] for forged_cases(), decoded by the oracle into 1 MiB"""
    out = []
    for base_name in BASES:
        base = BASES[base_name]()
        cl = T.from_blob(oracle, base)
        for name, b, j, nibs, want in forged_cases():
            if b != base_name:
                continue
            k0 = nibble_at(T, oracle, base, j) if j else 0
            rc, stream, _ = T.encode_forged(cl, [(k0 + o, v) for o, v in nibs], window_size=BASE_WINDOW)
            assert stream, name
            st, data = oracle.decode(stream, out_cap=1 << 20)
            out.append((name, stream, st, data, want))
    return out
