"""Hand-built DVCL command-list blobs (include/divans_b200.h) for the replay tests: a builder, and one blob per refusal rule of
divans_b200_replay_cmds_batch_* together with the status and out_len the rule gives; and two blobs the encoder refuses."""
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
