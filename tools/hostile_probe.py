"""Dev probe (not collected by pytest): corrupted streams with the CRC check skipped must come back with a status, never
hang or fault.  Run under `timeout`."""
import os, sys, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import divans_b200
from divans_b200 import synth
from oracle import oracle_py as O
from irfuzz import random_ir

rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 1)
import os
eng = divans_b200.Engine(0, 0, int(os.environ.get("DIVANS_B200_LPS", "16")))
text = synth.text_corpus(1 << 18)
base = []
for seed in range(16):
    c = O.Commands.from_ir(random_ir(O, seed, n_cmds=150, window=16, text=text))
    base.append(c.encode(O.options(window_size=16, dynamic_context_mixing=seed % 3)))
for k in range(8):
    r = text[k * 9000: k * 9000 + 20000]
    base.append(O.encode_raw(r, O.options(window_size=10 + k)))
tot = 0
for rnd in range(int(sys.argv[2]) if len(sys.argv) > 2 else 20):
    streams = []
    for s in base:
        b = bytearray(s)
        nmut = int(rng.integers(1, 6))
        for _ in range(nmut):
            pos = int(rng.integers(16, len(b) - 8))       # keep header + trailer framing, corrupt records / payload
            mode = int(rng.integers(0, 3))
            if mode == 0: b[pos] ^= 1 << int(rng.integers(0, 8))
            elif mode == 1: b[pos] = int(rng.integers(0, 256))
            else:
                ln = int(rng.integers(1, 64)); b[pos:pos + ln] = bytes(rng.integers(0, 256, min(ln, len(b) - 8 - pos)).astype(np.uint8))
        streams.append(bytes(b))
    res = eng.decode(streams, [1 << 20] * len(streams), flags=divans_b200.FLAG_SKIP_CRC if hasattr(divans_b200, "FLAG_SKIP_CRC") else 1)
    st = [r[0] for r in res]
    assert all(x in (0, 1, 2, 3) for x in st), st
    tot += len(streams)
    print("round", rnd, "statuses", {x: st.count(x) for x in set(st)}, flush=True)
# and the engine still works afterwards
(st, out), = eng.decode([base[-1]], [1 << 20])
assert st == 0 and out == text[7 * 9000: 7 * 9000 + 20000]
print("hostile probe ok:", tot, "corrupted streams")
