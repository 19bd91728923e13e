"""Reduced parity set for compute-sanitizer (memcheck / racecheck / initcheck): golden fixtures, the reference-held stream,
12 random-IR streams, one 64 KiB literal-only stream and one LZ77 stream, all lane layouts, the blend model, decode and encode, every result
checked against the oracle.  Usage: compute-sanitizer --tool memcheck python tools/sanitize_set.py"""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import divans_b200
from divans_b200 import synth
from oracle import oracle_py as O
import irfuzz

gold = json.load(open(os.path.join(ROOT, "tests", "golden", "golden.json")))
streams = [open(os.path.join(ROOT, "tests", "golden", e["name"] + ".divans"), "rb").read() for e in gold
           if e["name"] in ("alice29_priors_mix2", "truncated_dictionary", "random_then_unicode_ir")]
text = synth.text_corpus(1 << 18)
cmds = []
for seed in range(12):
    c = O.Commands.from_ir(irfuzz.random_ir(O, 100 + seed, n_cmds=80, window=[10, 14, 16, 22][seed % 4], text=text))
    cmds.append((c, O.options(window_size=[10, 14, 16, 22][seed % 4], dynamic_context_mixing=seed % 3)))
    streams.append(c.encode(cmds[-1][1]))
raw64 = text[5000:5000 + 65536]
streams.append(O.encode_raw(raw64))
streams.append(O.Commands.lz77(raw64, window=16).encode(O.options(window_size=16, dynamic_context_mixing=2)))
refs = [O.decode(s, out_cap=1 << 20) for s in streams]
assert all(rc == 0 for rc, _ in refs)
wasm = open(os.path.join(ROOT, "tests", "golden", "ref_wasm_example.divans"), "rb").read()
for lps in (8, 16):
    eng = divans_b200.Engine(0, 32, lps)
    res = eng.decode(streams, [len(r) + 64 for _, r in refs])
    assert all(st == 0 and out == r for (st, out), (_, r) in zip(res, refs)), "decode mismatch lps=%d" % lps
    st, out = eng.decode([wasm], [400], divans_b200.FLAG_MODEL_WASM_2018)[0]
    assert st == 0 and out.startswith(b"It snowed")
    if lps == 8:
        enc = eng.encode([raw64, raw64[:1000], b""], divans_b200.encode_options(dynamic_context_mixing=2))
        assert enc[0] == O.encode_raw(raw64, O.options(dynamic_context_mixing=2)) and enc[2] == O.encode_raw(b"", O.options(dynamic_context_mixing=2))
        for c, o in cmds[:6]:
            got = eng.encode([c.serialize()], divans_b200.encode_options(window_size=o.window_size, dynamic_context_mixing=o.dynamic_context_mixing), cmds=True)[0]
            assert got == c.encode(o)
    if lps == 16:   # the reference's feature="blend" probability model: its own decode / encode kernels
        from oracle import oracle_blend as OB
        braws = [raw64[:20000], raw64[:1], b"", text[70000:70000 + 9000]]
        for dcm in (0, 2):
            bs = [OB.encode_raw(r, OB.options(dynamic_context_mixing=dcm)) for r in braws]
            bs.append(OB.Commands.lz77(raw64[:30000], window=16).encode(OB.options(window_size=16, dynamic_context_mixing=dcm)))
            res = eng.decode(bs, [len(r) + 64 for r in braws] + [30064], divans_b200.FLAG_CDF_BLEND)
            assert all(st == 0 for st, _ in res) and all(out == r for (st, out), r in zip(res, braws + [raw64[:30000]]))
            enc = eng.encode(braws, divans_b200.encode_options(dynamic_context_mixing=dcm, cdf_model=divans_b200.CDF_BLEND))
            assert enc == bs[:len(braws)]
    eng.close()
print("sanitize set ok: %d streams, both lane layouts, decode + encode" % len(streams))
