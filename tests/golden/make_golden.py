#!/usr/bin/env python3
"""Regenerate tests/golden/*.  Usage: make_golden.py <reference tree> (reads its testdata/).

The reference holds no compressed golden vectors (SURVEY section 4), so the fixtures are made by feeding the
reference's own IR fixtures (testdata/*.ir, the input of src/bin/integration_test.rs:76-108) through the oracle
encoder; the EXPECTED OUTPUT side is pinned by the reference's raw testdata files (sha256 below), i.e. by real
reference data, not by the oracle.  Each entry: <name>.divans + an index line in golden.json.
"""
import hashlib, json, lzma, os, sys
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle_py as O

REF = os.path.join(sys.argv[1], "testdata", "")
CASES = [
    # name, ir file, raw file, options
    ("alice29_ir", "alice29.ir", "alice29", dict()),
    ("alice29_priors_mix2", "alice29-priors.ir", "alice29", dict(dynamic_context_mixing=2)),
    ("alice29_priors_nocm", "alice29-priors.ir", "alice29", dict(dynamic_context_mixing=0, use_context_map=0)),
    ("alice29_q11_mix1", "alice29-q11.ir", "alice29", dict(dynamic_context_mixing=1)),
    ("asyoulik_ir_mix2", "asyoulik.ir", "asyoulik", dict(dynamic_context_mixing=2)),
    ("random_then_unicode_ir", "random_then_unicode.ir", "random_then_unicode", dict(dynamic_context_mixing=1)),
    ("truncated_dictionary", "ends_with_truncated_dictionary.ir", "ends_with_truncated_dictionary", dict()),
    ("alice29_literal_only", None, "alice29", dict()),
]
index = []
for name, ir, rawf, opts in CASES:
    raw = open(REF + rawf, "rb").read()
    o = O.options(**opts)
    if ir is None:
        enc = O.encode_raw(raw, o)
    else:
        enc = O.Commands.from_ir(open(REF + ir, "rb").read()).encode(o)
    rc, dec = O.decode(enc, out_cap=len(raw) + 64)
    assert rc == 0 and dec == raw, name
    open(os.path.join(HERE, name + ".divans"), "wb").write(enc)
    index.append(dict(name=name, source_ir=ir, source_raw=rawf, options=opts, raw_len=len(raw),
                      raw_sha256=hashlib.sha256(raw).hexdigest(), divans_len=len(enc), divans_sha256=hashlib.sha256(enc).hexdigest()))
    print(name, len(enc), len(raw))
json.dump(index, open(os.path.join(HERE, "golden.json"), "w"), indent=1)
# one of the reference IR fixtures itself, for the tests of the IR text parser on a real file
open(os.path.join(HERE, "asyoulik.ir.xz"), "wb").write(lzma.compress(open(REF + "asyoulik.ir", "rb").read(), preset=9 | lzma.PRESET_EXTREME))
