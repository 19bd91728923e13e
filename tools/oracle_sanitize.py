"""Run the command-code catalogue, the forged streams and the record-limit cases on the CPU oracle built with
-fsanitize=undefined,address: the oracle library and the oracle_tally library (the oracle with the tally, forging and coverage
hooks) are both compiled instrumented into a temporary directory, and a child interpreter, with the ASan runtime preloaded,
runs the sets through them.  Any report aborts the child (halt_on_error, -fno-sanitize-recover), so exit status 0 is a clean
run.  Usage: python tools/oracle_sanitize.py"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r"""
import sys
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT + "/tests")
from oracle import oracle_py as O
from oracle_tally import tally_py as T
O._LIB_PATH = O_LIB; O.build = lambda force=False: O_LIB
T._lib_path = lambda blend: T_LIB; T.build = lambda force=False: None
import numpy as np
import cmd_codes as K
import dvcl as D
n = 0
for name, blob in K.lists():
    w = int(np.frombuffer(blob[20:24], np.uint32)[0])
    rc, stream, _ = T.encode_forged(T.from_blob(O, blob), window_size=w)
    assert rc == 0, name
    r = T.recode_blob(blob)
    assert O.decode_cmds(stream, out_cap=r[1] + 64)[0] == 0, name
    n += 1
rc, stream, _ = T.encode_forged(T.from_blob(O, K.huge_count()), window_size=16)
assert O.decode(stream, out_cap=1 << 16)[0] == 2
forged = K.forged(T, O)
for name, blob, carried in D.limit_cases() + D.long_literal_cases() + D.fuzzed_cmd_blobs():
    cl = T.from_blob(O, blob)
    if cl is not None:
        rc, stream, _ = T.encode_forged(cl, window_size=16)
        if rc == 0:
            O.decode(stream, out_cap=T.recode_blob(blob)[1] + 64)
print("clean: %d catalogue lists, the huge count, %d forged streams, the limit and fuzzed records" % (n, len(forged)))
"""


def main():
    from oracle_tally import tally_py as T
    T.build()   # writes the hooked source
    tmp = tempfile.mkdtemp(prefix="oracle_sanitize_")
    san = ["-O1", "-g", "-fsanitize=undefined,address", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer", "-fPIC", "-shared",
           "-pthread", "-I", os.path.join(ROOT, "oracle"), '-DDVO_TABLES_PATH="%s"' % T._TABLES]
    o_lib, t_lib = os.path.join(tmp, "liboracle.so"), os.path.join(tmp, "libtally.so")
    subprocess.check_call(["gcc"] + san + ["-o", o_lib, os.path.join(ROOT, "oracle", "divans_oracle.c")])
    subprocess.check_call(["gcc"] + san + ["-o", t_lib, T._SRC])
    asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    code = "ROOT = %r; O_LIB = %r; T_LIB = %r\n" % (ROOT, o_lib, t_lib) + CHILD
    return subprocess.call([sys.executable, "-c", code], env=env, cwd=ROOT)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    sys.exit(main())
