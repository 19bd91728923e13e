"""Compare the machine code of two builds of libdivans_b200.so, kernel by kernel.

    python tools/sass_compare.py OLD.so NEW.so [--rename OLD_MANGLED=NEW_MANGLED ...]

For every kernel present in both libraries (after applying the renames) it compares the SASS of `cuobjdump -sass` with
addresses and instruction encodings stripped, and the registers, stack, shared and local memory of `cuobjdump -res-usage`.
It also lists the kernels only one of the libraries has.  Exit status 0 when every common kernel is identical.
Needs only the CUDA toolkit: no GPU.  A refactor that claims to leave the generated code alone can show it with this.
"""
import argparse
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def _run(args):
    return subprocess.run([CUOBJDUMP] + args, check=True, capture_output=True, text=True).stdout


def sass(lib):
    """kernel -> list of normalised instructions"""
    out, cur = {}, None
    for line in _run(["-sass", lib]).splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        if line[:1] not in ("", " ", "\t"):   # the header of the next cubin ("Fatbin elf code:", "arch = ...")
            cur = None
        if cur is None:
            continue
        ins = re.sub(r"/\*.*?\*/", "", line).strip()
        if ins and not ins.startswith(".") and ins not in ("{", "}"):
            cur.append(ins)
    return out


def res_usage(lib):
    """kernel -> resource line (REG, STACK, SHARED, LOCAL, ...)"""
    out, cur = {}, None
    for line in _run(["-res-usage", lib]).splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur and "REG:" in line:
            out[cur] = " ".join(line.split())
            cur = None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", action="append", default=[], metavar="OLD=NEW", help="a kernel's mangled name in each build")
    a = ap.parse_args()
    ren = dict(r.split("=", 1) for r in a.rename)
    so, sn = sass(a.old), sass(a.new)
    ro, rn = res_usage(a.old), res_usage(a.new)
    back = {v: k for k, v in ren.items()}

    def new_name(k):
        return ren.get(k, k)

    def subst(lines):   # the new names inside instructions (calls), spelt the old way
        text = "\n".join(lines)
        for o, n in ren.items():
            text = text.replace(n, o)
        return text.splitlines()

    ok = True
    for k in sorted(so):
        n = new_name(k)
        if n not in sn:
            continue
        same_code = so[k] == subst(sn[n])
        same_res = ro.get(k) == rn.get(n)
        ok &= same_code and same_res
        label = k if n == k else "%s -> %s" % (k, n)
        print("%-10s %5d instructions  %s" % ("identical" if same_code and same_res else "DIFFERS", len(so[k]), label))
        print("           old: %s" % ro.get(k))
        if not same_res:
            print("           new: %s" % rn.get(n))
        if not same_code:
            import difflib
            for d in list(difflib.unified_diff(so[k], subst(sn[n]), lineterm="", n=1))[:40]:
                print("           " + d)
    only_old = sorted(k for k in so if new_name(k) not in sn)
    only_new = sorted(n for n in sn if back.get(n, n) not in so)
    for k in only_old:
        print("only in old: %s" % k)
    for n in only_new:
        print("only in new: %s" % n)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
