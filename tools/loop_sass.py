"""Account for every instruction of the 16-lane T2S plain literal loop, or of the 16-lane mixing-value loop, of the v2 decoder.

    python tools/loop_sass.py                 # compiles divans_b200/csrc/dv2_kernels.cu for sm_90a with -lineinfo
    python tools/loop_sass.py --cubin K.cubin # or reads a cubin built from the same sources
    python tools/loop_sass.py --list          # also prints the hot path, one instruction per line
    python tools/loop_sass.py --mixval        # the pair loop of mixval_run16 instead (two mixing values per iteration)

The loop is `literal_plain_loop_v2<16, true>` (dv2_core.cuh): the plain loop with the context read from T2S in shared
memory, which the flagship text batch runs for nearly all of its time.  The tool finds it in the SASS of
`decode_kernel_v2<16>` through the inlining chains of `nvdisasm --print-line-info-inline`: an instruction belongs to the
loop when one of its frames is a line of the loop's `for` body inlined at the call that instantiates the T2S loop.  The
loop's region runs from the target of its back edge to the back edge.  Inside it, a forward branch that skips code of a
rare case (a block under `__builtin_expect`, or the eager refill of a rANS state) leaves that code off the hot path: the
hot path is what one byte costs when every prior carries the stream's tag and neither state needs a payload word.

With --mixval the loop is the pair loop of `mixval_run16`, the out-of-line mixing-value run that `decode_kernel_v2<16>` calls:
its instructions carry the loop's lines as their outermost frame (the function is not inlined), and its hot path is one pair
of mixing values with no refill.

It prints the hot path's instruction count per byte, the count per source line of the loop and per opcode class, the
size of each rare block, and the kernel's registers, stack and local-memory accesses.  Needs only the CUDA toolkit.
It is a tool for reading the code the compiler made, not a test: counts move with the compiler and with unrelated edits.
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "divans_b200", "csrc")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
KERNEL = "_ZN2dv16decode_kernel_v2ILi16EEEvNS_12DecodeParamsE"
CORE = "dv2_core.cuh"

INS_RE = re.compile(r"^\s+/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;?\s*$")
FRAME_RE = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
LABEL_RE = re.compile(r"^(\.L_x_\d+):")
BRA_RE = re.compile(r"^(@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(?:UR\d+,\s*)?`\((\.L_x_\d+)\)")


def compile_cubin(csrc, out):
    nvcc = os.path.join(CUDA, "bin", "nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-cubin",
                    os.path.join(csrc, "dv2_kernels.cu"), "-o", out], check=True)


def disassemble(cubin):
    """[(address, text, frames)] of the kernel, labels -> address.  frames: [(file basename, line, caller)] innermost first,
    caller = (file basename, line) or None"""
    text = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "--print-line-info-inline", cubin],
                          check=True, capture_output=True, text=True).stdout
    ins, labels, frames, pending, inside = [], {}, [], [], False
    for line in text.splitlines():
        if line.startswith(".text."):
            inside = line[len(".text."):].rstrip(":") == KERNEL
            continue
        if not inside:
            continue
        m = FRAME_RE.search(line)
        if m:
            caller = (os.path.basename(m.group(3)), int(m.group(4))) if m.group(3) else None
            pending.append((os.path.basename(m.group(1)), int(m.group(2)), caller))
            continue
        m = LABEL_RE.match(line)
        if m:
            labels[m.group(1)] = None   # resolved to the next instruction
            continue
        m = INS_RE.match(line)
        if m:
            if pending:
                frames, pending = pending, []
            addr = int(m.group(1), 16)
            for k, v in labels.items():
                if v is None:
                    labels[k] = addr
            ins.append((addr, m.group(2), frames))
    if not ins:
        sys.exit("kernel %s not found in %s" % (KERNEL, cubin))
    return ins, labels


def block_end(src, start):
    """index of the line that closes the first brace opened on or after line `start` (0-based)"""
    depth, opened = 0, False
    for i in range(start, len(src)):
        for ch in src[i].split("//")[0]:
            if ch == "{":
                depth, opened = depth + 1, True
            elif ch == "}":
                depth -= 1
                if opened and depth == 0:
                    return i
    raise ValueError("unbalanced braces after line %d" % (start + 1))


# the loops: (function definition, its `for` line, the call that instantiates it -- None: an out-of-line function)
LOOPS = {
    "t2s": (r"\bbool literal_plain_loop_v2\(", r"for \(uint32_t i = 0; i < m; i\+\+\)", "literal_plain_loop_v2<LPG, LPG == 16>("),
    "mixval": (r"\bMixvalRun mixval_run16\(", r"for \(uint32_t j = 0; 2 \* j \+ 1 < m; j\+\+\)", None),
}


def source_map(csrc, loop):
    """1-based lines of dv2_core.cuh: the loop's `for` body, the call that instantiates it (None: not inlined), the rare lines"""
    fn_re, for_re, call_s = LOOPS[loop]
    src = open(os.path.join(csrc, CORE)).read().splitlines()
    fn = next(i for i, s in enumerate(src) if re.search(fn_re, s))
    fn_end = block_end(src, fn)
    fo = next(i for i in range(fn, fn_end) if re.search(for_re, src[i]))
    body = range(fo + 1, block_end(src, fo) + 2)                          # 1-based: the `for` line and its body
    call = next(i for i, s in enumerate(src) if call_s in s) + 1 if call_s else None
    rare = set()
    for i in range(fn, fn_end):
        if "__builtin_expect(" in src[i]:
            rare.update(range(i + 2, block_end(src, i) + 2))
    for er in (i for i, s in enumerate(src) if re.search(r"\bvoid (eager_refill|split_refill16)\(", s)):
        rare.update(range(er + 1, block_end(src, er) + 2))
    return src, body, call, rare


def loop_frame(frames, body, call):
    """the line of the loop body this instruction is charged to, or None"""
    for f, ln, caller in frames:
        if f == CORE and ln in body and caller == ((CORE, call) if call else None):
            return ln
    return None


def opclass(text):
    t = re.sub(r"^@!?U?P\w+\s+", "", text)
    op = t.split()[0]
    base = op.split(".")[0]
    args = t[len(op):]
    if base in ("LDG", "STG", "LDS", "STS", "LD", "ST", "LDL", "STL", "ATOM", "ATOMG", "RED", "LDC", "ULDC"):
        return "memory (LDG/STG/LDS)"
    if base in ("SHFL", "VOTE", "VOTEU", "MATCH", "REDUX"):
        return "SHFL/VOTE"
    if base in ("MUFU", "I2F", "F2I", "I2FP", "F2F", "FRND"):
        return "MUFU/convert"
    if base in ("BRA", "BSSY", "BSYNC", "WARPSYNC", "EXIT", "CALL", "RET", "BREAK", "NOP", "BAR"):
        return "branch/WARPSYNC"
    if base in ("MOV", "UMOV", "R2UR", "S2R", "S2UR", "CS2R") or op.startswith("IMAD.MOV"):
        return "move/R2UR"
    # halves of a 64-bit operation: carry in (.X / .EX), wide products, 64-bit shifts, adds that write a carry predicate
    if {"X", "EX", "WIDE", "U64"} & set(op.split(".")[1:]) or re.match(r"\s*R\w+,\s*P\d", args):
        return "64-bit pair"
    return "ALU"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cubin", help="a cubin of dv2_kernels.cu built with -lineinfo (default: compile one)")
    ap.add_argument("--csrc", default=CSRC, help="the sources the cubin is built from (default: this tree's)")
    ap.add_argument("--list", action="store_true", help="print the hot path")
    ap.add_argument("--mixval", action="store_true", help="the mixing-value pair loop (mixval_run16) instead of the T2S loop")
    a = ap.parse_args()
    loop = "mixval" if a.mixval else "t2s"
    with tempfile.TemporaryDirectory() as tmp:
        cubin = a.cubin
        if not cubin:
            cubin = os.path.join(tmp, "dv2_kernels.cubin")
            compile_cubin(a.csrc, cubin)
        ins, labels = disassemble(cubin)
        res = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-res-usage", cubin], check=True, capture_output=True,
                             text=True).stdout
    src, body, call, rare = source_map(a.csrc, loop)
    idx = {addr: i for i, (addr, _, _) in enumerate(ins)}
    mine = [loop_frame(fr, body, call) is not None for _, _, fr in ins]
    if not any(mine):
        sys.exit("no instruction of the %s loop found: was the cubin built with -lineinfo from these sources?" % loop)
    # the back edge: the shortest backward branch charged to the `for` line itself (the out-of-line divergent paths of the
    # loop's votes and shuffles branch back into it too, but from the lines of those votes)
    best = None
    for i, (addr, text, fr) in enumerate(ins):
        m = BRA_RE.match(text)
        if not m or loop_frame(fr, body, call) != body[0] or labels.get(m.group(2)) is None or labels[m.group(2)] > addr:
            continue
        lo = idx[labels[m.group(2)]]
        if best is None or i - lo < best[1] - best[0]:
            best = (lo, i)
    if best is None:
        sys.exit("the back edge of the %s loop was not found" % loop)
    lo, hi = best
    # forward branches that skip a rare block
    skipped, blocks = set(), []
    for i in range(lo, hi + 1):
        m = BRA_RE.match(ins[i][1])
        if not m or not m.group(1) or labels.get(m.group(2)) is None:
            continue
        j = idx[labels[m.group(2)]]
        if not (i < j <= hi + 1):
            continue
        span = range(i + 1, j)
        if any(f == CORE and ln in rare for k in span for f, ln, _ in ins[k][2][:1]):
            skipped.update(span)
            blocks.append((ins[i][0], len(span), sorted({loop_frame(ins[k][2], body, call) or 0 for k in span} - {0})))
    hot = [k for k in range(lo, hi + 1) if k not in skipped]

    if loop == "mixval":
        print("decode_kernel_v2<16>, mixing-value pair loop (mixval_run16): region 0x%04x-0x%04x, %d instructions"
              % (ins[lo][0], ins[hi][0], hi - lo + 1))
        print("hot path (no refill): %d warp instructions per pair of values, %.1f per value (two streams per warp)"
              % (len(hot), len(hot) / 2))
    else:
        print("decode_kernel_v2<16>, T2S plain loop (literal_plain_loop_v2<16, true>): region 0x%04x-0x%04x, %d instructions"
              % (ins[lo][0], ins[hi][0], hi - lo + 1))
        print("hot path (tags match, no refill): %d warp instructions per byte (two streams per warp)" % len(hot))
    for addr, n, lines in blocks:
        print("  rare block after the branch at 0x%04x: %3d instructions (loop lines %s)" % (addr, n, ", ".join(map(str, lines))))
    print()
    per_line = collections.Counter()
    for k in hot:
        per_line[loop_frame(ins[k][2], body, call) or 0] += 1
    print("per source line of the loop (%s):" % CORE)
    for ln in sorted(per_line):
        s = src[ln - 1].strip() if ln else "(not charged to a line of the loop body)"
        print("  %4s %4d  %s" % (ln or "-", per_line[ln], s[:100]))
    print()
    per_class = collections.Counter(opclass(ins[k][1]) for k in hot)
    print("per opcode class:")
    for c, n in per_class.most_common():
        print("  %-22s %4d" % (c, n))
    print()
    local_k = sum(1 for _, t, _ in ins if re.search(r"\b(LDL|STL)\b", t))
    local_l = sum(1 for k in range(lo, hi + 1) if re.search(r"\b(LDL|STL)\b", ins[k][1]))
    m = re.search(r"Function %s:\s*\n\s*(REG:.*)" % re.escape(KERNEL), res)
    print("kernel: %s" % (" ".join(m.group(1).split()) if m else "(no resource line)"))
    print("local-memory accesses: %d in the kernel, %d in the loop region" % (local_k, local_l))
    if a.list:
        print()
        for k in hot:
            print("  %04x  %-4s %s" % (ins[k][0], loop_frame(ins[k][2], body, call) or "-", ins[k][1]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
