"""Where a batch call's regions go: the layouts tests/test_gpu_placement.py sends every decode and encode entry point through.

The Engine convenience wrappers put every input at a 16-byte aligned offset and every output at a 256-byte aligned one, so in
nearly every other test a byte's address mod 8 is its stream position mod 8.  The layouts here break that on purpose.  One call
places all its regions (inputs, outputs, blobs) in one allocation whose every other byte holds CANARY:

  residue_r        every output region starts at an offset = r mod 8; inputs start at IN_RESIDUES (mod 16), cycled
  mixed            output residues MIXED, cycled: the streams of one warp store at different phases
  adjacent         each output region is exactly the stream's output, and the next one starts where it ends
  reversed         as adjacent, but region i lies after region i + 1
  tight_minus_one  each output region one byte short of the stream's output
  high             regions start at HIGH_BASE + r, r in HIGH_RESIDUES, inside one allocation of HIGH_BYTES (device calls only)

Blob regions (decode to command lists) take residues independent of the outputs'.  Every group of regions has at least G
canary bytes before and after it, and nothing is placed against the end of the allocation.  Offsets are relative to the start
of the allocation (cudaMalloc and numpy give it an alignment of at least 16 bytes, so an offset's residue is the address's).
tests/test_placement_layouts.py checks on the CPU that each layout is what its name says."""
import collections

import numpy as np

G = 64                  # canary bytes around every group of regions
CANARY = 0xA5
IN_RESIDUES = [0, 1, 2, 3, 5, 8, 13, 15]
MIXED = [0, 7, 1, 6, 2, 5, 3, 4]
HIGH_BASE = 1 << 32
HIGH_RESIDUES = [0, 3, 7]
HIGH_BYTES = HIGH_BASE + (64 << 20)
LAYOUTS = ["residue_%d" % r for r in range(8)] + ["mixed", "adjacent", "reversed", "tight_minus_one"]
CONTIGUOUS = ("adjacent", "reversed")
SLACK = [0, 1, 7, 64, 300]   # cap - exact of the free layouts' regions, cycled (some regions exactly full)

# lo: the first byte of the window that holds every region (0, or HIGH_BASE - G); total: the allocation's size in bytes
Plan = collections.namedtuple("Plan", "layout lo total in_off in_len out_off out_cap blob_off blob_cap")


def _at(pos, res, mod):
    """the first offset >= pos that is = res mod `mod`"""
    return pos + (res - pos) % mod


def _caps(layout, exact, caps, short):
    exact = [int(x) for x in exact]
    if layout in CONTIGUOUS:
        return exact
    if layout == "tight_minus_one":
        return [max(e - 1, 0) if s else e + SLACK[i % len(SLACK)] for i, (e, s) in enumerate(zip(exact, short))]
    return [int(c) for c in caps] if caps is not None else [e + SLACK[i % len(SLACK)] for i, e in enumerate(exact)]


def _residues(layout, n, shift):
    """the residue mod 8 of each region of a free layout (shift: blobs take another sequence than outputs)"""
    if layout.startswith("residue_"):
        r = int(layout[len("residue_"):])
        return [(3 * r + 5) % 8 if shift else r] * n     # 3r + 5 = r (mod 8) has no solution: blobs never share the outputs' residue
    if layout == "mixed":
        return [MIXED[(i + 3 * shift) % 8] for i in range(n)]
    if layout == "high":
        return [HIGH_RESIDUES[(i + shift) % len(HIGH_RESIDUES)] for i in range(n)]
    return [(5 * i + 1 + 3 * shift) % 8 for i in range(n)]   # tight_minus_one


def _group(layout, pos, caps, shift, align):
    """place one group of regions from `pos` on: (offsets, the first free offset after the group's trailing guard)"""
    n = len(caps)
    off = [0] * n
    if layout in CONTIGUOUS:
        pos = _at(pos, (3 + 2 * shift + 2 * (layout == "reversed")) % 8 & ~(align - 1), 8)
        for i in (range(n) if layout == "adjacent" else reversed(range(n))):
            off[i] = pos
            pos += caps[i]
        return off, pos + G
    for i, r in enumerate(_residues(layout, n, shift)):
        pos = _at(pos, r & ~(align - 1), 8)
        off[i] = pos
        pos += caps[i] + G
    return off, pos


def place(layout, in_lens, exact, caps=None, blob_exact=None, blob_caps=None, in_residues=IN_RESIDUES, blob_align=1):
    """The regions of one call under `layout`.

    in_lens: the input lengths; exact: each stream's exact output length, caps: the output capacities of the free layouts
    (default exact plus SLACK); blob_exact / blob_caps: the same for blob regions (decode to command lists, LZ77 lists), None
    for calls without them.  tight_minus_one makes the outputs of every stream short, or with blobs the outputs of odd and the
    blobs of even streams.  in_residues: the inputs' residues mod 16, cycled; blob_align: 4 for regions that must be 4-byte
    aligned (contiguous regions then get caps rounded up to it)."""
    n = len(in_lens)
    with_blobs = blob_exact is not None
    out_short = [not with_blobs or i % 2 == 1 for i in range(n)]
    out_cap = _caps(layout, exact, caps, out_short)
    lo = HIGH_BASE - G if layout == "high" else 0
    out_off, pos = _group(layout, lo + G, out_cap, 0, 1)
    blob_off, blob_cap = [], []
    if with_blobs:
        blob_cap = _caps(layout, blob_exact, blob_caps, [not s for s in out_short])
        if blob_align > 1 and layout in CONTIGUOUS:
            blob_cap = [(c + blob_align - 1) // blob_align * blob_align for c in blob_cap]
        blob_off, pos = _group(layout, pos, blob_cap, 1, blob_align)
    in_off = []
    for i, ln in enumerate(in_lens):
        pos = _at(pos, in_residues[i % len(in_residues)], 16)
        in_off.append(pos)
        pos += int(ln) + G
    total = pos + G
    assert layout != "high" or total <= HIGH_BYTES, total
    u64 = lambda a: np.array(a, np.uint64).reshape(-1)
    return Plan(layout, lo, total, u64(in_off), u64(in_lens), u64(out_off), u64(out_cap), u64(blob_off), u64(blob_cap))


def spans(plan):
    """(offset, length) of every region of the plan: inputs, outputs, blobs"""
    return [(int(o), int(c)) for o, c in zip(np.concatenate([plan.in_off, plan.out_off, plan.blob_off]),
                                                 np.concatenate([plan.in_len, plan.out_cap, plan.blob_cap]))]


def region_mask(plan):
    """bool over the window [plan.lo, plan.total): True inside some region"""
    m = np.zeros(plan.total - plan.lo, bool)
    for o, c in spans(plan):
        m[o - plan.lo:o - plan.lo + c] = True
    return m


def host_buffer(plan, inputs):
    """the window of the allocation as a numpy array, CANARY everywhere but in the input regions"""
    buf = np.full(plan.total - plan.lo, CANARY, np.uint8)
    for o, x in zip(plan.in_off, inputs):
        buf[int(o) - plan.lo:int(o) - plan.lo + len(x)] = np.frombuffer(bytes(x), np.uint8)
    return buf
