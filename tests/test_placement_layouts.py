"""CPU checks (no GPU) that every layout of tests/placement.py is what its name says: the residues, the adjacency, the short
regions, the regions past 2^32, and the canary bytes around every group of regions."""
import numpy as np
import pytest

import placement as P

IN_LENS = [0, 1, 7, 8, 9, 100, 1000, 4097, 3, 17, 20000]
EXACT = [31, 8, 13, 0, 1, 99, 1001, 5000, 7, 33, 20011]
BLOBS = [51268, 51300, 51301, 51299, 51270, 51269, 51290, 51400, 51271, 51277, 60000]


def _sorted_spans(plan):
    return sorted(P.spans(plan))


@pytest.mark.parametrize("blobs", [False, True])
@pytest.mark.parametrize("layout", P.LAYOUTS + ["high"])
def test_layout_is_what_its_name_says(layout, blobs):
    plan = P.place(layout, IN_LENS, EXACT, blob_exact=BLOBS if blobs else None)
    n = len(IN_LENS)
    out, cap = plan.out_off.astype(np.int64), plan.out_cap.astype(np.int64)
    assert [int(o) % 16 for o in plan.in_off] == [P.IN_RESIDUES[i % 8] for i in range(n)]
    if layout.startswith("residue_"):
        r = int(layout[-1])
        assert (out % 8 == r).all()
        if blobs:
            assert (plan.blob_off.astype(np.int64) % 8 != r).all()
    if layout == "mixed":
        assert list(out % 8) == [P.MIXED[i % 8] for i in range(n)]
    if layout in P.CONTIGUOUS:
        assert list(cap) == EXACT
        order = list(range(n)) if layout == "adjacent" else list(reversed(range(n)))
        seq = [int(out[i]) for i in order]
        caps = [int(cap[i]) for i in order]
        assert all(seq[k + 1] == seq[k] + caps[k] for k in range(n - 1)), "regions do not touch"
        if blobs:
            assert list(plan.blob_cap) == BLOBS
    if layout == "tight_minus_one":
        short = [True] * n if not blobs else [i % 2 == 1 for i in range(n)]
        assert all(int(c) == max(e - 1, 0) for c, e, s in zip(cap, EXACT, short) if s)
        if blobs:
            assert all(int(c) == e - 1 for i, (c, e) in enumerate(zip(plan.blob_cap, BLOBS)) if i % 2 == 0)
    if layout == "high":
        assert int(out[0]) == P.HIGH_BASE and plan.total <= P.HIGH_BYTES
        assert min(o for o, _ in P.spans(plan)) >= P.HIGH_BASE
        assert list(out % 8) == [P.HIGH_RESIDUES[i % 3] for i in range(n)]
    # no two regions overlap; a gap between two regions is either zero (contiguous layouts) or at least G canary bytes;
    # at least G canary bytes before the first region and after the last, inside the allocation
    sp = _sorted_spans(plan)
    assert sp[0][0] - plan.lo >= P.G and plan.total - (sp[-1][0] + sp[-1][1]) >= P.G
    for (a, la), (b, _) in zip(sp, sp[1:]):
        gap = b - (a + la)
        assert gap >= P.G or (gap == 0 and layout in P.CONTIGUOUS), (a, la, b)
    mask = P.region_mask(plan)
    assert mask.sum() == sum(c for _, c in sp)


def test_blob_alignment():
    for layout in P.LAYOUTS + ["high"]:
        plan = P.place(layout, IN_LENS, EXACT, blob_exact=BLOBS, blob_align=4)
        assert (plan.blob_off % np.uint64(4) == 0).all(), layout


def test_host_buffer_holds_inputs_and_canary():
    ins = [bytes([i]) * n for i, n in enumerate(IN_LENS)]
    plan = P.place("mixed", IN_LENS, EXACT)
    buf = P.host_buffer(plan, ins)
    for o, x in zip(plan.in_off, ins):
        assert buf[int(o):int(o) + len(x)].tobytes() == x
    assert (buf[~P.region_mask(plan)] == P.CANARY).all()
