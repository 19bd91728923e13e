"""GPU tests (-m gpu) of where the 16-lane mixing-value loop (dv2_core.cuh, mixval_run16) ends its runs and trips: runs of
every length around the 16-value trip, odd and even, changes of prior at value 256 and later, in one group or in its
warp-mate; a chunk restart inside a long run; command payloads that end at consecutive refill words; warps where the other
group is a dummy; and the recording decoder's command lists.  Every byte, status and list is compared with the CPU oracle."""
import functools

import pytest

import mixval_regimes as M
import regimes as R

pytestmark = pytest.mark.gpu

ONE_WARP = 2                       # slots of a one-warp engine at 16 lanes per stream
VALUES = [1, 4, 7, 2, 5, 8, 3, 6, 0]
# run lengths of the mixing values: every length up to three trips, both sides of 256, and one run to the end
LENGTHS = list(range(1, 50)) + [63, 64, 65, 255, 256, 257]


def run_values(shift, lengths=LENGTHS):
    """8192 mixing values in runs of the given lengths (cycled; the first run `shift` values shorter), each run a different
    value from the one before.  Value v >= 256 takes the prior of value v - 256, so the priors run the same lengths from 256 on"""
    mv, k = [], 0
    while len(mv) < 8192 + shift:
        mv += [VALUES[k % len(VALUES)]] * lengths[k % len(lengths)]
        k += 1
    return mv[shift:shift + 8192]


@functools.lru_cache(maxsize=None)
def runs_case(oracle, shift, mode="lsb6", model_rev=None):
    raw = R._txt(shift, 900, 23000)
    lines = [R.pm_line(mode, mix=run_values(shift)), R.insert(raw)]
    if model_rev is None:
        return R._good(oracle, R.from_ir(oracle, lines), raw)
    stream = R.from_ir(oracle, lines, model_rev=model_rev)
    rc, out, _ = oracle.decode_cmds(stream, model_rev=model_rev)
    assert rc == 0 and out == raw
    return R.Case(stream, raw, 0, 0, len(raw) + 64)


@functools.lru_cache(maxsize=None)
def chunk_in_run(oracle, at):
    """command-coder symbol 65535 at mixing value `at` of a PredictionMode command whose values are all 4: the chunk restart
    falls inside a run (as tests/mixval_regimes.chunk_at, which uses random values)"""
    want = 65535 - M._pm_head(oracle) - at
    src = R._txt(1, 40000, 27000)
    lines, pos = [], 0
    while M.cmd_nibbles(oracle, lines + [R.pm_line("lsb6")]) <= want:
        lines.append(R.pm_line("lsb6"))
    if (want - M.cmd_nibbles(oracle, lines)) % 2:
        lines.append(R.insert(src[pos:pos + 16])); pos += 16
    while lines and M.cmd_nibbles(oracle, lines) < want:
        n = (want - M.cmd_nibbles(oracle, lines)) // 2
        lines += [R.insert(src[pos + k:pos + k + 1]) for k in range(n)]; pos += n
    assert M.cmd_nibbles(oracle, lines) == want
    tail = R._txt(1, 700, 29000)
    lines += [R.pm_line("msb6", mix=4), R.insert(tail)]
    return R._good(oracle, R.from_ir(oracle, lines), src[:pos] + tail)


def _check(res, oracle, cases, what, flags=0):
    for i, ((st, out), c) in enumerate(zip(res, cases)):
        rc, ref = oracle.decode(c.stream, out_cap=c.cap, skip_crc=bool(flags & R.SKIP_CRC))
        assert st == rc, "%s: stream %d: status %d, oracle %d" % (what, i, st, rc)
        if rc == 0:
            assert out == ref, "%s: stream %d differs" % (what, i)


def _decode_check(eng, oracle, cases, what, flags=0):
    _check(eng.decode([c.stream for c in cases], [c.cap for c in cases], flags), oracle, cases, what, flags)


@pytest.fixture(scope="module")
def run_cases(oracle):
    return [runs_case(oracle, s) for s in range(4)] + [runs_case(oracle, 5, "utf8"), runs_case(oracle, 17, "msb6")]


@pytest.mark.parametrize("lanes", [16, 8])
def test_runs_of_every_length(oracle, run_cases, lanes):
    """runs of 1..49, 63..65 and 255..257 values, shifted so that each length starts at both parities and at every place in a
    trip; the warp-mates of a batch have different run boundaries, so a run also ends where the other group's prior changes"""
    import divans_b200
    eng = divans_b200.Engine(0, 0, lanes)
    try:
        _decode_check(eng, oracle, run_cases, "batch")
        _decode_check(eng, oracle, run_cases[::-1][:-1], "odd batch, reversed")
        assert eng.last_lanes() == lanes
    finally:
        eng.close()


def test_runs_next_to_a_dummy_and_each_other(oracle, run_cases):
    """one warp: each run pattern alone (the other group a dummy that codes against slot 16 of its own slot), and every pair of
    patterns, in both orders"""
    import divans_b200
    eng = divans_b200.Engine(0, ONE_WARP, 16)
    try:
        for i, c in enumerate(run_cases):
            _decode_check(eng, oracle, [c], "alone %d" % i)
        for i, a in enumerate(run_cases):
            for j, b in enumerate(run_cases):
                if i != j:
                    _decode_check(eng, oracle, [a, b], "pair %d %d" % (i, j))
        _decode_check(eng, oracle, [run_cases[0], R.build("lsb6", oracle), run_cases[1]], "next to plain literals, odd")
    finally:
        eng.close()


def test_wasm_2018_one_run(oracle):
    """under model revision WASM_2018 every value takes slot 16, whatever the mask holds: the whole command is one run"""
    import divans_b200
    cases = [runs_case(oracle, s, model_rev=oracle.MODEL_WASM_2018) for s in (0, 3)]
    eng = divans_b200.Engine(0, 0, 16)
    try:
        res = eng.decode([c.stream for c in cases] * 2 + [cases[0].stream], [c.cap for c in cases] * 2 + [cases[0].cap],
                         divans_b200.FLAG_MODEL_WASM_2018)
        for i, ((st, out), c) in enumerate(zip(res, cases * 2 + cases[:1])):
            assert st == 0 and out == c.raw, i
    finally:
        eng.close()


@pytest.mark.parametrize("at", [300, 301, 4000, 4001])
def test_chunk_restart_inside_a_run(oracle, at):
    """the chunk restart at a mixing value inside a run of one prior, at both parities: the run stops before symbol 65534 and
    the loop resumes after the generic path has coded the restart"""
    import divans_b200
    c = chunk_in_run(oracle, at)
    eng = divans_b200.Engine(0, ONE_WARP, 16)
    try:
        _decode_check(eng, oracle, [c], "alone")
        _decode_check(eng, oracle, [c, runs_case(oracle, 1)], "pair")
    finally:
        eng.close()


def test_payload_ends_at_each_refill(oracle):
    """the command payload cut at 48 consecutive 32-bit words inside the mixing values (after the first 256 values and
    well inside the runs): the payload runs dry at a refill of `a` alone, `b` alone and both, in either group of a warp"""
    import divans_b200
    base = runs_case(oracle, 2)
    cmd = oracle.demux(base.stream)[0]
    cuts = [len(cmd) // 3 + 4 * k for k in range(48)]
    bad = []
    for n in cuts:
        s = M._recode(oracle, base.stream, n)
        rc, out = oracle.decode(s, out_cap=base.cap)
        bad.append(R.Case(s, out if rc == 0 else None, 0, rc, base.cap))
    assert any(c.status != 0 for c in bad)
    eng = divans_b200.Engine(0, 0, 16)
    try:
        _decode_check(eng, oracle, bad, "cut")
        _decode_check(eng, oracle, [x for c in bad for x in (c, base)], "cut next to the whole stream")
    finally:
        eng.close()


def test_recorded_command_lists(oracle, run_cases):
    """the recording decoder (decode to command lists) runs the same loop: every list is the oracle's"""
    import divans_b200
    cases = run_cases + [chunk_in_run(oracle, 301)]
    eng = divans_b200.Engine(0, 0, 16)
    try:
        res = eng.decode_cmds([c.stream for c in cases], [c.cap for c in cases])
        for i, ((st, out, blob), c) in enumerate(zip(res, cases)):
            rc, ref, ref_cl = oracle.decode_cmds(c.stream, out_cap=c.cap)
            assert rc == 0 and st == 0 and out == ref, i
            assert blob == ref_cl.serialize(), "stream %d: command list differs" % i
    finally:
        eng.close()
