"""Stream builders for the mixing values of a PredictionMode command: the 8192 nibbles the v2 decoder codes in its converged
mixing-value loop (dv2_core.cuh, mixval_fast_v2).  Same conventions as tests/regimes.py: every builder is oracle-encoded and
deterministic and returns a regimes.Case.  tests/test_mixval_regimes.py checks on the CPU that each stream is what its name
says; tests/test_gpu_mixval_loop.py decodes them on the GPU."""
import functools

import numpy as np

import regimes as R

# command-coder symbol 65535 (the last one before the 16-byte re-initialisation, ans.rs:230-244) at these mixing values
CHUNK_AT = [0, 1, 255, 256, 8190, 8191]


def mixing_values(seed):
    """8192 random mixing values (0..8, as the per-context regime of tests/regimes.py): past value 255 the prior of almost
    every value differs from the one before; fixed, different values around positions 255/256 and 8190/8191"""
    mv = [int(x) for x in np.random.default_rng(seed).integers(0, 9, 8192)]
    mv[254:258] = [1, 7, 3, 6]
    mv[8189:8192] = [2, 5, 8]
    return mv


def _pm(seed, mode="lsb6"):
    return R.pm_line(mode, mix=mixing_values(seed))


@functools.lru_cache(maxsize=None)
def random_mix(oracle, variant=0):
    """one PredictionMode command with random mixing values, then 1500 bytes of text"""
    raw = R._txt(variant, 1500, 3000)
    return R._good(oracle, R.from_ir(oracle, [_pm(100 + variant), R.insert(raw)]), raw)


@functools.lru_cache(maxsize=None)
def multi_pm(oracle, variant=0):
    """three PredictionMode commands with literals between them: random values, all 4, random values again"""
    a, b, c = (R._txt(variant, 700, 5000 + 1000 * k) for k in range(3))
    lines = [_pm(200 + variant), R.insert(a), R.pm_line("msb6"), R.insert(b), _pm(300 + variant, "utf8"), R.insert(c)]
    return R._good(oracle, R.from_ir(oracle, lines), a + b + c)


@functools.lru_cache(maxsize=None)
def late_pm(oracle, variant=0):
    """`variant + 1` one-byte literals, then a PredictionMode command (all values 4) and 1000 bytes of text: warp-mates with
    different variants reach the mixing values at different nibbles"""
    pre = R._txt(variant, variant + 1, 9000)
    raw = R._txt(variant, 1000, 11000)
    lines = [R.insert(pre[k:k + 1]) for k in range(len(pre))] + [R.pm_line("lsb6"), R.insert(raw)]
    return R._good(oracle, R.from_ir(oracle, lines), pre + raw)


def cmd_nibbles(oracle, lines):
    """command-coder symbols of the stream of these IR lines, without the end-of-stream nibble"""
    rc, out, st = oracle.decode(R.from_ir(oracle, lines), out_cap=1 << 20, stats=True)
    assert rc == 0
    return st["cmd_nibbles"] - 1


@functools.lru_cache(maxsize=None)
def _pm_head(oracle):
    """command nibbles of a PredictionMode command (identity map, random values) before its first mixing value"""
    return cmd_nibbles(oracle, [_pm(0)]) - 8192


@functools.lru_cache(maxsize=None)
def chunk_at(oracle, at):
    """command-coder symbol 65535 falls at mixing value `at` of the last PredictionMode command: the list before it is padded
    with PredictionMode commands and literals of 1 byte (2 command nibbles) or 16 bytes (3 command nibbles)"""
    want = 65535 - _pm_head(oracle) - at                 # command nibbles before the last PredictionMode command
    src = R._txt(0, 40000, 13000)
    lines, pos = [], 0
    while cmd_nibbles(oracle, lines + [R.pm_line("lsb6")]) <= want:
        lines.append(R.pm_line("lsb6"))
    have = cmd_nibbles(oracle, lines)
    if (want - have) % 2:
        lines.append(R.insert(src[pos:pos + 16])); pos += 16
    while len(lines) and cmd_nibbles(oracle, lines) < want:
        n = (want - cmd_nibbles(oracle, lines)) // 2
        lines += [R.insert(src[pos + k:pos + k + 1]) for k in range(n)]; pos += n
    assert cmd_nibbles(oracle, lines) == want
    tail = R._txt(0, 900, 17000)
    lines += [_pm(400 + at), R.insert(tail)]
    return R._good(oracle, R.from_ir(oracle, lines), src[:pos] + tail)


@functools.lru_cache(maxsize=None)
def wasm_2018(oracle, variant=0):
    """(stream, plain) under model revision WASM_2018, where every mixing value is coded with prior slot 16: random values"""
    raw = R._txt(variant, 1200, 21000)
    cl = oracle.Commands.from_ir("window 16 0 0 0\n%s\n%s\n" % (_pm(500 + variant), R.insert(raw)))
    stream = cl.encode(oracle.options(window_size=16, model_rev=oracle.MODEL_WASM_2018))
    rc, plain, _ = oracle.decode_cmds(stream, model_rev=oracle.MODEL_WASM_2018)
    assert rc == 0 and plain == raw
    return cl, stream, raw


def _recode(oracle, stream, cmd_len):
    """`stream` with its command payload cut to cmd_len bytes (one record per coder, the CRC recomputed)"""
    cmd, lit = oracle.demux(stream)
    out = bytearray(stream[:16])
    for coder, pay in ((0, cmd[:cmd_len]), (1, lit)):
        for o in range(0, len(pay), 65536):
            n = min(65536, len(pay) - o)
            out += bytes([coder, (n - 1) & 0xFF, (n - 1) >> 8]) + pay[o:o + n]
    return R.close(oracle, bytes(out))


@functools.lru_cache(maxsize=None)
def truncated(oracle, frac):
    """random_mix with its command payload cut to `frac` of its length: the command coder runs dry inside the mixing values"""
    base = random_mix(oracle, 0)
    cmd = oracle.demux(base.stream)[0]
    s = _recode(oracle, base.stream, int(len(cmd) * frac))
    rc, out = oracle.decode(s, out_cap=base.cap)
    return R.Case(s, out if rc == 0 else None, 0, rc, base.cap)


@functools.lru_cache(maxsize=None)
def bitflip(oracle, seed):
    """random_mix with one bit flipped in the first 80 % of its command payload (the mixing values); CRC not checked"""
    base = random_mix(oracle, 0)
    cmd = oracle.demux(base.stream)[0]
    at = base.stream.find(cmd[:32])
    rng = np.random.default_rng(seed)
    b = bytearray(base.stream)
    b[at + 16 + int(rng.integers(0, len(cmd) * 4 // 5 - 16))] ^= 1 << int(rng.integers(0, 8))
    rc, out = oracle.decode(bytes(b), out_cap=base.cap, skip_crc=True)
    return R.Case(bytes(b), out if rc == 0 else None, R.SKIP_CRC, rc, base.cap)
