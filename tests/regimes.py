"""Named stream builders, one per regime the v2 decoder branches on (dv2_core.cuh, dv2_kernels.cu, dv_engine_kernel.cuh).

Every builder is oracle-encoded and deterministic and returns a ``Case``: ``stream`` (the .divans bytes), ``raw`` (what it
decodes to, None when it fails), ``flags`` (the decode flags it needs, FLAG_SKIP_CRC for corrupted payloads), plus the
``status`` the oracle reports and the output capacity ``cap`` to decode it with.  ``variant`` picks different text for the
same regime (a "twin" that touches the same priors).  tests/test_regimes.py checks on the CPU that each stream really is what
its name says; tests/test_gpu_slot_state.py sends them through one warp in every combination and succession."""
import collections
import ctypes
import functools
import itertools

import numpy as np

SKIP_CRC = 1
Case = collections.namedtuple("Case", "stream raw flags status cap")

# regimes that decode to their input; FAILING decode to a nonzero status
GOOD = ["lsb6", "msb6", "utf8", "sign", "dcm2", "per_context_mix", "mix2_flat", "wide_speeds", "wide_midstream", "short_literals",
        "lit_quirk_w10", "chunk_restart", "switches", "bt256", "no_predmode", "empty"]
FAILING = ["corrupt_status1", "corrupt_status3", "out_cap_small"]
ALL = GOOD + FAILING


@functools.lru_cache(maxsize=1)
def text():
    from divans_b200 import synth
    return synth.text_corpus(1 << 18)


def _txt(variant, n, base=0):
    o = (base + 7919 * variant) % (len(text()) - n)
    return text()[o:o + n]


def pm_line(mode="lsb6", lmap=None, mix=4, dmap=(0, 1, 2, 3), cm_speeds=None):
    """an IR `prediction` line: identity 64-entry literal map by default, one mixing value (int) or 8192 of them, and
    optionally one (inc, max) pair for both context-map speeds (the stride speeds keep their default)"""
    lmap = list(range(64)) if lmap is None else list(lmap)
    mv = [mix] * 8192 if isinstance(mix, int) else list(mix)
    s = "prediction %s lcontextmap %s dcontextmap %s mixingvalues %s" % (
        mode, " ".join(map(str, lmap)), " ".join(map(str, dmap)), " ".join(map(str, mv)))
    if cm_speeds is not None:
        s += " cmspeedinc %d %d cmspeedmax %d %d" % (cm_speeds[0], cm_speeds[0], cm_speeds[1], cm_speeds[1])
    return s


def insert(data):
    return "insert %d %s" % (len(data), data.hex())


def from_ir(oracle, lines, window=16, **opts):
    ir = "window %d 0 0 0\n" % window + "".join(l + "\n" for l in lines)
    return oracle.Commands.from_ir(ir).encode(oracle.options(window_size=window, **opts))


def _raw_mode(oracle, raw, pred_mode, mixing_value, **opts):
    blob = np.frombuffer(raw, np.uint8)
    out, off, ln = oracle.encode_batch(blob, [0], [len(raw)], oracle.options(**opts), 1, False, pred_mode, mixing_value)
    return out[: int(ln[0])].tobytes()


def _good(oracle, stream, raw=None):
    rc, out = oracle.decode(stream, out_cap=(len(raw) if raw is not None else 1 << 20) + 64)
    assert rc == 0, rc
    assert raw is None or out == raw
    return Case(stream, out, 0, 0, len(out) + 64)


def _corrupt(oracle, base, raw, want_status, seed, coder):
    """flip single bits inside the payload of one coder of `base` (0: commands, 1: literals; located through the oracle's
    demux, so that the mux framing stays intact and the failure happens inside the decoder) until the oracle, CRC skipped,
    reports `want_status` after decoding part of the literals"""
    pay = oracle.demux(base)[coder]
    at = base.find(pay[64:96])
    assert at > 0 and len(pay) > 200
    rng = np.random.default_rng(seed)
    for _ in range(4000):
        b = bytearray(base)
        for _k in range(int(rng.integers(1, 3))):
            b[at + int(rng.integers(len(pay) // 4, len(pay) - 96))] ^= 1 << int(rng.integers(0, 8))
        rc, out, st = oracle.decode(bytes(b), out_cap=len(raw) + 64, skip_crc=True, stats=True)
        if rc == want_status and 1000 < st["lit_nibbles"]:
            return Case(bytes(b), None, SKIP_CRC, rc, len(raw) + 64)
    raise AssertionError("no corruption with status %d found" % want_status)


@functools.lru_cache(maxsize=None)
def build(name, oracle, variant=0):
    t = lambda n, base=0: _txt(variant, n, base)
    if name in ("lsb6", "msb6", "utf8", "sign"):      # plain literals, mixing value 4: T2S (LSB6/MSB6) or global T2 (UTF8/SIGN)
        raw = t(2048)
        return _good(oracle, _raw_mode(oracle, raw, ["lsb6", "msb6", "utf8", "sign"].index(name), 4), raw)
    if name == "dcm2":                                  # dynamic context mixing 2, one mixing value: the mix loop
        raw = t(3000, 5000)
        return _good(oracle, _raw_mode(oracle, raw, 0, 4, dynamic_context_mixing=2), raw)
    if name == "per_context_mix":                       # mixing values per context (lit_cfg < 0): the generic path
        raw = t(3000, 11000)
        mv = [(i * 7 + i // 64) % 9 for i in range(8192)]
        return _good(oracle, from_ir(oracle, [pm_line("lsb6", mix=mv), insert(raw)]), raw)
    if name == "mix2_flat":                             # mixing value 2: the flat prior, never adapted
        raw = t(3000, 17000)
        return _good(oracle, _raw_mode(oracle, raw, 0, 2), raw)
    # wide speeds: context-map speeds that fail speed_is_small (dv_engine.cuh), so the slot's literal priors go untagged.  With
    # dynamic context mixing 0 the context-map priors are never coded with, so the stream still decodes to its input.
    if name == "wide_speeds":                           # from the start
        raw = t(2500, 23000)
        return _good(oracle, from_ir(oracle, [pm_line("lsb6", cm_speeds=WIDE), insert(raw)]), raw)
    if name == "wide_midstream":                        # small speeds and literals first: v2_make_untagged mid-stream
        a, b = t(1500, 29000), t(1500, 31000)
        return _good(oracle, from_ir(oracle, [pm_line("lsb6"), insert(a), pm_line("lsb6", cm_speeds=WIDE), insert(b)]), a + b)
    if name == "short_literals":                        # every literal below the 12 bytes the fast loops want
        src, lines, raw = t(4000, 37000), [pm_line("msb6")], b""
        pos = 0
        for k in range(150):
            n = 1 + k % 11
            lines.append(insert(src[pos:pos + n])); raw += src[pos:pos + n]; pos += n
            if k % 3 == 2:
                lines.append("copy 5 from 3 ctx 0"); raw += bytes(raw[len(raw) - 3 + (j % 3)] for j in range(5))
        return _good(oracle, from_ir(oracle, lines), raw)
    if name == "lit_quirk_w10":                         # window 10: literals that begin within 8 bytes of the ring start
        src, lines, raw = t(6000, 41000), [pm_line("lsb6")], b""
        pos = 0
        for start in (0, 1024 + 3, 2048 + 7, 3072 + 1):
            if len(raw) < start:                        # fill up to `start` with a copy
                n = start - len(raw)
                lines.append("copy %d from 700 ctx 0" % n)
                raw += bytes(raw[len(raw) - 700 + (j % 700)] for j in range(n))
            lines.append(insert(src[pos:pos + 700])); raw += src[pos:pos + 700]; pos += 700
        return _good(oracle, from_ir(oracle, lines, window=10), raw)
    if name == "chunk_restart":                         # one 40000-byte literal: 80000 literal nibbles, a restart in the fast loop
        raw = t(40000, 50000)
        return _good(oracle, oracle.encode_raw(raw, oracle.options(window_size=22)), raw)
    if name == "switches":                              # block switches and LSB6 -> UTF8 -> LSB6 between literals: T2 / T2S rebuilt
        lmap = [(i * 5 + i // 64 * 17) % 40 for i in range(192)]
        lines, raw = [], b""
        parts = [t(400, 61000 + 500 * k) for k in range(7)]
        lines += [pm_line("lsb6", lmap=lmap), insert(parts[0]), "ltype 1 1", insert(parts[1]), "ltype 2 2", insert(parts[2]),
                  pm_line("utf8", lmap=lmap), insert(parts[3]), "ltype 0 1", insert(parts[4]), pm_line("lsb6", lmap=lmap),
                  insert(parts[5]), "ltype 1 1", insert(parts[6])]
        return _good(oracle, from_ir(oracle, lines), b"".join(parts))
    if name == "bt256":                                 # 256 literal block types, the full 16384-byte literal context map
        lmap = [1 + (i * 37 + i // 64 * 11) % 255 for i in range(16384)]   # never 0: a map left behind is visible
        lines, parts = [pm_line("lsb6", lmap=lmap)], []
        for k, bt in enumerate([0, 255, 17, 128, 254, 3]):
            if k:
                lines.append("ltype %d 1" % bt)
            parts.append(t(300, 71000 + 400 * k)); lines.append(insert(parts[-1]))
        return _good(oracle, from_ir(oracle, lines), b"".join(parts))
    if name == "no_predmode":                           # no PredictionMode command at all: a zero map and mask, LSB6
        a, b = t(1200, 81000), t(900, 83000)
        raw = a + a[:300] + b
        return _good(oracle, from_ir(oracle, [insert(a), "copy 300 from %d ctx 0" % len(a), insert(b)]), raw)
    if name == "empty":                                 # no command: only the end-of-stream nibble
        return _good(oracle, from_ir(oracle, []), b"")
    if name == "corrupt_status1":                       # literal payload corrupted: the payload runs dry inside a literal
        raw = t(6000, 91000)
        base = oracle.encode_raw(raw, oracle.options(window_size=16))
        return _corrupt(oracle, base, raw, 1, seed=1 + variant, coder=1)
    if name == "corrupt_status3":                       # command payload corrupted: an invalid command after literals
        raw = t(6000, 91000)
        base = oracle.Commands.lz77(raw, window=16).encode(oracle.options(window_size=16))
        return _corrupt(oracle, base, raw, 3, seed=1 + variant, coder=0)
    if name == "out_cap_small":                         # the output region holds less than the stream decodes to: status 2
        raw = t(3000, 97000)
        return Case(oracle.encode_raw(raw), None, 0, 2, 1000)
    raise KeyError(name)


WIDE = (8192, 8192)    # 4 * (inc + 16) > 0x7fff: not speed_is_small (dv_engine.cuh), yet no i16 counter wraps


# ---- the command list and encoder options behind every GOOD regime (tests/test_gpu_encode.py sends them to the GPU encoder) ----
_RAW_DEFAULT = ("lsb6", "msb6", "utf8", "sign", "mix2_flat", "chunk_restart")   # raw mode, window 22


def encode_options(name):
    """oracle.options(**kw) / divans_b200.encode_options(**kw) arguments that encode command_list(name) to build(name).stream"""
    if name in _RAW_DEFAULT:
        return dict(window_size=22)
    if name == "dcm2":
        return dict(window_size=22, dynamic_context_mixing=2)
    return dict(window_size=10 if name == "lit_quirk_w10" else 16)


def command_list(name, oracle, variant=0):
    """the command list of regime `name` as the oracle decodes it from build(name).stream (a raw-mode regime's list is the
    PredictionMode and literal commands the raw encoder made).  Re-encoded under encode_options(name), it gives the stream
    back byte for byte (tests/test_regimes.py)."""
    case = build(name, oracle, variant)
    rc, out, cl = oracle.decode_cmds(case.stream, out_cap=case.cap)
    assert rc == 0
    return cl


# ---- framing and chunk edges: streams whose mux records or rANS chunks sit exactly on a boundary ----
# (the parameters were found with the oracle; tests/test_regimes.py checks that each stream still has its property)
#   name: (source, offset, length, property)   source "rnd" = random bytes under default options (raw mode),
#   "lz16" = the oracle's LZ77 of the text corpus, window 16
EDGES = {
    "lit4096": ("rnd", 0, 3824, ("lit_payload", 4096)),
    "lit16384": ("rnd", 1, 15178, ("lit_payload", 16384)),
    "lit65536": ("rnd", 3, 60786, ("lit_payload", 65536)),
    "lit69632": ("rnd", 0, 64594, ("lit_payload", 65536 + 4096)),
    "lit81920": ("rnd", 0, 76036, ("lit_payload", 65536 + 16384)),
    "lit131072": ("rnd", 0, 122248, ("lit_payload", 131072)),
    "cmd4096": ("lz16", 0, 16784, ("cmd_payload", 4096)),
    "cmd16384": ("lz16", 0, 59558, ("cmd_payload", 16384)),
    "nib65535": ("lz16", 3, 63352, ("cmd_nibbles", 65535)),
    "nib65536": ("lz16", 2, 63353, ("cmd_nibbles", 65536)),
    "nib65537": ("lz16", 11, 63347, ("cmd_nibbles", 65537)),   # the command coder's last chunk holds 1 symbol
    "both_over": ("both", 0, 125, ("both_over", 131073)),        # both payloads over 131073 bytes: 65536-byte records alternate
}
EDGE_NAMES = list(EDGES)
# The same properties under the blend model (oracle/oracle_blend.py), whose payloads differ in length for the same input: found
# by search_blend_edges below.  The command-nibble edges and both_over keep the parameters of EDGES (nibble counts depend on
# the command list alone).
BLEND_EDGES = {
    "lit4096": ("rnd", 0, 3703, ("lit_payload", 4096)),
    "lit16384": ("rnd", 1, 14855, ("lit_payload", 16384)),
    "lit65536": ("rnd", 3, 57870, ("lit_payload", 65536)),
    "lit69632": ("rnd", 0, 61486, ("lit_payload", 65536 + 4096)),
    "lit81920": ("rnd", 0, 72426, ("lit_payload", 65536 + 16384)),
    "lit131072": ("rnd", 0, 117133, ("lit_payload", 131072)),
    "cmd4096": ("lz16", 0, 16692, ("cmd_payload", 4096)),
    "cmd16384": ("lz16", 0, 59415, ("cmd_payload", 16384)),
    "nib65535": EDGES["nib65535"],
    "nib65536": EDGES["nib65536"],
    "nib65537": EDGES["nib65537"],
    "both_over": EDGES["both_over"],
}


def is_blend(oracle):
    return getattr(oracle, "_VARIANT", "") == "blend"


def edges(oracle):
    """the edge table of `oracle`'s probability model"""
    return BLEND_EDGES if is_blend(oracle) else EDGES


@functools.lru_cache(maxsize=1)
def _rnd():
    return np.random.default_rng(1).integers(0, 256, 400000).astype(np.uint8).tobytes()


@functools.lru_cache(maxsize=1)
def _corpus():
    from divans_b200 import synth
    return synth.text_corpus(1 << 20)


def edge_options(name, oracle=None):
    src = (EDGES if oracle is None else edges(oracle))[name][0]
    return dict(window_size=22) if src == "rnd" else dict(window_size=16)


def _edge_raw(src, off, n):
    if src == "rnd":
        return _rnd()[off:off + n]
    if src == "lz16":
        return _corpus()[off:off + n]
    # "both": n pieces of 5000 text bytes (copy-heavy) and 1000 random bytes (literal-heavy)
    return b"".join(_corpus()[k * 5000:(k + 1) * 5000] + _rnd()[k * 1000:(k + 1) * 1000] for k in range(n))


def edge_measure(oracle, src, off, n):
    """payload lengths and nibble counts of the stream an edge with these parameters makes under `oracle`"""
    raw = _edge_raw(src, off, n)
    if src == "rnd":
        stream = oracle.encode_raw(raw, oracle.options(window_size=22))
    else:
        stream = oracle.Commands.lz77(raw, window=16).encode(oracle.options(window_size=16))
    cmd, lit = oracle.demux(stream)
    rc, out, st = oracle.decode(stream, out_cap=len(raw) + 64, stats=True)
    assert rc == 0 and out == raw
    return dict(cmd_payload=len(cmd), lit_payload=len(lit), cmd_nibbles=st["cmd_nibbles"], lit_nibbles=st["lit_nibbles"])


def edge_has_property(got, prop):
    kind, want = prop
    if kind == "both_over":
        return got["cmd_payload"] > want and got["lit_payload"] > want
    return got[kind] == want


def search_blend_edges(oracle_blend, seed=5, tries=64):
    """the seeded search that found BLEND_EDGES (seconds; not run by the tests).  An edge whose EDGES parameters keep their
    property under the blend model keeps them.  Otherwise, for the EDGES offset and then seeded random offsets below 64, a
    bisection over the length finds the shortest input whose measured payload reaches the target, and the lengths around it
    are tried for an exact hit (payload lengths grow in steps of 4 bytes, and not quite monotonically).  Returns the table."""
    rng = np.random.default_rng(seed)
    table = {}
    for name, (src, off0, n0, prop) in EDGES.items():
        if edge_has_property(edge_measure(oracle_blend, src, off0, n0), prop):
            table[name] = (src, off0, n0, prop)
            continue
        kind, want = prop
        for t in range(tries):
            off = off0 if t == 0 else int(rng.integers(0, 64))
            lo, hi = n0 // 2, n0 * 2
            while lo < hi:
                mid = (lo + hi) // 2
                if edge_measure(oracle_blend, src, off, mid)[kind] >= want:
                    hi = mid
                else:
                    lo = mid + 1
            hit = next((n for n in range(lo - 16, lo + 17) if edge_measure(oracle_blend, src, off, n)[kind] == want), None)
            if hit is not None:
                table[name] = (src, off, hit, prop)
                break
        else:
            raise AssertionError("no blend parameters for edge %s" % name)
    return table


@functools.lru_cache(maxsize=None)
def edge(name, oracle):
    """(Commands, raw, stream) of framing edge `name` under `oracle`'s probability model"""
    src, off, n, _prop = edges(oracle)[name]
    raw = _edge_raw(src, off, n)
    if src == "rnd":
        stream = oracle.encode_raw(raw, oracle.options(**edge_options(name, oracle)))
        cl = oracle.decode_cmds(stream, out_cap=n + 64)[2]
        return cl, raw, stream
    cl = oracle.Commands.lz77(raw, window=16)
    return cl, raw, cl.encode(oracle.options(**edge_options(name, oracle)))


# ---- re-muxing: the same two coder payloads under another record chain ----
def mux_records(oracle, stream, plan):
    """`stream` with its record chain replaced by `plan`, a list of (coder, n, k): n bytes of coder 0 (commands) or 1
    (literals), in a three-byte record (k None) or a one-byte record of code k (n = 1024 << 2k).  Header, EOF marker and
    trailer as the mux writes them (mux.rs:29, codec/mod.rs:541-556); the CRC32C is recomputed by the oracle library."""
    pay = oracle.demux(stream)
    pos = [0, 0]
    out = bytearray(stream[:16])
    for coder, n, k in plan:
        if k is None:
            assert 1 <= n <= 65536
            out += bytes([coder, (n - 1) & 0xFF, (n - 1) >> 8])
        else:
            assert n == 1024 << (2 * k)
            out += bytes([coder | (k << 4)])
        out += pay[coder][pos[coder]:pos[coder] + n]
        pos[coder] += n
    assert pos == [len(pay[0]), len(pay[1])], (pos, len(pay[0]), len(pay[1]))
    return close(oracle, bytes(out))


def close(oracle, body):
    """header + records -> a complete stream: EOF marker, then the trailer with the CRC32C of everything before it"""
    body += b"\xff\xfe\xff"
    return body + oracle.crc32c(body).to_bytes(4, "little") + b"ans~"


def record_chain(stream):
    """the record chain of a well-formed stream as a plan (the inverse of mux_records): [(coder, n, k)]"""
    o, plan = 16, []
    while stream[o] != 0xFF:
        b = stream[o]
        if b < 2:
            n = (stream[o + 1] | stream[o + 2] << 8) + 1
            plan.append((b, n, None)); o += 3 + n
        else:
            k = b >> 4
            plan.append((b & 1, 1024 << (2 * k), k)); o += 1 + (1024 << (2 * k))
    return plan


def record_starts(plan):
    """offset in the stream of every record's first payload byte"""
    o, res = 16, []
    for _coder, n, k in plan:
        o += 3 if k is None else 1
        res.append(o)
        o += n
    return res


def _split(n, sizes):
    """cut n bytes into pieces of the given sizes (cycled), the last piece what is left"""
    out, i = [], 0
    while n:
        t = min(n, sizes[i % len(sizes)])
        out.append(t); n -= t; i += 1
    return out


def layout(name, lens, seed=0):
    """a record plan over payload lengths lens = (commands, literals)"""
    rng = np.random.default_rng(seed)
    if name == "one_byte":                      # every record carries one byte, coders alternating while both last
        q = [[(c, 1, None)] * lens[c] for c in (0, 1)]
        return [r for pair in itertools.zip_longest(*q) for r in pair if r is not None]
    if name == "random":                        # three-byte records of random sizes, coders in random order
        q = [[(c, n, None) for n in _split(lens[c], [int(x) for x in rng.integers(1, 9000, 64)])] for c in (0, 1)]
        return _interleave(q, rng)
    if name == "codes":                         # one-byte codes k = 3, 2, 1 while the payload allows, then a tail
        # (code 0 would be the byte 0x00 / 0x01, which is the first byte of a three-byte record: no stream can carry it)
        q = []
        for c in (0, 1):
            left, recs = lens[c], []
            for k in (3, 2, 1):
                while left >= 1024 << (2 * k) and (k == 1 or rng.random() < 0.7 or left < 2 * (1024 << (2 * k))):
                    recs.append((c, 1024 << (2 * k), k)); left -= 1024 << (2 * k)
            recs += [(c, n, None) for n in _split(left, [777])]
            q.append(recs)
        return _interleave(q, rng)
    if name == "lit_first":                     # every literal record before every command record
        return [(1, n, None) for n in _split(lens[1], [5000])] + [(0, n, None) for n in _split(lens[0], [3000])]
    if name == "align16":                       # sizes 1, 2, ..., 16, 1, ...: record starts at every offset mod 16
        q = [[(c, n, None) for n in _split(lens[c], list(range(1, 17)))] for c in (0, 1)]
        return [r for pair in itertools.zip_longest(*q) for r in pair if r is not None]
    raise KeyError(name)


LAYOUTS = ["one_byte", "random", "codes", "lit_first", "align16"]


def _interleave(q, rng):
    out, i = [], [0, 0]
    while i[0] < len(q[0]) or i[1] < len(q[1]):
        c = int(rng.integers(0, 2))
        if i[c] >= len(q[c]):
            c ^= 1
        out.append(q[c][i[c]]); i[c] += 1
    return out


# ---- one literal prior driven into a state whose CDF element exceeds its max, then coded at that element ----
# Literal speed (8192, 1920) (f8-representable, far outside speed_is_small) wraps the i16 counters of the high-nibble prior.
# The all-zero literal context map with mixing value 0 sends every high nibble to one prior (index_b = index_c = 0,
# codec/literal.rs:154-200).  The bytes were found by a seeded search over random high-nibble walks: the last byte's high
# nibble is coded at element c = 9377 of a CDF whose max is 6, a quotient (c << 15) / max of 51,210,922 (> 2^24, where fp32
# cannot even hold every integer), and every frequency the oracle encoder codes is > 0.
# Dynamic context mixing 2 keeps the same stride prior and walk (the context-map priors take small speeds, or the averaged
# CDF codes a frequency <= 0): a second path through the same prior state, whose frequency for the weights divides by that max.
C_OVER_MAX_BYTES = bytes.fromhex("f50a0918421d1eb063b121b1b416a2a5f4d9884b48d1d58ff66b")
C_OVER_MAX_SPEED = (8192, 1920)
C_OVER_MAX_OPTIONS = {
    "plain": dict(window_size=16, literal_adaptation=[C_OVER_MAX_SPEED] * 4),
    "dcm2": dict(window_size=16, dynamic_context_mixing=2,
                 literal_adaptation=[C_OVER_MAX_SPEED, C_OVER_MAX_SPEED, (16, 8192), (16, 8192)]),
}


def c_over_max(oracle, variant="plain"):
    """(Commands, stream) of the c > max regime: one PredictionMode command, then the literal bytes"""
    ir = "window 16 0 0 0\n%s\n%s\n" % (pm_line("lsb6", lmap=[0] * 64, mix=0), insert(C_OVER_MAX_BYTES))
    cl = oracle.Commands.from_ir(ir)
    return cl, cl.encode(oracle.options(**C_OVER_MAX_OPTIONS[variant]))


def fp32_cdf_div(c, d):
    """the fp32 path cdf_div took for every 0 <= c <= 0x7fff before kernel r2.16, emulated with a correctly rounded reciprocal in
    place of rcp.approx (which cannot be emulated bit for bit)"""
    n = np.uint32((c << 15) & 0xFFFFFFFF)
    q = int(np.uint32(np.float32(n) * (np.float32(1) / np.float32(d))))
    r = (int(n) - q * d) & 0xFFFFFFFF
    r = r - (1 << 32) if r >= 1 << 31 else r
    if r < 0:
        q, r = q - 1, r + d
    return q + 1 if r >= d else q


def search_c_over_max(oracle, seed=3, speed=C_OVER_MAX_SPEED, misdivides=None, trials=20000):
    """the seeded search that found C_OVER_MAX_BYTES (seed 3, trial 19585; about two minutes; not run by the tests).  Random
    64-nibble high-nibble walks under `speed`; at the first nibble coded at an element c above the max with a quotient >= 2^24
    that `misdivides(c, max)` (default: the fp32 emulation above differs from exact division; pass a set of measured
    mismatch pairs to aim at those), up to 20 random low-nibble choices are tried until the oracle encoder accepts the bytes
    under both C_OVER_MAX_OPTIONS.  Returns the bytes, or None."""
    misdivides = misdivides or (lambda c, m: fp32_cdf_div(c, m) != (c << 15) // m)
    rng = np.random.default_rng(seed)
    pm = pm_line("lsb6", lmap=[0] * 64, mix=0)
    for _trial in range(trials):
        hs = rng.integers(0, 16, 64).astype(np.uint8)
        tr = oracle.cdf_walks(np.array([speed], np.int16), hs[None, :])[0].astype(np.int64)
        for k in range(64):
            cdf, h = tr[k], int(hs[k])
            c, m = int(cdf[h]), int(cdf[15])
            if not (0 < m < c <= 0x7FFF and (c << 15) // m >= 1 << 24 and misdivides(c, m)):
                continue
            for _ in range(20):
                data = bytes(int(x) << 4 | int(l) for x, l in zip(hs[:k + 1], rng.integers(0, 16, k + 1)))
                try:
                    for opts in C_OVER_MAX_OPTIONS.values():
                        from_ir(oracle, [pm, insert(data)], **{k: v for k, v in opts.items() if k != "window_size"})
                    return data
                except ValueError:               # the oracle encoder refuses a frequency <= 0
                    continue
            break
    return None


def c_over_max_walk(oracle):
    """the high-nibble prior before each byte (the oracle's dvo_cdf_blend walk), as (n, 16) ints"""
    hs = np.frombuffer(C_OVER_MAX_BYTES, np.uint8) >> 4
    return oracle.cdf_walks(np.array([C_OVER_MAX_SPEED], np.int16), hs[None, :])[0, :-1].astype(np.int64)


def speed_is_small(inc, lim):
    """dv_engine.cuh speed_is_small: adaptive values of a prior with this speed stay inside [0, 0x7fff]"""
    return inc >= 0 and lim >= 0 and lim + inc + 16 <= 0x7FFF and 4 * (inc + 16) <= 0x7FFF


# ---- reading the command list the oracle decoded (oracle/divans_oracle.h dvo_cmd / dvo_predmode) ----
class _Cmd(ctypes.Structure):
    _fields_ = [("type", ctypes.c_uint32), ("a", ctypes.c_uint32), ("b", ctypes.c_uint32), ("c", ctypes.c_uint32), ("d", ctypes.c_uint32)]


class _PredMode(ctypes.Structure):
    _fields_ = [("pred_mode", ctypes.c_uint8), ("is_adv", ctypes.c_uint8), ("has_speeds", ctypes.c_uint8), ("pad", ctypes.c_uint8),
                ("cm_speed", (ctypes.c_uint16 * 2) * 2), ("stride_speed", (ctypes.c_uint16 * 2) * 2),
                ("combined_speed", (ctypes.c_uint16 * 2) * 2), ("lit_map_len", ctypes.c_uint32), ("dist_map_len", ctypes.c_uint32),
                ("lit_map", ctypes.c_uint8 * 16384), ("dist_map", ctypes.c_uint8 * 1024), ("mixing", ctypes.c_uint8 * 8192)]


COPY, DICT, LITERAL, BTYPE_L, BTYPE_C, BTYPE_D, PREDMODE = 1, 2, 3, 4, 5, 6, 7


def commands(cl):
    """(list of (type, a, b, c, d), list of prediction modes as dicts) of an oracle Commands object"""
    c = cl.c
    cmds = (_Cmd * c.n_cmds).from_address(c.cmds) if c.n_cmds else []
    pms = (_PredMode * c.n_pms).from_address(c.pms) if c.n_pms else []
    out_pms = []
    for p in pms:
        out_pms.append(dict(mode=p.pred_mode, lit_map=bytes(p.lit_map[: p.lit_map_len]), mixing=bytes(p.mixing),
                            speeds=[(p.stride_speed[k][0], p.stride_speed[k][1]) for k in range(2)] +
                                   [(p.cm_speed[k][0], p.cm_speed[k][1]) for k in range(2)]))
    return [(x.type, x.a, x.b, x.c, x.d) for x in cmds], out_pms


def literal_starts(cmds):
    """(output position, length) of every literal command"""
    pos, res = 0, []
    for ty, a, b, c, d in cmds:
        if ty == LITERAL:
            res.append((pos, b)); pos += b
        elif ty == COPY:
            pos += b
        elif ty == DICT:
            pos += d
    return res
