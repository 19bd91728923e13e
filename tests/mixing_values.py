"""Stream builders for the mixing values 0..15 of a PredictionMode record and for per-context mixing masks, in every literal
context mode (dv_engine_kernel.cuh mm_cfg and mixval_prior; dv_engine.cuh scan_literal_config; dv2_core.cuh literal_fast_v2).
Same conventions as tests/regimes.py: every builder is oracle-encoded and deterministic and returns a regimes.Case.

The IR grammar caps mixing values at 8 (as the reference's), so each list is built from IR and its masks are then written
with the oracle's dvo_cmdlist_set_mixing (oracle_tally).  Every builder takes the oracle module (oracle_py, or oracle_blend
for a blend-model twin) and the dynamic context mixing option: 0 and 1 code the same stream (force_stride 9 turns 0 into 1,
codec/interface.rs:360-366), 2 codes with the context-map priors, where value 2 reads the stride prior without adapting it
and value 3 clears fast_cm.  tests/test_mixing_values_oracle.py checks on the CPU that each stream is what its name says;
tests/test_gpu_mixing_values.py decodes and encodes them on the GPU."""
import functools

import numpy as np

import mixval_regimes as M
import regimes as R
from oracle_tally import tally_py as T

MODES = ["lsb6", "msb6", "utf8", "sign"]
DCMS = [0, 1, 2]
HALVES = [(2, 9), (9, 2), (3, 15), (1, 12), (0, 8)]
UNIFORM = list(range(9, 16))
MIX = T.MIX_ENTRIES
HIGH, LOW = slice(0, MIX // 2), slice(MIX // 2, MIX)   # entries of high nibbles (< 4096) and of low nibbles (the 4096 bit)

ALL16 = ["all16_" + m for m in MODES]
HALF_NAMES = ["halves_%d_%d" % ab for ab in HALVES]
PER_CONTEXT = ALL16 + HALF_NAMES + ["one_entry", "one_entry_unvisited", "switch"]
UNIFORM_NAMES = ["uniform_%d_%s" % (v, m) for m in MODES for v in UNIFORM]
CODING = ["mv16_0", "mv16_1"] + ["chunk_at_%d" % at for at in M.CHUNK_AT] + ["wasm_2018"]
ALL = PER_CONTEXT + UNIFORM_NAMES + CODING
BLEND_TWINS = ALL16 + ["halves_3_15", "switch", "uniform_9_lsb6", "uniform_15_utf8", "mv16_0"]

FLAG_WASM_2018 = 4                 # the decode flag of model revision WASM_2018 (divans_b200.FLAG_MODEL_WASM_2018)
ODD_ENTRY = 13                     # the value of one_entry's odd entry
UNVISITED = 63 | 15 << 8           # LSB6, identity map: a high nibble after the byte 0xff, which the text never holds
# a literal context map over three block types whose entries reach 255: the mask entries of contexts above 63 are coded with
LMAP = [(i * 37 + (i // 64) * 101 + 3) % 256 for i in range(192)]


def hash16(e):
    """value(e) of the all16 masks: the top nibble of a multiplicative hash"""
    return ((e * 0x9E3779B1) & 0xFFFFFFFF) >> 28


def all16_mask():
    return np.array([hash16(e) for e in range(MIX)], np.uint8)


def halves_mask(a, b):
    m = np.full(MIX, b, np.uint8)
    m[HIGH] = a
    return m


def rich23_mask():
    return np.array([[2, 3, 2, 3, 5][hash16(e) % 5] for e in range(MIX)], np.uint8)


def mv16(seed):
    """random values 0..15, with fixed, different values around entries 254..257 and 8189..8191: the values whose priors
    (mixval_prior: the value 256 entries back) are slots 9..15"""
    m = np.random.default_rng(seed).integers(0, 16, MIX).astype(np.uint8)
    m[254:258] = [9, 15, 3, 12]
    m[8189:8192] = [13, 10, 11]
    return m


def records(n, width, seed):
    """n bytes of `width`-byte records, each column a slow random walk"""
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n].tobytes()


def utf8_text(n, base):
    """Cyrillic UTF-8 text (two-byte sequences) made from the text corpus"""
    src = R._txt(0, n, base)
    return b"".join(chr(0x430 + (c % 26)).encode() if 97 <= c < 123 else bytes([c]) for c in src)[:n]


def mode_input(mode, n, base):
    """the input each mode is meant for: text, UTF-8 text, or 4-byte records for SIGN"""
    if mode == "utf8":
        return utf8_text(n, base)
    if mode == "sign":
        return records(n, 4, base)
    return R._txt(0, n, base)


def _spec(name, oracle):
    """(IR lines, masks: one per PredictionMode record, raw)"""
    if name.startswith("all16_"):
        parts = [R._txt(0, 1500, 101000), utf8_text(1500, 103000), records(1200, 2, 1), records(1200, 4, 2)]
        lines = [R.pm_line(name[6:], lmap=LMAP), R.insert(parts[0]), "ltype 1 1", R.insert(parts[1]), "ltype 2 2", R.insert(parts[2]),
                 "ltype 0 1", R.insert(parts[3])]
        return lines, [all16_mask()], b"".join(parts)
    if name.startswith("halves_"):
        a, b = (int(x) for x in name.split("_")[1:])
        parts = [R._txt(0, 1500, 107000 + 100 * a), records(1000, 4, 3 + b)]
        return [R.pm_line("msb6", lmap=LMAP), R.insert(parts[0]), "ltype 1 1", R.insert(parts[1])], [halves_mask(a, b)], \
            b"".join(parts)
    if name in ("one_entry", "one_entry_unvisited"):
        raw = R._txt(0, 2500, 113000)
        lines = [R.pm_line("lsb6"), R.insert(raw)]
        m = np.full(MIX, 4, np.uint8)
        m[one_entry_index(oracle) if name == "one_entry" else UNVISITED] = ODD_ENTRY
        return lines, [m], raw
    if name == "switch":
        src, lines, raw, masks = R._txt(0, 8000, 117000), [], b"", []
        pos = 0
        for mode, m in (("lsb6", np.full(MIX, 12, np.uint8)), ("msb6", all16_mask()), ("lsb6", np.full(MIX, 4, np.uint8)),
                        ("utf8", rich23_mask())):
            lines.append(R.pm_line(mode)); masks.append(m)
            for n in (1, 5, 11, 40, 3, 200, 12, 7, 90, 2, 13, 300):   # literals below and from the fast loops' 12 bytes
                lines.append(R.insert(src[pos:pos + n])); raw += src[pos:pos + n]; pos += n
        return lines, masks, raw
    if name.startswith("uniform_"):
        v, mode = name.split("_")[1:]
        raw = mode_input(mode, 2000, 121000 + 10 * int(v))
        return [R.pm_line(mode), R.insert(raw)], [np.full(MIX, int(v), np.uint8)], raw
    if name.startswith("mv16_"):
        raw = R._txt(0, 1500, 127000)
        return [R.pm_line("lsb6"), R.insert(raw)], [mv16(600 + int(name[5:]))], raw
    if name == "wasm_2018":
        raw = R._txt(0, 1200, 131000)
        return [R.pm_line("lsb6"), R.insert(raw)], [mv16(700)], raw
    raise KeyError(name)


@functools.lru_cache(maxsize=None)
def one_entry_index(oracle):
    """the high-nibble entry of one_entry's input that codes the most literal bits under uniform 4"""
    raw = R._txt(0, 2500, 113000)
    cl = oracle.Commands.from_ir(_ir([R.pm_line("lsb6"), R.insert(raw)]))
    rc, _cost, bins, _nb = T.tally_cmds_bins(cl, *T.KEEP, blend=R.is_blend(oracle), window_size=16)
    assert rc == 0
    return int(np.argmax(bins[HIGH]))


def _ir(lines, window=16):
    return "window %d 0 0 0\n" % window + "".join(l + "\n" for l in lines)


def command_list(name, oracle):
    """(oracle Commands with the masks written, masks, raw): the list that encode_options(name, dcm) encodes to
    build(name, oracle, dcm).stream"""
    if name.startswith("chunk_at_"):
        # mixval_regimes.chunk_at's list (command symbol 65535 at mixing value `at` of the last record); only the last record's
        # values change, and each value is one command nibble whatever it is, so the symbol stays where it was
        base = M.chunk_at(oracle, int(name[9:]))
        rc, raw, cl = oracle.decode_cmds(base.stream, out_cap=base.cap)
        assert rc == 0
        n = int(cl.c.n_pms)
        masks = [np.frombuffer(R.commands(cl)[1][k]["mixing"], np.uint8).copy() for k in range(n - 1)] + [mv16(800 + int(name[9:]))]
        assert T.cmdlist_set_mixing(cl, n - 1, masks[-1]) == T.SUCCESS
        return cl, masks, raw
    lines, masks, raw = _spec(name, oracle)
    cl = oracle.Commands.from_ir(_ir(lines))
    assert int(cl.c.n_pms) == len(masks)
    for k, m in enumerate(masks):
        assert T.cmdlist_set_mixing(cl, k, m) == T.SUCCESS
    return cl, masks, raw


def encode_options(name, dcm=1):
    """oracle.options(**kw) / divans_b200.encode_options(**kw) arguments of stream `name`"""
    kw = dict(window_size=16, dynamic_context_mixing=dcm)
    if name == "wasm_2018":
        kw["model_rev"] = 1
    return kw


@functools.lru_cache(maxsize=None)
def build(name, oracle, dcm=1):
    """the Case of stream `name` under dynamic context mixing `dcm`; `oracle` is oracle_py, or oracle_blend for the twin"""
    cl, masks, raw = command_list(name, oracle)
    kw = encode_options(name, dcm)
    stream = cl.encode(oracle.options(**kw))
    rc, out, _ = oracle.decode_cmds(stream, out_cap=len(raw) + 64, model_rev=kw.get("model_rev", 0))
    assert rc == 0 and out == raw, name
    return R.Case(stream, out, FLAG_WASM_2018 if name == "wasm_2018" else 0, 0, len(raw) + 64)


def masks_of(blob):
    """the 8192 mixing values of every PredictionMode record of a DVCL blob, as (n_pms, 8192) uint8"""
    h = np.frombuffer(bytes(blob[:32]), np.uint32)
    at = 32 + 20 * int(h[2])
    pmb = 32 + 16384 + 1024 + 8192
    b = np.frombuffer(bytes(blob), np.uint8)
    return np.stack([b[at + k * pmb + pmb - MIX:at + (k + 1) * pmb] for k in range(int(h[3]))]) if h[3] else np.zeros((0, MIX), np.uint8)
