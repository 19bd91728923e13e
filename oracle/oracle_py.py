"""ctypes binding of the CPU oracle (oracle/divans_oracle.c).

TEST INFRASTRUCTURE: imported only by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  Nothing under divans_b200/ may import this module.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# "" = the reference's default probability model; "blend" = its feature="blend" build (oracle/oracle_blend.py loads this same
# module a second time with _VARIANT preset: a compile-time switch in the reference, a second library here)
_VARIANT = globals().get("_VARIANT", "")
_LIB_PATH = os.path.join(_HERE, "_build", "libdivans_oracle%s.so" % ("_" + _VARIANT if _VARIANT else ""))

SUCCESS, NEEDS_MORE_INPUT, NEEDS_MORE_OUTPUT, FAILURE = 0, 1, 2, 3


def build(force=False):
    if force or not os.path.exists(_LIB_PATH) or (
        os.path.getmtime(_LIB_PATH) < os.path.getmtime(os.path.join(_HERE, "divans_oracle.c"))
    ):
        subprocess.check_call(["make", "-s", "-C", _HERE], stdout=subprocess.DEVNULL)
    return _LIB_PATH


class Speed(ctypes.Structure):
    _fields_ = [("inc", ctypes.c_int16), ("lim", ctypes.c_int16)]


class Cdf16(ctypes.Structure):
    _fields_ = [("c", ctypes.c_int16 * 16)] + ([("mix_rate", ctypes.c_int32), ("count", ctypes.c_int32)] if _VARIANT == "blend" else [])


class Options(ctypes.Structure):
    _fields_ = [
        ("window_size", ctypes.c_int),
        ("dynamic_context_mixing", ctypes.c_int),
        ("prior_depth", ctypes.c_int),
        ("use_context_map", ctypes.c_int),
        ("force_stride", ctypes.c_int),
        ("have_literal_adaptation", ctypes.c_int),
        ("literal_adaptation", Speed * 4),
        ("model_rev", ctypes.c_int),
    ]


class CmdList(ctypes.Structure):
    _fields_ = [
        ("cmds", ctypes.c_void_p), ("n_cmds", ctypes.c_size_t), ("cap_cmds", ctypes.c_size_t),
        ("lits", ctypes.c_void_p), ("n_lits", ctypes.c_size_t), ("cap_lits", ctypes.c_size_t),
        ("pms", ctypes.c_void_p), ("n_pms", ctypes.c_size_t), ("cap_pms", ctypes.c_size_t),
        ("window", ctypes.c_int),
    ]


class Weights(ctypes.Structure):
    _fields_ = [("w", ctypes.c_int32 * 2), ("mixing_param", ctypes.c_uint8), ("norm", ctypes.c_int16)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        u8p, szp = ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)
        L.dvo_decode.argtypes = [u8p, ctypes.c_size_t, u8p, ctypes.c_size_t, szp, ctypes.c_int]
        L.dvo_decode_ex.argtypes = [u8p, ctypes.c_size_t, u8p, ctypes.c_size_t, szp, ctypes.c_int, szp,
                                    ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]
        L.dvo_decode_cmds.argtypes = [u8p, ctypes.c_size_t, u8p, ctypes.c_size_t, szp, ctypes.c_int, ctypes.c_int,
                                      ctypes.POINTER(CmdList)]
        L.dvo_encode_raw.argtypes = [u8p, ctypes.c_size_t, ctypes.POINTER(Options), u8p, ctypes.c_size_t, szp]
        L.dvo_encode_cmds.argtypes = [ctypes.POINTER(CmdList), ctypes.POINTER(Options), u8p, ctypes.c_size_t, szp]
        L.dvo_parse_ir.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(CmdList)]
        L.dvo_recode.argtypes = [ctypes.POINTER(CmdList), ctypes.c_int, u8p, ctypes.c_size_t, szp]
        L.dvo_lz77_cmds.argtypes = [u8p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(CmdList)]
        L.dvo_cmdlist_serialize.argtypes = [ctypes.POINTER(CmdList), u8p, ctypes.c_size_t]
        L.dvo_cmdlist_serialize.restype = ctypes.c_size_t
        L.dvo_demux.argtypes = [u8p, ctypes.c_size_t, u8p, szp, u8p, szp, szp]
        L.dvo_mux_single.argtypes = [ctypes.c_int, u8p, ctypes.c_size_t, u8p, ctypes.c_size_t]
        L.dvo_mux_single.restype = ctypes.c_size_t
        L.dvo_crc32c.argtypes = [ctypes.c_uint32, u8p, ctypes.c_size_t]
        L.dvo_crc32c.restype = ctypes.c_uint32
        L.dvo_fast_divide.argtypes = [ctypes.c_int32, ctypes.c_int16]
        L.dvo_fast_divide.restype = ctypes.c_int32
        L.dvo_speed_to_u8.argtypes = [ctypes.c_int16]
        L.dvo_speed_to_u8.restype = ctypes.c_uint8
        L.dvo_u8_to_speed.argtypes = [ctypes.c_uint8]
        L.dvo_u8_to_speed.restype = ctypes.c_int16
        L.dvo_dict_word.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, u8p]
        L.dvo_cdf_lookup.argtypes = [ctypes.POINTER(Cdf16), ctypes.c_int16, ctypes.POINTER(ctypes.c_int16), ctypes.POINTER(ctypes.c_int16)]
        L.dvo_cdf_lookup.restype = ctypes.c_uint8
        L.dvo_cdf_sym_start_freq.argtypes = [ctypes.POINTER(Cdf16), ctypes.c_uint8, ctypes.POINTER(ctypes.c_int16), ctypes.POINTER(ctypes.c_int16)]
        L.dvo_cdf_blend.argtypes = [ctypes.POINTER(Cdf16), ctypes.c_uint8, Speed]
        L.dvo_cdf_average.argtypes = [ctypes.POINTER(Cdf16), ctypes.POINTER(Cdf16), ctypes.c_int32, ctypes.POINTER(Cdf16)]
        L.dvo_weights_update.argtypes = [ctypes.POINTER(Weights), ctypes.c_int16, ctypes.c_int16, ctypes.c_int16]
        L.dvo_weights_update_batch.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 8
        L.dvo_cdf_step_batch.argtypes = [ctypes.c_size_t, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 13
        L.dvo_cdf_walk_batch.argtypes = [ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        assert L.dvo_feature_blend() == (1 if _VARIANT == "blend" else 0)
        if _VARIANT == "blend":
            L.dvo_cdf_value.argtypes = [ctypes.POINTER(Cdf16), ctypes.c_uint8]
            L.dvo_cdf_value.restype = ctypes.c_int16
        u64p = ctypes.c_void_p
        L.dvo_decode_batch.argtypes = [u8p, u64p, u64p, u8p, u64p, u64p, u64p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int]
        L.dvo_encode_raw_batch.argtypes = [u8p, u64p, u64p, u8p, u64p, u64p, u64p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int,
                                           ctypes.POINTER(Options), ctypes.c_int, ctypes.c_int, ctypes.c_int]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _as_u8(b):
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b, dtype=np.uint8)
    return np.frombuffer(bytes(b), dtype=np.uint8) if len(b) else np.zeros(0, np.uint8)


MODEL_CURRENT, MODEL_WASM_2018 = 0, 1  # divans_oracle.h "model revisions"


def options(window_size=22, dynamic_context_mixing=0, prior_depth=0, use_context_map=1, force_stride=9,
            literal_adaptation=None, model_rev=MODEL_CURRENT):
    o = Options()
    lib().dvo_options_default(ctypes.byref(o))
    o.window_size, o.dynamic_context_mixing, o.prior_depth = window_size, dynamic_context_mixing, prior_depth
    o.use_context_map, o.force_stride = use_context_map, force_stride
    o.model_rev = model_rev
    if literal_adaptation is not None:
        o.have_literal_adaptation = 1
        for i, (a, b) in enumerate(literal_adaptation):
            o.literal_adaptation[i].inc, o.literal_adaptation[i].lim = a, b
    return o


def crc32c(data, crc=0):
    d = _as_u8(data)
    return lib().dvo_crc32c(crc, _ptr(d), d.size)


def decode(data, out_cap=None, skip_crc=False, stats=False):
    d = _as_u8(data)
    if out_cap is None:
        out_cap = max(1 << 16, d.size * 64)
    out = np.empty(out_cap, np.uint8)
    n = ctypes.c_size_t(0)
    consumed = ctypes.c_size_t(0)
    nc, nl = ctypes.c_uint64(0), ctypes.c_uint64(0)
    rc = lib().dvo_decode_ex(_ptr(d), d.size, _ptr(out), out_cap, ctypes.byref(n), int(skip_crc), ctypes.byref(consumed),
                             ctypes.byref(nc), ctypes.byref(nl))
    res = out[: min(n.value, out_cap)].tobytes()
    if stats:
        return rc, res, dict(consumed=consumed.value, cmd_nibbles=nc.value, lit_nibbles=nl.value)
    return rc, res


def decode_cmds(data, out_cap=None, skip_crc=False, model_rev=MODEL_CURRENT):
    """decode with an explicit model revision; returns (rc, bytes, Commands holding the decoded command list)."""
    d = _as_u8(data)
    if out_cap is None:
        out_cap = max(1 << 16, d.size * 64)
    out = np.empty(out_cap, np.uint8)
    n = ctypes.c_size_t(0)
    cl = Commands()
    rc = lib().dvo_decode_cmds(_ptr(d), d.size, _ptr(out), out_cap, ctypes.byref(n), int(skip_crc), model_rev,
                               ctypes.byref(cl.c))
    return rc, out[: min(n.value, out_cap)].tobytes(), cl


def encode_raw(data, opts=None):
    d = _as_u8(data)
    o = opts or options()
    cap = d.size + d.size // 2 + 65536
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    rc = lib().dvo_encode_raw(_ptr(d), d.size, ctypes.byref(o), _ptr(out), cap, ctypes.byref(n))
    assert rc == SUCCESS, rc
    return out[: n.value].tobytes()


class Commands:
    """An IR command list (owned C object)."""

    def __init__(self):
        self.c = CmdList()
        lib().dvo_cmdlist_init(ctypes.byref(self.c))

    def __del__(self):
        try:
            lib().dvo_cmdlist_free(ctypes.byref(self.c))
        except Exception:
            pass

    @classmethod
    def from_ir(cls, text):
        self = cls()
        t = text if isinstance(text, bytes) else text.encode()
        rc = lib().dvo_parse_ir(t, len(t), ctypes.byref(self.c))
        if rc != SUCCESS:
            raise ValueError("IR parse failed")
        return self

    @classmethod
    def lz77(cls, data, window=16, pred_mode=2, mixing_value=4):
        self = cls()
        d = _as_u8(data)
        lib().dvo_lz77_cmds(_ptr(d), d.size, window, pred_mode, mixing_value, ctypes.byref(self.c))
        return self

    @property
    def window(self):
        return self.c.window

    @property
    def n_cmds(self):
        return self.c.n_cmds

    def encode(self, opts=None, cap=None):
        o = opts or options()
        cap = cap or (self.c.n_lits * 2 + self.c.n_cmds * 16 + (1 << 20))
        out = np.empty(cap, np.uint8)
        n = ctypes.c_size_t(0)
        rc = lib().dvo_encode_cmds(ctypes.byref(self.c), ctypes.byref(o), _ptr(out), cap, ctypes.byref(n))
        if rc != SUCCESS:
            raise ValueError("encode failed rc=%d" % rc)
        return out[: n.value].tobytes()

    def recode(self, window, cap=1 << 24):
        out = np.empty(cap, np.uint8)
        n = ctypes.c_size_t(0)
        rc = lib().dvo_recode(ctypes.byref(self.c), window, _ptr(out), cap, ctypes.byref(n))
        return rc, out[: n.value].tobytes()

    def serialize(self):
        need = lib().dvo_cmdlist_serialize(ctypes.byref(self.c), None, 0)
        out = np.empty(need, np.uint8)
        got = lib().dvo_cmdlist_serialize(ctypes.byref(self.c), _ptr(out), need)
        assert got == need
        return out.tobytes()


def demux(stream):
    """(cmd_payload, lit_payload) of a complete .divans buffer."""
    d = _as_u8(stream)
    cmd = np.empty(d.size, np.uint8)
    lit = np.empty(d.size, np.uint8)
    cl, ll, cons = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_size_t(0)
    body = d[16:]
    rc = lib().dvo_demux(_ptr(body), body.size, _ptr(cmd), ctypes.byref(cl), _ptr(lit), ctypes.byref(ll), ctypes.byref(cons))
    assert rc == SUCCESS, rc
    return cmd[: cl.value].tobytes(), lit[: ll.value].tobytes()


def weights_update_batch(w0, w1, f_cm, f_nb, weighted):
    """codec/weights.rs update of every case (w0[i], w1[i]) with (f_cm, f_nb, weighted)[i]; returns (w0, w1, norm) arrays"""
    w0, w1 = np.ascontiguousarray(w0, np.int32), np.ascontiguousarray(w1, np.int32)
    p0, p1, wt = (np.ascontiguousarray(a, np.int16) for a in (f_cm, f_nb, weighted))
    o0, o1, on = np.empty_like(w0), np.empty_like(w1), np.empty(w0.size, np.int16)
    lib().dvo_weights_update_batch(w0.size, _ptr(w0), _ptr(w1), _ptr(p0), _ptr(p1), _ptr(wt), _ptr(o0), _ptr(o1), _ptr(on))
    return o0, o1, on


def cdf_steps(cdf, speeds, state=None, sym=None, cdf2=None, wts=None):
    """one coded literal nibble per case (dvo_cdf_step_batch): cdf (n, 16) i16, speeds (n, 2, 2) i16 [(stride inc, lim),
    (context-map inc, lim)], state (n,) u64 to decode or sym (n,) to encode, cdf2 (n, 16) and wts (n, 3) = (w0, w1, norm) to
    mix.  Returns a dict of sym, start, freq, state (decode), cdf, and cdf2, wts (mixing)"""
    cdf = np.ascontiguousarray(cdf, np.int16).reshape(-1, 16)
    n, mix, enc = cdf.shape[0], cdf2 is not None, sym is not None
    sp = np.ascontiguousarray(speeds, np.int16).reshape(n, 4)
    c2 = np.ascontiguousarray(cdf2 if mix else np.zeros((n, 16)), np.int16)
    w = np.ascontiguousarray(wts if mix else np.zeros((n, 3)), np.int32)
    st = np.ascontiguousarray(state if not enc else np.zeros(n), np.uint64)
    si = np.ascontiguousarray(sym if enc else np.zeros(n), np.uint8)
    out = dict(sym=np.empty(n, np.uint8), start=np.empty(n, np.int16), freq=np.empty(n, np.int16), state=np.zeros(n, np.uint64),
               cdf=np.empty((n, 16), np.int16), cdf2=np.zeros((n, 16), np.int16), wts=np.zeros((n, 3), np.int32))
    lib().dvo_cdf_step_batch(n, int(mix), int(enc), _ptr(cdf), _ptr(c2), _ptr(w), _ptr(sp), _ptr(st), _ptr(si), _ptr(out["sym"]),
                             _ptr(out["start"]), _ptr(out["freq"]), _ptr(out["state"]), _ptr(out["cdf"]), _ptr(out["cdf2"]), _ptr(out["wts"]))
    return out


def cdf_walks(speeds, syms):
    """symbol walks from the default CDF: speeds (n, 2) i16 (inc, lim), syms (n, steps) u8.  Returns (n, steps + 1, 16) i16:
    the CDF before each step, then the final one (frequentist_cdf.rs:74-85 through dvo_cdf_blend)"""
    sp = np.ascontiguousarray(speeds, np.int16).reshape(-1, 2)
    sy = np.ascontiguousarray(syms, np.uint8).reshape(sp.shape[0], -1)
    tr = np.empty((sp.shape[0], sy.shape[1] + 1, ctypes.sizeof(Cdf16) // 2), np.int16)
    lib().dvo_cdf_walk_batch(sp.shape[0], sy.shape[1], _ptr(sp), _ptr(sy), _ptr(tr))
    return tr[:, :, :16]


def decode_batch(blob, in_off, in_len, out_off, out_cap, n_threads=1, skip_crc=False):
    """blob: uint8 array; offsets/lengths: uint64 arrays.  returns (out array, out_len, status)."""
    blob = _as_u8(blob)
    in_off, in_len = np.ascontiguousarray(in_off, np.uint64), np.ascontiguousarray(in_len, np.uint64)
    out_off, out_cap = np.ascontiguousarray(out_off, np.uint64), np.ascontiguousarray(out_cap, np.uint64)
    n = in_off.size
    total = int((out_off + out_cap).max()) if n else 0
    out = np.zeros(total, np.uint8)
    out_len = np.zeros(n, np.uint64)
    status = np.zeros(n, np.int32)
    lib().dvo_decode_batch(_ptr(blob), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off), _ptr(out_cap), _ptr(out_len),
                           _ptr(status), n, n_threads, int(skip_crc))
    return out, out_len, status


def encode_raw_list(raws, opts=None, pred_mode=0, mixing_value=4):
    """(status, stream or None) per raw byte string: the literal-only encode under the PredictionMode record of (pred_mode,
    mixing_value), status 3 where the encoder refuses a symbol (dvo_encode_raw_batch)"""
    blob = np.frombuffer(b"".join(raws) or b"\0", np.uint8)
    in_len = np.array([len(r) for r in raws], np.uint64)
    in_off = np.concatenate([[0], np.cumsum(in_len)[:-1]]).astype(np.uint64)
    cap = in_len * np.uint64(2) + np.uint64(70000)
    out_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
    out = np.zeros(int(cap.sum()), np.uint8)
    out_len, status = np.zeros(len(raws), np.uint64), np.zeros(len(raws), np.int32)
    o = opts or options()
    lib().dvo_encode_raw_batch(_ptr(blob), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off), _ptr(cap), _ptr(out_len), _ptr(status),
                               len(raws), 1, ctypes.byref(o), 0, pred_mode, mixing_value)
    return [(int(s), out[int(a):int(a) + int(n)].tobytes() if s == 0 else None) for s, a, n in zip(status, out_off, out_len)]


def encode_batch(blob, in_off, in_len, opts=None, n_threads=1, lz77=False, pred_mode=0, mixing_value=4):
    blob = _as_u8(blob)
    in_off, in_len = np.ascontiguousarray(in_off, np.uint64), np.ascontiguousarray(in_len, np.uint64)
    n = in_off.size
    cap = (in_len + in_len // 2 + np.uint64(70000)).astype(np.uint64)
    out_off = np.zeros(n, np.uint64)
    if n:
        out_off[1:] = np.cumsum(cap)[:-1]
    out = np.zeros(int(cap.sum()), np.uint8)
    out_len = np.zeros(n, np.uint64)
    status = np.zeros(n, np.int32)
    o = opts or options()
    lib().dvo_encode_raw_batch(_ptr(blob), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off), _ptr(cap), _ptr(out_len),
                               _ptr(status), n, n_threads, ctypes.byref(o), int(lz77), pred_mode, mixing_value)
    assert (status == 0).all(), status
    return out, out_off, out_len
