"""divans_b200 -- host-side Python mirror of the H100-native divANS engine.

The compute lives in ``lib/libdivans_b200.so`` (hand-written sm_90a CUDA behind a C ABI, see
``include/divans_b200.h``).  This module only loads it and mirrors the reference's operator surface:

* :class:`DivansDecompressorReader`  -- reference ``src/reader.rs:298-320`` (``new(reader, buffer_size, skip_crc, multithread)``)
* :class:`DivansCompressorWriter`    -- reference ``src/writer.rs:267``
* :class:`Engine`                    -- the batch extension (N independent streams per call)

There is NO CPU fallback: if the shared library is missing or no CUDA device can be opened, importing
succeeds (so that CPU-only tooling can introspect symbols) but every compute entry point raises.
"""
import ctypes
import io
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libdivans_b200.so")

DIVANS_SUCCESS, DIVANS_NEEDS_MORE_INPUT, DIVANS_NEEDS_MORE_OUTPUT, DIVANS_FAILURE = 0, 1, 2, 3
FLAG_SKIP_CRC = 1
FLAG_NO_CRC_KERNEL = 2
FLAG_MODEL_WASM_2018 = 4   # include/divans_b200.h: the model revision of the reference-held stream wasm/wasm.html:98-107
MODEL_CURRENT, MODEL_WASM_2018 = 0, 1
FLAG_CDF_BLEND = 8         # include/divans_b200.h: streams coded with the reference's feature="blend" probability model
CDF_FREQUENTIST, CDF_BLEND = 0, 1

# symbols include/divans_b200.h declares (checked by the CPU test-suite)
REFERENCE_FFI_SYMBOLS = [
    "divans_new_decompressor", "divans_new_serial_decompressor", "divans_new_decompressor_with_custom_alloc",
    "divans_decode", "divans_free_decompressor", "divans_decompressor_malloc_u8", "divans_decompressor_free_u8",
    "divans_decompressor_malloc_usize", "divans_decompressor_free_usize", "divans_new_compressor",
    "divans_new_compressor_with_custom_alloc", "divans_set_option", "divans_encode", "divans_encode_flush",
    "divans_free_compressor", "divans_compressor_malloc_u8", "divans_compressor_free_u8",
    "divans_compressor_malloc_usize", "divans_compressor_free_usize",
]
BATCH_SYMBOLS = [
    "divans_b200_create", "divans_b200_destroy", "divans_b200_last_error", "divans_b200_launch_count",
    "divans_b200_last_kernel_ms", "divans_b200_last_main_kernel_ms", "divans_b200_decode_batch_host", "divans_b200_decode_batch_device",
    "divans_b200_synchronize", "divans_b200_encode_options_default", "divans_b200_encode_batch_host",
    "divans_b200_encode_cmds_batch_host", "divans_b200_encode_batch_device", "divans_b200_ir_to_cmds",
    "divans_b200_decode_batch_host_async", "divans_b200_decode_batch_host_wait", "divans_b200_lz77_cmds_batch", "divans_b200_kernel_version", "divans_b200_last_lanes",
    "divans_b200_debug_slot_header", "divans_b200_decode_cmds_batch_host", "divans_b200_decode_cmds_batch_device",
    "divans_b200_encode_cmds_batch_device", "divans_b200_encode_auto_batch_host", "divans_b200_encode_auto_batch_device",
    "divans_b200_encode_cmds_auto_batch_host", "divans_b200_encode_cmds_auto_batch_device",
    "divans_b200_replay_cmds_batch_host", "divans_b200_replay_cmds_batch_device", "divans_b200_lz77_cmds_batch_device",
    "divans_b200_encode_mixmap_batch_host", "divans_b200_encode_mixmap_batch_device", "divans_b200_encode_cmds_mixmap_batch_host",
    "divans_b200_encode_cmds_mixmap_batch_device",
    "divans_b200_encode_speeds_batch_host",
    "divans_b200_encode_speeds_batch_device",
    "divans_b200_encode_cmds_speeds_batch_host",
    "divans_b200_encode_cmds_speeds_batch_device",
    "divans_b200_lz77_cmds_batch_parse", "divans_b200_lz77_cmds_batch_device_parse", "divans_b200_encode_cmds_choose_batch_device",
]
PM_RECORD_BYTES = 32 + 16384 + 1024 + 8192   # one prediction-mode record of a DVCL blob (include/divans_b200.h)


class DivansError(RuntimeError):
    pass


class EncodeOptions(ctypes.Structure):
    _fields_ = [
        ("window_size", ctypes.c_int32), ("dynamic_context_mixing", ctypes.c_int32), ("prior_depth", ctypes.c_int32),
        ("use_context_map", ctypes.c_int32), ("force_stride", ctypes.c_int32), ("have_literal_adaptation", ctypes.c_int32),
        ("literal_adaptation", (ctypes.c_int16 * 2) * 4), ("literal_pred_mode", ctypes.c_int32),
        ("literal_mixing_value", ctypes.c_int32), ("model_rev", ctypes.c_int32), ("cdf_model", ctypes.c_int32),
    ]


class LiteralModel(ctypes.Structure):
    """divans_b200_literal_model: a candidate of encode_auto (literal context mode LSB6=0 MSB6=1 UTF8=2 SIGN=3, mixing value)"""
    _fields_ = [("literal_pred_mode", ctypes.c_int32), ("literal_mixing_value", ctypes.c_int32)]


# encode_auto's default candidates, (pred_mode, mixing_value).  Entry 0 is the encoder's default model, so no stream's cost
# under encode_auto exceeds its cost under the default.  The others are the models that code the survey corpora in the
# fewest bits (tools/auto_probe.py --survey, DESIGN.md section 4); mixing value 2 is left out (it decodes on the generic path).
DEFAULT_LITERAL_MODELS = [(0, 4), (2, 8), (2, 5), (2, 1), (2, 7), (3, 5), (0, 5), (2, 4)]

# DIVANS_B200_LITERAL_MODEL_KEEP: the candidate of the command-list calls (encode_cmds_auto_*, transcode*) that keeps a list's own
# PredictionMode records.  Their default candidates are [LITERAL_MODEL_KEEP] + DEFAULT_LITERAL_MODELS: ties go to the lowest
# index, and a pair whose list would outgrow the encoder's logs costs the maximum, so a list the plain call encodes is encoded,
# and by the tally at no higher cost than under its own records.
LITERAL_MODEL_KEEP = (-1, -1)

# encode_mixmap's default mixing values, chosen per literal context (mixing-mask entry) under the options' context mode.  The
# values the survey corpora pick most per entry (tools/mixmap_probe.py --survey, DESIGN.md section 4, "Per-context mixing
# values"); 4 first, the encoder's default value, so unvisited entries keep it.
DEFAULT_MIXING_VALUES = [4, 5, 8, 1, 7, 0]
MIX_ENTRIES = 8192

# The reference encoder's speed palette (Speed::ENCODER_DEFAULT_PALETTE), (inc, lim) pairs.
LITERAL_SPEED_PALETTE = [(0, 1024), (2, 1024), (1, 128), (1, 16384), (2, 2048), (4, 1024), (8, 8192), (16, 48), (16, 8192), (32, 4096),
                         (64, 16384), (128, 256), (128, 16384), (512, 16384), (1664, 16384)]
# encode_speeds' default candidates: MUD (16, 8192), the speed every stream is coded with otherwise, first, then the palette
# speeds the real-text survey picks (DESIGN.md section 4, "Literal speeds").
DEFAULT_LITERAL_SPEEDS = [(16, 8192), (32, 4096), (64, 16384), (128, 16384), (512, 16384), (1664, 16384)]


class Lz77Parse(ctypes.Structure):
    """divans_b200_lz77_parse: the LZ77 generator's minimum copy (4..32) and lazy lookahead steps (0..2)"""
    _fields_ = [("min_match", ctypes.c_int32), ("lazy", ctypes.c_int32)]


# compress_device's default parses, (min_match, lazy): (4, 0), the generator's own parse, first, so no stream costs more than
# under it; then the parses a greedy survey of the corpora picks (tools/lz77_parse_probe.py --survey, DESIGN.md section 4,
# "Choosing the LZ77 parse").
DEFAULT_LZ77_PARSES = [(4, 0), (7, 2), (10, 2), (6, 2)]


class CAllocator(ctypes.Structure):
    _fields_ = [("alloc_func", ctypes.c_void_p), ("free_func", ctypes.c_void_p), ("opaque", ctypes.c_void_p)]


_lib = None


def load_library():
    """dlopen libdivans_b200.so (raises DivansError if it has not been built: no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DivansError("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (make -C divans_b200/csrc). "
                          "divans_b200 has no CPU implementation." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, sz, u8p = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p
    szp = ctypes.POINTER(ctypes.c_size_t)
    L.divans_b200_create.argtypes = [ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32]
    L.divans_b200_create.restype = vp
    L.divans_b200_destroy.argtypes = [vp]
    L.divans_b200_last_error.argtypes = [vp]
    L.divans_b200_last_error.restype = ctypes.c_char_p
    L.divans_b200_kernel_version.restype = ctypes.c_char_p
    L.divans_b200_last_lanes.argtypes = [vp]
    L.divans_b200_launch_count.argtypes = [vp]
    L.divans_b200_launch_count.restype = ctypes.c_uint64
    L.divans_b200_last_kernel_ms.argtypes = [vp]
    L.divans_b200_last_kernel_ms.restype = ctypes.c_float
    L.divans_b200_last_main_kernel_ms.argtypes = [vp]
    L.divans_b200_last_main_kernel_ms.restype = ctypes.c_float
    L.divans_b200_synchronize.argtypes = [vp]
    L.divans_b200_synchronize.restype = ctypes.c_uint8
    L.divans_b200_debug_slot_header.argtypes = [vp, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32 * 4)]
    L.divans_b200_debug_slot_header.restype = ctypes.c_uint8
    batch = [vp, sz, vp, vp, vp, vp, vp, vp, vp, vp]
    L.divans_b200_decode_batch_host.argtypes = batch + [ctypes.c_uint32]
    L.divans_b200_decode_batch_host.restype = ctypes.c_uint8
    L.divans_b200_decode_batch_host_async.argtypes = batch + [ctypes.c_uint32, ctypes.POINTER(ctypes.c_int32)]
    L.divans_b200_decode_batch_host_async.restype = ctypes.c_uint8
    L.divans_b200_decode_batch_host_wait.argtypes = [vp, ctypes.c_int32]
    L.divans_b200_decode_batch_host_wait.restype = ctypes.c_uint8
    L.divans_b200_decode_batch_device.argtypes = batch + [ctypes.c_uint64, ctypes.c_uint32, vp]
    L.divans_b200_decode_batch_device.restype = ctypes.c_uint8
    L.divans_b200_decode_cmds_batch_host.argtypes = batch[:-2] + [vp, vp, vp, vp, vp, vp, ctypes.c_uint32]
    L.divans_b200_decode_cmds_batch_host.restype = ctypes.c_uint8
    L.divans_b200_decode_cmds_batch_device.argtypes = batch[:-2] + [vp, vp, vp, vp, vp, vp, ctypes.c_uint64, ctypes.c_uint32, vp]
    L.divans_b200_decode_cmds_batch_device.restype = ctypes.c_uint8
    L.divans_b200_encode_options_default.argtypes = [ctypes.POINTER(EncodeOptions)]
    L.divans_b200_encode_batch_host.argtypes = batch + [ctypes.POINTER(EncodeOptions)]
    L.divans_b200_encode_batch_host.restype = ctypes.c_uint8
    L.divans_b200_encode_cmds_batch_host.argtypes = batch + [ctypes.POINTER(EncodeOptions)]
    L.divans_b200_encode_cmds_batch_host.restype = ctypes.c_uint8
    L.divans_b200_encode_batch_device.argtypes = [vp, sz, vp, vp, vp, ctypes.c_uint64, vp, vp, vp, vp, vp, ctypes.POINTER(EncodeOptions), vp]
    L.divans_b200_encode_batch_device.restype = ctypes.c_uint8
    L.divans_b200_encode_cmds_batch_device.argtypes = [vp, sz, vp, vp, vp, ctypes.c_uint64, ctypes.c_uint64, vp, vp, vp, vp, vp,
                                                       ctypes.POINTER(EncodeOptions), vp]
    L.divans_b200_encode_cmds_batch_device.restype = ctypes.c_uint8
    # the selection calls: a batch, the options and k candidates, then the selection's outputs (device calls: and the CUDA stream)
    for stem, n_outs in (("auto", 2), ("mixmap", 4), ("speeds", 3)):
        sel = [ctypes.POINTER(EncodeOptions), vp, ctypes.c_uint32] + [vp] * n_outs
        for cmds in (False, True):
            name = "divans_b200_encode_%s%s_batch_" % ("cmds_" if cmds else "", stem)
            getattr(L, name + "host").argtypes = batch + sel
            getattr(L, name + "device").argtypes = [vp, sz, vp, vp, vp] + [ctypes.c_uint64] * (2 if cmds else 1) + [vp] * 5 + sel + [vp]
            getattr(L, name + "host").restype = getattr(L, name + "device").restype = ctypes.c_uint8
    L.divans_b200_replay_cmds_batch_host.argtypes = batch + [ctypes.c_int32]
    L.divans_b200_replay_cmds_batch_host.restype = ctypes.c_uint8
    L.divans_b200_replay_cmds_batch_device.argtypes = batch + [ctypes.c_int32, vp]
    L.divans_b200_replay_cmds_batch_device.restype = ctypes.c_uint8
    L.divans_b200_ir_to_cmds.argtypes = [ctypes.c_char_p, sz, vp, sz, szp, ctypes.POINTER(ctypes.c_int32)]
    L.divans_b200_ir_to_cmds.restype = ctypes.c_uint8
    L.divans_b200_lz77_cmds_batch.argtypes = [sz, vp, vp, vp, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, vp, sz, vp, vp, szp, ctypes.c_int32]
    L.divans_b200_lz77_cmds_batch.restype = ctypes.c_uint8
    L.divans_b200_lz77_cmds_batch_device.argtypes = [vp, sz, vp, vp, vp, ctypes.c_uint64, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, vp, vp,
                                                     vp, vp, vp, vp]
    L.divans_b200_lz77_cmds_batch_device.restype = ctypes.c_uint8
    L.divans_b200_lz77_cmds_batch_parse.argtypes = L.divans_b200_lz77_cmds_batch.argtypes + [ctypes.POINTER(Lz77Parse)]
    L.divans_b200_lz77_cmds_batch_parse.restype = ctypes.c_uint8
    L.divans_b200_lz77_cmds_batch_device_parse.argtypes = L.divans_b200_lz77_cmds_batch_device.argtypes[:-1] + [ctypes.POINTER(Lz77Parse), vp]
    L.divans_b200_lz77_cmds_batch_device_parse.restype = ctypes.c_uint8
    L.divans_b200_encode_cmds_choose_batch_device.argtypes = [vp, sz, ctypes.c_uint32, vp, vp, vp, ctypes.c_uint64, ctypes.c_uint64, vp, vp, vp,
                                                              vp, vp, ctypes.POINTER(EncodeOptions), vp, vp, vp]
    L.divans_b200_encode_cmds_choose_batch_device.restype = ctypes.c_uint8
    # reference FFI
    L.divans_new_decompressor.restype = vp
    L.divans_new_serial_decompressor.restype = vp
    L.divans_new_decompressor_with_custom_alloc.argtypes = [CAllocator, ctypes.c_uint8, ctypes.c_uint8]
    L.divans_new_decompressor_with_custom_alloc.restype = vp
    L.divans_decode.argtypes = [vp, u8p, sz, szp, u8p, sz, szp]
    L.divans_decode.restype = ctypes.c_uint8
    L.divans_free_decompressor.argtypes = [vp]
    L.divans_new_compressor.restype = vp
    L.divans_set_option.argtypes = [vp, ctypes.c_uint8, ctypes.c_uint32]
    L.divans_set_option.restype = ctypes.c_uint8
    L.divans_encode.argtypes = [vp, u8p, sz, szp, u8p, sz, szp]
    L.divans_encode.restype = ctypes.c_uint8
    L.divans_encode_flush.argtypes = [vp, u8p, sz, szp]
    L.divans_encode_flush.restype = ctypes.c_uint8
    L.divans_free_compressor.argtypes = [vp]
    _lib = L
    return L


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _u8(b):
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b, dtype=np.uint8)
    return np.frombuffer(bytes(b), dtype=np.uint8) if len(b) else np.zeros(0, np.uint8)


def _pack(bufs):
    """Byte strings -> (blob, off, len) of one input blob: each at a 16-byte aligned offset, and 16 bytes of zeros at the end."""
    bufs = [_u8(b) for b in bufs]
    ln = np.array([b.size for b in bufs], np.uint64)
    pad = (ln + np.uint64(15)) & ~np.uint64(15)
    off = np.zeros(len(bufs), np.uint64)
    off[1:] = np.cumsum(pad)[:-1]
    blob = np.zeros(int(pad.sum()) + 16, np.uint8)
    for b, o in zip(bufs, off):
        blob[int(o):int(o) + b.size] = b
    return blob, off, ln


def _regions(caps):
    """Output regions of caps[i] bytes, back to back at 256-byte aligned offsets -> (off, total bytes)."""
    pad = (np.asarray(caps, np.uint64) + np.uint64(255)) & ~np.uint64(255)
    off = np.zeros(pad.size, np.uint64)
    off[1:] = np.cumsum(pad)[:-1]
    return off, int(pad.sum())


def _encoded_cap(in_len):
    """The output region an encode of in_len bytes (raw bytes or a command list) gets: half as much again plus a fixed
    headroom, rounded up to 256 bytes."""
    L = np.asarray(in_len, np.uint64)
    return (L + L // np.uint64(2) + np.uint64(70000 + 255)) & ~np.uint64(255)


def _host_batch(*desc):
    """The descriptor arrays of a host call as contiguous uint64 arrays, then its out_len and status arrays."""
    n = len(desc[0])
    return [np.ascontiguousarray(a, np.uint64) for a in desc] + [np.zeros(n, np.uint64), np.full(n, DIVANS_FAILURE, np.int32)]


def ir_to_cmds(text):
    """Reference IR text (src/bin/divans.rs:191-483) -> (DVCL command-list blob, window size).  Host-side parser of the
    C ABI (divans_b200_ir_to_cmds); feed the blob to ``Engine.encode(..., cmds=True)``."""
    L = load_library()
    t = text if isinstance(text, bytes) else text.encode()
    need, win = ctypes.c_size_t(0), ctypes.c_int32(0)
    rc = L.divans_b200_ir_to_cmds(t, len(t), None, 0, ctypes.byref(need), ctypes.byref(win))
    if rc == DIVANS_FAILURE:
        raise ValueError("IR parse failed")
    out = np.zeros(need.value, np.uint8)
    rc = L.divans_b200_ir_to_cmds(t, len(t), _ptr(out), out.size, ctypes.byref(need), ctypes.byref(win))
    if rc != DIVANS_SUCCESS:
        raise ValueError("IR parse failed")
    return out.tobytes(), int(win.value)


def kernel_version():
    return load_library().divans_b200_kernel_version().decode()


def _parse(parse):
    """(min_match, lazy) -> a Lz77Parse (the C calls refuse one outside min_match 4..32, lazy 0..2)"""
    mm, lz = parse
    return Lz77Parse(int(mm), int(lz))


def lz77_cmds_batch(blob, in_off, in_len, window=16, pred_mode=2, mixing_value=4, n_threads=None, parse=None):
    """Raw buffers -> DVCL command lists by the library's greedy LZ77 (divans_b200_lz77_cmds_batch): returns
    (blobs uint8 array, blob_off, blob_len) ready for Engine.encode_batch_host(..., cmds=True).  ``parse`` (min_match, lazy):
    the parse of divans_b200_lz77_cmds_batch_parse (include/divans_b200.h); None is (4, 0)."""
    L = load_library()
    if parse is not None:
        ps = _parse(parse)
        if not (4 <= ps.min_match <= 32 and 0 <= ps.lazy <= 2):
            raise ValueError("lz77_cmds_batch: parse (%d, %d) is outside min_match 4..32, lazy 0..2" % (ps.min_match, ps.lazy))
        fn = lambda *a: L.divans_b200_lz77_cmds_batch_parse(*a, ctypes.byref(ps))
    else:
        fn = L.divans_b200_lz77_cmds_batch
    blob = _u8(blob)
    in_off, in_len = np.ascontiguousarray(in_off, np.uint64), np.ascontiguousarray(in_len, np.uint64)
    n = len(in_off)
    boff, blen = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    total = ctypes.c_size_t(0)
    nt = int(n_threads or os.cpu_count() or 1)
    rc = fn(n, _ptr(blob), _ptr(in_off), _ptr(in_len), window, pred_mode, mixing_value, None, 0, _ptr(boff), _ptr(blen), ctypes.byref(total), nt)
    if rc != DIVANS_NEEDS_MORE_OUTPUT and not (rc == DIVANS_SUCCESS and total.value == 0):
        raise ValueError("lz77_cmds_batch failed")
    out = np.zeros(max(1, total.value), np.uint8)
    rc = fn(n, _ptr(blob), _ptr(in_off), _ptr(in_len), window, pred_mode, mixing_value, _ptr(out), out.size, _ptr(boff), _ptr(blen),
            ctypes.byref(total), nt)
    if rc != DIVANS_SUCCESS:
        raise ValueError("lz77_cmds_batch failed")
    return out, boff, blen


def lz77_blob_cap(in_len):
    """The blob region that always holds the LZ77 command list of in_len raw bytes (lz77_cmds_batch, and
    Engine.lz77_cmds_batch_device): header, one PredictionMode command and at most 2 + 2 * floor(in_len / 5) Literal / Copy
    commands, the record, and the literal pool, which is the raw bytes.  The count: with a Copies that have a Literal just
    before them and b that do not, there are at most a + 1 Literal runs (never two in a row), and 5a + 4b <= in_len (a Copy
    covers at least 4 bytes, a Literal at least 1), so 2a + b + 1 <= floor(2 in_len / 5) + 1 <= 2 floor(in_len / 5) + 2."""
    L = np.asarray(in_len, np.uint64)
    return np.uint64(32 + PM_RECORD_BYTES) + np.uint64(20) * (np.uint64(3) + np.uint64(2) * (L // np.uint64(5))) + L


def first_blob_cap(out_cap):
    """The blob region decoding to a command list tries first, for streams of up to ``out_cap`` decoded bytes: header, one
    prediction-mode record, every byte a literal byte plus a few commands per 64 bytes.  Lists with more commands than that
    report the exact size they need and are decoded once more."""
    out_cap = np.asarray(out_cap, np.uint64)
    return np.uint64(32 + PM_RECORD_BYTES + 4096) + out_cap + out_cap // np.uint64(4)


def encode_options(**kw):
    o = EncodeOptions()
    load_library().divans_b200_encode_options_default(ctypes.byref(o))
    adapt = kw.pop("literal_adaptation", None)
    for k, v in kw.items():
        setattr(o, k, v)
    if adapt is not None:
        o.have_literal_adaptation = 1
        for i, (a, b) in enumerate(adapt):
            o.literal_adaptation[i][0], o.literal_adaptation[i][1] = a, b
    return o


class Engine:
    """Batch engine bound to one GPU.  ``lanes_per_stream``: 0 = by batch size (16, or 8 where their residency holds the batch in fewer passes; never on an 80 GB H100, whose slot memory caps both), 16 / 8 = the v2
    engine with two / four streams per warp; any other value means 16 (include/divans_b200.h)."""

    def __init__(self, device=0, max_resident=0, lanes_per_stream=0):
        self._L = load_library()
        self._h = self._L.divans_b200_create(int(device), int(max_resident), int(lanes_per_stream))
        if not self._h:
            raise DivansError("divans_b200_create(device=%d) failed: no usable sm_90a CUDA device (no CPU fallback)" % device)
        self.device = device
        self._inflight = {}     # ticket -> every buffer the C side still reads or writes for that pipelined batch

    def close(self):
        if getattr(self, "_h", None):
            self._L.divans_b200_destroy(self._h)   # drains the pipelined batches (their buffers are still referenced here)
            self._h = None
            self._inflight.clear()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- info
    @property
    def launch_count(self):
        return int(self._L.divans_b200_launch_count(self._h))

    def last_lanes(self):
        return int(self._L.divans_b200_last_lanes(self._h))

    def last_kernel_ms(self):
        return float(self._L.divans_b200_last_kernel_ms(self._h))

    def last_main_kernel_ms(self):
        return float(self._L.divans_b200_last_main_kernel_ms(self._h))

    def synchronize(self):
        if self._L.divans_b200_synchronize(self._h) != DIVANS_SUCCESS:
            raise DivansError(self._L.divans_b200_last_error(self._h).decode())

    def _err(self):
        return self._L.divans_b200_last_error(self._h).decode()

    def slot_header(self, i):
        """Tests and diagnostics: the four persistent header words of arena slot ``i`` (include/divans_b200.h,
        divans_b200_debug_slot_header) after the context's last call: [generation counter, untagged-tables flag,
        literal-context-map high-water mark, stale-mixing-mask flag]."""
        out = (ctypes.c_uint32 * 4)()
        if self._L.divans_b200_debug_slot_header(self._h, int(i), ctypes.byref(out)) != DIVANS_SUCCESS:
            raise DivansError("slot_header(%d): %s" % (i, self._err()))
        return [int(v) for v in out]

    # -- host-buffer paths (numpy arrays; `in_blob`/`out` may be pinned)
    def decode_batch_host(self, in_blob, in_off, in_len, out, out_off, out_cap, flags=0):
        n = len(in_off)
        in_off, in_len, out_off, out_cap, out_len, status = _host_batch(in_off, in_len, out_off, out_cap)
        rc = self._L.divans_b200_decode_batch_host(self._h, n, _ptr(in_blob), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off),
                                                   _ptr(out_cap), _ptr(out_len), _ptr(status), flags)
        if rc != DIVANS_SUCCESS:
            raise DivansError("decode_batch_host: " + self._err())
        return out_len, status

    def decode_batch_host_async(self, in_blob, in_off, in_len, out, out_off, out_cap, flags=0):
        """Pipelined host-buffer decode: returns a pending-batch handle; ``handle.wait()`` -> (out_len, status).  At most two
        batches in flight; pass pinned ``in_blob`` / ``out`` (e.g. torch pinned tensors' numpy views) for the copies to
        overlap the kernels of the neighbouring batches."""
        n = len(in_off)
        *keep, out_len, status = _host_batch(in_off, in_len, out_off, out_cap)
        ticket = ctypes.c_int32(-1)
        rc = self._L.divans_b200_decode_batch_host_async(self._h, n, _ptr(in_blob), _ptr(keep[0]), _ptr(keep[1]), _ptr(out), _ptr(keep[2]),
                                                         _ptr(keep[3]), _ptr(out_len), _ptr(status), flags, ctypes.byref(ticket))
        if rc != DIVANS_SUCCESS:
            raise DivansError("decode_batch_host_async: " + self._err())
        eng = self
        # The C side writes out / out_len / status when the batch is retired (wait(), the async call that reuses the lane,
        # or destroy): the engine itself keeps them alive until then, also when the caller drops the handle.
        if ticket.value >= 0:
            eng._inflight[ticket.value] = (keep, in_blob, out, out_len, status)

        class _Pending:
            def wait(self_inner):
                if eng._L.divans_b200_decode_batch_host_wait(eng._h, ticket.value) != DIVANS_SUCCESS:
                    raise DivansError("decode_batch_host_wait: " + eng._err())
                if eng._inflight.get(ticket.value, (None,) * 5)[3] is out_len:
                    del eng._inflight[ticket.value]
                return out_len, status
        return _Pending()

    def decode_batch_device(self, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, n, in_total_bytes, flags=0, stream=None):
        """All arguments are raw device pointers (ints), e.g. ``tensor.data_ptr()``.  Asynchronous."""
        rc = self._L.divans_b200_decode_batch_device(self._h, n, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status,
                                                     int(in_total_bytes), flags, stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("decode_batch_device: " + self._err())

    def decode(self, streams, out_caps, flags=0):
        """Convenience: list of bytes -> list of (status, bytes)."""
        blob, in_off, in_len = _pack(streams)
        out_cap = np.array(out_caps, np.uint64)
        out_off, out_total = _regions(out_cap)
        out = np.zeros(out_total, np.uint8)
        out_len, status = self.decode_batch_host(blob, in_off, in_len, out, out_off, out_cap, flags)
        return [(int(st), out[int(o):int(o) + int(n)].tobytes()) for st, o, n in zip(status, out_off, out_len)]

    # -- decoding to command lists (DVCL blobs, include/divans_b200.h)
    def decode_cmds_batch_host(self, in_blob, in_off, in_len, out, out_off, out_cap, blobs, blob_off, blob_cap, flags=0):
        """decode_batch_host that also records every stream's command list into blobs[blob_off[i] .. +blob_cap[i]): returns
        (out_len, blob_len, status).  Status 2 with blob_len > blob_cap: the blob region was too small, blob_len is the size it
        needs (the stream was still decoded)."""
        n = len(in_off)
        in_off, in_len, out_off, out_cap, blob_off, blob_cap, out_len, status = _host_batch(in_off, in_len, out_off, out_cap, blob_off,
                                                                                            blob_cap)
        blob_len = np.zeros(n, np.uint64)
        rc = self._L.divans_b200_decode_cmds_batch_host(self._h, n, _ptr(in_blob), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off),
                                                        _ptr(out_cap), _ptr(out_len), _ptr(blobs), _ptr(blob_off), _ptr(blob_cap),
                                                        _ptr(blob_len), _ptr(status), flags)
        if rc != DIVANS_SUCCESS:
            raise DivansError("decode_cmds_batch_host: " + self._err())
        return out_len, blob_len, status

    def decode_cmds_batch_device(self, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_blobs, d_blob_off, d_blob_cap,
                                 d_blob_len, d_status, n, in_total_bytes, flags=0, stream=None):
        """decode_cmds_batch_host with raw device pointers (ints).  Asynchronous, like decode_batch_device."""
        rc = self._L.divans_b200_decode_cmds_batch_device(self._h, n, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_cap, d_out_len,
                                                          d_blobs, d_blob_off, d_blob_cap, d_blob_len, d_status, int(in_total_bytes),
                                                          flags, stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("decode_cmds_batch_device: " + self._err())

    def decode_cmds(self, streams, out_caps, flags=0):
        """Convenience: list of .divans bytes -> list of (status, decoded bytes, DVCL blob bytes).  A stream whose blob did not fit
        the first guess is decoded once more with the exact size the first call reported."""
        blob, in_off, in_len = _pack(streams)
        n = in_len.size
        out_cap = np.array(out_caps, np.uint64).reshape(n)
        blob_cap = first_blob_cap(out_cap)
        res = [None] * n
        todo = np.arange(n)
        for attempt in range(2):
            idx = todo
            (out_off, out_total), (blob_off, blobs_total) = _regions(out_cap[idx]), _regions(blob_cap[idx])
            out, blobs = np.zeros(out_total, np.uint8), np.zeros(blobs_total, np.uint8)
            out_len, blob_len, status = self.decode_cmds_batch_host(blob, in_off[idx], in_len[idx], out, out_off, out_cap[idx], blobs,
                                                                   blob_off, blob_cap[idx], flags)
            retry = []
            for k, i in enumerate(idx):
                if status[k] == DIVANS_NEEDS_MORE_OUTPUT and blob_len[k] > blob_cap[i] and attempt == 0:
                    blob_cap[i] = blob_len[k]
                    retry.append(i)
                    continue
                raw = out[int(out_off[k]):int(out_off[k]) + int(out_len[k])].tobytes()
                res[i] = (int(status[k]), raw, blobs[int(blob_off[k]):int(blob_off[k]) + int(blob_len[k])].tobytes() if status[k] == 0 else b"")
            if not retry:
                break
            todo = np.array(retry)
        return res

    def transcode(self, streams, out_caps, opts=None, flags=0, candidates=None):
        """Re-encode .divans streams under other entropy options: decode_cmds (``flags`` as for decode: the model and revision the
        streams were written with), then encode(..., cmds=True) with ``opts`` (encode_options; a window_size of 0, the
        default when ``opts`` is None, keeps each stream's own window).  Returns the new streams; raises DivansError naming the
        first stream that does not decode.  With ``candidates`` (a list, see encode_cmds_auto_batch_host) each list is coded
        under the cheapest of them instead, and the call returns (streams, chosen, cost)."""
        dec = self.decode_cmds(streams, out_caps, flags)
        for i, (st, _, _) in enumerate(dec):
            if st != DIVANS_SUCCESS:
                raise DivansError("transcode: stream %d does not decode (status %d)" % (i, st))
        o = opts if opts is not None else encode_options(window_size=0)
        wins = [int(np.frombuffer(b[20:24], np.uint32)[0]) if o.window_size == 0 else int(o.window_size) for _, _, b in dec]
        auto = candidates is not None
        res = [None] * len(dec)
        chosen = np.zeros(len(dec), np.uint32)
        cost = np.zeros((len(dec), len(candidates) if auto else 0), np.uint64)
        for w in sorted(set(wins)):
            idx = [i for i, x in enumerate(wins) if x == w]
            ow = EncodeOptions.from_buffer_copy(o)
            ow.window_size = w
            st, outs, *sel = self._encode_lists([dec[i][2] for i in idx], ow, True, *((self._auto_host, candidates) if auto else ()))
            if (st != 0).any():
                raise DivansError("encode failed for streams %s" % np.array(idx)[np.nonzero(st)[0][:8]])
            for k, i in enumerate(idx):
                res[i] = outs[k]
            if auto:
                chosen[idx], cost[idx] = sel
        return (res, chosen, cost) if auto else res

    def encode_batch_host(self, in_blob, in_off, in_len, out, out_off, out_cap, opts=None, cmds=False):
        n = len(in_off)
        in_off, in_len, out_off, out_cap, out_len, status = _host_batch(in_off, in_len, out_off, out_cap)
        o = opts or encode_options()
        fn = self._L.divans_b200_encode_cmds_batch_host if cmds else self._L.divans_b200_encode_batch_host
        rc = fn(self._h, n, _ptr(in_blob), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off), _ptr(out_cap), _ptr(out_len),
                _ptr(status), ctypes.byref(o))
        if rc != DIVANS_SUCCESS:
            raise DivansError("encode_batch_host: " + self._err())
        return out_len, status

    def encode_batch_device(self, n, d_in, d_in_off, d_in_len, max_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, opts=None,
                            stream=None):
        """All arguments are raw device pointers (ints).  Asynchronous on ``stream``."""
        o = opts or encode_options()
        rc = self._L.divans_b200_encode_batch_device(self._h, n, d_in, d_in_off, d_in_len, int(max_in_len), d_out, d_out_off, d_out_cap,
                                                     d_out_len, d_status, ctypes.byref(o), stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("encode_batch_device: " + self._err())

    @staticmethod
    def _cands(candidates, cmds=False):
        cs = candidates if candidates is not None else [LITERAL_MODEL_KEEP] + DEFAULT_LITERAL_MODELS if cmds else DEFAULT_LITERAL_MODELS
        arr = (LiteralModel * max(1, len(cs)))()
        for i, (pm, mv) in enumerate(cs):
            arr[i].literal_pred_mode, arr[i].literal_mixing_value = int(pm), int(mv)
        return arr, len(cs)

    def _select_host(self, stem, cmds, in_blob, in_off, in_len, out, out_off, out_cap, opts, cands, k, outs):
        """The host call of selection ``stem`` (auto, mixmap or speeds; ``cmds``: its command-list call) with the candidates
        ``cands`` (a pointer), ``k`` of them, and the output arrays ``outs`` (None: not wanted).  Returns (out_len, status)."""
        name = "encode_%s%s" % ("cmds_" if cmds else "", stem)
        n = len(in_off)
        in_off, in_len, out_off, out_cap, out_len, status = _host_batch(in_off, in_len, out_off, out_cap)
        rc = getattr(self._L, "divans_b200_%s_batch_host" % name)(
            self._h, n, _ptr(in_blob), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off), _ptr(out_cap), _ptr(out_len), _ptr(status),
            ctypes.byref(opts or encode_options()), cands, k, *(None if a is None else _ptr(a) for a in outs))
        if rc != DIVANS_SUCCESS:
            raise DivansError("%s_batch_host: %s" % (name, self._err()))
        return out_len, status

    def _select_device(self, stem, cmds, batch, opts, cands, k, outs, stream):
        """The device call of selection ``stem`` on ``batch`` (its arguments from n to d_status) with device outputs ``outs``."""
        name = "encode_%s%s" % ("cmds_" if cmds else "", stem)
        rc = getattr(self._L, "divans_b200_%s_batch_device" % name)(self._h, *batch, ctypes.byref(opts or encode_options()), cands, k, *outs,
                                                                    stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("%s_batch_device: %s" % (name, self._err()))

    def _auto_host(self, cmds, in_blob, in_off, in_len, out, out_off, out_cap, opts, candidates):
        cands, nc = self._cands(candidates, cmds)
        chosen, cost = np.zeros(len(in_off), np.uint32), np.zeros((len(in_off), nc), np.uint64)
        return self._select_host("auto", cmds, in_blob, in_off, in_len, out, out_off, out_cap, opts, ctypes.addressof(cands), nc,
                                 (chosen, cost)) + (chosen, cost)

    def encode_auto_batch_host(self, in_blob, in_off, in_len, out, out_off, out_cap, opts=None, candidates=None):
        """encode_batch_host with each stream's literal model chosen among ``candidates`` ((pred_mode, mixing_value) pairs,
        default DEFAULT_LITERAL_MODELS) by its coding cost.  Returns (out_len, status, chosen, cost): cost[i, c] is stream i's
        cost under candidate c in 1/65536 bit (2**64 - 1 where that pass failed)."""
        return self._auto_host(False, in_blob, in_off, in_len, out, out_off, out_cap, opts, candidates)

    def encode_cmds_auto_batch_host(self, blobs, blob_off, blob_len, out, out_off, out_cap, opts=None, candidates=None):
        """encode_batch_host(..., cmds=True) with each command list coded under the cheapest of ``candidates``: (pred_mode,
        mixing_value) pairs whose PredictionMode record replaces every record of the list, or LITERAL_MODEL_KEEP for the list's
        own (default [LITERAL_MODEL_KEEP] + DEFAULT_LITERAL_MODELS).  Returns (out_len, status, chosen, cost) as
        encode_auto_batch_host; stream i equals encode_batch_host(..., cmds=True) on the list under candidate chosen[i]."""
        return self._auto_host(True, blobs, blob_off, blob_len, out, out_off, out_cap, opts, candidates)

    def encode_auto_batch_device(self, n, d_in, d_in_off, d_in_len, max_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, d_chosen,
                                 d_cost=None, opts=None, candidates=None, stream=None):
        """encode_auto_batch_host with raw device pointers (ints; d_chosen u32 [n], d_cost u64 [n * C] or None).  Asynchronous
        on ``stream``."""
        cands, nc = self._cands(candidates)
        self._select_device("auto", False, (n, d_in, d_in_off, d_in_len, int(max_in_len), d_out, d_out_off, d_out_cap, d_out_len, d_status), opts,
                            ctypes.addressof(cands), nc, (d_chosen, d_cost), stream)

    def encode_cmds_auto_batch_device(self, n, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap,
                                      d_out_len, d_status, d_chosen, d_cost=None, opts=None, candidates=None, stream=None):
        """encode_cmds_batch_device with each list coded under the cheapest of ``candidates`` (as encode_cmds_auto_batch_host;
        d_chosen u32 [n], d_cost u64 [n * C] or None).  Asynchronous on ``stream``."""
        cands, nc = self._cands(candidates, cmds=True)
        self._select_device("auto", True, (n, d_blobs, d_blob_off, d_blob_len, int(max_blob_len), int(max_raw_len), d_out, d_out_off, d_out_cap,
                                           d_out_len, d_status), opts, ctypes.addressof(cands), nc, (d_chosen, d_cost), stream)

    def _encode_lists(self, bufs, opts, cmds, host=None, *args):
        """Byte strings (raw, or command lists with ``cmds``) through encode_batch_host, or through the selection's host call
        ``host`` (_auto_host, _mixmap_host or _speeds_host, with ``args`` after the options): (status, list of bytes or None,
        then the selection's other results)."""
        blob, in_off, in_len = _pack(bufs)
        out_cap = _encoded_cap(in_len)
        out_off, out_total = _regions(out_cap)
        out = np.zeros(out_total, np.uint8)
        if host is None:
            out_len, status, *rest = self.encode_batch_host(blob, in_off, in_len, out, out_off, out_cap, opts, cmds)
        else:
            out_len, status, *rest = host(cmds, blob, in_off, in_len, out, out_off, out_cap, opts, *args)
        return (status, [out[int(o):int(o) + int(n)].tobytes() if s == DIVANS_SUCCESS else None for s, o, n in zip(status, out_off, out_len)],
                *rest)

    def encode_auto(self, raws, opts=None, candidates=None):
        """Convenience: list of raw byte strings -> list of (status, .divans bytes or None, chosen candidate index)."""
        status, outs, chosen, _ = self._encode_lists(raws, opts, False, self._auto_host, candidates)
        return [(int(s), b, int(c)) for s, b, c in zip(status, outs, chosen)]

    def encode_cmds_auto(self, blobs, opts=None, candidates=None):
        """Convenience: list of DVCL command-list blobs -> list of (status, .divans bytes or None, chosen candidate index), each
        list coded under the cheapest of ``candidates`` (encode_cmds_auto_batch_host)."""
        status, outs, chosen, _ = self._encode_lists(blobs, opts, True, self._auto_host, candidates)
        return [(int(s), b, int(c)) for s, b, c in zip(status, outs, chosen)]

    # ---- per-context mixing values (include/divans_b200.h) ----
    @staticmethod
    def _values(values):
        v = np.ascontiguousarray(DEFAULT_MIXING_VALUES if values is None else values, np.int32)
        return (v if v.size else np.zeros(1, np.int32)), int(v.size)

    def _mixmap_host(self, cmds, in_blob, in_off, in_len, out, out_off, out_cap, opts, values, want_bins):
        n = len(in_off)
        v, k = self._values(values)
        chosen, mixing, cost = np.zeros(n, np.uint32), np.zeros((n, MIX_ENTRIES), np.uint8), np.zeros((n, k + 1), np.uint64)
        bins = np.zeros((n, k, MIX_ENTRIES), np.uint64) if want_bins else None
        return self._select_host("mixmap", cmds, in_blob, in_off, in_len, out, out_off, out_cap, opts, _ptr(v), k,
                                 (chosen, mixing, cost, bins)) + (chosen, mixing, cost, bins)

    def encode_mixmap_batch_host(self, in_blob, in_off, in_len, out, out_off, out_cap, opts=None, values=None, bins=False):
        """encode_batch_host with each stream's mixing values chosen per literal context among ``values`` (default
        DEFAULT_MIXING_VALUES) under opts.literal_pred_mode.  Returns (out_len, status, chosen, mixing [n, 8192], cost [n, k + 1],
        bins [n, k, 8192] or None): chosen[i] == k is the mixed record, cost[i] = the k uniform costs then the mixed one."""
        return self._mixmap_host(False, in_blob, in_off, in_len, out, out_off, out_cap, opts, values, bins)

    def encode_cmds_mixmap_batch_host(self, blobs, blob_off, blob_len, out, out_off, out_cap, opts=None, values=None, bins=False):
        """encode_mixmap_batch_host for command lists: every PredictionMode record of a list is replaced."""
        return self._mixmap_host(True, blobs, blob_off, blob_len, out, out_off, out_cap, opts, values, bins)

    def encode_mixmap_batch_device(self, n, d_in, d_in_off, d_in_len, max_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status,
                                   d_chosen=None, d_mixing=None, d_cost=None, d_bins=None, opts=None, values=None, stream=None):
        """encode_mixmap_batch_host with raw device pointers (ints, or None for an output not wanted).  Asynchronous."""
        v, k = self._values(values)
        self._select_device("mixmap", False, (n, d_in, d_in_off, d_in_len, int(max_in_len), d_out, d_out_off, d_out_cap, d_out_len, d_status),
                            opts, _ptr(v), k, (d_chosen, d_mixing, d_cost, d_bins), stream)

    def encode_cmds_mixmap_batch_device(self, n, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap,
                                        d_out_len, d_status, d_chosen=None, d_mixing=None, d_cost=None, d_bins=None, opts=None, values=None,
                                        stream=None):
        """encode_cmds_mixmap_batch_host with raw device pointers (ints, or None for an output not wanted).  Asynchronous."""
        v, k = self._values(values)
        self._select_device("mixmap", True, (n, d_blobs, d_blob_off, d_blob_len, int(max_blob_len), int(max_raw_len), d_out, d_out_off, d_out_cap,
                                             d_out_len, d_status), opts, _ptr(v), k, (d_chosen, d_mixing, d_cost, d_bins), stream)

    def encode_mixmap(self, raws, opts=None, values=None):
        """Convenience: list of raw byte strings -> list of (status, .divans bytes or None, chosen): chosen < k is the uniform
        value values[chosen], k the per-context record (encode_mixmap_batch_host)."""
        status, outs, chosen, _, _, _ = self._encode_lists(raws, opts, False, self._mixmap_host, values, False)
        return [(int(s), b, int(c)) for s, b, c in zip(status, outs, chosen)]

    def encode_cmds_mixmap(self, blobs, opts=None, values=None):
        """Convenience: encode_mixmap for DVCL command-list blobs (encode_cmds_mixmap_batch_host)."""
        status, outs, chosen, _, _, _ = self._encode_lists(blobs, opts, True, self._mixmap_host, values, False)
        return [(int(s), b, int(c)) for s, b, c in zip(status, outs, chosen)]

    # ---- literal speeds (include/divans_b200.h) ----
    @staticmethod
    def _speeds(values):
        v = np.ascontiguousarray(DEFAULT_LITERAL_SPEEDS if values is None else values, np.int16).reshape(-1, 2)
        return (v if v.size else np.zeros((1, 2), np.int16)), int(v.shape[0])

    def _speeds_host(self, cmds, in_blob, in_off, in_len, out, out_off, out_cap, opts, values):
        n = len(in_off)
        v, k = self._speeds(values)
        chosen, cost, halves = np.zeros((n, 3), np.uint32), np.zeros((n, k + 1), np.uint64), np.zeros((n, k, 2), np.uint64)
        return self._select_host("speeds", cmds, in_blob, in_off, in_len, out, out_off, out_cap, opts, _ptr(v), k,
                                 (chosen, cost, halves)) + (chosen, cost, halves)

    def encode_speeds_batch_host(self, in_blob, in_off, in_len, out, out_off, out_cap, opts=None, values=None):
        """encode_batch_host with each stream's literal speeds chosen among ``values`` ((inc, lim) pairs, default
        DEFAULT_LITERAL_SPEEDS).  Returns (out_len, status, chosen [n, 3], cost [n, k + 1], halves [n, k, 2]): stream i is coded
        with literal_adaptation (v[a], v[a], v[b], v[c]) for (a, b, c) = chosen[i]."""
        return self._speeds_host(False, in_blob, in_off, in_len, out, out_off, out_cap, opts, values)

    def encode_cmds_speeds_batch_host(self, blobs, blob_off, blob_len, out, out_off, out_cap, opts=None, values=None):
        """encode_speeds_batch_host for command lists: the speeds override every record's."""
        return self._speeds_host(True, blobs, blob_off, blob_len, out, out_off, out_cap, opts, values)

    def encode_speeds_batch_device(self, n, d_in, d_in_off, d_in_len, max_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status,
                                   d_chosen=None, d_cost=None, d_halves=None, opts=None, values=None, stream=None):
        """encode_speeds_batch_host with raw device pointers (ints, or None for an output not wanted).  Asynchronous."""
        v, k = self._speeds(values)
        self._select_device("speeds", False, (n, d_in, d_in_off, d_in_len, int(max_in_len), d_out, d_out_off, d_out_cap, d_out_len, d_status),
                            opts, _ptr(v), k, (d_chosen, d_cost, d_halves), stream)

    def encode_cmds_speeds_batch_device(self, n, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap,
                                        d_out_len, d_status, d_chosen=None, d_cost=None, d_halves=None, opts=None, values=None, stream=None):
        """encode_cmds_speeds_batch_host with raw device pointers (ints, or None for an output not wanted).  Asynchronous."""
        v, k = self._speeds(values)
        self._select_device("speeds", True, (n, d_blobs, d_blob_off, d_blob_len, int(max_blob_len), int(max_raw_len), d_out, d_out_off, d_out_cap,
                                             d_out_len, d_status), opts, _ptr(v), k, (d_chosen, d_cost, d_halves), stream)

    def _speeds_lists(self, bufs, opts, cmds, values):
        status, outs, chosen, cost, _ = self._encode_lists(bufs, opts, cmds, self._speeds_host, values)
        v, _ = self._speeds(values)
        res = []
        for i, (s, b) in enumerate(zip(status, outs)):
            a, b2, c = (int(x) for x in chosen[i])
            res.append((int(s), b, [tuple(int(x) for x in v[j]) for j in (a, a, b2, c)], [int(x) for x in cost[i]]))
        return res

    def encode_speeds(self, raws, opts=None, values=None):
        """Convenience: list of raw byte strings -> list of (status, .divans bytes or None, speeds, cost): speeds = the four
        (inc, lim) literal speeds the stream was coded with, cost = its k uniform costs then the verify cost
        (encode_speeds_batch_host)."""
        return self._speeds_lists(raws, opts, False, values)

    def encode_cmds_speeds(self, blobs, opts=None, values=None):
        """Convenience: encode_speeds for DVCL command-list blobs (encode_cmds_speeds_batch_host)."""
        return self._speeds_lists(blobs, opts, True, values)

    def encode_cmds_batch_device(self, n, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap, d_out_len,
                                 d_status, opts=None, stream=None):
        """encode_batch_host(..., cmds=True) with raw device pointers (ints): command lists resident in HBM, blob offsets 4-byte
        aligned.  ``max_blob_len`` >= every blob length sizes the symbol logs, ``max_raw_len`` >= every list's decoded length the
        replay window; a ``window_size`` of 0 takes each list's own window.  Asynchronous on ``stream``."""
        o = opts or encode_options()
        rc = self._L.divans_b200_encode_cmds_batch_device(self._h, n, d_blobs, d_blob_off, d_blob_len, int(max_blob_len), int(max_raw_len), d_out,
                                                          d_out_off, d_out_cap, d_out_len, d_status, ctypes.byref(o), stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("encode_cmds_batch_device: " + self._err())

    def transcode_device(self, d_in, in_off, in_len, out_caps, opts=None, flags=0, stream=None, candidates=None):
        """transcode without leaving the GPU: ``d_in`` is a CUDA uint8 tensor of concatenated .divans streams, stream i at
        in_off[i] .. +in_len[i] (host arrays), decoding to at most out_caps[i] bytes.  decode_cmds_batch_device then
        encode_cmds_batch_device on one CUDA stream, ordered after the work queued on ``stream`` (a torch.cuda.Stream, default
        the current one), the command
        lists staying in a device tensor.  Streams whose list did not fit the first guess (first_blob_cap) run once more with
        the exact size.  Returns (d_new, new_off, new_len, status): a CUDA uint8 tensor holding the re-encoded streams and host
        arrays; status[i] is the decode status where that failed, else the encode status.  ``opts`` as for transcode.
        With ``candidates`` (a list) the encode step is encode_cmds_auto_batch_device, and the call returns (d_new, new_off,
        new_len, status, chosen, cost) with chosen [n] and cost [n, C] host arrays (a stream that did not decode: every pass
        failed, chosen 0)."""
        import torch
        n = len(in_off)
        in_off, in_len = np.ascontiguousarray(in_off, np.uint64).reshape(n), np.ascontiguousarray(in_len, np.uint64).reshape(n)
        out_cap = np.array(out_caps, np.uint64).reshape(n)
        o = opts if opts is not None else encode_options(window_size=0)
        dev = d_in.device
        # the calls run on a stream of their own, ordered after the work already queued on `stream` (a default stream has no
        # handle the library could take: NULL would mean the context's stream)
        caller = stream if stream is not None else torch.cuda.current_stream(dev)
        s = torch.cuda.Stream(dev)
        s.wait_stream(caller)
        u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev, non_blocking=False)
        self.last_transcode_retried = 0
        auto = candidates is not None
        nc = len(candidates) if auto else 0
        if n == 0:
            empty = torch.zeros(0, dtype=torch.uint8, device=dev), np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.int32)
            return empty + (np.zeros(0, np.uint32), np.zeros((0, nc), np.uint64)) if auto else empty

        def run(idx, blob_cap, d_new=None):
            """decode + encode of streams idx on the device, one synchronisation: (d_new, new_off, new_len, status, blob_len,
            decode status, chosen, cost).  The new streams go to `d_new` when given (at least the total of
            _regions(_encoded_cap(blob_cap)) bytes)."""
            m = len(idx)
            ocap, bcap = out_cap[idx], blob_cap
            new_cap = _encoded_cap(bcap)
            (out_off, out_total), (blob_off, blobs_total), (new_off, new_total) = _regions(ocap), _regions(bcap), _regions(new_cap)
            with torch.cuda.stream(s):
                d_meta = u64(np.concatenate([in_off[idx], in_len[idx], out_off, ocap, blob_off, bcap, new_off, new_cap]))
                M = [d_meta[k * m:(k + 1) * m] for k in range(8)]
                d_out = torch.empty(out_total, dtype=torch.uint8, device=dev)
                d_blobs = torch.empty(blobs_total, dtype=torch.uint8, device=dev)
                if d_new is None:
                    d_new = torch.empty(new_total, dtype=torch.uint8, device=dev)
                # out_len | blob_len | new_len | both statuses (| candidates: cost [m * C] | chosen)
                d_res = torch.zeros((4 + (nc + 1 if auto else 0)) * m, dtype=torch.int64, device=dev)
                d_st = d_res[3 * m:4 * m].view(torch.int32)
                d_dec_st, d_enc_st = d_st[:m], d_st[m:]
                self.decode_cmds_batch_device(d_in.data_ptr(), M[0].data_ptr(), M[1].data_ptr(), d_out.data_ptr(), M[2].data_ptr(), M[3].data_ptr(),
                                              d_res.data_ptr(), d_blobs.data_ptr(), M[4].data_ptr(), M[5].data_ptr(), d_res[m:].data_ptr(),
                                              d_dec_st.data_ptr(), m, int(in_len[idx].sum()), flags, s.cuda_stream)
                # a stream that did not decode reaches the encoder with no blob (status 2's blob_len is larger than its region)
                d_enc_len = torch.where(d_dec_st == 0, d_res[m:2 * m], torch.zeros_like(d_res[m:2 * m]))
                enc = (m, d_blobs.data_ptr(), M[4].data_ptr(), d_enc_len.data_ptr(), int(bcap.max()), int(ocap.max()), d_new.data_ptr(),
                       M[6].data_ptr(), M[7].data_ptr(), d_res[2 * m:].data_ptr(), d_enc_st.data_ptr())
                if auto:
                    self.encode_cmds_auto_batch_device(*enc, d_res[(4 + nc) * m:].data_ptr(), d_res[4 * m:(4 + nc) * m].data_ptr(), o,
                                                       candidates, s.cuda_stream)
                else:
                    self.encode_cmds_batch_device(*enc, o, s.cuda_stream)
                res = d_res.cpu()   # (the one synchronisation of the pass)
            r = res.numpy()
            st = r[3 * m:4 * m].view(np.int32)
            dec_st, enc_st = st[:m], st[m:]
            chosen = r[(4 + nc) * m:].view(np.uint32)[:m].copy() if auto else None
            cost = r[4 * m:(4 + nc) * m].view(np.uint64).reshape(m, nc).copy() if auto else None
            return d_new, new_off, r[2 * m:3 * m].view(np.uint64).copy(), np.where(dec_st != 0, dec_st, enc_st).astype(np.int32), \
                r[m:2 * m].view(np.uint64).copy(), dec_st.copy(), chosen, cost

        cap1 = first_blob_cap(out_cap)
        d_new, new_off, new_len, status, blob_len, dec_st, chosen, cost = run(np.arange(n), cap1)
        retry = np.nonzero((dec_st == DIVANS_NEEDS_MORE_OUTPUT) & (blob_len > cap1))[0]
        self.last_transcode_retried = int(retry.size)   # (streams of the most recent call that ran twice)
        if retry.size:
            # one output tensor: the first pass's streams move into it before the second pass allocates its buffers, and the
            # second pass encodes straight into its tail
            base = d_new.numel()
            with torch.cuda.stream(s):
                out = torch.empty(base + _regions(_encoded_cap(blob_len[retry]))[1], dtype=torch.uint8, device=dev)
                out[:base].copy_(d_new)
            del d_new
            _, off2, len2, st2, _, _, ch2, co2 = run(retry, blob_len[retry], out[base:])
            d_new = out
            new_off[retry] = off2 + np.uint64(base)
            new_len[retry], status[retry] = len2, st2
            if auto:
                chosen[retry], cost[retry] = ch2, co2
        caller.wait_stream(s)
        d_new.record_stream(caller)   # (allocated on the private stream, used on the caller's from here on)
        return (d_new, new_off, new_len, status, chosen, cost) if auto else (d_new, new_off, new_len, status)

    # -- generating LZ77 command lists on the GPU (include/divans_b200.h, divans_b200_lz77_cmds_batch_device)
    def lz77_cmds_batch_device(self, n, d_in, d_in_off, d_in_len, max_in_len, window, pred_mode, mixing_value, d_blobs, d_blob_off,
                               d_blob_cap, d_blob_len, d_status, stream=None, parse=None):
        """lz77_cmds_batch on the GPU, with raw device pointers (ints): the blob of stream i goes to d_blobs[d_blob_off[i] ..
        +d_blob_cap[i]) (4-byte aligned; lz77_blob_cap always suffices).  Status 0: d_blob_len[i] bytes equal to lz77_cmds_batch's
        blob; 2: the region is too small and d_blob_len[i] is the size needed; 3: refused (misaligned region, in_len > max_in_len
        or >= 2**31).  Asynchronous on ``stream``; regions are not cleared first.  ``parse`` (min_match, lazy) as for
        lz77_cmds_batch (divans_b200_lz77_cmds_batch_device_parse); None is (4, 0)."""
        args = (self._h, n, d_in, d_in_off, d_in_len, int(max_in_len), int(window), int(pred_mode), int(mixing_value), d_blobs, d_blob_off,
                d_blob_cap, d_blob_len, d_status)
        if parse is None:
            rc = self._L.divans_b200_lz77_cmds_batch_device(*args, stream)
        else:
            rc = self._L.divans_b200_lz77_cmds_batch_device_parse(*args, ctypes.byref(_parse(parse)), stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("lz77_cmds_batch_device: " + self._err())

    def encode_cmds_choose_batch_device(self, n, k, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap,
                                        d_out_len, d_status, d_chosen, d_cost=None, opts=None, stream=None):
        """divans_b200_encode_cmds_choose_batch_device with raw device pointers (ints): k command lists per stream, list c of
        stream i at d_blob_off[c * n + i] / d_blob_len[c * n + i]; each stream is encoded from the list that costs least under its
        own records (d_chosen u32 [n], d_cost u64 [n * k] or None), exactly as encode_cmds_batch_device encodes that list.
        d_out None: the choice only.  Asynchronous on ``stream``."""
        rc = self._L.divans_b200_encode_cmds_choose_batch_device(self._h, n, int(k), d_blobs, d_blob_off, d_blob_len, int(max_blob_len),
                                                                 int(max_raw_len), d_out, d_out_off, d_out_cap, d_out_len, d_status,
                                                                 ctypes.byref(opts or encode_options()), d_chosen, d_cost, stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("encode_cmds_choose_batch_device: " + self._err())

    def compress_device(self, d_in, in_off, in_len, window=16, pred_mode=2, mixing_value=4, opts=None, candidates=None, stream=None,
                        sub_batch=None, parses=None):
        """Compress raw buffers held in HBM with copy commands, without leaving the GPU: ``d_in`` is a CUDA uint8 tensor, buffer
        i at in_off[i] .. +in_len[i] (host arrays).  lz77_cmds_batch_device (``window``, ``pred_mode``, ``mixing_value`` as for
        lz77_cmds_batch) into regions of lz77_blob_cap, one synchronisation to read the blob lengths, then
        encode_cmds_batch_device with ``opts`` (default: window_size 0, each list coded with its header window) -- the streams
        Engine.encode(lz77 blobs, opts, cmds=True) returns.  With ``candidates`` the encode step is
        encode_cmds_auto_batch_device and the call also returns chosen [n] and cost [n, C], as transcode_device.
        The calls run on a private CUDA stream ordered after ``stream`` (default the current one).  The encoder's symbol logs
        of a launch are one allocation, so the lists are encoded in as many sub-batches as memory needs: at most ``sub_batch``
        streams each (default all), halved while the encoder cannot allocate them.  Returns (d_new, new_off, new_len, status):
        status[i] is the generator's status where that failed (the list then reaches the encoder with length 0), else the
        encoder's.
        With ``parses`` (a list of 1..16 (min_match, lazy) pairs, e.g. DEFAULT_LZ77_PARSES) the generator makes one list per
        parse and stream, and encode_cmds_choose_batch_device encodes each stream from the list that codes cheapest under its own
        record; with ``candidates`` too, the literal model is then chosen on that list (encode_cmds_auto_batch_device).  The call
        then also returns chosen_parse [n] (an index into ``parses``) and parse_cost [n, k] last."""
        import torch
        n = len(in_off)
        in_off, in_len = np.ascontiguousarray(in_off, np.uint64).reshape(n), np.ascontiguousarray(in_len, np.uint64).reshape(n)
        o = opts if opts is not None else encode_options(window_size=0)
        if parses is not None:
            return self._compress_parses(d_in, in_off, in_len, window, pred_mode, mixing_value, o, candidates, stream, sub_batch, list(parses))
        auto = candidates is not None
        nc = len(candidates) if auto else 0
        dev = d_in.device
        if n == 0:
            empty = torch.zeros(0, dtype=torch.uint8, device=dev), np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.int32)
            return empty + (np.zeros(0, np.uint32), np.zeros((0, nc), np.uint64)) if auto else empty
        caller = stream if stream is not None else torch.cuda.current_stream(dev)
        s = torch.cuda.Stream(dev)
        s.wait_stream(caller)
        u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev, non_blocking=False)
        max_in = int(in_len.max())
        bcap = lz77_blob_cap(in_len)
        blob_off, blob_total = _regions(bcap)
        with torch.cuda.stream(s):
            d_meta = u64(np.concatenate([in_off, in_len, blob_off, bcap]))
            M = [d_meta[k * n:(k + 1) * n] for k in range(4)]
            d_blobs = torch.empty(blob_total, dtype=torch.uint8, device=dev)
            d_gen = torch.zeros(2 * n, dtype=torch.int64, device=dev)   # blob_len | status (int32 pairs)
            self.lz77_cmds_batch_device(n, d_in.data_ptr(), M[0].data_ptr(), M[1].data_ptr(), max_in, window, pred_mode, mixing_value,
                                        d_blobs.data_ptr(), M[2].data_ptr(), M[3].data_ptr(), d_gen.data_ptr(), d_gen[n:].data_ptr(),
                                        s.cuda_stream)
            g = d_gen.cpu().numpy()   # (the synchronisation that reads the blob lengths)
        gen_st = g[n:].view(np.int32)[:n].copy()
        blob_len = np.where(gen_st == 0, g[:n].view(np.uint64), np.uint64(0))
        new_cap = _encoded_cap(blob_len)
        new_off, new_total = _regions(new_cap)
        max_blob = int(blob_len.max())
        with torch.cuda.stream(s):
            d_enc = u64(np.concatenate([blob_len, new_off, new_cap]))
            d_new = torch.empty(new_total, dtype=torch.uint8, device=dev)
            # new_len | status (| candidates: cost [n * C] | chosen)
            d_res = torch.zeros((2 + (nc + 1 if auto else 0)) * n, dtype=torch.int64, device=dev)
            m = n if sub_batch is None else max(1, int(sub_batch))
            i0 = 0
            self.last_compress_sub_batches = 0   # (encode launches of the most recent call)
            while i0 < n:
                k = min(m, n - i0)
                at = lambda t, esz=8: t.data_ptr() + i0 * esz
                enc = (k, d_blobs.data_ptr(), at(M[2]), at(d_enc[:n]), max_blob, max_in, d_new.data_ptr(), at(d_enc[n:2 * n]),
                       at(d_enc[2 * n:]), at(d_res), at(d_res[n:], 4))
                try:
                    if auto:
                        self.encode_cmds_auto_batch_device(*enc, at(d_res[(2 + nc) * n:], 4), at(d_res[2 * n:], 8 * nc), o, candidates,
                                                           s.cuda_stream)
                    else:
                        self.encode_cmds_batch_device(*enc, o, s.cuda_stream)
                except DivansError as e:
                    if k == 1 or not ("cannot allocate" in str(e) or "out of memory" in str(e)):
                        raise
                    m = k // 2   # the logs of k streams did not fit next to what the GPU holds
                    continue
                i0 += k
                self.last_compress_sub_batches += 1
            r = d_res.cpu().numpy()
        enc_st = r[n:2 * n].view(np.int32)[:n]
        status = np.where(gen_st != 0, gen_st, enc_st).astype(np.int32)
        new_len = r[:n].view(np.uint64).copy()
        caller.wait_stream(s)
        d_new.record_stream(caller)   # (allocated on the private stream, used on the caller's from here on)
        if auto:
            chosen = r[(2 + nc) * n:].view(np.uint32)[:n].copy()
            cost = r[2 * n:(2 + nc) * n].view(np.uint64).reshape(n, nc).copy()
            return d_new, new_off, new_len, status, chosen, cost
        return d_new, new_off, new_len, status

    def _compress_parses(self, d_in, in_off, in_len, window, pred_mode, mixing_value, o, candidates, stream, sub_batch, parses):
        """compress_device with ``parses``: k lists per stream, candidate-major (list c of stream i is list v = c * n + i), in
        regions of lz77_blob_cap each; one synchronisation reads their lengths; then each sub-batch chooses and encodes."""
        import torch
        n, k = len(in_off), len(parses)
        if not 1 <= k <= 16:
            raise ValueError("compress_device: 1..16 parses are required")
        auto = candidates is not None
        nc = len(candidates) if auto else 0
        dev = d_in.device
        if n == 0:
            empty = torch.zeros(0, dtype=torch.uint8, device=dev), np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.int32)
            return empty + ((np.zeros(0, np.uint32), np.zeros((0, nc), np.uint64)) if auto else ()) + \
                (np.zeros(0, np.uint32), np.zeros((0, k), np.uint64))
        caller = stream if stream is not None else torch.cuda.current_stream(dev)
        s = torch.cuda.Stream(dev)
        s.wait_stream(caller)
        u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev, non_blocking=False)
        max_in = int(in_len.max())
        bcap = np.tile(lz77_blob_cap(in_len), k)
        blob_off, blob_total = _regions(bcap)
        with torch.cuda.stream(s):
            d_meta = u64(np.concatenate([in_off, in_len, blob_off, bcap]))
            d_in_off, d_in_len, d_boff, d_bcap = d_meta[:n], d_meta[n:2 * n], d_meta[2 * n:2 * n + k * n], d_meta[2 * n + k * n:]
            d_blobs = torch.empty(blob_total, dtype=torch.uint8, device=dev)
            d_gen = torch.zeros(2 * k * n, dtype=torch.int64, device=dev)   # blob_len [k * n] | status (int32 pairs)
            for c, ps in enumerate(parses):
                v = c * n
                self.lz77_cmds_batch_device(n, d_in.data_ptr(), d_in_off.data_ptr(), d_in_len.data_ptr(), max_in, window, pred_mode, mixing_value,
                                            d_blobs.data_ptr(), d_boff[v:].data_ptr(), d_bcap[v:].data_ptr(), d_gen[v:].data_ptr(),
                                            d_gen[k * n:].data_ptr() + 4 * v, s.cuda_stream, parse=ps)
            g = d_gen.cpu().numpy()   # (the synchronisation that reads the blob lengths)
        gen_st = g[k * n:].view(np.int32)[:k * n].reshape(k, n)
        blob_len = np.where(gen_st == 0, g[:k * n].view(np.uint64).reshape(k, n), np.uint64(0))
        gen_st = np.where((gen_st != 0).any(axis=0), gen_st.max(axis=0), 0).astype(np.int32)   # (a refusal refuses every parse)
        new_cap = _encoded_cap(blob_len.max(axis=0))
        new_off, new_total = _regions(new_cap)
        max_blob = int(blob_len.max())
        boff2 = blob_off.reshape(k, n)
        with torch.cuda.stream(s):
            d_enc = u64(np.concatenate([new_off, new_cap]))
            d_new = torch.empty(new_total, dtype=torch.uint8, device=dev)
            # new_len | status | parse cost [n * k] | chosen parse (| candidates: cost [n * C] | chosen)
            d_res = torch.zeros((2 + k + 1 + (nc + 1 if auto else 0)) * n, dtype=torch.int64, device=dev)
            d_pcost, d_pch = d_res[2 * n:(2 + k) * n], d_res[(2 + k) * n:(3 + k) * n]
            d_cost, d_ch = d_res[(3 + k) * n:(3 + k + nc) * n], d_res[(3 + k + nc) * n:]
            m = n if sub_batch is None else max(1, int(sub_batch))
            i0 = 0
            self.last_compress_sub_batches = 0
            while i0 < n:
                kk = min(m, n - i0)
                at = lambda t, esz=8: t.data_ptr() + i0 * esz
                # the sub-batch's lists, candidate-major
                d_sub = u64(np.concatenate([boff2[:, i0:i0 + kk].reshape(-1), blob_len[:, i0:i0 + kk].reshape(-1)]))
                try:
                    if auto:
                        self.encode_cmds_choose_batch_device(kk, k, d_blobs.data_ptr(), d_sub.data_ptr(), d_sub[k * kk:].data_ptr(), max_blob, max_in,
                                                             None, None, None, None, None, at(d_pch, 4), at(d_pcost, 8 * k), o, s.cuda_stream)
                        ch = d_pch.view(torch.int32)[i0:i0 + kk].long()
                        d_pick = torch.cat([d_sub[:k * kk].view(k, kk).gather(0, ch[None])[0], d_sub[k * kk:].view(k, kk).gather(0, ch[None])[0]])
                        self.encode_cmds_auto_batch_device(kk, d_blobs.data_ptr(), d_pick.data_ptr(), d_pick[kk:].data_ptr(), max_blob, max_in,
                                                           d_new.data_ptr(), at(d_enc[:n]), at(d_enc[n:]), at(d_res), at(d_res[n:], 4), at(d_ch, 4),
                                                           at(d_cost, 8 * nc), o, candidates, s.cuda_stream)
                    else:
                        self.encode_cmds_choose_batch_device(kk, k, d_blobs.data_ptr(), d_sub.data_ptr(), d_sub[k * kk:].data_ptr(), max_blob, max_in,
                                                             d_new.data_ptr(), at(d_enc[:n]), at(d_enc[n:]), at(d_res), at(d_res[n:], 4),
                                                             at(d_pch, 4), at(d_pcost, 8 * k), o, s.cuda_stream)
                except DivansError as e:
                    if kk == 1 or not ("cannot allocate" in str(e) or "out of memory" in str(e)):
                        raise
                    m = kk // 2   # the logs of kk streams (and the slots of their kk * k pairs) did not fit next to what the GPU holds
                    continue
                i0 += kk
                self.last_compress_sub_batches += 1
            r = d_res.cpu().numpy()
        enc_st = r[n:2 * n].view(np.int32)[:n]
        status = np.where(gen_st != 0, gen_st, enc_st).astype(np.int32)
        new_len = r[:n].view(np.uint64).copy()
        caller.wait_stream(s)
        d_new.record_stream(caller)   # (allocated on the private stream, used on the caller's from here on)
        chosen_parse = r[(2 + k) * n:(3 + k) * n].view(np.uint32)[:n].copy()
        parse_cost = r[2 * n:(2 + k) * n].view(np.uint64).reshape(n, k).copy()
        if auto:
            chosen = r[(3 + k + nc) * n:].view(np.uint32)[:n].copy()
            cost = r[(3 + k) * n:(3 + k + nc) * n].view(np.uint64).reshape(n, nc).copy()
            return d_new, new_off, new_len, status, chosen, cost, chosen_parse, parse_cost
        return d_new, new_off, new_len, status, chosen_parse, parse_cost

    # -- replaying command lists to raw bytes (include/divans_b200.h, divans_b200_replay_cmds_batch_*)
    def replay_cmds_batch_host(self, blobs, blob_off, blob_len, out, out_off, out_cap, window_size=0):
        """Realise the DVCL command lists blobs[blob_off[i] .. +blob_len[i]) as raw bytes in out[out_off[i] .. +out_cap[i]):
        returns (out_len, status).  ``window_size`` 0 takes each list's header window; status 2: out_len is the exact length
        and the region holds its first out_cap bytes (out_cap 0 measures lengths only); status 3: the list is refused."""
        n = len(blob_off)
        blob_off, blob_len, out_off, out_cap, out_len, status = _host_batch(blob_off, blob_len, out_off, out_cap)
        rc = self._L.divans_b200_replay_cmds_batch_host(self._h, n, _ptr(blobs), _ptr(blob_off), _ptr(blob_len), _ptr(out), _ptr(out_off),
                                                        _ptr(out_cap), _ptr(out_len), _ptr(status), int(window_size))
        if rc != DIVANS_SUCCESS:
            raise DivansError("replay_cmds_batch_host: " + self._err())
        return out_len, status

    def replay_cmds_batch_device(self, n, d_blobs, d_blob_off, d_blob_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, window_size=0,
                                 stream=None):
        """replay_cmds_batch_host with raw device pointers (ints); blobs 4-byte aligned.  Asynchronous on ``stream``; regions
        are not cleared first."""
        rc = self._L.divans_b200_replay_cmds_batch_device(self._h, n, d_blobs, d_blob_off, d_blob_len, d_out, d_out_off, d_out_cap,
                                                          d_out_len, d_status, int(window_size), stream)
        if rc != DIVANS_SUCCESS:
            raise DivansError("replay_cmds_batch_device: " + self._err())

    def replay(self, blobs, window_size=0, max_bytes=1 << 32):
        """Convenience: list of DVCL command-list blobs -> list of (status, raw bytes).  A length pass (out_cap 0), then one
        exact pass over the lists it measured; a refused list gives (3, b"").  The exact pass holds the whole output in host
        memory and in HBM, and a short list can describe gigabytes (one copy record: up to 4 GiB), so when the measured lengths
        add up to more than ``max_bytes`` the call raises DivansError instead of allocating them; pass a larger bound knowingly,
        or replay such lists with replay_cmds_batch_host / _device into regions of your own."""
        n = len(blobs)
        if n == 0:
            return []
        blob, off, ln = _pack(blobs)
        out_len, status = self.replay_cmds_batch_host(blob, off, ln, np.zeros(1, np.uint8), np.zeros(n, np.uint64), np.zeros(n, np.uint64),
                                                      window_size)
        res = [(DIVANS_FAILURE, b"")] * n
        idx = np.nonzero(status != DIVANS_FAILURE)[0]
        if idx.size:
            cap = out_len[idx]
            if sum(int(c) for c in cap) > max_bytes:
                raise DivansError("replay: the lists measure %d bytes in all, more than max_bytes = %d" % (sum(int(c) for c in cap), max_bytes))
            out_off, total = _regions(cap)
            out = np.zeros(max(total, 1), np.uint8)
            ln2, st2 = self.replay_cmds_batch_host(blob, off[idx], ln[idx], out, out_off, cap, window_size)
            for k, i in enumerate(idx):
                res[i] = (int(st2[k]), out[int(out_off[k]):int(out_off[k]) + int(ln2[k])].tobytes())
        return res

    def encode(self, raws, opts=None, cmds=False):
        """Convenience: list of raw byte strings (or DVCL command-list blobs with cmds=True) -> list of .divans bytes."""
        status, outs = self._encode_lists(raws, opts, cmds)
        if (status != 0).any():
            raise DivansError("encode failed for streams %s" % np.nonzero(status)[0][:8])
        return outs


class DivansDecompressorReader(io.RawIOBase):
    """Mirror of the reference's ``DivansDecompressorReader::new(reader, buffer_size, skip_crc, multithread)``
    (src/reader.rs:298-320): wraps a readable of .divans bytes and yields the decompressed bytes, driving the
    C-ABI ``divans_decode`` exactly like ``GenReader::read`` (src/reader.rs:45-109)."""

    def __init__(self, reader, buffer_size=65536, skip_crc=False, multithread=True):
        super().__init__()
        self._L = load_library()
        self._reader = reader
        self._buf_size = max(1, int(buffer_size))
        alloc = CAllocator(None, None, None)
        self._state = self._L.divans_new_decompressor_with_custom_alloc(alloc, int(bool(skip_crc)), int(bool(multithread)))
        if not self._state:
            raise DivansError("divans_new_decompressor failed")
        self._in = np.zeros(0, np.uint8)
        self._in_off = ctypes.c_size_t(0)
        self._eof_in = False
        self._done = False

    def readable(self):
        return True

    def close(self):
        if getattr(self, "_state", None):
            self._L.divans_free_decompressor(self._state)
            self._state = None
        super().close()

    def readinto(self, b):
        if self._done or len(b) == 0:
            return 0
        out = np.frombuffer(b, dtype=np.uint8) if not isinstance(b, np.ndarray) else b
        out_off = ctypes.c_size_t(0)
        while True:
            if self._in_off.value == self._in.size and not self._eof_in:
                chunk = self._reader.read(self._buf_size)
                if not chunk:
                    self._eof_in = True
                    self._in = np.zeros(0, np.uint8)
                else:
                    self._in = np.frombuffer(chunk, dtype=np.uint8)
                self._in_off = ctypes.c_size_t(0)
            rc = self._L.divans_decode(self._state, _ptr(self._in) if self._in.size else None, self._in.size, ctypes.byref(self._in_off),
                                       ctypes.c_void_p(out.ctypes.data), out.size, ctypes.byref(out_off))
            if rc == DIVANS_FAILURE:
                raise ValueError("divans: invalid data")                  # io::ErrorKind::InvalidData, reader.rs:96-98
            if rc == DIVANS_SUCCESS:
                self._done = True
                return out_off.value
            if rc == DIVANS_NEEDS_MORE_OUTPUT:
                return out_off.value
            if rc == DIVANS_NEEDS_MORE_INPUT and self._eof_in and self._in_off.value == self._in.size:
                raise EOFError("divans: unexpected end of input")          # UnexpectedEof, reader.rs:279-281


class DivansCompressorWriter(io.RawIOBase):
    """Mirror of the reference's ``DivansBrotliHybridCompressorWriter``/``DivansExperimentalCompressorWriter``
    (src/writer.rs:267): bytes written are compressed into ``writer`` on close()."""

    def __init__(self, writer, options=None):
        super().__init__()
        self._L = load_library()
        self._writer = writer
        self._state = self._L.divans_new_compressor()
        for sel, val in (options or {}).items():
            if self._L.divans_set_option(self._state, sel, val) != DIVANS_SUCCESS:
                raise ValueError("bad option %r=%r" % (sel, val))

    def writable(self):
        return True

    def write(self, b):
        data = _u8(b)
        off = ctypes.c_size_t(0)
        oo = ctypes.c_size_t(0)
        rc = self._L.divans_encode(self._state, _ptr(data) if data.size else None, data.size, ctypes.byref(off), None, 0, ctypes.byref(oo))
        if rc == DIVANS_FAILURE:
            raise DivansError("divans_encode failed")
        return data.size

    def close(self):
        if getattr(self, "_state", None):
            buf = np.zeros(1 << 16, np.uint8)
            while True:
                oo = ctypes.c_size_t(0)
                rc = self._L.divans_encode_flush(self._state, _ptr(buf), buf.size, ctypes.byref(oo))
                if oo.value:
                    self._writer.write(buf[: oo.value].tobytes())
                if rc == DIVANS_SUCCESS:
                    break
                if rc == DIVANS_FAILURE:
                    self._L.divans_free_compressor(self._state)
                    self._state = None
                    raise DivansError("divans_encode_flush failed")
            self._L.divans_free_compressor(self._state)
            self._state = None
        super().close()
