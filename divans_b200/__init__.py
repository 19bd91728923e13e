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
    "divans_b200_debug_slot_header",
]


class DivansError(RuntimeError):
    pass


class EncodeOptions(ctypes.Structure):
    _fields_ = [
        ("window_size", ctypes.c_int32), ("dynamic_context_mixing", ctypes.c_int32), ("prior_depth", ctypes.c_int32),
        ("use_context_map", ctypes.c_int32), ("force_stride", ctypes.c_int32), ("have_literal_adaptation", ctypes.c_int32),
        ("literal_adaptation", (ctypes.c_int16 * 2) * 4), ("literal_pred_mode", ctypes.c_int32),
        ("literal_mixing_value", ctypes.c_int32), ("model_rev", ctypes.c_int32), ("cdf_model", ctypes.c_int32),
    ]


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
    L.divans_b200_encode_options_default.argtypes = [ctypes.POINTER(EncodeOptions)]
    L.divans_b200_encode_batch_host.argtypes = batch + [ctypes.POINTER(EncodeOptions)]
    L.divans_b200_encode_batch_host.restype = ctypes.c_uint8
    L.divans_b200_encode_cmds_batch_host.argtypes = batch + [ctypes.POINTER(EncodeOptions)]
    L.divans_b200_encode_cmds_batch_host.restype = ctypes.c_uint8
    L.divans_b200_encode_batch_device.argtypes = [vp, sz, vp, vp, vp, ctypes.c_uint64, vp, vp, vp, vp, vp, ctypes.POINTER(EncodeOptions), vp]
    L.divans_b200_encode_batch_device.restype = ctypes.c_uint8
    L.divans_b200_ir_to_cmds.argtypes = [ctypes.c_char_p, sz, vp, sz, szp, ctypes.POINTER(ctypes.c_int32)]
    L.divans_b200_ir_to_cmds.restype = ctypes.c_uint8
    L.divans_b200_lz77_cmds_batch.argtypes = [sz, vp, vp, vp, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, vp, sz, vp, vp, szp, ctypes.c_int32]
    L.divans_b200_lz77_cmds_batch.restype = ctypes.c_uint8
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


def lz77_cmds_batch(blob, in_off, in_len, window=16, pred_mode=2, mixing_value=4, n_threads=None):
    """Raw buffers -> DVCL command lists by the library's greedy LZ77 (divans_b200_lz77_cmds_batch): returns
    (blobs uint8 array, blob_off, blob_len) ready for Engine.encode_batch_host(..., cmds=True)."""
    L = load_library()
    blob = _u8(blob)
    in_off, in_len = np.ascontiguousarray(in_off, np.uint64), np.ascontiguousarray(in_len, np.uint64)
    n = len(in_off)
    boff, blen = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    total = ctypes.c_size_t(0)
    nt = int(n_threads or os.cpu_count() or 1)
    rc = L.divans_b200_lz77_cmds_batch(n, _ptr(blob), _ptr(in_off), _ptr(in_len), window, pred_mode, mixing_value, None, 0, _ptr(boff), _ptr(blen),
                                       ctypes.byref(total), nt)
    if rc != DIVANS_NEEDS_MORE_OUTPUT and not (rc == DIVANS_SUCCESS and total.value == 0):
        raise ValueError("lz77_cmds_batch failed")
    out = np.zeros(max(1, total.value), np.uint8)
    rc = L.divans_b200_lz77_cmds_batch(n, _ptr(blob), _ptr(in_off), _ptr(in_len), window, pred_mode, mixing_value, _ptr(out), out.size, _ptr(boff),
                                       _ptr(blen), ctypes.byref(total), nt)
    if rc != DIVANS_SUCCESS:
        raise ValueError("lz77_cmds_batch failed")
    return out, boff, blen


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
        in_off, in_len = np.ascontiguousarray(in_off, np.uint64), np.ascontiguousarray(in_len, np.uint64)
        out_off, out_cap = np.ascontiguousarray(out_off, np.uint64), np.ascontiguousarray(out_cap, np.uint64)
        out_len = np.zeros(n, np.uint64)
        status = np.full(n, DIVANS_FAILURE, np.int32)
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
        keep = [np.ascontiguousarray(in_off, np.uint64), np.ascontiguousarray(in_len, np.uint64),
                np.ascontiguousarray(out_off, np.uint64), np.ascontiguousarray(out_cap, np.uint64)]
        out_len = np.zeros(n, np.uint64)
        status = np.full(n, DIVANS_FAILURE, np.int32)
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
        bufs = [_u8(s) for s in streams]
        in_len = np.array([b.size for b in bufs], np.uint64)
        in_off = np.zeros(len(bufs), np.uint64)
        pad = (in_len + np.uint64(15)) & ~np.uint64(15)
        if len(bufs) > 1:
            in_off[1:] = np.cumsum(pad)[:-1]
        blob = np.zeros(int(pad.sum()) + 16, np.uint8)
        for b, o in zip(bufs, in_off):
            blob[int(o):int(o) + b.size] = b
        out_cap = np.array(out_caps, np.uint64)
        opad = (out_cap + np.uint64(255)) & ~np.uint64(255)
        out_off = np.zeros(len(bufs), np.uint64)
        if len(bufs) > 1:
            out_off[1:] = np.cumsum(opad)[:-1]
        out = np.zeros(int(opad.sum()) + 256, np.uint8)
        out_len, status = self.decode_batch_host(blob, in_off, in_len, out, out_off, out_cap, flags)
        return [(int(st), out[int(o):int(o) + int(n)].tobytes()) for st, o, n in zip(status, out_off, out_len)]

    def encode_batch_host(self, in_blob, in_off, in_len, out, out_off, out_cap, opts=None, cmds=False):
        n = len(in_off)
        in_off, in_len = np.ascontiguousarray(in_off, np.uint64), np.ascontiguousarray(in_len, np.uint64)
        out_off, out_cap = np.ascontiguousarray(out_off, np.uint64), np.ascontiguousarray(out_cap, np.uint64)
        out_len = np.zeros(n, np.uint64)
        status = np.full(n, DIVANS_FAILURE, np.int32)
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

    def encode(self, raws, opts=None, cmds=False):
        """Convenience: list of raw byte strings (or DVCL command-list blobs with cmds=True) -> list of .divans bytes."""
        bufs = [_u8(s) for s in raws]
        in_len = np.array([b.size for b in bufs], np.uint64)
        in_off = np.zeros(len(bufs), np.uint64)
        pad = (in_len + np.uint64(15)) & ~np.uint64(15)
        if len(bufs) > 1:
            in_off[1:] = np.cumsum(pad)[:-1]
        blob = np.zeros(int(pad.sum()) + 16, np.uint8)
        for b, o in zip(bufs, in_off):
            blob[int(o):int(o) + b.size] = b
        out_cap = (in_len + in_len // np.uint64(2) + np.uint64(70000 + 255)) & ~np.uint64(255)
        out_off = np.zeros(len(bufs), np.uint64)
        if len(bufs) > 1:
            out_off[1:] = np.cumsum(out_cap)[:-1]
        out = np.zeros(int(out_cap.sum()), np.uint8)
        out_len, status = self.encode_batch_host(blob, in_off, in_len, out, out_off, out_cap, opts, cmds)
        if (status != 0).any():
            raise DivansError("encode failed for streams %s" % np.nonzero(status)[0][:8])
        return [out[int(o):int(o) + int(n)].tobytes() for o, n in zip(out_off, out_len)]


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
