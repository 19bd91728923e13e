"""Drivers of the reference FFI entry points of libdivans_b200.so (divans_new_compressor .. divans_encode_flush, divans_decode)
through ctypes, for tests/test_gpu_ffi_oracle.py and the child processes it starts.  ctypes releases the GIL for the length of
each call, so host threads running these drive the library concurrently.  Every call's cursors are checked against its
buffers; a contract violation raises AssertionError."""
import ctypes

import numpy as np

import divans_b200 as D

SUCCESS, NEEDS_MORE_INPUT, NEEDS_MORE_OUTPUT, FAILURE = 0, 1, 2, 3


def _arr(b):
    return np.frombuffer(bytes(b), np.uint8) if len(b) else np.zeros(1, np.uint8)


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def compress(options, data, cuts=(), out_window=65536):
    """Set `options` [(selector, value)], feed `data` in pieces ending at each of `cuts` (then at len(data)), each call entered
    with *input_offset at the piece's start of the whole buffer (a repeated cut is a zero-length call), then flush through
    `out_window`-byte windows.  Returns (set_option results, flush result, stream bytes or None on FAILURE)."""
    L = D.load_library()
    st = L.divans_new_compressor()
    assert st, "divans_new_compressor returned NULL"
    try:
        rcs = [L.divans_set_option(st, sel, val) for sel, val in options]
        buf = _arr(data)
        pos = 0
        for end in list(cuts) + [len(data)]:
            off, oo = ctypes.c_size_t(pos), ctypes.c_size_t(0)
            rc = L.divans_encode(st, _p(buf), end, ctypes.byref(off), None, 0, ctypes.byref(oo))
            assert rc == NEEDS_MORE_INPUT and off.value == end and oo.value == 0, (rc, pos, end, off.value, oo.value)
            pos = end
        out, win = bytearray(), np.zeros(out_window, np.uint8)
        while True:
            oo = ctypes.c_size_t(0)
            rc = L.divans_encode_flush(st, _p(win), out_window, ctypes.byref(oo))
            assert oo.value <= out_window
            out += win[:oo.value].tobytes()
            if rc == FAILURE:
                assert not out
                return rcs, rc, None
            assert rc in (SUCCESS, NEEDS_MORE_OUTPUT), rc
            assert rc == SUCCESS or oo.value == out_window, "NEEDS_MORE_OUTPUT with room left in the window"
            if rc == SUCCESS:
                return rcs, rc, bytes(out)
    finally:
        L.divans_free_compressor(st)


def decompress(data, cuts=(), out_window=65536, skip_crc=False, state=None):
    """Feed `data` in pieces ending at each of `cuts` (then at len(data)), each call entered with *input_offset where the previous
    one stopped, every piece drained through `out_window`-byte windows before the next.  Returns (last result, output, input
    consumed, index of the piece whose call returned the last result)."""
    L = D.load_library()
    own = state is None
    if own:
        state = L.divans_new_decompressor_with_custom_alloc(D.CAllocator(None, None, None), int(skip_crc), 1)
        assert state, "divans_new_decompressor returned NULL"
    try:
        buf, win = _arr(data), np.zeros(out_window, np.uint8)
        out, pos, rc = bytearray(), 0, None
        for k, end in enumerate(list(cuts) + [len(data)]):
            end = max(end, pos)
            while True:
                off, oo = ctypes.c_size_t(pos), ctypes.c_size_t(0)
                rc = L.divans_decode(state, _p(buf), end, ctypes.byref(off), _p(win), out_window, ctypes.byref(oo))
                assert pos <= off.value <= end and oo.value <= out_window, (pos, off.value, end, oo.value)
                out += win[:oo.value].tobytes()
                pos = off.value
                if rc == NEEDS_MORE_INPUT:
                    assert pos == end, "NEEDS_MORE_INPUT with input left"
                    break
                if rc in (SUCCESS, FAILURE):
                    return rc, bytes(out), pos, k
                assert rc == NEEDS_MORE_OUTPUT and oo.value == out_window, (rc, oo.value)
        return rc, bytes(out), pos, k
    finally:
        if own:
            L.divans_free_decompressor(state)
