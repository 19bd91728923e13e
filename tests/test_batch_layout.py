"""The batch layout the convenience calls build (Engine.decode, decode_cmds, encode, encode_auto, encode_cmds_auto,
transcode_device): inputs at 16-byte aligned offsets with a 16-byte tail, output regions at 256-byte aligned offsets, and the
encoder's output capacity L + L // 2 + 70000 rounded up to 256.  The expected offsets are written out by hand."""
import numpy as np

from divans_b200 import _encoded_cap, _pack, _regions


def _check_pack(bufs, off, total):
    blob, got_off, got_len = _pack(bufs)
    assert got_off.dtype == np.uint64 and got_len.dtype == np.uint64 and blob.dtype == np.uint8
    assert got_off.tolist() == off
    assert got_len.tolist() == [len(b) for b in bufs]
    assert blob.size == total
    want = np.zeros(total, np.uint8)
    for b, o in zip(bufs, off):
        want[o:o + len(b)] = np.frombuffer(b, np.uint8)
    assert blob.tobytes() == want.tobytes()


def test_pack_empty_list():
    _check_pack([], [], 16)


def test_pack_zero_length_items():
    _check_pack([b""], [0], 16)
    _check_pack([b"", b""], [0, 0], 16)
    _check_pack([b"a", b"", b"b" * 17, b""], [0, 16, 16, 48], 64)


def test_pack_lengths_around_16():
    bufs = [b"\x01", bytes(range(1, 16)), bytes(range(16, 32)), bytes(range(32, 49))]   # 1, 15, 16, 17 bytes
    _check_pack(bufs, [0, 16, 32, 48], 96)


def test_pack_accepts_arrays():
    _check_pack([np.arange(17, dtype=np.uint8), bytearray(b"xyz")], [0, 32], 64)


def _check_regions(caps, off, total):
    got_off, got_total = _regions(np.array(caps, np.uint64))
    assert got_off.dtype == np.uint64
    assert got_off.tolist() == off
    assert got_total == total


def test_regions_empty_and_zero_caps():
    _check_regions([], [], 0)
    _check_regions([0], [0], 0)
    _check_regions([0, 0, 5], [0, 0, 0], 256)


def test_regions_small_caps():
    _check_regions([1, 15, 16, 17], [0, 256, 512, 768], 1024)
    _check_regions([257, 1], [0, 512], 768)


def test_regions_caps_already_multiples_of_256():
    _check_regions([256, 512, 0, 256], [0, 256, 768, 768], 1024)
    _check_regions([70144, 71680], [0, 70144], 141824)


def test_encoded_cap():
    assert _encoded_cap(np.zeros(0, np.uint64)).tolist() == []
    # L + L // 2 + 70000: 70000, 70001, 70022, 70024, 70025 -> 70144 (274 * 256)
    assert _encoded_cap(np.array([0, 1, 15, 16, 17], np.uint64)).tolist() == [70144] * 5
    # 96 + 48 + 70000 = 70144 exactly; 1000 -> 71500 -> 71680; 2**20 -> 1642864 -> 1643008
    assert _encoded_cap(np.array([96, 1000, 1 << 20], np.uint64)).tolist() == [70144, 71680, 1643008]
    assert _encoded_cap(np.array([5], np.uint64)).dtype == np.uint64
