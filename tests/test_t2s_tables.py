"""The 16-lane literal loop reads the context of LSB6 / MSB6 streams from a 256-entry class-free table (T2S, dv2_core.cuh).
That is exact only because those modes have no classes: lut1 of the shipped context tables must be all zeros for them."""
import os

import numpy as np

TABLES = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "divans_b200", "csrc", "brotli_tables.bin")
TB_CTX = 184   # dv_common.cuh: per mode, lut0 (256 bytes) then lut1 (256 bytes)


def _lut1(mode):
    t = np.fromfile(TABLES, dtype=np.uint8)
    return t[TB_CTX + 512 * mode + 256: TB_CTX + 512 * mode + 512]


def test_lsb6_msb6_have_no_classes():
    for mode in (0, 1):   # LSB6, MSB6: the modes t2s_mode() accepts
        assert not _lut1(mode).any()


def test_utf8_signed_use_classes():
    # the modes that keep the full T2 in the slot: their classes really are used
    assert set(_lut1(2).tolist()) == {0, 1, 2, 3}
    assert set(_lut1(3).tolist()) == set(range(8))
