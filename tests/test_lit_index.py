"""The v2 decoder's literal prior order (dv_common.cuh: lit_index_hi / lit_index_lo), compiled for the host with g++.

Every v2 access to the literal tables goes through these two functions: each must map the 256 x 256 priors of a `which`
block one-to-one onto that block, or two priors would share storage.  The dense order exists for one property: under LSB6
with the identity context map and mixing value 4 (stride byte = the previous byte), the 256 high-nibble priors a stream can
use are one contiguous run, so its hot priors share cache lines."""
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "divans_b200", "csrc")
CUDA_INCLUDE = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")   # dv_common.cuh includes cuda_runtime.h


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("lit_index") / "lit_index_dump")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-I", CSRC, "-I", CUDA_INCLUDE, "-o", exe,
                           os.path.join(HERE, "c_client", "lit_index_dump.cpp")])
    raw = subprocess.run([exe], check=True, capture_output=True).stdout
    t = np.frombuffer(raw, dtype="<u4").reshape(2, 3, 256, 256)   # [hi, lo][which][index_c][index_b]
    return {"hi": t[0], "lo": t[1]}


@pytest.mark.parametrize("table", ["hi", "lo"])
@pytest.mark.parametrize("which", [0, 1, 2])
def test_index_is_a_bijection_onto_its_block(tables, table, which):
    idx = tables[table][which].ravel()
    assert idx.max() < 65536
    assert np.unique(idx).size == 65536


def test_lsb6_identity_map_mixing4_high_priors_are_one_run(tables):
    prev = np.arange(256)
    # mixing value 4: which 1, index_b = the stride byte = prev; LSB6 with the identity context map: index_c = prev & 63
    idx = np.sort(tables["hi"][1][prev & 63, prev])
    assert (np.diff(idx) == 1).all(), "the 256 high priors of the flagship configuration are not contiguous"
