"""The CPU oracle's per-context mixing values (oracle_tally): the binned tally and dvo_encode_mixmap / dvo_encode_cmds_mixmap."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from divans_b200 import synth  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402

VALUES = [4, 5, 8, 1, 7, 0]


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _text(n, seed=3):
    blob, off, ln = synth.text_streams(1, n, seed=seed)
    return blob.tobytes()


def _records(n, width, seed=5):
    rng = np.random.default_rng(seed)
    cols = [(np.cumsum(rng.integers(-1, 2, n // width + 1)) + 60 * j) & 255 for j in range(width)]
    return (np.stack(cols, 1).astype(np.uint8).reshape(-1)[:n]).tobytes()


def _corpora():
    utf8 = "".join(chr(0x430 + (c % 26)) if 97 <= c < 123 else chr(c) for c in _text(2000, 8)).encode()[:2000]
    return {"empty": b"", "one": b"Q", "text": _text(3000), "utf8": utf8, "rec2": _records(3000, 2), "rec4": _records(3000, 4),
            "rec8": _records(3000, 8), "text+rec4": _text(1500, 4) + _records(1500, 4, 6),
            "random": np.random.default_rng(1).integers(0, 256, 1500, dtype=np.uint8).tobytes()}


@pytest.mark.parametrize("blend", [False, True])
@pytest.mark.parametrize("name", sorted(_corpora()))
def test_bins_sum_to_the_tally(name, blend):
    data = _corpora()[name]
    for pm, mv in ((0, 4), (2, 8), (3, 1)):
        rc, cost, bins, nobin = T.tally_raw_bins(data, pm, mv, blend, window_size=10)
        assert rc == 0 and cost == T.tally_raw(data, pm, mv, blend, window_size=10)[1]
        assert int(bins.sum()) + nobin == cost
        assert nobin > 0   # the command nibbles and the end-of-stream nibble
        assert (int(bins.sum()) > 0) == (len(data) > 0)


def test_uniform_map_gives_the_uniform_stream():
    """one value: the mixed record equals the uniform one, the mixed pass costs the same, and the tie keeps the uniform record"""
    for data in _corpora().values():
        for v in (4, 8):
            rc, out, ch, mixing, cost, bins = T.encode_mixmap(data, 2, [v])
            assert rc == 0 and ch == 0 and cost[1] == cost[0] and (mixing == v).all()
            assert out == T.encode_raw_model(data, 2, v)[1]


@pytest.mark.parametrize("blend", [False, True])
@pytest.mark.parametrize("dcm", [0, 1, 2])
def test_mixmap_streams_decode_and_never_cost_more(oracle, blend, dcm):
    from oracle import oracle_blend
    O = oracle_blend if blend else oracle
    mixed_seen = False
    for name, data in _corpora().items():
        for pm in (0, 2):
            rc, out, ch, mixing, cost, bins = T.encode_mixmap(data, pm, VALUES, blend, window_size=10, dynamic_context_mixing=dcm)
            assert rc == 0, name
            u = cost[:len(VALUES)]
            cstar = int(np.argmin(u))
            assert ch in (cstar, len(VALUES))
            if ch == len(VALUES):
                mixed_seen = True
                assert cost[-1] < u[cstar], name
            else:
                assert cost[-1] >= u[cstar]
                assert out == T.encode_raw_model(data, pm, VALUES[ch], blend, window_size=10, dynamic_context_mixing=dcm)[1]
            # the per-entry choice: lowest bin, ties to the lowest index
            want = np.array(VALUES, np.uint8)[np.argmin(bins, axis=0)]
            if ch == len(VALUES):
                assert (mixing == want).all()
            assert O.decode(out, out_cap=len(data) + 64)[1] == data, name
    assert mixed_seen


def test_cmds_mixmap(oracle):
    """LZ77 lists: the bins of every record-replaced pass sum to its tally, and the choice decodes to the list's bytes"""
    for name, data in _corpora().items():
        cmds = oracle.Commands.lz77(data, 16, 0, 4)
        for pm, mv in ((0, 4), (2, 5)):
            rc, cost, bins, nobin = T.tally_cmds_bins(cmds, pm, mv)
            assert rc == 0 and int(bins.sum()) + nobin == cost
        rc, out, ch, mixing, cost, bins = T.encode_cmds_mixmap(cmds, 2, VALUES)
        assert rc == 0
        if ch == len(VALUES):
            assert cost[-1] < cost[:-1].min()
        assert oracle.decode(out, out_cap=len(data) + 64)[1] == data, name
