"""The Python pipelines that keep their data in HBM, Engine.compress_device in each of its four modes and
Engine.transcode_device: the library launches each call makes, the shapes and dtypes of what it returns, also for an empty
batch, and the parse lists compress_device refuses.

Launches: a decode to command lists is 5, an encode 4, a literal-model choice (encode_cmds_auto) 7, a parse choice that also
encodes (encode_cmds_choose) 7, one that only chooses 2, and each generated list 1.  Every test takes a context of its own
and makes its first encode before counting: a context's first encode also builds its reciprocal table, one launch more."""
import numpy as np
import pytest

import divans_b200
from divans_b200 import synth

pytestmark = pytest.mark.gpu

CANDS = [divans_b200.LITERAL_MODEL_KEEP] + divans_b200.DEFAULT_LITERAL_MODELS
PARSES = divans_b200.DEFAULT_LZ77_DICT_PARSES     # pairs and triples: every generator call a parse reaches
N = 12                                            # streams: sub_batch=7 runs them in two sub-batches


@pytest.fixture
def eng():
    import torch
    e = divans_b200.Engine(0, 64, 16)
    e.encode([b"the context's first encode"])
    yield e
    e.close()
    torch.cuda.empty_cache()


def _launches(eng, f):
    """(library launches f makes, f's result)"""
    import torch
    before = eng.launch_count
    res = f()
    torch.cuda.synchronize()
    return eng.launch_count - before, res


def _raws(n=N):
    rng = np.random.default_rng(7)
    corpus = synth.text_corpus(1 << 18, seed=7)
    out = []
    for _ in range(n):
        k = int(rng.integers(1000, 6000))
        o = int(rng.integers(0, len(corpus) - k))
        out.append(corpus[o:o + k])
    return out


def _on_device(bufs):
    import torch
    blob, off, ln = divans_b200._pack(bufs)
    return torch.from_numpy(blob).to("cuda:0"), off, ln


def _check_result(res, d_in, n, choices):
    """(d_new, new_off, new_len, status), then (chosen u32 [n], cost u64 [n, c]) for each c in ``choices``"""
    import torch
    assert len(res) == 4 + 2 * len(choices)
    d_new, new_off, new_len, status = res[:4]
    assert isinstance(d_new, torch.Tensor) and d_new.dtype == torch.uint8 and d_new.dim() == 1 and d_new.device == d_in.device
    assert (new_off.dtype, new_off.shape) == (np.uint64, (n,))
    assert (new_len.dtype, new_len.shape) == (np.uint64, (n,))
    assert (status.dtype, status.shape) == (np.int32, (n,))
    for j, c in enumerate(choices):
        chosen, cost = res[4 + 2 * j:6 + 2 * j]
        assert (chosen.dtype, chosen.shape) == (np.uint32, (n,))
        assert (cost.dtype, cost.shape) == (np.uint64, (n, c))
    if n:
        assert (status == 0).all()
    else:
        assert d_new.numel() == 0


# compress_device's modes: keywords, launches per call given S sub-batches, and the choices the call returns
K, C = len(PARSES), len(CANDS)
MODES = {
    "plain": (dict(), lambda s: 1 + 4 * s, []),
    "candidates": (dict(candidates=CANDS), lambda s: 1 + 7 * s, [C]),
    "parses": (dict(parses=PARSES), lambda s: K + 7 * s, [K]),
    "both": (dict(candidates=CANDS, parses=PARSES), lambda s: K + 9 * s, [C, K]),
}


@pytest.mark.parametrize("sub_batch", [None, 7])
@pytest.mark.parametrize("mode", list(MODES))
def test_compress_device_launches(eng, mode, sub_batch):
    kw, launches, choices = MODES[mode]
    d_in, off, ln = _on_device(_raws())
    got, res = _launches(eng, lambda: eng.compress_device(d_in, off, ln, sub_batch=sub_batch, **kw))
    s = 1 if sub_batch is None else 2
    assert eng.last_compress_sub_batches == s
    assert got == launches(s)
    _check_result(res, d_in, N, choices)


@pytest.mark.parametrize("retry", [False, True])
@pytest.mark.parametrize("auto", [False, True])
def test_transcode_device_launches(eng, auto, retry):
    """9 launches per pass, 12 with candidates; streams whose command list outgrows first_blob_cap (the LZ77 lists of 64 KiB
    of text) run a second pass"""
    raws = _raws(4)
    streams = eng.encode(raws)
    if retry:
        blob, off, ln = synth.text_streams(2, 65536)
        big = [blob[int(o):int(o + n)].tobytes() for o, n in zip(off, ln)]
        lists, loff, llen = divans_b200.lz77_cmds_batch(*divans_b200._pack(big))
        streams += eng.encode([lists[int(o):int(o + n)].tobytes() for o, n in zip(loff, llen)], cmds=True)
        raws += big
    d_in, in_off, in_len = _on_device(streams)
    caps = [len(r) + 64 for r in raws]
    kw = dict(candidates=CANDS) if auto else {}
    got, res = _launches(eng, lambda: eng.transcode_device(d_in, in_off, in_len, caps, **kw))
    assert eng.last_transcode_retried == (2 if retry else 0)
    assert got == (12 if auto else 9) * (2 if retry else 1)
    _check_result(res, d_in, len(streams), [C] if auto else [])


def test_empty_batches(eng):
    """n = 0 in every return shape, with no launch"""
    import torch
    d_in = torch.zeros(16, dtype=torch.uint8, device="cuda:0")
    none = np.zeros(0, np.uint64)
    for kw, _, choices in MODES.values():
        got, res = _launches(eng, lambda: eng.compress_device(d_in, none, none, **kw))
        assert got == 0
        _check_result(res, d_in, 0, choices)
    for kw, choices in ((dict(), []), (dict(candidates=CANDS), [C])):
        got, res = _launches(eng, lambda: eng.transcode_device(d_in, none, none, [], **kw))
        assert got == 0 and eng.last_transcode_retried == 0
        _check_result(res, d_in, 0, choices)


@pytest.mark.parametrize("n", [0, 3])
def test_parse_count_refused(eng, n):
    """1..16 parses, also for an empty batch and with candidates; nothing is launched"""
    d_in, off, ln = _on_device(_raws(3))
    for parses in ([], [(4, 0)] * 17):
        for kw in (dict(), dict(candidates=CANDS)):
            before = eng.launch_count
            with pytest.raises(ValueError, match="compress_device: 1..16 parses are required"):
                eng.compress_device(d_in, off[:n], ln[:n], parses=parses, **kw)
            assert eng.launch_count == before
