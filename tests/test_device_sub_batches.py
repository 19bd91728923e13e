"""The sub-batch loop of Engine.compress_device (divans_b200._sub_batches) with a fake step: the (i0, kk) sequence it runs, how it
halves on an allocation failure, and which errors it raises.  Needs no GPU."""
import pytest

from divans_b200 import DivansError, _sub_batches

ALLOC = "encode_cmds_batch_device: divans_b200: cannot allocate the symbol logs of %d command lists of up to 9000 bytes: 1 bytes"
OOM = "encode_cmds_batch_device: cudaMalloc: out of memory (%d streams)"


def _run(n, sub_batch, fits=None, msg=ALLOC):
    """(sub-batches run, every (i0, kk) the step was called with); the step fails with ``msg`` above ``fits`` streams"""
    calls = []

    def step(i0, kk):
        calls.append((i0, kk))
        if fits is not None and kk > fits:
            raise DivansError(msg % kk)
    return _sub_batches(n, sub_batch, step), calls


@pytest.mark.parametrize("msg", [ALLOC, OOM])
def test_halves_while_it_cannot_allocate(msg):
    runs, calls = _run(100, None, fits=20, msg=msg)
    assert calls == [(0, 100), (0, 50), (0, 25)] + [(i0, 12) for i0 in range(0, 96, 12)] + [(96, 4)]
    assert runs == 9


def test_halving_starts_from_sub_batch():
    runs, calls = _run(30, 16, fits=5)
    assert calls == [(0, 16), (0, 8), (0, 4)] + [(i0, 4) for i0 in range(4, 28, 4)] + [(28, 2)]
    assert runs == 8


def test_sub_batch_sizes():
    assert _run(100, 7) == (15, [(i0, 7) for i0 in range(0, 98, 7)] + [(98, 2)])
    assert _run(100, None) == (1, [(0, 100)])
    assert _run(3, 0) == (3, [(0, 1), (1, 1), (2, 1)])
    assert _run(3, -5) == (3, [(0, 1), (1, 1), (2, 1)])
    assert _run(5, 64) == (1, [(0, 5)])
    assert _run(0, None) == (0, [])


def test_other_errors_are_raised():
    calls = []

    def step(i0, kk):
        calls.append((i0, kk))
        raise DivansError("encode_cmds_batch_device: batch too large")
    with pytest.raises(DivansError, match="batch too large"):
        _sub_batches(100, None, step)
    assert calls == [(0, 100)]

    def not_divans(i0, kk):
        raise RuntimeError("cannot allocate")
    with pytest.raises(RuntimeError):
        _sub_batches(100, None, not_divans)


@pytest.mark.parametrize("msg", [ALLOC, OOM])
def test_allocation_failure_of_one_stream_is_raised(msg):
    with pytest.raises(DivansError, match="cannot allocate|out of memory"):
        _run(10, None, fits=0, msg=msg)
    calls = []

    def step(i0, kk):
        calls.append((i0, kk))
        if i0 == 3:
            raise DivansError(msg % kk)
    with pytest.raises(DivansError):
        _sub_batches(10, 1, step)
    assert calls == [(0, 1), (1, 1), (2, 1), (3, 1)]

