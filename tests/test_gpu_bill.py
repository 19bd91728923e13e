"""Billing by coder state on the GPU (divans_b200_bill_*, include/divans_b200.h): the bill of every stream equals the CPU oracle's
row for row, sums to the cost pass's cost, and follows the conventions of the encode calls."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import divans_b200  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402
import bill_corpora as B  # noqa: E402

gpu = pytest.mark.gpu
S = len(divans_b200.BILL_STATES)


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="module")
def eng():
    """16 resident streams: every batch below has more streams than slots, so slots are reused"""
    e = divans_b200.Engine(0, 16, 16)
    yield e
    e.close()


def _u64(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to("cuda:0")


def _bill_device(eng, items, opts, cmds=False, max_raw=None, max_in=None, shift=None):
    """Engine.bill_device of byte strings packed as Engine.bill packs them; ``shift``: stream index whose bytes move one byte on"""
    import torch
    blob, off, ln = divans_b200._pack(items)
    if shift is not None:   # a copy of the stream's bytes at an odd offset past the others
        moved = blob[int(off[shift]):int(off[shift] + ln[shift])].copy()
        off = off.copy()
        off[shift] = np.uint64(blob.size + 1)
        blob = np.concatenate([blob, np.zeros(1, np.uint8), moved, np.zeros(16, np.uint8)])
    n = len(items)
    d_b = torch.from_numpy(blob).to("cuda:0")
    d_off, d_len = _u64(off), _u64(ln)
    d_bill = torch.full((max(n, 1) * S * 2,), -1, dtype=torch.int64, device="cuda:0")
    d_st = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda:0")
    torch.cuda.current_stream().synchronize()
    eng.bill_device(n, d_b.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()) if max_in is None else max_in, d_bill.data_ptr(),
                    d_st.data_ptr(), opts, cmds, max_raw)
    eng.synchronize()
    return d_bill.cpu().numpy().view(np.uint64).reshape(-1, S, 2)[:n], d_st.cpu().numpy()[:n]


def _raw_len(blob, window):
    """the bytes the list replays to at ``window``"""
    rc, n, _ = T.recode_blob(blob, window)
    assert rc in (0, 2), rc
    return n


def _check_lists(eng, lists, kw, blend, reps=1):
    """host and device bills of the lists (oracle Commands), each ``reps`` times, under the oracle options kw: the oracle's rows
    and statuses"""
    opts = divans_b200.encode_options(cdf_model=int(blend), **kw)
    blobs = [cl.serialize() for cl in lists] * reps
    ref = [T.bill_cmds(cl, blend=blend, **kw) for cl in lists] * reps
    bill, st = eng.bill(blobs, opts, cmds=True)
    dbill, dst = _bill_device(eng, blobs, opts, cmds=True, max_raw=max(_raw_len(b, kw["window_size"]) for b, r in zip(blobs, ref) if r[0] == 0))
    for i, (rc, cost, rows) in enumerate(ref):
        assert st[i] == dst[i] == rc, i
        assert (bill[i] == rows).all() and (dbill[i] == rows).all(), "stream %d: bill differs from the oracle's" % i
    return bill, st


@gpu
@pytest.mark.parametrize("blend", [False, True], ids=["frequentist", "blend"])
def test_lists_equal_oracle(eng, oracle, blend):
    groups = {}
    for name, cl, kw in B.golden_lists(oracle) + B.parse_lists(oracle, T) + B.fuzz_lists(oracle, 12):
        if blend and kw.get("model_rev"):
            continue
        groups.setdefault(tuple(sorted(kw.items())), []).append(cl)
    for key, lists in groups.items():
        _check_lists(eng, lists, dict(key), blend, reps=1 + 17 // len(lists))   # more lists than the 16 slots
    # LZ77 lists of 24 texts under the 2018 revision, and a refused list among them
    lz = [T.lz77_dict_parse(oracle, B.text(3000 + 500 * k, seed=k), 6, 1, 4, window=16) for k in range(24)]
    lz[5] = T.from_blob(oracle, B.refused_blob(oracle))
    _, st = _check_lists(eng, lz, dict(window_size=16, dynamic_context_mixing=1, model_rev=0 if blend else 1), blend)
    assert st[5] == 3 and (st != 3).sum() == 23


@gpu
@pytest.mark.parametrize("blend", [False, True], ids=["frequentist", "blend"])
def test_raw_equal_oracle(eng, oracle, blend):
    raws = [B.text(200 * k, seed=k) for k in range(20)]
    for pm, mv in B.RAW_MODELS:
        kw = dict(window_size=12, dynamic_context_mixing=(pm + mv) % 3)
        opts = divans_b200.encode_options(literal_pred_mode=pm, literal_mixing_value=mv, cdf_model=int(blend), **kw)
        bill, st = eng.bill(raws, opts)
        dbill, dst = _bill_device(eng, raws, opts)
        for i, r in enumerate(raws):
            rc, cost, rows = T.bill_raw(r, pm, mv, blend=blend, **kw)
            assert st[i] == dst[i] == rc and (bill[i] == rows).all() and (dbill[i] == rows).all(), (pm, mv, i)


@gpu
def test_equals_cost_pass(eng, oracle):
    """the cost column sums to encode_cmds_choose's d_cost and encode_auto's cost"""
    import torch
    lists = [cl for _, cl, _ in B.fuzz_lists(oracle, 10)] + [T.lz77_parse(oracle, B.text(9000, seed=k), 4 + k, k % 3) for k in range(10)]
    blobs = [cl.serialize() for cl in lists] + [B.refused_blob(oracle)]
    opts = divans_b200.encode_options(window_size=16, dynamic_context_mixing=2)
    bill, st = eng.bill(blobs, opts, cmds=True)
    blob, off, ln = divans_b200._pack(blobs)
    n = len(blobs)
    d_b, d_off, d_len = torch.from_numpy(blob).to("cuda:0"), _u64(off), _u64(ln)
    d_ch = torch.zeros(n, dtype=torch.int32, device="cuda:0")
    d_cost = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    torch.cuda.current_stream().synchronize()
    eng.encode_cmds_choose_batch_device(n, 1, d_b.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()),
                                        max(_raw_len(b, 16) for b in blobs[:-1]), None, 0, 0, 0, 0, d_ch.data_ptr(), d_cost.data_ptr(), opts)
    eng.synchronize()
    cost = d_cost.cpu().numpy().view(np.uint64)
    sums = bill[:, :, 0].sum(axis=1, dtype=np.uint64)
    assert list(st == 0) == [True] * (n - 1) + [False]
    assert (np.where(st == 0, sums, np.uint64(T.TALLY_FAILED)) == cost).all()
    raws = [B.text(3000 * k, seed=k) for k in range(20)]
    for pm, mv in ((0, 4), (2, 8), (3, 5)):
        o = divans_b200.encode_options(literal_pred_mode=pm, literal_mixing_value=mv)
        bill, st = eng.bill(raws, o)
        blob, off, ln = divans_b200._pack(raws)
        out_cap = divans_b200._encoded_cap(ln)
        out_off, total = divans_b200._regions(out_cap)
        _, ast, _, acost = eng.encode_auto_batch_host(blob, off, ln, np.zeros(total, np.uint8), out_off, out_cap, o, [(pm, mv)])
        assert (st == 0).all() and (ast == 0).all()
        assert (bill[:, :, 0].sum(axis=1, dtype=np.uint64) == acost[:, 0]).all()


@gpu
def test_slot_hygiene(eng, oracle):
    """encode, bill, encode on one context: the streams are a fresh context's, and the bill is a fresh context's"""
    raws = [B.text(4000 + 700 * k, seed=40 + k) for k in range(20)]
    lists = [cl.serialize() for _, cl, _ in B.fuzz_lists(oracle, 12)] * 2
    o_enc = divans_b200.encode_options(window_size=16)
    o_bill = divans_b200.encode_options(window_size=16, dynamic_context_mixing=2, literal_adaptation=[(32, 4096)] * 4)
    fresh = divans_b200.Engine(0, 16, 16)
    try:
        ref_enc, ref_bill = fresh.encode(raws, o_enc), fresh.bill(lists, o_bill, cmds=True)[0]
        fresh2 = divans_b200.Engine(0, 16, 16)
        ref_bill2 = fresh2.bill(lists, o_bill, cmds=True)[0]
        fresh2.close()
    finally:
        fresh.close()
    assert (ref_bill == ref_bill2).all()
    a = eng.encode(raws, o_enc)
    bill, st = eng.bill(lists, o_bill, cmds=True)
    c = eng.encode(raws, o_enc)
    assert a == ref_enc and c == ref_enc
    assert (st == 0).all() and (bill == ref_bill).all()


@gpu
def test_device_conventions(eng, oracle):
    """misaligned blobs and blobs longer than max_blob_len: status 3; lists replaying past max_raw_len: status 2; all with zero
    bills, next to streams billed as usual.  n == 0 succeeds; a NULL bill array is refused."""
    lists = []
    for k in range(20):   # lists whose headers name window 16
        b = bytearray(T.lz77_parse(oracle, B.text(2000 + 300 * k, seed=k), 6, 1).serialize())
        b[20:24] = np.uint32(16).tobytes()
        lists.append(bytes(b))
    opts = divans_b200.encode_options(window_size=0)   # each list's header window
    ref, rst = eng.bill(lists, divans_b200.encode_options(window_size=16), cmds=True)
    assert (rst == 0).all()
    max_raw = max(_raw_len(b, 16) for b in lists)
    bill, st = _bill_device(eng, lists, opts, cmds=True, max_raw=max_raw, shift=3)
    assert st[3] == 3 and not bill[3].any()
    keep = np.arange(20) != 3
    assert (st[keep] == 0).all() and (bill[keep] == ref[keep]).all()
    longest = int(np.argmax([len(b) for b in lists]))
    bill, st = _bill_device(eng, lists, opts, cmds=True, max_raw=max_raw, max_in=len(lists[longest]) - 1)
    assert st[longest] == 3 and not bill[longest].any()
    big = int(np.argmax([_raw_len(b, 16) for b in lists]))
    bill, st = _bill_device(eng, lists, opts, cmds=True, max_raw=_raw_len(lists[big], 16) - 64)
    assert st[big] == 2 and not bill[big].any()
    assert (bill[st == 0] == ref[st == 0]).all() and (st == 0).sum() >= 10
    eng.bill_device(0, 0, 0, 0, 0, 0, 0, opts, True, 0)
    with pytest.raises(divans_b200.DivansError, match="bill array"):
        eng.bill_device(1, 0, 0, 0, 64, None, 0, opts, True, 64)


@gpu
@pytest.mark.parametrize("blend", [False, True], ids=["frequentist", "blend"])
def test_stored_streams(eng, oracle, blend):
    """streams the GPU encoder wrote, decoded to lists and billed under the options they were written with: the original's bill"""
    lists = [cl.serialize() for _, cl, _ in B.fuzz_lists(oracle, 8)] + \
        [T.lz77_words_parse(oracle, B.text(5000, seed=k), 4, 0, 4, 1, window=16).serialize() for k in range(10)]
    opts = divans_b200.encode_options(window_size=16, dynamic_context_mixing=1, cdf_model=int(blend))
    ref, rst = eng.bill(lists, opts, cmds=True)
    streams = eng.encode(lists, opts, cmds=True)
    dec = eng.decode_cmds(streams, [_raw_len(b, 16) + 64 for b in lists], divans_b200.FLAG_CDF_BLEND if blend else 0)
    assert all(s == 0 for s, _, _ in dec)
    bill, st = eng.bill([b for _, _, b in dec], opts, cmds=True)
    assert (rst == 0).all() and (st == 0).all() and (bill == ref).all()
