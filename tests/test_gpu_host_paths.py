"""The host marshalling of the batch calls: calls on different CUDA streams are serialised on the device, the host encode
calls write nothing outside the bytes they return, and every entry point runs the launches it is documented to run."""
import numpy as np
import pytest

import divans_b200
from divans_b200 import _encoded_cap, _pack, _regions

pytestmark = pytest.mark.gpu

CANARY = 0xA5


def _texts(n, seed, lo=1500, hi=6000):
    rng = np.random.default_rng(seed)
    words = [bytes(w, "ascii") for w in "the quick brown fox jumps over a lazy dog while seven wizards quietly hex jolly \
bold zebras near 1024 old mills and 77 new barns".split()]
    out = []
    for _ in range(n):
        k = int(rng.integers(lo, hi))
        s = b" ".join(words[int(i)] for i in rng.integers(0, len(words), k // 4))
        out.append(s[:k])
    return out


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()


def _lists(raws):
    """each raw buffer as a DVCL command list of the library's LZ77"""
    blob, off, ln = _pack(raws)
    blobs, boff, blen = divans_b200.lz77_cmds_batch(blob, off, ln)
    return [blobs[int(o):int(o) + int(n)].tobytes() for o, n in zip(boff, blen)]


def test_raw_device_encodes_on_two_streams_keep_their_own_literal_models():
    """Two raw encode_batch_device calls with different literal models, enqueued back to back on two CUDA streams with no host
    synchronisation, more streams than the context's encoder slots: each call's bytes equal encode_batch_host under its own
    options.  The second call may set up its PredictionMode record only after the first call's model pass is done with it."""
    import torch
    eng = divans_b200.Engine(0, 64, 16)
    try:
        raws = _texts(400, 11)
        blob, in_off, in_len = _pack(raws)
        out_cap = _encoded_cap(in_len)
        out_off, total = _regions(out_cap)
        opts = [divans_b200.encode_options(literal_pred_mode=0, literal_mixing_value=4),
                divans_b200.encode_options(literal_pred_mode=2, literal_mixing_value=8)]
        want = []
        for o in opts:
            out = np.zeros(total, np.uint8)
            ol, st = eng.encode_batch_host(blob, in_off, in_len, out, out_off, out_cap, o)
            assert (st == 0).all()
            want.append([out[int(a):int(a) + int(b)].tobytes() for a, b in zip(out_off, ol)])
        assert want[0] != want[1]
        n = len(raws)
        d_in, d_in_off, d_in_len, d_out_off, d_out_cap = _dev(blob), _dev(in_off), _dev(in_len), _dev(out_off), _dev(out_cap)
        d_out = [torch.zeros(total, dtype=torch.uint8, device="cuda") for _ in opts]
        d_len = [torch.zeros(n, dtype=torch.int64, device="cuda") for _ in opts]
        d_st = [torch.full((n,), 3, dtype=torch.int32, device="cuda") for _ in opts]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        for k, (o, s) in enumerate(zip(opts, streams)):
            eng.encode_batch_device(n, d_in.data_ptr(), d_in_off.data_ptr(), d_in_len.data_ptr(), int(in_len.max()), d_out[k].data_ptr(),
                                    d_out_off.data_ptr(), d_out_cap.data_ptr(), d_len[k].data_ptr(), d_st[k].data_ptr(), o, s.cuda_stream)
        torch.cuda.synchronize()
        for k in range(len(opts)):
            st, ol, out = d_st[k].cpu().numpy(), d_len[k].cpu().numpy(), d_out[k].cpu().numpy()
            assert (st == 0).all()
            got = [out[int(a):int(a) + int(b)].tobytes() for a, b in zip(out_off, ol)]
            bad = [i for i in range(n) if got[i] != want[k][i]]
            assert not bad, "call %d: %d of %d streams differ from encode_batch_host, first %s" % (k, len(bad), n, bad[:8])
    finally:
        eng.close()


def _canary_layout(lens, cap_of):
    """regions of cap_of(len) bytes, some exactly adjacent and some with gaps, behind a 77-byte lead"""
    cap = cap_of(np.array(lens, np.uint64))
    gap = np.array([0 if i % 3 else 50 + 7 * i for i in range(len(lens))], np.uint64)
    off = np.zeros(len(lens), np.uint64)
    off[0] = 77
    for i in range(1, len(lens)):
        off[i] = off[i - 1] + cap[i - 1] + gap[i]
    return off, cap, int(off[-1] + cap[-1]) + 333


@pytest.mark.parametrize("call", ["encode", "encode_cmds", "encode_auto", "encode_cmds_auto"])
def test_host_encode_writes_only_the_returned_bytes(engine, call):
    """The host encode calls copy back out_len bytes of each successful stream and nothing else: canary bytes between, around
    and inside the regions past out_len survive, with regions that are exactly adjacent among them."""
    raws = _texts(9, 5)
    cmds = call in ("encode_cmds", "encode_cmds_auto")
    items = _lists(raws) if cmds else raws
    blob, in_off, in_len = _pack(items)
    out_off, out_cap, total = _canary_layout(in_len, _encoded_cap)
    out = np.full(total, CANARY, np.uint8)
    if call in ("encode", "encode_cmds"):
        ol, st = engine.encode_batch_host(blob, in_off, in_len, out, out_off, out_cap, cmds=cmds)
        want = engine.encode(items, cmds=cmds)
    else:
        fn = engine.encode_cmds_auto_batch_host if cmds else engine.encode_auto_batch_host
        ol, st, _, _ = fn(blob, in_off, in_len, out, out_off, out_cap)
        want = [b for _, b, _ in (engine.encode_cmds_auto(items) if cmds else engine.encode_auto(items))]
    assert (st == 0).all()
    written = np.zeros(total, bool)
    for o, n, w in zip(out_off, ol, want):
        assert out[int(o):int(o) + int(n)].tobytes() == w
        written[int(o):int(o) + int(n)] = True
    assert (out[~written] == CANARY).all()


def test_launch_count_of_each_entry_point():
    """Launches per small call: decode 4, decode to command lists 5, encode 4, encode_auto / encode_cmds_auto 7, and one more
    on a context's first encode (its reciprocal table).  Host and device variants alike."""
    import torch
    eng = divans_b200.Engine(0, 64, 16)
    try:
        raws = _texts(3, 9)
        lists = _lists(raws)
        rblob, r_off, r_len = _pack(raws)
        lblob, l_off, l_len = _pack(lists)
        e_cap = _encoded_cap(r_len)
        e_off, e_total = _regions(e_cap)

        def delta(f):
            before = eng.launch_count
            f()
            torch.cuda.synchronize()
            return eng.launch_count - before

        streams = []
        assert delta(lambda: streams.extend(eng.encode(raws))) == 5          # first encode: + the reciprocal table
        assert delta(lambda: eng.encode(raws)) == 4
        assert delta(lambda: eng.encode(lists, cmds=True)) == 4
        assert delta(lambda: eng.encode_auto(raws)) == 7
        assert delta(lambda: eng.encode_cmds_auto(lists)) == 7

        n = len(raws)
        d_out, d_len, d_st, d_ch = (torch.zeros(e_total, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda"),
                                    torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"))
        d_eoff, d_ecap = _dev(e_off), _dev(e_cap)
        dr = (_dev(rblob), _dev(r_off), _dev(r_len))
        dl = (_dev(lblob), _dev(l_off), _dev(l_len))
        outs = (d_out.data_ptr(), d_eoff.data_ptr(), d_ecap.data_ptr(), d_len.data_ptr(), d_st.data_ptr())
        raw_in = (n, dr[0].data_ptr(), dr[1].data_ptr(), dr[2].data_ptr(), int(r_len.max()))
        lst_in = (n, dl[0].data_ptr(), dl[1].data_ptr(), dl[2].data_ptr(), int(l_len.max()), int(r_len.max()))
        assert delta(lambda: eng.encode_batch_device(*raw_in, *outs)) == 4
        assert delta(lambda: eng.encode_cmds_batch_device(*lst_in, *outs)) == 4
        assert delta(lambda: eng.encode_auto_batch_device(*raw_in, *outs, d_ch.data_ptr())) == 7
        assert delta(lambda: eng.encode_cmds_auto_batch_device(*lst_in, *outs, d_ch.data_ptr())) == 7
        assert (d_st.cpu().numpy() == 0).all()

        sblob, s_off, s_len = _pack(streams)
        d_cap = np.array([len(r) for r in raws], np.uint64)
        d_off, d_total = _regions(d_cap)
        b_cap = divans_b200.first_blob_cap(d_cap)
        b_off, b_total = _regions(b_cap)
        out, blobs = np.zeros(d_total, np.uint8), np.zeros(b_total, np.uint8)
        assert delta(lambda: eng.decode(streams, d_cap)) == 4
        assert delta(lambda: eng.decode_batch_host(sblob, s_off, s_len, out, d_off, d_cap)) == 4
        assert delta(lambda: eng.decode_batch_host_async(sblob, s_off, s_len, out, d_off, d_cap).wait()) == 4
        assert delta(lambda: eng.decode_cmds_batch_host(sblob, s_off, s_len, out, d_off, d_cap, blobs, b_off, b_cap)) == 5

        ds = (_dev(sblob), _dev(s_off), _dev(s_len))
        dd_out, dd_off, dd_cap = torch.zeros(d_total, dtype=torch.uint8, device="cuda"), _dev(d_off), _dev(d_cap)
        db, db_off, db_cap = torch.zeros(b_total, dtype=torch.uint8, device="cuda"), _dev(b_off), _dev(b_cap)
        db_len = torch.zeros(n, dtype=torch.int64, device="cuda")
        dec = (ds[0].data_ptr(), ds[1].data_ptr(), ds[2].data_ptr(), dd_out.data_ptr(), dd_off.data_ptr(), dd_cap.data_ptr(), d_len.data_ptr())
        assert delta(lambda: eng.decode_batch_device(*dec, d_st.data_ptr(), n, int(s_len.sum()))) == 4
        assert (d_st.cpu().numpy() == 0).all()
        assert delta(lambda: eng.decode_cmds_batch_device(*dec, db.data_ptr(), db_off.data_ptr(), db_cap.data_ptr(), db_len.data_ptr(),
                                                          d_st.data_ptr(), n, int(s_len.sum()))) == 5
        assert (d_st.cpu().numpy() == 0).all()
        got = dd_out.cpu().numpy()
        for o, r in zip(d_off, raws):
            assert got[int(o):int(o) + len(r)].tobytes() == r
    finally:
        eng.close()
