"""Billing by coder state (include/divans_b200.h, "billing each stream's coding cost by coder state"): where the bits go, and what
the bill costs on the GPU.
    python tools/bill_probe.py --survey                      # CPU (oracle): alice29, the q11 list against the library's parse
    python tools/bill_probe.py [--n 4096] [--len 65536] [--reps 5] [--chunk 1024] [--out FILE]   # H100: bill against the cost pass
--survey bills alice29 on the CPU oracle twice, at window 22 with dynamic context mixing 1: the reference's quality-11 command list
(tests/golden/alice29_q11_mix1.divans, decoded to its list) and the list the library chooses from DEFAULT_LZ77_WORD_PARSES (the
host generator's list of each parse, the cheapest by the oracle's tally).  It prints both bills side by side, by the groups of
divans_b200.bill_summary and row by row, in bytes (cost / 2^19).
The GPU mode takes the bench's n synthetic text streams of --len bytes and their literal-only lists (the raw encoder's streams
decoded to command lists) and LZ77 lists (the GPU generator, parse (4, 0)), and times, alternately, on one CUDA stream:
  * bill_ms: Engine.bill_device of the lists;
  * cost_ms: the plain cost pass of the same lists, encode_cmds_choose_batch_device with k = 1 and no output;
  * raw_bill_ms: Engine.bill_device of the raw buffers.
Each call takes --chunk streams at a time (the cost pass of a command-list call sizes the encoder's logs for all of its lists).
Medians of --reps after one warm-up; every bill's cost column is checked against the cost pass's cost.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from auto_probe import fixture_streams, gpu_info  # noqa: E402

BYTES = float(1 << 19)   # 1/65536 bit -> bytes


def survey():
    import divans_b200
    from oracle import oracle_py as O
    from oracle_tally import tally_py as T
    kw = dict(window_size=22, dynamic_context_mixing=1)
    alice = fixture_streams()["alice29"][0]
    g = os.path.join(ROOT, "tests", "golden", "alice29_q11_mix1.divans")
    rc, raw, q11 = O.decode_cmds(open(g, "rb").read(), out_cap=len(alice) + 64)
    assert rc == 0 and raw == alice
    blob, off, ln = divans_b200._pack([alice])
    best = None
    for ps in divans_b200.DEFAULT_LZ77_WORD_PARSES:
        out, bo, bl = divans_b200.lz77_cmds_batch(blob, off, ln, 22, 2, 4, parse=ps)
        cl = T.from_blob(O, out[int(bo[0]):int(bo[0] + bl[0])].tobytes())
        rc, cost = T.tally_cmds(cl, **kw)
        if rc == 0 and (best is None or cost < best[0]):
            best = (cost, ps, cl)
    bills = {}
    for name, cl in (("q11", q11), ("library %s" % (best[1],), best[2])):
        rc, cost, rows = T.bill_cmds(cl, **kw)
        assert rc == 0 and int(rows[:, 0].sum()) == cost
        bills[name] = rows
    (na, a), (nb, b) = bills.items()
    print("alice29 (%d bytes), window 22, dynamic context mixing 1; bytes = cost / 2^19" % len(alice))
    print("%-18s %12s %12s %10s %10s %10s" % ("group", na, nb, "diff", "nib " + na, "nib lib"))
    sa, sb = divans_b200.bill_summary(a), divans_b200.bill_summary(b)
    for (g1, c1, n1), (_, c2, n2) in zip(sa, sb):
        print("%-18s %12.1f %12.1f %+10.1f %10d %10d" % (g1, c1 / BYTES, c2 / BYTES, (c2 - c1) / BYTES, n1, n2))
    print("%-18s %12.1f %12.1f %+10.1f" % ("total", a[:, 0].sum() / BYTES, b[:, 0].sum() / BYTES, (b[:, 0].sum() - a[:, 0].sum()) / BYTES))
    print()
    for r, name in enumerate(divans_b200.BILL_STATES):
        if a[r].any() or b[r].any():
            print("%-18s %12.1f %12.1f %+10.1f %10d %10d" % (name, a[r, 0] / BYTES, b[r, 0] / BYTES, (int(b[r, 0]) - int(a[r, 0])) / BYTES,
                                                             a[r, 1], b[r, 1]))
    print(json.dumps({"alice29_w22_mix1": {k: {n: [int(c), int(m)] for n, c, m in divans_b200.bill_summary(v)} for k, v in bills.items()}}))


def gpu(args):
    import torch
    import divans_b200
    from divans_b200 import synth
    eng = divans_b200.Engine(0)
    n, L = args.n, args.len
    blob, off, ln = synth.text_streams(n, L)
    raws = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]
    opts = divans_b200.encode_options(window_size=16)
    strm = torch.cuda.Stream()
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).cuda()
    # literal-only lists: the raw encoder's streams decoded to their lists
    streams = eng.encode(raws, opts)
    lit = [b for _, _, b in eng.decode_cmds(streams, [L + 64] * n)]
    del streams
    # LZ77 lists from the GPU generator
    d_raw = torch.from_numpy(blob).cuda()
    cap = divans_b200.lz77_blob_cap(ln)
    boff, btot = divans_b200._regions(cap)
    d_lz = torch.zeros(btot, dtype=torch.uint8, device="cuda")
    d_res = torch.zeros(2 * n, dtype=torch.int64, device="cuda")
    d_roff, d_rlen, d_boff, d_cap = t64(off), t64(ln), t64(boff), t64(cap)
    torch.cuda.synchronize()
    eng.lz77_cmds_batch_device(n, d_raw.data_ptr(), d_roff.data_ptr(), d_rlen.data_ptr(), L, 16, 2, 4, d_lz.data_ptr(), d_boff.data_ptr(),
                               d_cap.data_ptr(), d_res.data_ptr(), d_res[n:].data_ptr())
    eng.synchronize()
    lz_len = d_res[:n].cpu().numpy().view(np.uint64).copy()
    assert (d_res[n:].cpu().numpy().view(np.int32)[:n] == 0).all()
    lb, loff, llen = divans_b200._pack(lit)
    corpora = {"literal_only": (torch.from_numpy(lb).cuda(), t64(loff), t64(llen), int(llen.max())),
               "lz77": (d_lz, d_boff, t64(lz_len), int(lz_len.max()))}
    d_bill = torch.zeros(n * len(divans_b200.BILL_STATES) * 2, dtype=torch.int64, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_ch = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_cost = torch.zeros(n, dtype=torch.int64, device="cuda")
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def timed(fn):
        a, b = ev(), ev()
        a.record(strm)
        fn()
        b.record(strm)
        torch.cuda.synchronize()
        return a.elapsed_time(b)

    res = dict(gpu=gpu_info(), n=n, len=L, chunk=args.chunk)
    S2 = len(divans_b200.BILL_STATES) * 2
    for name, (d_in, d_off, d_len, mx) in corpora.items():
        # in chunks of --chunk streams: the cost pass's call sizes the encoder's logs for every list of a call, from max_blob_len
        def bill():
            for i in range(0, n, args.chunk):
                k = min(args.chunk, n - i)
                eng.bill_device(k, d_in.data_ptr(), d_off[i:].data_ptr(), d_len[i:].data_ptr(), mx, d_bill[i * S2:].data_ptr(),
                                d_st[i:].data_ptr(), opts, True, L, strm.cuda_stream)

        def cost():
            for i in range(0, n, args.chunk):
                k = min(args.chunk, n - i)
                eng.encode_cmds_choose_batch_device(k, 1, d_in.data_ptr(), d_off[i:].data_ptr(), d_len[i:].data_ptr(), mx, L, None, 0, 0, 0, 0,
                                                    d_ch[i:].data_ptr(), d_cost[i:].data_ptr(), opts, strm.cuda_stream)
        tb, tc = [], []
        for rep in range(args.reps + 1):
            b_ms, c_ms = timed(bill), timed(cost)
            if rep == 0:
                rows = d_bill.cpu().numpy().view(np.uint64).reshape(n, -1, 2)
                assert (d_st.cpu().numpy() == 0).all()
                assert (rows[:, :, 0].sum(axis=1, dtype=np.uint64) == d_cost.cpu().numpy().view(np.uint64)).all(), name
                summary = divans_b200.bill_summary(rows)
            else:
                tb.append(b_ms)
                tc.append(c_ms)
        res[name] = dict(bill_ms=float(np.median(tb)), cost_ms=float(np.median(tc)), ratio=round(float(np.median(tb) / np.median(tc)), 3),
                         bill_ms_all=[round(x, 2) for x in tb], cost_ms_all=[round(x, 2) for x in tc],
                         bytes=int(sum(c for _, c, _ in summary) / BYTES), groups={g: [c, m] for g, c, m in summary})
        print(name, json.dumps(res[name]), flush=True)
    d_in = torch.from_numpy(blob).cuda()
    rb = lambda: eng.bill_device(n, d_in.data_ptr(), d_roff.data_ptr(), d_rlen.data_ptr(), L, d_bill.data_ptr(), d_st.data_ptr(), opts,
                                 False, None, strm.cuda_stream)
    tr = [timed(rb) for _ in range(args.reps + 1)][1:]
    res["raw_bill_ms"] = float(np.median(tr))
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)
    eng.close()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--survey", action="store_true")
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    survey() if a.survey else gpu(a)
