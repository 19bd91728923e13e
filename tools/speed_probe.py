"""Literal speeds: what encode_speeds buys on real text, and what it costs on an H100.
    python tools/speed_probe.py --survey                          # CPU (oracle): exact sizes of every palette speed
    python tools/speed_probe.py [--n 4096] [--len 65536] [--reps 3]
--survey is the sweep divans_b200.DEFAULT_LITERAL_SPEEDS was chosen by (DESIGN.md section 4, "Literal speeds").
The GPU mode prints the card's name and power limit, then
  * bytes of alice29 and asyoulik (decoded from the golden fixtures) cut into --len pieces and encoded, at dynamic context mixing 2
    and the UTF8 context mode, by the plain encoder (MUD speeds), encode_auto and encode_speeds with DEFAULT_LITERAL_SPEEDS;
  * encode times of the three calls on n streams of --len bytes in HBM (the fixture text repeated), CUDA events, medians of
    --reps, the three alternating;
  * decode times of the streams encode_speeds and the plain encoder made, which should match: every accepted speed keeps the
    decoder on its fast literal loops.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import auto_probe  # noqa: E402


def survey():
    """CPU (oracle): exact costs of every palette speed on the fixture text.  For each (text, mode, dynamic mixing) it prints
    MUD's stream size, the best uniform speed and its gain, and, at dynamic mixing 2, the gain of the speeds encode_speeds
    chooses from the whole palette.  Then how often each palette speed is chosen for S0, S2 or S3."""
    import collections
    from oracle_tally import tally_py as T
    import divans_b200
    P = divans_b200.LITERAL_SPEED_PALETTE
    fx = auto_probe.fixture_streams()
    texts = {"alice29[:64K]": fx["alice29"][0][:65536], "asyoulik[:64K]": fx["asyoulik"][0][:65536], "alice29[:8K]": fx["alice29"][0][:8192]}
    picks = collections.Counter()
    print("%-15s %4s %5s %9s %-14s %8s %8s" % ("input", "dcm", "mode", "MUD B", "best uniform", "gain", "tuned"))
    for dcm, mode in ((1, 2), (2, 2), (2, 0)):
        for name, d in texts.items():
            mud = T.tally_raw(d, mode, 4, dynamic_context_mixing=dcm, literal_adaptation=[(16, 8192)] * 4)[1]
            rc, out, ch, cost, halves = T.encode_speeds(d, mode, 4, P, dynamic_context_mixing=dcm)
            k = len(P)
            c = int(ch[0])
            picks.update([P[c], P[int(ch[1])], P[int(ch[2])]])
            print("%-15s %4d %5s %9.0f %-14s %7.2f%% %7.2f%%" % (name, dcm, ("LSB6", "MSB6", "UTF8", "SIGN")[mode], mud / 65536 / 8, P[c],
                                                              100 * (1 - cost[c] / mud), 100 * (1 - min(cost[k], cost[c]) / mud)))
    print("chosen (S0, S2, S3 counted once each per row):", ", ".join("%s: %d" % (s, n) for s, n in picks.most_common()))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--survey", action="store_true")
    a = ap.parse_args()
    if a.survey:
        survey()
        return
    import torch
    import divans_b200
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    eng = divans_b200.Engine(0)
    opts = divans_b200.encode_options(literal_pred_mode=2, dynamic_context_mixing=2)
    fx = auto_probe.fixture_streams()
    text = fx["alice29"][0] + fx["asyoulik"][0]
    pieces = [text[i:i + a.len] for i in range(0, len(text), a.len)]
    plain = eng.encode(pieces, opts)
    auto = [x[1] for x in eng.encode_auto(pieces, opts)]
    spd = eng.encode_speeds(pieces, opts)
    print("real text, %d pieces, %d B: plain %d  auto %d  speeds %d bytes" % (len(pieces), len(text), sum(map(len, plain)),
                                                                            sum(map(len, auto)), sum(len(x[1]) for x in spd)))
    print("chosen speeds:", sorted(set(tuple(map(tuple, x[2])) for x in spd)), flush=True)

    big = text * (a.n * a.len // len(text) + 1)
    streams = [big[i * a.len:(i + 1) * a.len] for i in range(a.n)]
    blob, off, ln = divans_b200._pack(streams)
    cap = divans_b200._encoded_cap(ln)
    oo, tot = divans_b200._regions(cap)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_in, d_off, d_len, d_oo, d_cap = dev(blob), dev(off.view(np.int64)), dev(ln.view(np.int64)), dev(oo.view(np.int64)), dev(cap.view(np.int64))
    n = len(streams)
    kinds = ("plain", "auto", "speeds")
    outs = {k: torch.zeros(tot, dtype=torch.uint8, device="cuda") for k in kinds}
    olen = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in kinds}
    st = {k: torch.zeros(n, dtype=torch.int32, device="cuda") for k in kinds}
    ch = torch.zeros(3 * n, dtype=torch.int32, device="cuda")
    ts = torch.cuda.Stream()
    sp = ts.cuda_stream

    def run(kind):
        x = (n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), a.len, outs[kind].data_ptr(), d_oo.data_ptr(), d_cap.data_ptr(),
             olen[kind].data_ptr(), st[kind].data_ptr())
        if kind == "speeds":
            eng.encode_speeds_batch_device(*x, d_chosen=ch.data_ptr(), opts=opts, stream=sp)
        elif kind == "auto":
            eng.encode_auto_batch_device(*x, ch.data_ptr(), opts=opts, stream=sp)
        else:
            eng.encode_batch_device(*x, opts=opts, stream=sp)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record(ts); fn(); e1.record(ts); torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for k in kinds:
        run(k)
    enc = {k: [] for k in kinds}
    for _ in range(a.reps):
        for k in kinds:
            enc[k].append(timed(lambda: run(k)))
    for k in kinds:
        run(k)
    torch.cuda.synchronize()
    assert all(int((st[k] != 0).sum()) == 0 for k in kinds)
    dout = torch.zeros(n * a.len + 4096, dtype=torch.uint8, device="cuda")
    doff = dev((np.arange(n, dtype=np.uint64) * np.uint64(a.len)).view(np.int64))
    dcap = dev(np.full(n, a.len, np.int64))
    dl, ds = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    dec = {"plain": [], "speeds": []}
    for _ in range(a.reps + 1):
        for k in dec:
            dec[k].append(timed(lambda: eng.decode_batch_device(outs[k].data_ptr(), d_oo.data_ptr(), olen[k].data_ptr(), dout.data_ptr(),
                                                                doff.data_ptr(), dcap.data_ptr(), dl.data_ptr(), ds.data_ptr(), n, tot, stream=sp)))
            assert int((ds != 0).sum()) == 0
    med = lambda x: float(np.median(x))
    print("n %d x %d B: bytes plain %d  auto %d  speeds %d" % (n, a.len, int(olen["plain"].sum()), int(olen["auto"].sum()), int(olen["speeds"].sum())))
    print("encode ms: plain %.1f  auto %.1f  speeds %.1f;  decode ms (first run dropped): plain %.1f  speeds %.1f" % (
        med(enc["plain"]), med(enc["auto"]), med(enc["speeds"]), med(dec["plain"][1:]), med(dec["speeds"][1:])))


if __name__ == "__main__":
    main()
