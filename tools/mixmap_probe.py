"""Per-context mixing values: what encode_mixmap buys, and what it costs.

    python tools/mixmap_probe.py --survey [--streams 2] [--len 16384]   # CPU (oracle): exact stream sizes per corpus
    python tools/mixmap_probe.py [--n 4096] [--len 65536] [--reps 3]      # H100: encode and decode times

--survey encodes a few streams of each corpus of DESIGN.md's candidate table (text, UTF-8, records of 2, 4 and 8 bytes,
alice29, asyoulik) and of two mixed corpora (text then 4-byte records in one stream; 2-byte then 8-byte records) with the CPU
oracle, and prints bytes per input byte of three encoders: the default model (LSB6, 4), encode_auto with
DEFAULT_LITERAL_MODELS, and encode_mixmap with all 16 values under each context mode; then the same for the oracle's LZ77
lists (window 16).  It also counts, over all corpora, how many literal nibbles' worth of cost each value wins per entry, which
is how divans_b200.DEFAULT_MIXING_VALUES was chosen.

The GPU mode times encode_mixmap_batch_device with DEFAULT_MIXING_VALUES against encode_auto_batch_device with
DEFAULT_LITERAL_MODELS (every context mode) on n streams in HBM -- text then 4-byte records, 2-byte then 8-byte records, text, 4-byte records --
under the UTF8 context mode, the survey's best single mode, then the decode of the streams each produced (CUDA events,
the two sides alternating, medians).
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import auto_probe  # noqa: E402


def corpora(n, length):
    cs = auto_probe.corpora(n, length)
    cs.update({k: [s[:length] for s in v] for k, v in auto_probe.fixture_streams().items()})
    half = length // 2
    cs["text+rec4"] = [t[:half] + r[:half] for t, r in zip(cs["text"], cs["stride4"])]
    cs["rec2+rec8"] = [a[:half] + b[:half] for a, b in zip(cs["stride2"], cs["stride8"])]
    return cs


def survey(n, length):
    import divans_b200
    from oracle import oracle_py as O
    from oracle_tally import tally_py as T
    allv = list(range(16))
    wins = np.zeros(16)
    print("%-10s %8s %8s %8s %s" % ("corpus", "", "default", "auto", "mixmap LSB6 / MSB6 / UTF8 / SIGN"))
    for name, streams in corpora(n, length).items():
        raw = sum(len(s) for s in streams)
        for lz in (False, True):
            d = a = 0
            m = np.zeros(4)
            for s in streams:
                if lz:
                    cmds = O.Commands.lz77(s, 16, 0, 4)
                    d += len(T.encode_cmds_auto(cmds, [(0, 4)])[1])
                    a += len(T.encode_cmds_auto(cmds, divans_b200.DEFAULT_LITERAL_MODELS)[1])
                else:
                    d += len(T.encode_raw_model(s, 0, 4)[1])
                    a += len(T.encode_auto(s, divans_b200.DEFAULT_LITERAL_MODELS)[1])
                for p in range(4):
                    rc, out, ch, mixing, cost, bins = T.encode_cmds_mixmap(cmds, p, allv) if lz else T.encode_mixmap(s, p, allv)
                    m[p] += len(out)
                    if not lz:   # the cost each value saves per entry against the entry's worst value
                        ok = bins.max(axis=1) != T.TALLY_FAILED
                        b = bins[ok].astype(np.float64)
                        wins += np.bincount(np.argmin(b, axis=0), weights=b.max(axis=0) - b.min(axis=0), minlength=16) / 65536 / 8
            print("%-10s %8s %8.4f %8.4f %s" % (name, "lz77" if lz else "literal", d / raw, a / raw, " / ".join("%.4f" % (x / raw) for x in m)))
    order = np.argsort(-wins)
    print("bytes saved per value (winning entries, against the entry's worst value):",
          ", ".join("%d: %.0f" % (v, wins[v]) for v in order))


def gpu(args):
    import torch
    import divans_b200
    eng = divans_b200.Engine(0)
    per = args.n // 4
    cs = corpora(per, args.len)
    streams = (cs["text+rec4"] + cs["rec2+rec8"] + cs["text"] + cs["stride4"])[:args.n]
    blob, off, ln = divans_b200._pack(streams)
    cap = divans_b200._encoded_cap(ln)
    oo, tot = divans_b200._regions(cap)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_in, d_off, d_len, d_oo, d_cap = dev(blob), dev(off.view(np.int64)), dev(ln.view(np.int64)), dev(oo.view(np.int64)), dev(cap.view(np.int64))
    n = len(streams)
    outs = {k: torch.zeros(tot, dtype=torch.uint8, device="cuda") for k in ("mixmap", "auto")}
    olen = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in outs}
    st = {k: torch.zeros(n, dtype=torch.int32, device="cuda") for k in outs}
    ch = torch.zeros(n, dtype=torch.int32, device="cuda")
    k = len(divans_b200.DEFAULT_MIXING_VALUES)
    ts = torch.cuda.Stream()
    sp = ts.cuda_stream   # every call runs on this stream, and the events that time it are recorded there

    def run(kind):
        a = (n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), args.len, outs[kind].data_ptr(), d_oo.data_ptr(), d_cap.data_ptr(),
             olen[kind].data_ptr(), st[kind].data_ptr())
        if kind == "mixmap":
            eng.encode_mixmap_batch_device(*a, d_chosen=ch.data_ptr(), opts=divans_b200.encode_options(literal_pred_mode=2), stream=sp)
        else:
            eng.encode_auto_batch_device(*a, ch.data_ptr(), stream=sp)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record(ts); fn(); e1.record(ts); torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    enc = {"mixmap": [], "auto": []}
    for _ in range(args.reps):
        for kind in enc:
            enc[kind].append(timed(lambda: run(kind)))
    run("mixmap"); torch.cuda.synchronize()
    chosen = ch.cpu().numpy()
    dec = {"mixmap": [], "auto": []}
    dout = torch.zeros(n * args.len + 4096, dtype=torch.uint8, device="cuda")
    doff = dev((np.arange(n, dtype=np.uint64) * np.uint64(args.len)).view(np.int64))
    dcap = dev(np.full(n, args.len, np.int64))
    dl, ds = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    for kind in dec:
        run(kind)
    for _ in range(args.reps):
        for kind in dec:
            dec[kind].append(timed(lambda: eng.decode_batch_device(outs[kind].data_ptr(), d_oo.data_ptr(), olen[kind].data_ptr(), dout.data_ptr(),
                                                                   doff.data_ptr(), dcap.data_ptr(), dl.data_ptr(), ds.data_ptr(), n, tot, stream=sp)))
            assert int((ds != 0).sum()) == 0
    med = lambda x: float(np.median(x))
    print("n %d x %d B, %d mixed records of %d; bytes mixmap %d auto %d" % (n, args.len, int((chosen == k).sum()), n,
                                                                             int(olen["mixmap"].sum()), int(olen["auto"].sum())))
    print("encode ms: mixmap %.1f  auto %.1f;  decode ms: mixmap %.1f  auto %.1f" % (med(enc["mixmap"]), med(enc["auto"]),
                                                                                    med(dec["mixmap"]), med(dec["auto"])))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--survey", action="store_true")
    ap.add_argument("--streams", type=int, default=2)
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if a.survey:
        survey(a.streams, a.len or 16384)
    else:
        a.len = a.len or 65536
        gpu(a)


if __name__ == "__main__":
    main()
