"""Choosing the LZ77 parse per stream by coding cost: what it buys, and what it costs.

    python tools/lz77_parse_probe.py --survey [--streams 3]      # CPU (oracle): exact sizes of every parse on each corpus
    python tools/lz77_parse_probe.py [--n 4096] [--len 65536] [--reps 3]   # H100: times, bytes, decode time

--survey generates the list of every parse (min_match 4..32, lazy 0..2; include/divans_b200.h, "the LZ77 parse") with the CPU
oracle (dvo_lz77_cmds_parse) for a few streams of each corpus of tools/auto_probe.py (the bench's text, UTF-8 text, records of
2, 4 and 8 bytes) and for alice29 and asyoulik, encodes it with the oracle under compress_device's default options (each list's
window, 16; dynamic context mixing 0) and prints the bytes and commands per parse.  It then picks parses greedily: starting from
(4, 0), the parse that most lowers the sum over corpora of the per-stream best size (relative to the corpus's size with (4, 0)),
while it gains at least 0.1 %.  That is how divans_b200.DEFAULT_LZ77_PARSES was chosen.

The GPU mode, for n streams of the bench's text and of the mixed corpus (the five synthetic corpora in turn), reports:
  * gen_ms: the generator's kernel time per parse (CUDA events of the library, median of --reps);
  * compress_ms: wall time of compress_device with DEFAULT_LZ77_PARSES against compress_device with (4, 0) only (the Z
    streams), CUDA events on the caller's stream, medians;
  * bytes of both, and how often each parse was chosen;
  * decode_ms of the chosen streams against the (4, 0) streams (decode_batch_device, alternating, medians).
Every output is decoded on the GPU and compared with its raw input; a difference fails.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from auto_probe import corpora, fixture_streams, gpu_info  # noqa: E402

ALL_PARSES = [(m, z) for m in range(4, 33) for z in range(3)]


def survey(n_streams, length, parses=ALL_PARSES, min_gain=0.001, max_k=4):
    from oracle import oracle_py as O
    from oracle_tally import tally_py as T
    cs = corpora(n_streams, length)
    cs.update(fixture_streams())
    opts = O.options(window_size=16, dynamic_context_mixing=0)
    size = {}   # corpus -> [parse, stream] bytes
    for name, streams in cs.items():
        tab = np.zeros((len(parses), len(streams)), np.int64)
        cmds = np.zeros(len(parses), np.int64)
        for k, (mm, lz) in enumerate(parses):
            for j, s in enumerate(streams):
                cl = T.lz77_parse(O, s, mm, lz, window=16)
                tab[k, j] = len(cl.encode(opts))
                cmds[k] += cl.n_cmds
        size[name] = tab
        base = tab[0].sum()
        best = sorted(range(len(parses)), key=lambda k: tab[k].sum())[:5]
        print("%-9s %8d B  (4,0) %d B / %d cmds  best %s" % (name, sum(len(s) for s in streams), base, cmds[0],
                                                           ", ".join("%s %d / %d" % (parses[k], tab[k].sum(), cmds[k]) for k in best)), flush=True)
    # greedy: the sum over corpora of the per-stream best, relative to (4, 0)
    chosen = [0]
    score = lambda ks: sum(t[ks].min(0).sum() / t[0].sum() for t in size.values())
    cur = score(chosen)
    while len(chosen) < max_k:
        k = min((k for k in range(len(parses)) if k not in chosen), key=lambda k: score(chosen + [k]))
        s = score(chosen + [k])
        if (cur - s) / len(size) < min_gain:
            break
        chosen.append(k)
        cur = s
        print("pick %s: mean size %.4f of (4, 0)" % (parses[k], cur / len(size)), flush=True)
    picks = [parses[k] for k in chosen]
    print(json.dumps(dict(picks=picks, per_corpus={name: dict(base=int(t[0].sum()), chosen=int(t[chosen].min(0).sum()))
                                                   for name, t in size.items()})))
    return picks


def gpu(args):
    import torch
    import divans_b200
    eng = divans_b200.Engine(0)
    parses = divans_b200.DEFAULT_LZ77_PARSES
    L = args.len
    cs = corpora(args.n, L)
    mixed = [cs[("text", "utf8", "stride2", "stride4", "stride8")[k % 5]][k] for k in range(args.n)]
    sets = {"text": cs["text"], "mixed": mixed}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).cuda()
    out = {}
    for name, raws in sets.items():
        n = len(raws)
        blob, off, ln = divans_b200._pack(raws)
        d_in = torch.from_numpy(blob).cuda()
        strm = torch.cuda.Stream()

        def timed(fn):
            a, b = ev(), ev()
            a.record(strm)
            r = fn()
            b.record(strm)
            torch.cuda.synchronize()
            return a.elapsed_time(b), r

        # the generator per parse (kernel time, library events)
        cap = divans_b200.lz77_blob_cap(ln)
        boff, btot = divans_b200._regions(cap)
        d_off, d_len, d_boff, d_cap = t64(off), t64(ln), t64(boff), t64(cap)
        d_blobs = torch.empty(btot, dtype=torch.uint8, device="cuda")
        d_res = torch.zeros(2 * n, dtype=torch.int64, device="cuda")
        gen = {}
        for ps in parses:
            ks = []
            for _ in range(args.reps + 1):
                eng.lz77_cmds_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), L, 16, 2, 4, d_blobs.data_ptr(),
                                           d_boff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), d_res[n:].data_ptr(), strm.cuda_stream, parse=ps)
                torch.cuda.synchronize()   # (the library's events are on strm)
                ks.append(eng.last_kernel_ms())
            assert (d_res[n:].cpu().numpy().view(np.int32)[:n] == 0).all()
            gen["%d,%d" % ps] = float(np.median(ks[1:]))
        del d_blobs
        torch.cuda.empty_cache()
        # compress: chosen parses against (4, 0) only, alternating
        tz, tc = [], []
        for _ in range(args.reps):
            ms, z = timed(lambda: eng.compress_device(d_in, off, ln, stream=strm))
            tz.append(ms)
            ms, c = timed(lambda: eng.compress_device(d_in, off, ln, stream=strm, parses=parses))
            tc.append(ms)
            del z, c
        _, z = timed(lambda: eng.compress_device(d_in, off, ln, stream=strm))
        _, c = timed(lambda: eng.compress_device(d_in, off, ln, stream=strm, parses=parses))
        assert (z[3] == 0).all() and (c[3] == 0).all()
        r = dict(raw=int(ln.sum()), gen_kernel_ms=gen, compress_z_ms=float(np.median(tz)), compress_parses_ms=float(np.median(tc)),
                 bytes_z=int(z[2].sum()), bytes_parses=int(c[2].sum()),
                 chosen_hist=np.bincount(c[4], minlength=len(parses)).tolist())
        # decode: chosen streams against Z streams, alternating; every output equals the input
        ocap = np.array(ln, np.uint64)
        doff, dtot = divans_b200._regions(ocap)
        d_doff, d_dcap = t64(doff), t64(ocap)
        d_dec = torch.empty(dtot, dtype=torch.uint8, device="cuda")
        d_ol = torch.zeros(n, dtype=torch.int64, device="cuda")
        d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
        want = np.frombuffer(b"".join(raws), np.uint8)
        td = {"z": [], "parses": []}
        for rep in range(args.reps + 1):
            for tag, res in (("z", z), ("parses", c)):
                d_new, new_off, new_len = res[0], t64(res[1]), t64(res[2])
                ms, _ = timed(lambda: eng.decode_batch_device(d_new.data_ptr(), new_off.data_ptr(), new_len.data_ptr(), d_dec.data_ptr(),
                                                              d_doff.data_ptr(), d_dcap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), n,
                                                              int(d_new.numel()), 0, strm.cuda_stream))
                if rep == 0:
                    h = d_dec.cpu().numpy()
                    assert (d_st.cpu().numpy() == 0).all(), "%s %s: a stream failed to decode" % (name, tag)
                    assert all((h[int(a):int(a) + int(l)] == want[int(o):int(o) + int(l)]).all()
                               for a, o, l in zip(doff, np.concatenate([[0], np.cumsum(ln)[:-1]]), ln)), "%s %s: output differs" % (name, tag)
                else:
                    td[tag].append(ms)
        r["decode_z_ms"], r["decode_parses_ms"] = float(np.median(td["z"])), float(np.median(td["parses"]))
        out[name] = r
        print(name, json.dumps(r), flush=True)
        del z, c, d_dec
        torch.cuda.empty_cache()
    print(json.dumps(dict(gpu=gpu_info(), n=args.n, len=L, reps=args.reps, parses=parses, results=out)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--survey", action="store_true")
    ap.add_argument("--streams", type=int, default=3)
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if args.survey:
        survey(args.streams, args.len)
    else:
        gpu(args)


if __name__ == "__main__":
    main()
