"""Dictionary words in the LZ77 parse: what they buy, and what they cost.

    python tools/lz77_dict_probe.py --survey                     # CPU (oracle): exact sizes, and the pick of the default parses
    python tools/lz77_dict_probe.py [--n 4096] [--compress-n 1024] [--len 65536] [--reps 5]   # H100: times and bytes

--survey generates, with the library's host generator (equal to the oracle's dvo_lz77_cmds_dict_parse, tests/
test_lz77_dict_oracle.py), the list of every parse of DEFAULT_LZ77_PARSES and of each of them with dict_min 4, 5, 6, 8, 10, 12 or
16 (include/divans_b200.h, "dictionary words in the LZ77 parse"), for: 16 streams of the bench's synthetic text (64 KiB),
alice29, asyoulik, their 1, 4, 16 and 64 KiB prefixes, and a buffer built from dictionary words (tests/lz77_dict_corpora.py).
Each list is encoded by the oracle under compress_device's default options (window 16, dynamic context mixing 0), and a stream
costs the least of its parses' sizes.  The pick starts from DEFAULT_LZ77_PARSES and adds, greedily, the dictionary parse that most
lowers the mean over corpora of the size relative to DEFAULT_LZ77_PARSES, while it gains at least 0.05 %.  It prints the exact
sizes (bytes per input byte) under DEFAULT_LZ77_PARSES and the picked set.  That is how DEFAULT_LZ77_DICT_PARSES was chosen.

The GPU mode, for n streams of the bench's text (the first --compress-n of them for compress_device, whose k lists per stream
are held in HBM at once), reports:
  * gen_kernel_ms: the generator's kernel time for (4, 0), (4, 0, 4), (6, 2) and (6, 2, 6), run alternately (CUDA events of the
    library, medians of --reps);
  * compress_ms and bytes of compress_device with DEFAULT_LZ77_PARSES and with DEFAULT_LZ77_DICT_PARSES, alternating, medians;
  * how often each parse was chosen.
Every compressed stream is decoded on the GPU (512 at a time) and compared with its input; a difference fails.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from auto_probe import fixture_streams, gpu_info  # noqa: E402

DICT_MINS = (4, 5, 6, 8, 10, 12, 16)


def survey_corpora():
    import lz77_dict_corpora as C
    from divans_b200 import synth
    blob, off, ln = synth.text_streams(16, 65536)
    fx = fixture_streams()
    alice, ayl = fx["alice29"][0], fx["asyoulik"][0]
    cs = {"text": [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)], "alice29": [alice], "asyoulik": [ayl]}
    for k in (1, 4, 16, 64):
        cs["prefix%dk" % k] = [alice[:k << 10], ayl[:k << 10]]
    cs["words"] = [C.word_buffer(3000, 1)]
    return cs


def survey(min_gain=0.0005, max_add=4):
    import divans_b200
    from oracle import oracle_py as O
    from oracle_tally import tally_py as T
    base = divans_b200.DEFAULT_LZ77_PARSES
    parses = list(base) + [tuple(p) + (dm,) for p in base for dm in DICT_MINS]
    opts = O.options(window_size=16, dynamic_context_mixing=0)
    size, raw = {}, {}
    for name, streams in survey_corpora().items():
        blob, off, ln = divans_b200._pack(streams)
        tab = np.zeros((len(parses), len(streams)), np.int64)
        for k, ps in enumerate(parses):
            out, bo, bl = divans_b200.lz77_cmds_batch(blob, off, ln, 16, 2, 4, parse=ps)
            for j in range(len(streams)):
                tab[k, j] = len(T.from_blob(O, out[int(bo[j]):int(bo[j] + bl[j])].tobytes()).encode(opts))
        size[name], raw[name] = tab, int(ln.sum())
        nb = len(base)
        print("%-10s %8d B  base %d B  best single dict parse %s" % (
            name, raw[name], tab[:nb].min(0).sum(), min(parses[nb:], key=lambda p: tab[parses.index(p)].sum())), flush=True)
    nb = len(base)
    chosen = list(range(nb))
    score = lambda ks: np.mean([t[ks].min(0).sum() / t[:nb].min(0).sum() for t in size.values()])
    cur = score(chosen)
    while len(chosen) < nb + max_add:
        k = min((k for k in range(nb, len(parses)) if k not in chosen), key=lambda k: score(chosen + [k]))
        s = score(chosen + [k])
        if cur - s < min_gain:
            break
        chosen.append(k)
        cur = s
        print("pick %s: mean size %.5f of DEFAULT_LZ77_PARSES" % (parses[k], cur), flush=True)
    picks = [parses[k] for k in chosen]
    current = [parses.index(tuple(p)) for p in divans_b200.DEFAULT_LZ77_DICT_PARSES]
    rows = {name: dict(raw=raw[name], base=int(t[:nb].min(0).sum()), picked=int(t[chosen].min(0).sum()),
                       default_dict=int(t[current].min(0).sum()),
                       base_bpb=round(float(t[:nb].min(0).sum()) / raw[name], 5),
                       default_dict_bpb=round(float(t[current].min(0).sum()) / raw[name], 5)) for name, t in size.items()}
    print(json.dumps(dict(picks=picks, per_corpus=rows)))
    return picks


def gpu(args):
    import torch
    import divans_b200
    from divans_b200 import synth
    eng = divans_b200.Engine(0)
    L, n = args.len, args.n
    blob, off, ln = synth.text_streams(n, L)
    raws = [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)]
    d_in = torch.from_numpy(blob).cuda()
    strm = torch.cuda.Stream()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).cuda()

    def timed(fn):
        a, b = ev(), ev()
        a.record(strm)
        r = fn()
        b.record(strm)
        torch.cuda.synchronize()
        return a.elapsed_time(b), r

    cap = divans_b200.lz77_blob_cap(ln)
    boff, btot = divans_b200._regions(cap)
    d_off, d_len, d_boff, d_cap = t64(off), t64(ln), t64(boff), t64(cap)
    d_blobs = torch.empty(btot, dtype=torch.uint8, device="cuda")
    d_res = torch.zeros(2 * n, dtype=torch.int64, device="cuda")
    gen_parses = [(4, 0), (4, 0, 4), (6, 2), (6, 2, 6)]
    gen = {ps: [] for ps in gen_parses}
    n_words = {}
    for rep in range(args.reps + 1):
        for ps in gen_parses:
            eng.lz77_cmds_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), L, 16, 2, 4, d_blobs.data_ptr(),
                                       d_boff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), d_res[n:].data_ptr(), strm.cuda_stream, parse=ps)
            torch.cuda.synchronize()
            if rep:
                gen[ps].append(eng.last_kernel_ms())
            else:
                assert (d_res[n:].cpu().numpy().view(np.int32)[:n] == 0).all()
                h = d_blobs.cpu().numpy()
                recs = [np.frombuffer(h[int(b) + 32:int(b) + 32 + 20 * int(h[int(b) + 8:int(b) + 12].view(np.uint32)[0])], np.uint32) for b in boff[:64]]
                n_words["%s" % (ps,)] = int(sum((r.reshape(-1, 5)[:, 0] == 2).sum() for r in recs))
    del d_blobs
    eng.close()   # (its generator scratch; compress_device gets a context of its own)
    torch.cuda.empty_cache()
    eng = divans_b200.Engine(0)
    n = min(n, args.compress_n)
    off, ln, raws = off[:n], ln[:n], raws[:n]
    res = dict(gen_kernel_ms={"%s" % (ps,): float(np.median(v)) for ps, v in gen.items()}, words_in_first_64_lists=n_words)
    sets = {"parses": divans_b200.DEFAULT_LZ77_PARSES, "dict_parses": divans_b200.DEFAULT_LZ77_DICT_PARSES}
    times = {k: [] for k in sets}
    last = {}
    for rep in range(args.reps + 1):
        for tag, ps in sets.items():
            ms, c = timed(lambda: eng.compress_device(d_in, off, ln, stream=strm, parses=ps))
            assert (c[3] == 0).all()
            if rep:
                times[tag].append(ms)
            else:
                last[tag] = (int(c[2].sum()), np.bincount(c[4], minlength=len(ps)).tolist())
                h = c[0].cpu().numpy()
                for k0 in range(0, n, 512):   # (in slices: the generator's scratch still holds device memory)
                    got = eng.decode([h[int(o):int(o + l)].tobytes() for o, l in zip(c[1][k0:k0 + 512], c[2][k0:k0 + 512])],
                                     [len(r) + 64 for r in raws[k0:k0 + 512]])
                    assert all(s == 0 and b == r for (s, b), r in zip(got, raws[k0:k0 + 512])), tag
                del h, got
            del c
    for tag in sets:
        res[tag] = dict(compress_ms=float(np.median(times[tag])), bytes=last[tag][0], chosen_hist=last[tag][1])
    print(json.dumps(dict(gpu=gpu_info(), gen_n=args.n, compress_n=n, len=L, reps=args.reps, compress_raw=int(ln.sum()), results=res)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--survey", action="store_true")
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=65536)
    ap.add_argument("--compress-n", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if args.survey:
        survey()
    else:
        gpu(args)


if __name__ == "__main__":
    main()
