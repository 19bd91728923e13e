"""Dictionary words under every RFC 7932 transform in the LZ77 parse: what they buy, and what they cost.

    python tools/lz77_words_probe.py --survey                    # CPU (oracle): exact sizes, and the pick of the default parses
    python tools/lz77_words_probe.py [--n 4096] [--compress-n 1024] [--len 65536] [--reps 3]   # H100: times and bytes

--survey generates, with the library's host generator (equal to the oracle's dvo_lz77_cmds_words_parse, tests/
test_lz77_words_oracle.py), the list of every parse of DEFAULT_LZ77_DICT_PARSES and of each parse of DEFAULT_LZ77_PARSES with
dict_min 4, 5, 6, 8, 10, 12 or 16 under every transform (transforms 1; include/divans_b200.h, "dictionary words under every
transform in the LZ77 parse"), for the corpora of tools/lz77_dict_probe.py --survey.  Each list is encoded by the oracle under
compress_device's default options (window 16, dynamic context mixing 0), and a stream costs the least of its parses' sizes.  The
pick starts from DEFAULT_LZ77_DICT_PARSES and adds, greedily, the parse that most lowers the mean over corpora of the size
relative to DEFAULT_LZ77_DICT_PARSES, while it gains at least 0.05 % and the set has at most 16 parses.  That is how
DEFAULT_LZ77_WORD_PARSES was chosen.  It also codes alice29 whole at window 22 with dynamic context mixing 1, under each set,
against the 47,601 bytes of the stream of the reference's quality-11 command list (tests/golden/alice29_q11_mix1.divans).

The GPU mode, for n streams of the bench's text and n 16 KiB slices of alice29 and asyoulik (the first --compress-n of each for
compress_device), reports:
  * gen_kernel_ms: the generator's kernel time for (4, 0, 4) and (7, 2, 4), each with the 44-member set (transforms 0) and every
    transform (transforms 1), on both corpora, run alternately (CUDA events of the library, medians of --reps);
  * compress_ms and bytes of compress_device with DEFAULT_LZ77_DICT_PARSES and with DEFAULT_LZ77_WORD_PARSES, alternating,
    medians, on both corpora;
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
from lz77_dict_probe import DICT_MINS, survey_corpora  # noqa: E402

Q11_BYTES = 47601   # tests/golden/alice29_q11_mix1.divans: alice29, window 22, dynamic context mixing 1


def _sizes(streams, parses, window, opts):
    """[parse, stream] oracle-coded bytes of the host generator's lists"""
    import divans_b200
    from oracle import oracle_py as O
    from oracle_tally import tally_py as T
    blob, off, ln = divans_b200._pack(streams)
    tab = np.zeros((len(parses), len(streams)), np.int64)
    for k, ps in enumerate(parses):
        out, bo, bl = divans_b200.lz77_cmds_batch(blob, off, ln, window, 2, 4, parse=ps)
        for j in range(len(streams)):
            tab[k, j] = len(T.from_blob(O, out[int(bo[j]):int(bo[j] + bl[j])].tobytes()).encode(opts))
    return tab


def survey(min_gain=0.0005, max_parses=16):
    import divans_b200
    from oracle import oracle_py as O
    base = [tuple(p) for p in divans_b200.DEFAULT_LZ77_DICT_PARSES]
    parses = base + [tuple(p[:2]) + (dm, 1) for p in divans_b200.DEFAULT_LZ77_PARSES for dm in DICT_MINS]
    opts = O.options(window_size=16, dynamic_context_mixing=0)
    size, raw = {}, {}
    nb = len(base)
    for name, streams in survey_corpora().items():
        tab = _sizes(streams, parses, 16, opts)
        size[name], raw[name] = tab, sum(len(s) for s in streams)
        print("%-10s %8d B  dict %d B  best single words parse %s" % (
            name, raw[name], tab[:nb].min(0).sum(), min(parses[nb:], key=lambda p: tab[parses.index(p)].sum())), flush=True)
    chosen = list(range(nb))
    score = lambda ks: np.mean([t[ks].min(0).sum() / t[:nb].min(0).sum() for t in size.values()])
    cur = score(chosen)
    while len(chosen) < max_parses:
        k = min((k for k in range(nb, len(parses)) if k not in chosen), key=lambda k: score(chosen + [k]))
        s = score(chosen + [k])
        if cur - s < min_gain:
            break
        chosen.append(k)
        cur = s
        print("pick %s: mean size %.5f of DEFAULT_LZ77_DICT_PARSES" % (parses[k], cur), flush=True)
    picks = [parses[k] for k in chosen]
    current = [parses.index(tuple(p)) for p in divans_b200.DEFAULT_LZ77_WORD_PARSES]
    rows = {name: dict(raw=raw[name], dict=int(t[:nb].min(0).sum()), picked=int(t[chosen].min(0).sum()),
                       default_words=int(t[current].min(0).sum()),
                       dict_bpb=round(float(t[:nb].min(0).sum()) / raw[name], 5),
                       default_words_bpb=round(float(t[current].min(0).sum()) / raw[name], 5)) for name, t in size.items()}
    # alice29 at window 22, dynamic context mixing 1, against the reference's quality-11 list
    alice = fixture_streams()["alice29"][0]
    q = _sizes([alice], parses, 22, O.options(window_size=22, dynamic_context_mixing=1))[:, 0]
    w22 = dict(q11=Q11_BYTES, dict=int(q[:nb].min()), picked=int(q[chosen].min()), default_words=int(q[current].min()),
               best_dict_parse=str(parses[int(np.argmin(q[:nb]))]), best_parse=str(parses[int(np.argmin(q))]), best=int(q.min()))
    print(json.dumps(dict(picks=picks, per_corpus=rows, alice29_w22_mix1=w22)))
    return picks


def gpu(args):
    import torch
    import divans_b200
    from divans_b200 import synth
    eng = divans_b200.Engine(0)
    L, n = args.len, args.n
    blob, off, ln = synth.text_streams(n, L)
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

    fx = fixture_streams()
    books = b"".join(fx["alice29"] + fx["asyoulik"])
    slice_of = lambda k: books[(k * 16384) % (len(books) - 16384):][:16384]
    gen_parses = [(4, 0, 4, 0), (4, 0, 4, 1), (7, 2, 4, 0), (7, 2, 4, 1)]
    gen_ms = {}
    for cname, raws in (("text", None), ("books16k", [slice_of(k) for k in range(n)])):
        if raws is None:
            g_in, g_off, g_len, g_max = d_in, off, ln, L
        else:
            gb, g_off, g_len = divans_b200._pack(raws)
            g_in, g_max = torch.from_numpy(gb).cuda(), 16384
        cap = divans_b200.lz77_blob_cap(g_len)
        boff, btot = divans_b200._regions(cap)
        d_off, d_len, d_boff, d_cap = t64(g_off), t64(g_len), t64(boff), t64(cap)
        d_blobs = torch.empty(btot, dtype=torch.uint8, device="cuda")
        d_res = torch.zeros(2 * n, dtype=torch.int64, device="cuda")
        gen = {ps: [] for ps in gen_parses}
        for rep in range(args.reps + 1):
            for ps in gen_parses:
                eng.lz77_cmds_batch_device(n, g_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), g_max, 16, 2, 4, d_blobs.data_ptr(),
                                           d_boff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), d_res[n:].data_ptr(), strm.cuda_stream,
                                           parse=ps)
                torch.cuda.synchronize()
                if rep:
                    gen[ps].append(eng.last_kernel_ms())
                else:
                    assert (d_res[n:].cpu().numpy().view(np.int32)[:n] == 0).all()
        gen_ms[cname] = {"%s" % (ps,): float(np.median(v)) for ps, v in gen.items()}
        del d_blobs
    eng.close()   # (its generator scratch; compress_device gets a context of its own)
    torch.cuda.empty_cache()
    res = dict(gen_kernel_ms=gen_ms)
    nc = min(n, args.compress_n)
    corpora = {"text": [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off[:nc], ln[:nc])],
               "books16k": [slice_of(k) for k in range(nc)]}
    eng = divans_b200.Engine(0)
    sets = {"dict_parses": divans_b200.DEFAULT_LZ77_DICT_PARSES, "word_parses": divans_b200.DEFAULT_LZ77_WORD_PARSES}
    for cname, raws in corpora.items():
        cb, coff, cln = divans_b200._pack(raws)
        c_in = torch.from_numpy(cb).cuda()
        times = {k: [] for k in sets}
        last = {}
        for rep in range(args.reps + 1):
            for tag, ps in sets.items():
                ms, c = timed(lambda: eng.compress_device(c_in, coff, cln, stream=strm, parses=ps))
                assert (c[3] == 0).all()
                if rep:
                    times[tag].append(ms)
                else:
                    last[tag] = (int(c[2].sum()), np.bincount(c[4], minlength=len(ps)).tolist())
                    h = c[0].cpu().numpy()
                    for k0 in range(0, nc, 512):
                        got = eng.decode([h[int(o):int(o + l)].tobytes() for o, l in zip(c[1][k0:k0 + 512], c[2][k0:k0 + 512])],
                                         [len(r) + 64 for r in raws[k0:k0 + 512]])
                        assert all(s == 0 and b == r for (s, b), r in zip(got, raws[k0:k0 + 512])), (cname, tag)
                    del h, got
                del c
        res[cname] = {tag: dict(compress_ms=float(np.median(times[tag])), bytes=last[tag][0], chosen_hist=last[tag][1],
                                raw=int(cln.sum())) for tag in sets}
        del c_in
    print(json.dumps(dict(gpu=gpu_info(), gen_n=n, compress_n=nc, len=L, reps=args.reps, all_decoded=True, results=res)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--survey", action="store_true")
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=65536)
    ap.add_argument("--compress-n", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if args.survey:
        survey()
    else:
        gpu(args)


if __name__ == "__main__":
    main()
