"""Literal model selection: what encode_auto buys, and what it costs.

    python tools/auto_probe.py --survey [--streams 8]        # CPU (oracle): the cost of every literal model on each corpus
    python tools/auto_probe.py [--n 4096] [--len 65536] [--reps 3]   # H100: ratio, pick accuracy, encode and decode times
    python tools/auto_probe.py --transcode [--n 4096] [--lz-n 512]   # H100: transcode_device with and without candidates

--survey tallies every (pred_mode, mixing value) pair, mixing value 2 included, with the CPU oracle on a few streams of each
corpus and prints the table DESIGN.md section 4 quotes; it is how divans_b200.DEFAULT_LITERAL_MODELS was chosen.

The GPU mode, for the bench's text streams and for a mixed corpus (text, UTF-8 text, records of 2, 4 and 8 bytes), reports:
  * compressed bytes with the default model (LSB6, 4), with encode_auto and DEFAULT_LITERAL_MODELS, and with the per-stream
    exact optimum (every candidate encoded, the shortest stream kept), and how often the tally picked the exact optimum;
  * wall time of encode_auto_batch_device against C x encode_batch_device (inputs already in HBM);
  * decode time of the auto-encoded corpus against the default-encoded one.
Times alternate the two sides run by run and report medians (CUDA events around each call).

--transcode stores the same two corpora with the default model (literal-only streams, n of them) and as LZ77 lists from
divans_b200.lz77_cmds_batch (window 16, the generator's model (UTF8, 4); --lz-n of them: an LZ77 transcode needs a blob
region per stream on top of the encoder's logs), then reports the bytes and wall time of Engine.transcode_device without
candidates and with [LITERAL_MODEL_KEEP] + DEFAULT_LITERAL_MODELS, and the decode time of both outputs.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from divans_b200 import synth  # noqa: E402


def utf8_streams(n, length, seed=7):
    """the bench's text with every lowercase letter written as a two-byte Cyrillic letter (U+0430 + k)"""
    blob, off, ln = synth.text_streams(n, length, seed=seed)
    lut = [bytes([c]) for c in range(256)]
    for k in range(26):
        lut[ord("a") + k] = chr(0x430 + k).encode()
    out = []
    for i in range(n):
        s = b"".join(lut[c] for c in blob[int(off[i]):int(off[i]) + length].tobytes())
        out.append(s[:length])
    return out


def record_streams(n, length, width, seed=11):
    """fixed-width binary records: column j of every record is a slowly drifting small value of its own (a counter, flags,
    a level), so the byte `width` positions back predicts the next one far better than the byte before"""
    rng = np.random.default_rng(seed + width)
    out = []
    n_rec = (length + width - 1) // width
    for _ in range(n):
        cols = []
        for j in range(width):
            base = int(rng.integers(0, 256))
            step = rng.integers(-2, 3, n_rec) * (1 if j % 2 == 0 else 0) + (rng.random(n_rec) < 0.05) * rng.integers(0, 256, n_rec)
            cols.append((base + np.cumsum(step)) & 0xFF if j % 3 != 2 else rng.choice([0, 1, 3, 7, 0x80], n_rec))
        rec = np.stack(cols, 1).astype(np.uint8).reshape(-1)
        out.append(rec[:length].tobytes())
    return out


def fixture_streams():
    """alice29.txt and asyoulik.txt, decoded from the golden fixtures"""
    import lzma
    from oracle import oracle_py as O
    g = os.path.join(ROOT, "tests", "golden")
    rc, alice = O.decode(open(os.path.join(g, "alice29_literal_only.divans"), "rb").read(), out_cap=1 << 20)
    assert rc == 0
    ir = lzma.decompress(open(os.path.join(g, "asyoulik.ir.xz"), "rb").read())
    rc, ayl = O.Commands.from_ir(ir).recode(22)
    assert rc == 0
    return {"alice29": [alice], "asyoulik": [ayl]}


def corpora(n, length):
    blob, off, ln = synth.text_streams(n, length)
    c = {"text": [blob[int(o):int(o) + int(l)].tobytes() for o, l in zip(off, ln)], "utf8": utf8_streams(n, length)}
    for w in (2, 4, 8):
        c["stride%d" % w] = record_streams(n, length, w)
    return c


def survey(n_streams, length):
    from oracle_tally import tally_py as T
    cs = corpora(n_streams, length)
    cs.update(fixture_streams())
    models = [(pm, mv) for pm in range(4) for mv in range(16)]
    res = {}
    for name, streams in cs.items():
        tot = np.zeros(len(models))
        for s in streams:
            for k, (pm, mv) in enumerate(models):
                rc, c = T.tally_raw(s, pm, mv)
                tot[k] += c / 65536 / 8 if rc == 0 else np.inf
        raw = sum(len(s) for s in streams)
        res[name] = {"%d,%d" % m: round(t / raw, 4) for m, t in zip(models, tot)}
        best = sorted(range(len(models)), key=lambda k: tot[k])[:6]
        print("%-9s %8d B  default %.4f  best %s" % (name, raw, tot[models.index((0, 4))] / raw,
                                                      ", ".join("(%d,%d) %.4f" % (models[k] + (tot[k] / raw,)) for k in best)))
    print(json.dumps(res))


def gpu(args):
    import torch
    import divans_b200
    eng = divans_b200.Engine(0)
    cands = divans_b200.DEFAULT_LITERAL_MODELS
    L = args.len
    cs = corpora(args.n, L)
    mixed = []
    for k in range(args.n):
        mixed.append(cs[("text", "utf8", "stride2", "stride4", "stride8")[k % 5]][k])
    sets = {"text": cs["text"], "mixed": mixed}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    out = {}
    for name, raws in sets.items():
        n = len(raws)
        d_in = torch.from_numpy(np.frombuffer(b"".join(raws), np.uint8).copy()).cuda()
        in_off = np.arange(n, dtype=np.uint64) * np.uint64(L)
        in_len = np.array([len(r) for r in raws], np.uint64)
        cap = np.full(n, L + L // 2 + 70000, np.uint64)
        out_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
        d_off, d_len, d_oo, d_cap = t(in_off), t(in_len), t(out_off), t(cap)
        d_out = torch.empty(int(cap.sum()), dtype=torch.uint8, device="cuda")
        d_ol = torch.zeros(n, dtype=torch.int64, device="cuda")
        d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
        d_ch = torch.zeros(n, dtype=torch.int32, device="cuda")
        d_cost = torch.zeros(n * len(cands), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        strm = torch.cuda.Stream()   # the library's calls and the events on one stream of our own (NULL would be the context's stream)
        st = strm.cuda_stream

        def plain(pm, mv):
            eng.encode_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), L, d_out.data_ptr(), d_oo.data_ptr(),
                                    d_cap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(),
                                    divans_b200.encode_options(literal_pred_mode=pm, literal_mixing_value=mv), st)

        def auto():
            eng.encode_auto_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), L, d_out.data_ptr(), d_oo.data_ptr(),
                                         d_cap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), d_ch.data_ptr(), d_cost.data_ptr(),
                                         None, cands, st)

        def streams():
            torch.cuda.synchronize()
            o, ln_ = d_out.cpu().numpy(), d_ol.cpu().numpy()
            assert (d_st.cpu().numpy() == 0).all()
            return [o[int(a):int(a) + int(b)].tobytes() for a, b in zip(out_off, ln_)]

        # sizes: every candidate, then auto
        per = []
        for pm, mv in cands:
            plain(pm, mv)
            per.append([len(s) for s in streams()])
        per = np.array(per)
        auto()
        a_streams = streams()
        chosen = d_ch.cpu().numpy()
        plain(*cands[0])
        d_streams = streams()
        exact = per.argmin(0)
        r = dict(raw=int(in_len.sum()), default=int(per[0].sum()), auto=int(sum(len(s) for s in a_streams)),
                 optimum=int(per.min(0).sum()), picks_optimum=float((per[chosen, np.arange(n)] == per.min(0)).mean()),
                 chosen_hist=np.bincount(chosen, minlength=len(cands)).tolist(), exact_hist=np.bincount(exact, minlength=len(cands)).tolist())

        def timed(fn):
            a, b = ev(), ev()
            a.record(strm)
            fn()
            b.record(strm)
            torch.cuda.synchronize()
            return a.elapsed_time(b)

        # encode: auto against C plain encodes, alternating
        ta, tc = [], []
        for _ in range(args.reps):
            ta.append(timed(auto))
            tc.append(timed(lambda: [plain(pm, mv) for pm, mv in cands]))
        r["encode_auto_ms"], r["encode_C_plain_ms"] = float(np.median(ta)), float(np.median(tc))
        # decode: the auto-encoded corpus against the default-encoded one, alternating
        dec = {}
        for tag, ss in (("default", d_streams), ("auto", a_streams)):
            lens = np.array([len(s) for s in ss], np.uint64)
            offs = np.concatenate([[0], np.cumsum((lens + np.uint64(15)) & ~np.uint64(15))[:-1]]).astype(np.uint64)
            buf = np.zeros(int(offs[-1] + lens[-1]) + 16, np.uint8)
            for s, o in zip(ss, offs):
                buf[int(o):int(o) + len(s)] = np.frombuffer(s, np.uint8)
            dec[tag] = (torch.from_numpy(buf).cuda(), t(offs), t(lens))
        ocap = np.full(n, L, np.uint64)
        d_doff, d_dcap = t(np.arange(n, dtype=np.uint64) * np.uint64(L)), t(ocap)
        d_dec = torch.empty(n * L, dtype=torch.uint8, device="cuda")
        td = {"default": [], "auto": []}
        for _ in range(args.reps):
            for tag in ("default", "auto"):
                b, o_, l_ = dec[tag]
                td[tag].append(timed(lambda: eng.decode_batch_device(b.data_ptr(), o_.data_ptr(), l_.data_ptr(), d_dec.data_ptr(), d_doff.data_ptr(),
                                                                     d_dcap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), n, int(b.numel()), 0, st)))
                assert (d_st.cpu().numpy() == 0).all() and bytes(d_dec.cpu().numpy()) == b"".join(raws)
        r["decode_default_ms"], r["decode_auto_ms"] = float(np.median(td["default"])), float(np.median(td["auto"]))
        out[name] = r
        print(name, json.dumps(r), flush=True)
    props = torch.cuda.get_device_properties(0)
    print(json.dumps(dict(device=props.name, n=args.n, len=L, reps=args.reps, candidates=cands, results=out)))


def gpu_info():
    """the card, its power limit and its SM clock, read in the same process as the timings"""
    import subprocess
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return dict(device=torch.cuda.get_device_properties(0).name, power_limit_clock_sm_max_sm=q)


def transcode(args):
    import time
    import torch
    import divans_b200
    cands = [divans_b200.LITERAL_MODEL_KEEP] + divans_b200.DEFAULT_LITERAL_MODELS
    L = args.len
    cs = corpora(args.n, L)
    mixed = [cs[("text", "utf8", "stride2", "stride4", "stride8")[k % 5]][k] for k in range(args.n)]
    out = {}
    for name, raws in (("text", cs["text"]), ("mixed", mixed)):
        for kind in ("literal", "lz77"):
            rs = raws if kind == "literal" else raws[:args.lz_n]
            n = len(rs)
            eng = divans_b200.Engine(0)   # (one per corpus: the transcode's logs are freed before the decodes allocate theirs)
            if kind == "literal":
                stored = eng.encode(rs)
            else:
                blob = np.frombuffer(b"".join(rs), np.uint8)
                bl, boff, blen = divans_b200.lz77_cmds_batch(blob, np.arange(n, dtype=np.uint64) * np.uint64(L),
                                                            np.array([len(r) for r in rs], np.uint64), window=16)
                stored = eng.encode([bl[int(o):int(o + l)] for o, l in zip(boff, blen)], divans_b200.encode_options(window_size=16),
                                    cmds=True)
            lens = np.array([len(s) for s in stored], np.uint64)
            offs = np.concatenate([[0], np.cumsum((lens + np.uint64(15)) & ~np.uint64(15))[:-1]]).astype(np.uint64)
            buf = np.zeros(int(offs[-1] + lens[-1]) + 16, np.uint8)
            for s, o in zip(stored, offs):
                buf[int(o):int(o) + len(s)] = np.frombuffer(s, np.uint8)
            d_in = torch.from_numpy(buf).cuda()
            caps = [L + 64] * n

            def run(c):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = eng.transcode_device(d_in, offs, lens, caps, candidates=c)
                torch.cuda.synchronize()
                return time.perf_counter() - t0, res

            tp, ta = [], []
            for _ in range(args.reps):
                t, rp = run(None)
                tp.append(t)
                t, ra = run(cands)
                ta.append(t)
            r = dict(n=n, raw=int(sum(len(x) for x in rs)), stored=int(lens.sum()), plain=int(rp[2].sum()), auto=int(ra[2].sum()),
                     transcode_plain_ms=1e3 * float(np.median(tp)), transcode_auto_ms=1e3 * float(np.median(ta)),
                     chosen_hist=np.bincount(ra[4], minlength=len(cands)).tolist())
            assert (rp[3] == 0).all() and (ra[3] == 0).all()
            eng.close()
            torch.cuda.empty_cache()
            eng = divans_b200.Engine(0)
            # decode both outputs, alternating
            td = {"plain": [], "auto": []}
            d_doff = torch.from_numpy((np.arange(n, dtype=np.uint64) * np.uint64(L)).view(np.int64)).cuda()
            d_dcap = torch.from_numpy(np.full(n, L, np.uint64).view(np.int64)).cuda()
            d_dec = torch.empty(n * L, dtype=torch.uint8, device="cuda")
            d_ol = torch.zeros(n, dtype=torch.int64, device="cuda")
            d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
            for _ in range(args.reps):
                for tag, res in (("plain", rp), ("auto", ra)):
                    d_new, new_off, new_len = res[0], res[1], res[2]
                    d_o = torch.from_numpy(new_off.view(np.int64)).cuda()
                    d_l = torch.from_numpy(new_len.view(np.int64)).cuda()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    eng.decode_batch_device(d_new.data_ptr(), d_o.data_ptr(), d_l.data_ptr(), d_dec.data_ptr(), d_doff.data_ptr(),
                                            d_dcap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), n, int(d_new.numel()), 0)
                    eng.synchronize()
                    td[tag].append(time.perf_counter() - t0)
                    assert (d_st.cpu().numpy() == 0).all() and bytes(d_dec.cpu().numpy()) == b"".join(rs)   # (every stream is L bytes)
            r["decode_plain_ms"], r["decode_auto_ms"] = 1e3 * float(np.median(td["plain"])), 1e3 * float(np.median(td["auto"]))
            eng.close()
            out[name + " " + kind] = r
            print(name, kind, json.dumps(r), flush=True)
    print(json.dumps(dict(gpu_info(), n=args.n, lz_n=args.lz_n, len=L, reps=args.reps, results=out)))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--survey", action="store_true")
    ap.add_argument("--streams", type=int, default=6)
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--transcode", action="store_true")
    ap.add_argument("--lz-n", type=int, default=512)
    a = ap.parse_args()
    if a.survey:
        survey(a.streams, a.len)
    elif a.transcode:
        transcode(a)
    else:
        gpu(a)
