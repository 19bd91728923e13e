"""The GPU LZ77 command generator (divans_b200_lz77_cmds_batch_device) and Engine.compress_device against the host route.

    python tools/lz77_probe.py [--n 4096] [--len 65536] [--mixed-n 512] [--reps 5] [--out FILE]

For the bench's synthetic text (n streams of len bytes) and for the mixed corpus of tools/auto_probe.py (text, UTF-8 text,
records of 2, 4 and 8 bytes; mixed-n streams of each), with the GPU's name, power limit and SM clock read in the same run:
  * gen_kernel_ms: the generator's kernel time (CUDA events of the library, median of --reps after a warm-up);
  * host_lz77_s: the host generator's wall time (divans_b200_lz77_cmds_batch on every host thread);
  * compress_device_s against host_route_s, wall time: compress_device on buffers in HBM, against D2H of the raw bytes, the
    host generator, H2D of the lists and encode_cmds_batch_device (both end in a synchronisation);
  * output bytes of the two routes.
Every GPU blob is compared with the host generator's and every compressed stream with the host route's; a difference fails.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import divans_b200  # noqa: E402
from divans_b200 import synth  # noqa: E402


def run_corpus(eng, name, raws, reps):
    import torch
    n = len(raws)
    blob, off, ln = divans_b200._pack(raws)
    dev = torch.device("cuda:0")
    u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev)
    d_in = torch.from_numpy(blob).to(dev)
    cap = divans_b200.lz77_blob_cap(ln)
    boff, btot = divans_b200._regions(cap)
    d_off, d_len, d_boff, d_cap = u64(off), u64(ln), u64(boff), u64(cap)
    d_blobs = torch.empty(btot, dtype=torch.uint8, device=dev)
    d_res = torch.zeros(2 * n, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()

    def gen():
        eng.lz77_cmds_batch_device(n, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(ln.max()), 16, 2, 4, d_blobs.data_ptr(),
                                   d_boff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), d_res[n:].data_ptr())
        eng.synchronize()
        return eng.last_kernel_ms()

    gen()   # warm-up (scratch allocation)
    kms = [gen() for _ in range(reps)]
    t0 = time.perf_counter()
    hb, hoff, hlen = divans_b200.lz77_cmds_batch(blob, off, ln, 16, 2, 4)
    host_lz77_s = time.perf_counter() - t0
    r = d_res.cpu().numpy()
    st, blen = r[n:].view(np.int32)[:n], r[:n].view(np.uint64)
    assert (st == 0).all() and (blen == hlen).all(), "%s: status or length differs" % name
    g = d_blobs.cpu().numpy()
    for i in range(n):
        if not np.array_equal(g[int(boff[i]):int(boff[i] + blen[i])], hb[int(hoff[i]):int(hoff[i] + hlen[i])]):
            raise SystemExit("%s: GPU blob %d differs from the host generator's" % (name, i))
    del d_blobs, g   # (the encoder's slots and logs need the memory)
    torch.cuda.empty_cache()

    opts = divans_b200.encode_options(window_size=16)

    def host_route(m):
        """D2H of the raw bytes, the host generator, H2D of the lists, encode_cmds_batch_device in sub-batches of m streams"""
        raw = d_in.cpu().numpy()
        lb, lo, ll = divans_b200.lz77_cmds_batch(raw, off, ln, 16, 2, 4)
        d_lb = torch.from_numpy(lb).to(dev)
        new_cap = divans_b200._encoded_cap(ll)
        new_off, new_tot = divans_b200._regions(new_cap)
        d_m = u64(np.concatenate([lo, ll, new_off, new_cap]))
        d_new = torch.empty(new_tot, dtype=torch.uint8, device=dev)
        d_r = torch.zeros(2 * n, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()   # (the library's calls run on the context's stream)
        for i0 in range(0, n, m):
            k = min(m, n - i0)
            at = lambda t, esz=8: t.data_ptr() + i0 * esz
            eng.encode_cmds_batch_device(k, d_lb.data_ptr(), at(d_m), at(d_m[n:]), int(ll.max()), int(ln.max()), d_new.data_ptr(),
                                         at(d_m[2 * n:]), at(d_m[3 * n:]), at(d_r), at(d_r[n:], 4), opts)
        eng.synchronize()
        rr = d_r.cpu().numpy()
        return d_new, new_off, rr[:n].view(np.uint64).copy(), rr[n:].view(np.int32)[:n].copy()

    def device_route():
        d_new, new_off, new_len, status = eng.compress_device(d_in, off, ln, opts=opts)
        torch.cuda.synchronize()
        return d_new, new_off, new_len, status

    out = {}
    for label in ("compress_device", "host_route"):
        # the host route encodes in the sub-batches compress_device found its logs need
        fn = device_route if label == "compress_device" else lambda: host_route(-(-n // eng.last_compress_sub_batches))
        res = fn()   # warm-up: the encoder's slots and logs
        del res
        torch.cuda.empty_cache()
        t0 = time.perf_counter()
        res = fn()
        t = time.perf_counter() - t0
        out[label] = (t, (res[0].cpu().numpy(),) + tuple(res[1:]))
        del res
        torch.cuda.empty_cache()
    (hs, (hh, ho, hl, hst)), (ds, (dh, do, dl, dst)) = out["host_route"], out["compress_device"]
    assert (hst == 0).all() and (dst == 0).all(), "%s: an encode failed" % name
    assert (hl == dl).all(), "%s: stream lengths differ" % name
    for i in range(n):
        if not np.array_equal(hh[int(ho[i]):int(ho[i] + hl[i])], dh[int(do[i]):int(do[i] + dl[i])]):
            raise SystemExit("%s: stream %d differs between the routes" % (name, i))
    return dict(corpus=name, streams=n, raw_bytes=int(ln.sum()), list_bytes=int(hlen.sum()), gen_kernel_ms=statistics.median(kms),
                gen_kernel_ms_all=[round(k, 3) for k in kms], host_lz77_s=round(host_lz77_s, 3), host_threads=os.cpu_count(),
                host_route_s=round(hs, 3), compress_device_s=round(ds, 3), compress_device_sub_batches=eng.last_compress_sub_batches,
                out_bytes=int(dl.sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--len", type=int, default=65536)
    ap.add_argument("--mixed-n", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import auto_probe
    info = auto_probe.gpu_info()
    eng = divans_b200.Engine(0, 0, 16)
    blob, off, ln = synth.text_streams(args.n, args.len)
    results = [run_corpus(eng, "text", [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)], args.reps)]
    mixed = [r for rs in auto_probe.corpora(args.mixed_n, args.len).values() for r in rs]
    results.append(run_corpus(eng, "mixed", mixed, args.reps))
    eng.close()
    line = json.dumps(dict(info, results=results))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
