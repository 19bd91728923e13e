"""Cost of decoding to command lists against a plain decode, and of whole transcodes, on the bench's two populations:
4096 x 64 KiB synthetic text encoded by the literal-only generator (the flagship) and its LZ77 command streams (window 16).

    python tools/decode_cmds_probe.py [n_streams] [reps]

Per population it prints, as JSON lines: the device time of the plain decode and of the recording decode + pack kernel
(divans_b200_last_kernel_ms: framing through the last kernel, host copies excluded), the wall time of a transcode to
dynamic_context_mixing = 2, and the same for the blend-coded streams transcoded to the frequentist model.  The
`transcode_device_*` columns time Engine.transcode_device for the same two transcodes, streams already in HBM (`_streams`: the
batch measured, `_retried`: the streams whose command list did not fit the first guess).  Medians over `reps` after one
warm-up call.  The GPU's name, power limit and SM clock are printed with them."""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import divans_b200  # noqa: E402
from divans_b200 import synth  # noqa: E402


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def median(f, reps):
    f()
    return statistics.median(f() for _ in range(reps))


def transcode_device(eng, caps, reps, src, flags, o):
    """(median wall ms, streams per call, streams that ran twice): the streams already in HBM, the new ones left there.
    When the command lists of the whole batch do not fit in HBM next to the arena, the largest power-of-two share
    that does is measured, and reported as such."""
    m = len(src)
    while True:
        sub = src[:m]
        in_len = np.array([len(s) for s in sub], np.uint64)
        in_off = np.concatenate([[0], np.cumsum(in_len)[:-1]]).astype(np.uint64)
        d_in = torch.from_numpy(np.frombuffer(b"".join(sub), np.uint8).copy()).to("cuda:0")

        def f():
            torch.cuda.synchronize()
            t = time.perf_counter()
            _, _, _, st = eng.transcode_device(d_in, in_off, in_len, caps[:m], o, flags)
            ms = (time.perf_counter() - t) * 1e3
            assert (st == 0).all()
            return ms
        try:
            r = median(f, reps), m, eng.last_transcode_retried
            del d_in
            torch.cuda.empty_cache()
            return r
        except (divans_b200.DivansError, torch.OutOfMemoryError) as e:
            print(json.dumps({"transcode_device_failed_at": m, "error": str(e)}), flush=True)
            del d_in
            torch.cuda.empty_cache()
            if m == 1:
                raise
            m //= 2


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    eng = divans_b200.Engine(0, 0, 16)
    blob, off, ln = synth.text_streams(n, 65536, seed=0xD1FA15)
    raws = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]
    caps = [len(r) + 64 for r in raws]
    cb, co, cl = divans_b200.lz77_cmds_batch(blob, off, ln, 16, 2, 4)
    lz = [cb[int(o):int(o + l)].tobytes() for o, l in zip(co, cl)]
    pops = {
        "flagship_literal_only": (raws, divans_b200.encode_options(), False),
        "Z_lz77_window16": (lz, divans_b200.encode_options(window_size=16), True),
    }
    print(json.dumps({"gpu": gpu_info(), "streams": n, "reps": reps}))
    # every population's streams first: the device transcodes leave the symbol logs of a whole batch allocated
    coded = {}
    for name, (inp, opts, cmds) in pops.items():
        bopts = divans_b200.encode_options(window_size=opts.window_size, cdf_model=divans_b200.CDF_BLEND)
        coded[name] = (eng.encode(inp, opts, cmds=cmds), eng.encode(inp, bopts, cmds=cmds))
    # the device transcodes before any host-side one: the host calls keep their grow-only scratch on the context
    dev_cols = {}
    for name in pops:
        streams, blend = coded[name]
        row = dev_cols[name] = {}
        for col, src, flags, o in (("transcode_device_to_mix2", streams, 0, divans_b200.encode_options(window_size=0, dynamic_context_mixing=2)),
                                   ("transcode_device_blend_to_frequentist", blend, divans_b200.FLAG_CDF_BLEND, None)):
            ms, m, retried = transcode_device(eng, caps, reps, src, flags, o)
            row[col + "_ms"], row[col + "_streams"], row[col + "_retried"] = round(ms, 1), m, retried
    for name, (inp, opts, cmds) in pops.items():
        streams, blend = coded[name]

        def plain():
            res = eng.decode(streams, caps)
            assert all(st == 0 for st, _ in res)
            return eng.last_kernel_ms()

        def rec():
            res = eng.decode_cmds(streams, caps)
            assert all(st == 0 for st, _, _ in res)
            return eng.last_kernel_ms()

        def transcode(src, flags, o):
            def f():
                t = time.perf_counter()
                eng.transcode(src, caps, o, flags)
                return (time.perf_counter() - t) * 1e3
            return f

        plain_ms, rec_ms = median(plain, reps), median(rec, reps)
        # correctness at the measured size: the recovered lists re-encode to the streams
        back = eng.encode([b for _, _, b in eng.decode_cmds(streams[:64], caps[:64])], opts, cmds=True)
        assert back == streams[:64]
        row = {
            "population": name,
            "decode_kernel_ms": round(plain_ms, 3),
            "decode_cmds_kernel_ms": round(rec_ms, 3),
            "overhead": round(rec_ms / plain_ms - 1, 4),
            "transcode_to_mix2_ms": round(median(transcode(streams, 0, divans_b200.encode_options(window_size=0, dynamic_context_mixing=2)), reps), 1),
            "transcode_blend_to_frequentist_ms": round(median(transcode(blend, divans_b200.FLAG_CDF_BLEND, None), reps), 1),
        }
        row.update(dev_cols[name])
        print(json.dumps(row), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
