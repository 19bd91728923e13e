"""Device replay of command lists to raw bytes (divans_b200_replay_cmds_batch_device), on the bench's text:
4096 x 64 KiB synthetic text streams as LZ77 lists at window 16, and as the literal-only lists decode_cmds returns for the
bench's literal-only streams.

    python tools/replay_probe.py [n_streams] [reps]

Per population it prints, as a JSON line: the replay time (CUDA events around the call, lists and regions already in HBM),
its output rate, the time of the same batch's length pass (out_cap = 0), and for context the device decode time of the same
lists' encoded streams (events around divans_b200_decode_batch_device).  Medians over `reps` (>= 5) timed calls after one
warm-up call; every replay is checked against the raw input.  The GPU's name, power limit and SM clock are printed first,
from the same run."""
import json
import os
import statistics
import subprocess
import sys

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


def timed(fn, reps, s):
    """median device ms of fn() between two events on stream s, after one warm-up call"""
    fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        fn()
        b.record(s)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    reps = max(5, int(sys.argv[2]) if len(sys.argv) > 2 else 7)
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream(dev)
    u64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).to(dev)
    raw_blob, raw_off, raw_len = synth.text_streams(n, 65536, seed=0xD1FA15)
    raws = [raw_blob[int(o):int(o + l)].tobytes() for o, l in zip(raw_off, raw_len)]
    caps = np.array([len(r) for r in raws], np.uint64)
    lz_blob, lz_off, lz_len = divans_b200.lz77_cmds_batch(raw_blob, raw_off, raw_len, 16, 2, 4)
    lz = [lz_blob[int(o):int(o + l)].tobytes() for o, l in zip(lz_off, lz_len)]
    # the inputs on a context of their own, closed before the measured one is made: an engine sizes its slots from the memory
    # that is free when it is created, so every buffer of the measurement is allocated before that
    prep = divans_b200.Engine(0, 0, 16)
    bench_streams = prep.encode(raws)
    dec = prep.decode_cmds(bench_streams, caps + np.uint64(64))
    assert all(st == 0 for st, _, _ in dec)
    pops = {
        "Z_lz77_window16": (lz, prep.encode(lz, divans_b200.encode_options(window_size=16), cmds=True)),
        "literal_only_decoded": ([b for _, _, b in dec], bench_streams),
    }
    prep.close()
    del dec
    print(json.dumps({"gpu": gpu_info(), "streams": n, "stream_bytes": 65536, "reps": reps}), flush=True)
    out_off, out_total = divans_b200._regions(caps)
    want = np.concatenate([np.frombuffer(r, np.uint8) for r in raws])
    d_out = torch.empty(out_total, dtype=torch.uint8, device=dev)
    d_oo, d_cap, d_zero = u64(out_off), u64(caps), u64(np.zeros(n, np.uint64))
    d_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_st = torch.zeros(n, dtype=torch.int32, device=dev)
    dec_off, dec_total = divans_b200._regions(caps + np.uint64(64))
    d_dout, d_doff, d_dcap = torch.empty(dec_total, dtype=torch.uint8, device=dev), u64(dec_off), u64(caps + np.uint64(64))
    dev_pops = {}
    for name, (blobs, streams) in pops.items():
        packed, boff, blen = divans_b200._pack(blobs)
        sp, so, sl = divans_b200._pack(streams)
        dev_pops[name] = (torch.from_numpy(packed).to(dev), u64(boff), u64(blen), int(blen.sum()),
                          torch.from_numpy(sp).to(dev), u64(so), u64(sl), int(sl.sum()))
    torch.cuda.synchronize()
    eng = divans_b200.Engine(0, 0, 16)
    for name, (d_b, d_bo, d_bl, blob_bytes, d_s, d_so, d_sl, stream_bytes) in dev_pops.items():

        def replay(cap):
            eng.replay_cmds_batch_device(n, d_b.data_ptr(), d_bo.data_ptr(), d_bl.data_ptr(), d_out.data_ptr(), d_oo.data_ptr(), cap.data_ptr(),
                                         d_len.data_ptr(), d_st.data_ptr(), 0, s.cuda_stream)

        d_out.zero_()
        torch.cuda.synchronize()
        replay_ms = timed(lambda: replay(d_cap), reps, s)
        kernel_ms = eng.last_kernel_ms()
        assert (d_st.cpu().numpy() == 0).all() and (d_len.cpu().numpy() == caps.astype(np.int64)).all()
        o = d_out.cpu().numpy()
        got = np.concatenate([o[int(a):int(a) + int(c)] for a, c in zip(out_off, caps)])
        assert np.array_equal(got, want), name
        length_ms = timed(lambda: replay(d_zero), reps, s)
        assert (d_st.cpu().numpy() == 2).all() and (d_len.cpu().numpy() == caps.astype(np.int64)).all()
        # the decode of the same lists' encoded streams, in HBM

        def decode():
            eng.decode_batch_device(d_s.data_ptr(), d_so.data_ptr(), d_sl.data_ptr(), d_dout.data_ptr(), d_doff.data_ptr(), d_dcap.data_ptr(),
                                    d_len.data_ptr(), d_st.data_ptr(), n, stream_bytes, 0, s.cuda_stream)
        decode_ms = timed(decode, reps, s)
        assert (d_st.cpu().numpy() == 0).all()
        total = int(caps.sum())
        print(json.dumps({
            "population": name, "lists": n, "blob_bytes": blob_bytes, "out_bytes": total,
            "replay_ms": round(replay_ms, 3), "replay_kernel_ms": round(kernel_ms, 3), "replay_out_GBps": round(total / replay_ms / 1e6, 1),
            "length_pass_ms": round(length_ms, 3), "decode_ms": round(decode_ms, 3),
        }), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
