"""Dev probe (not a test, not the bench): device time of decode/encode for several stream populations.
  python tools/perf_probe.py [n_streams] [--l-only] [--lz-all] [--decode-once]     (DIVANS_B200_LPS selects the lane layout)
  python tools/perf_probe.py --sweep [n1,n2,...]     literal-only text decode kernel time per decoded byte per stream, by batch size
                                                     (default 132,528,1056,2112,4224: 1/8 to 4 warps per scheduler on 132 SMs)
  python tools/perf_probe.py --prelude [n1,n2,...]   decode kernel time of the bench's text streams cut to 16 bytes (the fixed
                                                     per-stream cost) next to the full 64 KiB streams, by batch size"""
import os, subprocess, sys, time, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import divans_b200
from divans_b200 import synth

once = "--decode-once" in sys.argv


def card_line():
    import torch
    prop = torch.cuda.get_device_properties(0)
    try:
        card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:
        card = "%s (nvidia-smi: %s)" % (prop.name, e)
    print("card: %s | %d SMs | kernel %s" % (card, prop.multi_processor_count, divans_b200.kernel_version()), flush=True)
    return prop


def sweep(sizes):
    """Is the literal loop bound by its dependency chain (time per byte flat in the warps per scheduler), by issue (time grows
    with them), or by memory (a step where the batch's literal priors, ~28 KB per stream, outgrow the L2)?"""
    prop = card_line()
    eng = divans_b200.Engine(0, 0, 16)
    blob, off, ln = synth.text_streams(max(sizes), 65536, seed=3)
    raws_all = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]
    for n in sizes:
        raws = raws_all[:n]
        streams = eng.encode(raws, divans_b200.encode_options())
        caps = [len(r) + 64 for r in raws]
        ms = []
        for _ in range(4):
            res = eng.decode(streams, caps)
            ms.append(eng.last_main_kernel_ms())
        ok = all(st == 0 and out == r for (st, out), r in zip(res, raws))
        kms = float(np.median(ms[1:]))
        wps = (n / 2) / (prop.multi_processor_count * 4)   # 16 lanes per stream: two streams per warp
        print("streams %5d  warps/scheduler %5.2f  decode kernel %8.2f ms (min %8.2f max %8.2f)  %7.1f ns/byte/stream  ok=%s"
              % (n, wps, kms, min(ms[1:]), max(ms[1:]), kms * 1e6 / 65536, ok), flush=True)
    eng.close()


def prelude(sizes):
    """The fixed per-stream cost: the bench's text streams cut to their first 16 bytes (per-stream setup, the PredictionMode
    command with its 8192 mixing values, a 16-byte literal) against the full 64 KiB streams, decode kernel time by batch size.
    A third column codes the same 16 bytes without the PredictionMode command: setup and literal only."""
    card_line()
    eng = divans_b200.Engine(0, 0, int(os.environ.get("DIVANS_B200_LPS", "16")))
    blob, off, ln = synth.text_streams(max(sizes), 65536)     # bench.py's seed
    full_all = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]

    def kernel_ms(raws, no_pm=False):
        if no_pm:
            cl = [divans_b200.ir_to_cmds("window 22 0 0 0\ninsert %d %s\n" % (len(r), r.hex()))[0] for r in raws]
            streams = eng.encode(cl, divans_b200.encode_options(), cmds=True)
        else:
            streams = eng.encode(raws, divans_b200.encode_options())
        caps = [len(r) + 64 for r in raws]
        ms = []
        for _ in range(4):
            res = eng.decode(streams, caps)
            ms.append(eng.last_main_kernel_ms())
        ok = all(st == 0 and out == r for (st, out), r in zip(res, raws))
        return float(np.median(ms[1:])), min(ms[1:]), max(ms[1:]), ok

    for n in sizes:
        full = full_all[:n]
        fm, fmin, fmax, fok = kernel_ms(full)
        pm, pmin, pmax, pok = kernel_ms([r[:16] for r in full])
        nm, nmin, nmax, nok = kernel_ms([r[:16] for r in full], no_pm=True)
        print("streams %5d  lanes %2d  64 KiB decode kernel %8.3f ms (min %8.3f max %8.3f)  16 B decode kernel %7.3f ms "
              "(min %7.3f max %7.3f)  prelude share %5.1f %%  16 B without PredictionMode %7.3f ms (min %7.3f max %7.3f)  ok=%s/%s/%s"
              % (n, eng.last_lanes(), fm, fmin, fmax, pm, pmin, pmax, 100.0 * pm / fm, nm, nmin, nmax, fok, pok, nok), flush=True)
    eng.close()


for mode, default, fn in (("--sweep", "132,528,1056,2112,4224", sweep), ("--prelude", "132,1056,4096,4224", prelude)):
    if mode in sys.argv:
        i = sys.argv.index(mode)
        spec = sys.argv[i + 1] if i + 1 < len(sys.argv) and not sys.argv[i + 1].startswith("--") else default
        fn([int(x) for x in spec.split(",")])
        sys.exit(0)

def run(name, raws, opts, eng, cmds=None):
    streams = eng.encode(cmds if cmds is not None else raws, opts, cmds=cmds is not None)
    enc_ms = eng.last_kernel_ms(); enc_model = eng.last_main_kernel_ms()
    caps = [len(r) + 64 for r in raws]
    for _ in range(1 if once else 2):
        res = eng.decode(streams, caps)
    dec_ms = eng.last_kernel_ms(); dec_main = eng.last_main_kernel_ms()
    ok = all(st == 0 and out == r for (st, out), r in zip(res, raws))
    tot = sum(len(r) for r in raws); comp = sum(len(s) for s in streams)
    print("%-34s n=%5d raw %7.1f MB ratio %.3f | decode %8.2f ms (main %8.2f) %7.0f MB/s | encode %8.2f ms (model %8.2f) %7.0f MB/s | ok=%s"
          % (name, len(raws), tot / 1e6, comp / tot, dec_ms, dec_main, tot / dec_ms / 1e3, enc_ms, enc_model, tot / enc_ms / 1e3, ok), flush=True)

eng = divans_b200.Engine(0, 0, int(os.environ.get("DIVANS_B200_LPS", "16")))
args = [a for a in sys.argv[1:] if not a.startswith("--")]
n = int(args[0]) if args else 4096
blob, off, ln = synth.text_streams(n, 65536, seed=3)
raws = [blob[int(o):int(o + l)].tobytes() for o, l in zip(off, ln)]
run("text 64KiB default", raws, divans_b200.encode_options(), eng)
if "--l-only" in sys.argv:
    sys.exit(0)
run("text 64KiB dcm=1", raws, divans_b200.encode_options(dynamic_context_mixing=1), eng)
run("text 64KiB dcm=2", raws, divans_b200.encode_options(dynamic_context_mixing=2), eng)
run("text 64KiB utf8 mix=1 ", raws, divans_b200.encode_options(literal_pred_mode=2, literal_mixing_value=1), eng)
if "--lz" in sys.argv or "--lz-all" in sys.argv:
    m = n if "--lz-all" in sys.argv else min(n, 512)
    cb, co, cl = divans_b200.lz77_cmds_batch(blob, off[:m], ln[:m], 16, 2, 4)
    cmds = [cb[int(o):int(o + l)].tobytes() for o, l in zip(co, cl)]
    run("text 64KiB lz77 cmds (w16)", raws[:m], divans_b200.encode_options(window_size=16), eng, cmds=cmds)
for p in (0.5, 0.9, 0.99):
    b2, o2, l2 = synth.bernoulli_streams(max(8, n // 16), 1 << 20, p, seed=5)
    r2 = [b2[int(o):int(o + l)].tobytes() for o, l in zip(o2, l2)]
    run("bernoulli p=%.2f 1MiB" % p, r2, divans_b200.encode_options(), eng)
