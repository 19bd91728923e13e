"""CPU tests: the C-ABI library builds, loads and exports every symbol include/divans_b200.h declares; the host-side
mirror refuses to compute without a GPU (no fallback); synthetic generators and the shard partition are deterministic."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib_path():
    import __graft_entry__ as g
    import divans_b200
    if not os.path.exists(divans_b200.LIB_PATH):
        g.build()
    return divans_b200.LIB_PATH


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b(divans_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_header_symbols_are_exported(lib_path):
    import divans_b200
    names = _declared_functions()
    assert len(names) >= 30
    out = subprocess.check_output(["nm", "-D", "--defined-only", lib_path]).decode()
    exported = set(l.split()[-1] for l in out.splitlines() if " T " in l)
    missing = [n for n in names if n not in exported]
    assert not missing, missing
    assert set(divans_b200.REFERENCE_FFI_SYMBOLS) <= exported and set(divans_b200.BATCH_SYMBOLS) <= exported


def test_library_loads_and_has_sm90a_code(lib_path):
    lib = ctypes.CDLL(lib_path)
    assert lib.divans_decode and lib.divans_b200_decode_batch_device
    sass = subprocess.run(["cuobjdump", "-lelf", lib_path], capture_output=True, text=True).stdout
    assert "sm_90a" in sass


def test_no_cpu_fallback_without_gpu(lib_path):
    import divans_b200
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        pytest.skip("GPU present")
    with pytest.raises(divans_b200.DivansError):
        divans_b200.Engine(0)


def test_product_does_not_reference_the_oracle():
    # the product tree must not import / link / read anything under oracle/
    bad = []
    for base, _, files in os.walk(os.path.join(ROOT, "divans_b200")):
        if base.endswith("lib") or "/lib/" in base:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", "Makefile")):
                txt = open(os.path.join(base, f), errors="ignore").read()
                if re.search(r"oracle_py|divans_oracle|from oracle|import oracle|oracle/", txt):
                    bad.append(os.path.join(base, f))
    assert not bad, bad


def test_synth_is_deterministic():
    from divans_b200 import synth
    a, off, ln = synth.text_streams(8, 4096)
    b, _, _ = synth.text_streams(8, 4096)
    assert (a == b).all() and a.size == 8 * 4096 and (ln == 4096).all()
    assert a[:4096].tobytes() != a[4096:8192].tobytes()
    x, _, _ = synth.bernoulli_streams(4, 1024, 0.9)
    ones = np.unpackbits(x).mean()
    assert 0.07 < ones < 0.13


def test_shard_partition_balances_by_bytes():
    from divans_b200 import sharding
    lens = np.array([10, 10, 10, 1000, 10, 10, 500, 500], np.uint64)
    parts = sharding.partition_by_bytes(lens, 3)
    assert parts[0][0] == 0 and parts[-1][1] == len(lens)
    assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
    sums = [int(lens[a:b].sum()) for a, b in parts]
    assert max(sums) <= 1100
    assert sharding.partition_by_bytes(lens, 1) == [(0, 8)]
    assert sharding.partition_by_bytes(np.zeros(0, np.uint64), 4) == [(0, 0)] * 4


def _gloo_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from divans_b200 import sharding
    lens = np.arange(1, 101, dtype=np.uint64)
    a, b = sharding.partition_by_bytes(lens, world)[rank]
    # every rank "processes" its shard; the job total is the sum over ranks, the job time the max over ranks
    done = torch.tensor([float(lens[a:b].sum())], dtype=torch.float64)
    t = torch.tensor([1.0 + rank], dtype=torch.float64)
    tot, tmax = sharding.reduce_job(done, t)
    q.put((rank, a, b, tot, tmax))
    dist.destroy_process_group()


def test_world_size_2_gloo_sharding():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 1000)
    ps = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(60) for p in ps]
    assert res[0][1] == 0 and res[0][2] == res[1][1] and res[1][2] == 100
    assert res[0][3] == res[1][3] == 5050.0 and res[0][4] == res[1][4] == 2.0


def _sharded_worker(rank, world, port, q):
    """world_size-2 gloo job: the root's host batch is scattered, decoded per rank (stand-in decoder: the CPU oracle), gathered"""
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from divans_b200 import sharding, synth
    from oracle import oracle_py as O

    def oracle_decode(d_in, in_off, in_len, d_out, out_off, out_cap):
        out, out_len, status = O.decode_batch(d_in.numpy(), in_off.numpy().astype(np.uint64), in_len.numpy().astype(np.uint64),
                                              out_off.numpy().astype(np.uint64), out_cap.numpy().astype(np.uint64), 2)
        d_out[: out.size] = torch.from_numpy(out)
        return torch.from_numpy(out_len.astype(np.int64)), torch.from_numpy(status)

    dec = sharding.ShardedDecoder(device="cpu", decode_fn=oracle_decode)
    if rank == 0:
        text = synth.text_corpus(1 << 16)
        raws = [text[i * 900: i * 900 + 400 + 350 * (i % 7)] for i in range(23)] + [b""]
        streams = [O.encode_raw(r, O.options(window_size=12)) for r in raws]
        in_len = np.array([len(s) for s in streams], np.uint64)
        in_off = np.concatenate([[0], np.cumsum(in_len)[:-1]]).astype(np.uint64)
        out, out_off, out_len, status = dec.decode(np.frombuffer(b"".join(streams), np.uint8).copy(), in_off, in_len,
                                                   np.array([len(r) + 5 for r in raws], np.uint64))
        ok = bool((status == 0).all()) and all(out[int(o): int(o) + int(l)].numpy().tobytes() == r for o, l, r in zip(out_off, out_len, raws))
        q.put((ok, dec.last["parts"], dec.last["shard_bytes"]))
    else:
        assert dec.decode() is None
    dist.destroy_process_group()


def test_world_size_2_gloo_sharded_decoder():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + ((os.getpid() + 311) % 1000)
    ps = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    ok, parts, shard_bytes = q.get(timeout=180)
    [p.join(60) for p in ps]
    assert ok
    assert parts[0][0] == 0 and parts[0][1] == parts[1][0] and parts[1][1] == 24 and 0 < parts[0][1] < 24
    assert abs(shard_bytes[0] - shard_bytes[1]) < 0.2 * sum(shard_bytes)      # balanced by compressed bytes


def test_ir_front_end_matches_oracle_parser(oracle):
    """The product's C++ IR parser (divans_b200_ir_to_cmds) yields the same command-list blob as the oracle's parser --
    which is pinned to the reference by replaying the reference's testdata/*.ir fixtures (tests/test_oracle_kat.py)."""
    import divans_b200
    from divans_b200 import synth
    from irfuzz import random_ir
    text = synth.text_corpus(1 << 16)
    for seed in range(12):
        ir = random_ir(oracle, seed, n_cmds=80, window=16 if seed % 2 else 22, text=text)
        blob, win = divans_b200.ir_to_cmds(ir)
        ref = oracle.Commands.from_ir(ir)
        assert win == ref.window
        assert blob == ref.serialize(), "seed %d" % seed
    edge = "window 18 0 0 0\r\n\ninsert 0 \ncopy 0 from 5 ctx 3\nrndins 2 00ff\nltype 3\nltype 1 8\nctype 200\ndtype 2\n" \
           "copy 7 from 2 ctx 0\ndict 5 word 4,9 6161 func 3 00 ctx 0\nprediction sign lcontextmap 1 2  3 dcontextmap 0 1 mixingvalues 4 4 stspeedinc 2 4 stspeedmax 1024 16384\n"
    blob, win = divans_b200.ir_to_cmds(edge)
    ref = oracle.Commands.from_ir(edge)
    assert win == 18 and blob == ref.serialize()
    for bad in ["bogus 1 2", "insert 3 00ff", "copy x from 1", "prediction nope", "insert 1 zz", "ltype 1 9", "dict 5 word 49 61 func 3"]:
        with pytest.raises(ValueError):
            divans_b200.ir_to_cmds(bad + "\n")
        with pytest.raises(ValueError):
            oracle.Commands.from_ir(bad + "\n")
