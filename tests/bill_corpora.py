"""Command lists and raw buffers shared by the tests of billing by coder state (include/divans_b200.h, "billing each stream's
coding cost by coder state"): every golden list, LZ77 lists with and without dictionary words, random IR with block switches and
several PredictionMode records, and a list with a refused record."""
import json
import os

import numpy as np

from divans_b200 import synth
from irfuzz import random_ir
import lz77_words_corpora as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def text(n, seed=3):
    blob, _, _ = synth.text_streams(1, n, seed=seed)
    return blob.tobytes()


def golden_lists(oracle):
    """(name, Commands, option keywords) of every golden stream, decoded to its list, with the options it was written with"""
    out = []
    for e in json.load(open(os.path.join(GOLDEN, "golden.json"))):
        stream = open(os.path.join(GOLDEN, e["name"] + ".divans"), "rb").read()
        rc, raw, cl = oracle.decode_cmds(stream, out_cap=e["raw_len"] + 64)
        assert rc == 0 and len(raw) == e["raw_len"], e["name"]
        out.append((e["name"], cl, dict(e["options"], window_size=cl.window)))
    wasm = json.load(open(os.path.join(GOLDEN, "ref_wasm_example.json")))
    stream = open(os.path.join(GOLDEN, "ref_wasm_example.divans"), "rb").read()
    rc, raw, cl = oracle.decode_cmds(stream, out_cap=(1 << 20), model_rev=oracle.MODEL_WASM_2018)
    assert rc == 0, wasm
    out.append(("ref_wasm_example", cl, dict(window_size=cl.window, model_rev=oracle.MODEL_WASM_2018)))
    return out


def parse_lists(oracle, T):
    """(name, Commands, option keywords) of LZ77 lists: the plain parse, dictionary words, and words under every transform"""
    t, words = text(24000, seed=11), W.forms_buffer(200, seed=4)
    return [
        ("lz77", T.lz77_parse(oracle, t, 7, 2, window=16), dict(window_size=16, dynamic_context_mixing=1)),
        ("lz77_dict", T.lz77_dict_parse(oracle, t, 7, 2, 4, window=16), dict(window_size=16)),
        ("lz77_words", T.lz77_words_parse(oracle, words, 4, 0, 4, 1, window=16), dict(window_size=16, dynamic_context_mixing=2)),
    ]


def fuzz_lists(oracle, n=6):
    """(name, Commands, option keywords) of random IR: copies, dictionary words, block switches, several PredictionMode records"""
    t = text(40000, seed=21)
    return [("irfuzz%d" % s, oracle.Commands.from_ir(random_ir(oracle, 3100 + s, n_cmds=150, window=16, text=t)),
             dict(window_size=16, dynamic_context_mixing=s % 3)) for s in range(n)]


def refused_blob(oracle):
    """an LZ77 list whose PredictionMode record has pred_mode 5: every encoder refuses it (status 3)"""
    b = bytearray(oracle.Commands.lz77(text(3000, seed=2), window=16).serialize())
    n_cmds = int(np.frombuffer(bytes(b[8:12]), np.uint32)[0])
    b[32 + 20 * n_cmds] = 5
    return bytes(b)


RAW_MODELS = [(pm, mv) for pm in range(4) for mv in range(16)]   # every literal prediction mode and mixing value
