"""Billing by coder state on the CPU oracle (oracle_tally: dvo_bill_cmds, dvo_bill_raw; include/divans_b200.h, "billing each
stream's coding cost by coder state"): the rows sum to the cost pass's tally exactly, and their counts are the list's structure."""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import divans_b200  # noqa: E402
from oracle_tally import tally_py as T  # noqa: E402
import bill_corpora as B  # noqa: E402

R = {name: i for i, name in enumerate(T.BILL_ROWS)}


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _check_total(rc, cost, rows, ref_rc, ref_cost):
    assert rc == ref_rc
    if rc == 0:
        assert int(rows[:, 0].sum(dtype=np.uint64)) == cost == ref_cost
    else:
        assert not rows.any()


def test_rows_are_the_header_table():
    """the oracle's rows, the Python names and the header's table are one list, in one order"""
    assert T.BILL_ROWS == divans_b200.BILL_STATES
    h = open(os.path.join(ROOT, "include", "divans_b200.h")).read()
    assert int(re.search(r"#define DIVANS_B200_BILL_STATES (\d+)", h).group(1)) == len(T.BILL_ROWS)
    table = re.findall(r"^ \*\s+(\d+) ([A-Z_]+)\s", h.split("* Rows (index")[1].split("#define DIVANS_B200_BILL_STATES")[0], re.M)
    assert [(int(i), n) for i, n in table] == list(enumerate(T.BILL_ROWS))


@pytest.mark.parametrize("blend", [False, True])
def test_totals_golden(oracle, blend):
    for name, cl, kw in B.golden_lists(oracle):
        if blend and kw.get("model_rev"):
            continue   # (the 2018 revision is a frequentist stream)
        rc, cost, rows = T.bill_cmds(cl, blend=blend, **kw)
        _check_total(rc, cost, rows, *T.tally_cmds(cl, blend=blend, **kw))
        assert rc == 0, name


@pytest.mark.parametrize("blend", [False, True])
def test_totals_parses_and_fuzz(oracle, blend):
    for name, cl, kw in B.parse_lists(oracle, T) + B.fuzz_lists(oracle):
        for extra in ({}, {"model_rev": 1}):
            rc, cost, rows = T.bill_cmds(cl, blend=blend, **kw, **extra)
            _check_total(rc, cost, rows, *T.tally_cmds(cl, blend=blend, **kw, **extra))
            assert rc == 0, name


@pytest.mark.parametrize("blend", [False, True])
def test_totals_raw_every_model(oracle, blend):
    data = B.text(6000, seed=9)
    for pm, mv in B.RAW_MODELS:
        for kw in ({}, {"dynamic_context_mixing": 2}, {"model_rev": 1}):
            rc, cost, rows = T.bill_raw(data, pm, mv, blend=blend, window_size=12, **kw)
            _check_total(rc, cost, rows, *T.tally_raw(data, pm, mv, blend=blend, window_size=12, **kw))
            assert rc == 0 and rows[R["LIT_HI"], 1] == rows[R["LIT_LO"], 1] == len(data)


def test_literal_counts(oracle):
    """a literal-only list of m bytes: m high and m low literal nibbles, one command-type nibble per command and the end"""
    for m in (0, 1, 17, 5000):
        data = B.text(m + 1, seed=m)[:m]
        rc, cost, rows = T.bill_raw(data, 2, 4, window_size=10)
        assert rc == 0
        assert rows[R["LIT_HI"], 1] == rows[R["LIT_LO"], 1] == m
        n_lit_cmds = (m + 1023) // 1024
        assert rows[R["CMD_TYPE"], 1] == 1 + n_lit_cmds + 1
        assert rows[R["PM_MIXVAL"], 1] == 8192


def _types(cl):
    blob = cl.serialize()
    n = int(np.frombuffer(blob[8:12], np.uint32)[0])
    return np.frombuffer(blob[32:32 + 20 * n], np.uint32).reshape(n, 5)[:, 0]


def test_command_counts(oracle):
    """command-type nibbles = commands + the end marker; small copy counts = copies; 8192 mixing values per PredictionMode
    command; no dictionary nibbles in a list without dictionary words"""
    for name, cl, kw in B.golden_lists(oracle) + B.parse_lists(oracle, T) + B.fuzz_lists(oracle):
        types = _types(cl)
        rc, cost, rows = T.bill_cmds(cl, **kw)
        assert rc == 0, name
        assert rows[R["CMD_TYPE"], 1] == len(types) + 1, name
        assert rows[R["CP_COUNT_SMALL"], 1] == (types == 1).sum(), name
        assert rows[R["PM_MIXVAL"], 1] == 8192 * (types == 7).sum(), name
        assert rows[R["PM_MODE"], 1] == (types == 7).sum(), name
        assert rows[R["PM_SPEED"], 1] == 16 * (types == 7).sum(), name
        if not (types == 2).any():
            assert not rows[R["DC_SIZE_BEG"]:R["DC_TR_LO"] + 1].any(), name
        else:
            assert rows[R["DC_TR_HI"], 1] == rows[R["DC_TR_LO"], 1] == (types == 2).sum(), name


def test_mixing_values_without_context_map(oracle):
    """with use_context_map 0 the record's mixing values are still coded, all of them as 4: 8192 nibbles per record"""
    cl = oracle.Commands.lz77(B.text(20000, seed=5), window=16)
    for ucm in (0, 1):
        rc, cost, rows = T.bill_cmds(cl, window_size=16, use_context_map=ucm)
        assert rc == 0 and rows[R["PM_MIXVAL"], 1] == 8192 * (_types(cl) == 7).sum()


def test_refused_record(oracle):
    """a record the encoder refuses: status 3 and a zero bill"""
    cl = T.from_blob(oracle, B.refused_blob(oracle))
    for blend in (False, True):
        rc, cost, rows = T.bill_cmds(cl, blend=blend, window_size=16)
        assert rc == 3 and cost == T.TALLY_FAILED and not rows.any()
        assert T.tally_cmds(cl, blend=blend, window_size=16) == (3, T.TALLY_FAILED)


def test_summary_groups():
    """bill_summary's groups take every row once"""
    keys = [k for _, ks in divans_b200.BILL_GROUPS for k in ks]
    assert sorted(keys) == sorted(divans_b200.BILL_STATES)
    rows = np.arange(64, dtype=np.uint64).reshape(32, 2)
    s = divans_b200.bill_summary(rows)
    assert sum(c for _, c, _ in s) == int(rows[:, 0].sum()) and sum(n for _, _, n in s) == int(rows[:, 1].sum())
