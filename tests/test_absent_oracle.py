"""CPU: the absent() restatement (tests/absent_oracle.py) reproduces the reference's printed tables and AbsentExec's unit
vectors, and its cursor walk agrees with "no valid cell at step k" on random grids."""
import json
import os

import numpy as np
import pytest

from tests import absent_oracle as ao
from tests.helpers import GOLDEN_DIR

with open(os.path.join(GOLDEN_DIR, "reference_absent_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}
UNITS = {u["name"]: u for u in G["unit"]}
LOOKBACK = G["lookback"]


def child_series(case):
    """The series the argument's selector matches (none for a table that does not exist)."""
    if case["table"] is None:
        return []
    t = G["tables"][case["table"]]
    return [s for s in t["series"] if ao.matches({k: s[k] for k in t["tags"]}, case["matchers"])]


def names(case):
    """(time index, value column) of the node: the table's, or the planner's defaults without a table"""
    if case["table"] is None:
        return "time", "value"
    t = G["tables"][case["table"]]
    return t["time_index"], t["field"]


def test_every_printed_table_and_unit_vector_is_a_case():
    assert sorted(CASES) == sorted(["absent_job1", "absent_job2", "absent_job3", "absent_nonexistent_table",
                                    "absent_nonexistent_job", "absent_job1_at_1000s", "absent_two_equal_matchers",
                                    "absent_regex_matchers"])
    assert len(UNITS) == 4


@pytest.mark.parametrize("name", sorted(CASES))
def test_rows_reproduce_the_golden(name):
    case = CASES[name]
    s, e, i = case["start"], case["end"], case["interval"]
    present = ao.present_steps(child_series(case), s, e, i, LOOKBACK)
    labels = ao.fake_labels(case["matchers"])
    got = [[t, 1.0, dict(labels)] for t in ao.absent_stream(s, e, i, present)]
    assert got == case["expected"]
    if case["columns"] is not None:
        assert case["columns"] == list(names(case)) + [n for n, _ in labels]
    else:
        assert got == []


@pytest.mark.parametrize("name", sorted(UNITS))
def test_unit_vectors(name):
    u = UNITS[name]
    assert ao.absent_stream(u["start"], u["end"], u["step"], u["present"]) == u["expected"]
    # the same as a grid: one row whose cells are the present steps
    ts = ao.grid(u["start"], u["end"], u["step"])
    ok = np.array([[t in u["present"] for t in ts]])
    assert ao.absent_steps(u["start"], u["end"], u["step"], ok) == u["expected"]


@pytest.mark.parametrize("seed", range(40))
def test_cursor_walk_equals_no_valid_cell(seed):
    rng = np.random.default_rng(seed)
    step = int(rng.integers(1, 7))
    start = int(rng.integers(-50, 50))
    end = start + int(rng.integers(-3, 80))  # (start > end included: nothing is emitted)
    T = len(ao.grid(start, end, step))
    rows = int(rng.integers(0, 6))
    ok = rng.random((rows, T)) < rng.choice([0.0, 0.05, 0.3, 0.9, 1.0])
    want = ao.absent_steps(start, end, step, ok)
    if rows == 0:
        assert want == ao.grid(start, end, step)
    ts = ao.grid(start, end, step)
    present = sorted({ts[k] for k in range(T) if ok[:, k].any()})
    assert ao.absent_stream(start, end, step, present) == want
    # timestamps off the grid or outside it never hide a step
    stray = [start - step - 1, end + step + 1] + [t + 1 for t in present if step > 1]
    assert ao.absent_stream(start, end, step, sorted(set(present) | set(stray))) == want
    out, words = ao.absent_words(ok, T)
    assert [t for t, v in zip(ts, out) if v == 1.0] == want
    assert int(sum(bin(int(w)).count("1") for w in words)) == len(want)


def test_fake_labels():
    m = [["job", "=", "a"], ["z", "=", ""], ["Job", "=", "b"], ["job", "=", "c"], ["x", "=~", "y"], ["ä", "=", "1"],
         ["w", "!=", "v"]]
    # the last job wins, "" is kept, names in byte order ("J" < "j" < "z" < "ä"), non-equality matchers dropped
    assert ao.fake_labels(m) == [("Job", "b"), ("job", "c"), ("z", ""), ("ä", "1")]
    assert ao.fake_labels([]) == []
