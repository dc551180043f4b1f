"""CPU: the subquery restatement (tests/subquery_oracle.py) reproduces every table of the reference's subquery.result,
digit for digit, and its grid -> rows step keeps NaN cells and value bits."""
import json
import os

import numpy as np
import pytest

from tests import subquery_oracle as sqo
from tests.helpers import GOLDEN_DIR

with open(os.path.join(GOLDEN_DIR, "reference_subquery_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}


def golden_child(c):
    """the case's inner grid and the instant selector metric_total on it"""
    t = G["tables"]["metric_total"]
    s, step, T_in = sqo.inner_grid(c["start"], c["end"], c["interval"], c["range"], c["step"])
    vals, valid = sqo.instant_child(t["ts"], t["val"], s, c["end"], step, G["lookback"])
    assert vals.shape == (1, T_in)
    return s, step, vals, valid


@pytest.mark.parametrize("name", sorted(CASES))
def test_row_literal_reproduces_the_golden_tables(name):
    c = CASES[name]
    s, step, vals, valid = golden_child(c)
    fn = c["function"][len("prom_"):]
    out, ov = sqo.subquery(fn, c["start"], c["end"], c["interval"], c["range"], s, step, vals, valid)
    got = [[c["start"] + k * c["interval"], repr(float(out[0, k]))] for k in range(out.shape[1]) if (ov[0, k >> 5] >> (k & 31)) & 1]
    assert got == [[ts, repr(float(v))] for ts, v in c["expected"]]


def test_the_six_printed_values():
    assert [e[1] for c in G["cases"] for e in c["expected"]] == [3.0, 4.0, 10.0, 2.0, 0.1, 0.06666666666666667]


def test_grid_to_rows_keeps_nan_and_bits():
    vals = np.array([[np.nan, -0.0, 1.0, 2.0], [5.0, 6.0, 7.0, 8.0]])
    nan_payload = np.array([0x7FF800000000BEEF], np.uint64).view(np.float64)[0]
    vals[0, 3] = nan_payload
    valid = np.array([[0b1011], [0b0000]], np.uint32)
    ts, val, offsets = sqo.grid_to_rows(vals, valid, -30_000, 10_000)
    assert ts.tolist() == [-30_000, -20_000, 0]
    assert val.view(np.uint64).tolist() == [vals[0, 0:1].view(np.uint64)[0], np.float64(-0.0).view(np.uint64),
                                            nan_payload.view(np.uint64)]
    assert offsets.tolist() == [0, 3, 3]


def test_nan_cells_are_samples():
    """count_over_time over a row whose cells are all NaN counts them: no SeriesNormalize filters the child"""
    vals = np.full((1, 6), np.nan)
    valid = np.array([[0b111111]], np.uint32)
    out, ov = sqo.subquery("count_over_time", 50_000, 50_000, 1000, 60_000, 0, 10_000, vals, valid)
    assert ov[0, 0] & 1 and out[0, 0] == 6.0
