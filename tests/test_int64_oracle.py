"""CPU: the Int64 restatement (tests/int64_oracle.py) prints every BIGINT golden table digit for digit, and its unit
rows: wrapping sum at INT64_MAX, min / max at INT64_MIN, and i64 values whose bits are NaN doubles."""
import json
import os

import numpy as np
import pytest

from tests import int64_oracle as io

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_int64_vectors.json")))


ROW_CASES = [c for c in GOLDEN["cases"] if "expr" not in c]
EXPR_CASES = [c for c in GOLDEN["cases"] if "expr" in c]


@pytest.mark.parametrize("case", ROW_CASES, ids=[c["query"] for c in ROW_CASES])
def test_oracle_prints_the_golden_table(case):
    assert io.evaluate(case, GOLDEN["tables"][case["table"]]) == case["rows"]


@pytest.mark.parametrize("case", EXPR_CASES, ids=[c["query"] for c in EXPR_CASES])
def test_oracle_prints_the_golden_expression(case):
    got = io.print_rows(case["expr"], GOLDEN["tables"])
    if case["sorted"]:  # (the reference sorted its printed rows as text)
        got, want = sorted(got), sorted(case["rows"])
    else:
        want = case["rows"]
    assert got == want


@pytest.mark.parametrize("case", EXPR_CASES, ids=[c["query"] for c in EXPR_CASES])
def test_promotion_types(case):
    """topk / bottomk over Int64 (and over sum of Int64) print integers; scalar(), arithmetic with a scalar or literal
    operand and clamp* print Float64"""
    col = 0 if case["expr"][0] == "topk" else case["header"].index(
        next(h for h in case["header"] if h not in ("ts", "host", "idc")))
    for row in case["rows"]:
        assert ("." in row[col] or row[col] == "NaN") == (case["expr"][0] != "topk"), row


@pytest.mark.parametrize("case", ROW_CASES, ids=[c["query"] for c in ROW_CASES])
def test_golden_value_columns_have_the_pinned_type(case):
    """sort, topk, sum and count_values' count and label print as integers; quantile prints with a decimal point"""
    col = 0 if case["query"].startswith(("topk", "count_values")) else case["header"].index(
        next(h for h in case["header"] if "(" in h or h == "val"))
    want_float = case["query"].startswith("quantile")
    for row in case["rows"]:
        assert ("." in row[col]) == want_float, row
        if case["query"].startswith("count_values"):
            assert "." not in row[-1]


def test_sum_wraps_at_int64_max():
    assert io.fold("sum", [io.INT64_MAX, 1]) == (io.INT64_MIN, "Int64")
    assert io.fold("sum", [io.INT64_MIN, -1]) == (io.INT64_MAX, "Int64")
    # associative: any order gives the same bits
    xs = [io.INT64_MAX, 5, io.INT64_MAX, -3, io.INT64_MIN]
    assert io.fold("sum", xs) == io.fold("sum", xs[::-1])


def test_min_max_at_int64_min():
    assert io.fold("min", [0, io.INT64_MIN, io.INT64_MAX]) == (io.INT64_MIN, "Int64")
    assert io.fold("max", [io.INT64_MIN, io.INT64_MIN]) == (io.INT64_MIN, "Int64")
    assert io.fold("max", [io.INT64_MIN, -1]) == (-1, "Int64")


def test_nan_pattern_i64_is_an_ordinary_integer():
    nan_bits = np.array([np.nan, -np.nan], np.float64).view(np.int64)  # 0x7FF8.. and 0xFFF8..
    a, b = int(nan_bits[0]), int(nan_bits[1])
    assert a > 0 > b
    assert io.fold("max", [a, b, 0]) == (a, "Int64")
    assert io.fold("min", [a, b, 0]) == (b, "Int64")
    vals = np.array([[a, b, 1]], np.int64)
    ok = np.ones((1, 3), bool)
    assert io.value_order(vals, ok, False) == [1, 2, 0]
    assert io.count_values(vals.T.copy(), np.ones((3, 1), bool), [0, 0, 0], 1)[0, 0] == [(b, 1), (1, 1), (a, 1)]


def test_avg_reads_double_of_i64():
    big = (1 << 53) + 1  # exact in Int64, rounded as a double
    assert io.fold("avg", [big]) == (float(big), "Float64") and float(big) != big
