"""CPU-only: the binary-operator oracle (tests/binary_oracle.py).  Its row-literal restatement of the reference's join +
projection / filter (binary_rows) reproduces the printed sqlness values, the dense restatement (series match +
binary_op) agrees with it on random label sets, and the comparisons follow IEEE 754 totalOrder."""
import math
import random

import numpy as np
import pytest

from tests import binary_oracle as bor
from tests.binary_helpers import (count_rows, dense_rows, expected_rows, load_binary, oracle_node, sum_rate_table)

G = load_binary()
CASES = {c["name"]: c for c in G["cases"]}


def _rows(table, case, **kw):
    return dense_rows(*oracle_node(table, case["start"], case["end"], case["interval"], **kw))


def test_sum_rate_times_scalar():
    c = CASES["sum_rate_times_100"]
    tags, rows = _rows(sum_rate_table(), c, fn="rate", range_ms=60000, agg="sum")
    assert sorted(bor.scalar_rows(rows, "*", 100.0)) == expected_rows(c, tags)
    c = CASES["sum_by_host_rate_times_60"]
    tags, rows = _rows(sum_rate_table(), c, fn="rate", range_ms=60000, agg="sum", by=("host",))
    assert sorted(bor.scalar_rows(rows, "*", 60.0)) == expected_rows(c, tags)


@pytest.mark.parametrize("name,fn", [("selector_plus_selector_two_tables", None),
                                     ("avg_over_time_plus_avg_over_time_two_tables", "avg_over_time")])
def test_vector_plus_vector_across_tables(name, fn):
    c = CASES[name]
    kw = dict(fn=fn, range_ms=c.get("range"))
    lhs = _rows(G["tables"]["host_sec"], c, **kw)
    rhs = _rows(G["tables"]["host_micro"], c, **kw)
    tags, rows = bor.binary_rows(lhs, rhs, "+", label_side="rhs")
    assert sorted(rows) == expected_rows(c, tags)


def test_tsid_keyed_division():
    c = CASES["tsid_div"]
    lhs = _rows(G["tables"]["tsid_binary_join_left"], c)
    rhs = _rows(G["tables"]["tsid_binary_join_right"], c)
    tags, rows = bor.binary_rows(lhs, rhs, "/")
    assert tags == ["host", "job"] and sorted(rows) == expected_rows(c, tags)


def _ratio_filtered():
    c = CASES["ratio_filtered_count"]
    rate_a = _rows(G["tables"]["metric_a"], c, fn="rate", range_ms=c["range"])
    b = _rows(G["tables"]["metric_b"], c)
    ratio = bor.binary_rows(rate_a, b, "/", on=["l3", "l4"], label_side="rhs")
    return rate_a, (ratio[0], bor.scalar_rows(ratio[1], ">", 0.50))


def test_ratio_repro():
    rate_a, (_, kept) = _ratio_filtered()
    assert count_rows(kept) == expected_rows(CASES["ratio_filtered_count"], [])
    total = count_rows(rate_a[1])
    assert bor.scalar_rows(total, "/", 2.0) == expected_rows(CASES["ratio_count_div_2"], [])
    _, ratio = bor.binary_rows(([], count_rows(kept)), ([], total), "/")
    assert bor.scalar_rows(ratio, "*", 100.0) == expected_rows(CASES["ratio_times_100"], [])


def test_missing_key_column_is_a_planning_error():
    with pytest.raises(KeyError, match="No field named job"):
        bor.binary_rows((["host"], [("a", 0, 1.0)]), (["host", "job"], [("a", "j", 0, 1.0)]), "+")


# ---- total order of the comparisons (arrow-rs cmp kernels on f64, third-party semantics the reference does not pin) ----
NEG_NAN = np.array([0xFFF8000000000000], np.uint64).view(np.float64)[0]


@pytest.mark.parametrize("a,op,b,kept", [
    (math.nan, ">", 1.0, True), (math.nan, "==", math.nan, True), (math.nan, "!=", math.nan, False),
    (-0.0, "==", 0.0, False), (-0.0, "<", 0.0, True), (0.0, ">", -0.0, True), (-0.0, "!=", 0.0, True),
    (NEG_NAN, "<", -math.inf, True), (NEG_NAN, "<", math.nan, True), (math.inf, "<", math.nan, True),
    (1.0, "<=", 1.0, True), (2.0, ">=", 3.0, False),
])
def test_comparisons_use_total_order(a, op, b, kept):
    v = bor.binary_value(op, a, b)
    assert (v is not None) == kept
    if kept:  # a filter keeps the lhs value bit for bit
        assert np.float64(v).view(np.uint64) == np.float64(a).view(np.uint64)
    assert bor.binary_value(op, a, b, return_bool=True) == (1.0 if kept else 0.0)


def test_ieee_arithmetic_is_not_an_error():
    assert bor.binary_value("/", 1.0, 0.0) == math.inf and bor.binary_value("/", -1.0, 0.0) == -math.inf
    assert math.isnan(bor.binary_value("/", 0.0, 0.0)) and math.isnan(bor.binary_value("%", 1.0, 0.0))
    assert bor.binary_value("%", -7.5, 2.0) == -1.5 and bor.binary_value("%", 7.5, -2.0) == 1.5
    assert bor.binary_value("^", math.nan, 0.0) == 1.0 and bor.binary_value("^", 1.0, math.nan) == 1.0
    assert bor.binary_value("atan2", 1.0, 0.0) == math.pi / 2  # y is the lhs


# ---- dense restatement (host series match + binary_op) against the row-literal join --------------------------------------
def _random_side(rng, tags, n_series, T, values):
    labels = sorted({tuple(rng.choice(values[t]) for t in tags) for _ in range(n_series)})
    out = np.array([[rng.choice([0.5, 1.0, 2.0, -3.0, 0.0, math.nan]) for _ in range(T)] for _ in labels]).reshape(len(labels), T)
    valid = np.zeros((len(labels), (T + 31) // 32), np.uint32)
    for r in range(len(labels)):
        for k in range(T):
            if rng.random() < 0.7:
                valid[r, k // 32] |= np.uint32(1 << (k % 32))
    return labels, out, valid


@pytest.mark.parametrize("seed", range(12))
def test_dense_restatement_matches_row_literal(seed):
    rng = random.Random(seed)
    values = {"a": ["x", "y"], "b": ["1", "2", "3"], "c": ["p", "q"], "d": ["u"]}
    shapes = [(["a", "b"], ["a", "b"], {}), (["a", "b", "c"], ["a", "b"], dict(on=["a"])),
              (["a", "b", "c"], ["a", "b", "d"], dict(ignoring=["d", "b"])), (["a", "c"], ["a"], {}),
              ([], ["a", "b"], {}), (["a", "b"], [], {}), (["a", "b"], ["a", "b"], dict(on=[]))]
    ltags, rtags, match = shapes[seed % len(shapes)]
    T = rng.choice([1, 5, 33, 40])
    eval_ts = 1000 * np.arange(T, dtype=np.int64)
    n_l, n_r = rng.choice([0, 1, 4, 9]), rng.choice([0, 1, 3, 7])
    ll, lo, lv = _random_side(rng, ltags, n_l, T, values)
    rl, ro, rv = _random_side(rng, rtags, n_r, T, values)
    for op, rb in [("/", False), ("-", False), (">", False), ("<=", True), ("==", False)]:
        for side in ("lhs", "rhs"):
            exp_tags, exp = bor.binary_rows(dense_rows(ltags, ll, lo, lv, eval_ts), dense_rows(rtags, rl, ro, rv, eval_ts),
                                            op, return_bool=rb, label_side=side, **match)
            lrow, rrow = bor.binary_pairs(ltags, ll, rtags, rl, **match)
            out, ov = bor.binary_op(op, lo.reshape(len(ll), T), lv, lrow, ro.reshape(len(rl), T), rv, rrow, return_bool=rb)
            from_lhs = side == "lhs" or (op in ("==", ">") and not rb)
            got_labels = [ll[i] if from_lhs else rl[j] for i, j in zip(lrow, rrow)]
            got_tags, got = dense_rows(ltags if from_lhs else rtags, got_labels, out, ov, eval_ts)
            assert got_tags == exp_tags
            key = lambda r: tuple(str(x) for x in r)  # NaN-safe order; values compared bit for bit below
            g, e = sorted(got, key=key), sorted(exp, key=key)
            assert len(g) == len(e), (op, side)
            for x, y in zip(g, e):
                assert x[:-1] == y[:-1] and np.float64(x[-1]).view(np.uint64) == np.float64(y[-1]).view(np.uint64)
