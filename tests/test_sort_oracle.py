"""CPU: the sort / sort_desc / sort_by_label / sort_by_label_desc restatement (tests/sort_oracle.py) reproduces the
reference's printed tables, and its value key follows the f64 total order on a hand-ordered list of special values."""
import json
import os
import struct

import numpy as np
import pytest

from tests import sort_oracle as so
from tests.helpers import GOLDEN_DIR

with open(os.path.join(GOLDEN_DIR, "reference_sort_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}
LOOKBACK = 300_000


def f64(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


# already in the f64 total order, every entry a different bit pattern
TOTAL_ORDER = [
    f64(0xFFF8000000000000),   # -NaN
    float("-inf"),
    -1e308,
    f64(0x8000000000000001),   # the smallest negative subnormal
    -0.0,
    0.0,
    f64(0x0000000000000001),   # the smallest positive subnormal
    1e308,
    float("inf"),
    f64(0x7FF8000000000000),   # +NaN
    f64(0x7FF800000000BEEF),   # +NaN, a larger payload
]


def child_rows(case):
    """The child's exported rows (value, {tag: label}, ts) in row-major order: the instant selector over the matched
    series (each visible from its sample for the lookback), or the sum by the listed labels with groups in label order."""
    t = G["tables"][case["input"]["table"]]
    series = [s for s in t["series"] if all(s[k] == v for k, v in case["input"]["match"].items())]
    steps = range(case["start"], case["end"] + 1, case["interval"])

    def at(s, step):
        seen = [(ts, v) for ts, v in zip(s["ts"], s["val"]) if ts <= step and step - ts <= LOOKBACK]
        return max(seen)[1] if seen else None

    if case["input"]["aggregate"] is None:
        return [(at(s, k), {tag: s[tag] for tag in t["tags"]}, k) for s in series for k in steps if at(s, k) is not None]
    assert case["input"]["aggregate"] == "sum"
    by = case["input"]["by"]
    groups = sorted({tuple(s[b] for b in by) for s in series})
    rows = []
    for g in groups:
        members = [s for s in series if tuple(s[b] for b in by) == g]
        for k in steps:
            vs = [at(s, k) for s in members if at(s, k) is not None]
            if vs:
                rows.append((float(sum(vs)), dict(zip(by, g)), k))
    return rows


def comparable(rows, masked):
    return [(lab, None if "ts" in masked else ts, None if "val" in masked else v) for v, lab, ts in rows]


def test_every_printed_table_is_a_case():
    assert sorted(CASES) == sorted(["sort_test_host1", "sort_desc_test_host1", "sort_sum_by_idc_host2",
                                    "sort_desc_sum_by_idc_host2", "sort_by_label_idc_host", "sort_by_label_desc_idc_host"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_rows_reproduce_the_golden(name):
    case = CASES[name]
    got = so.sort_rows(case["function"], child_rows(case), case["labels"])
    assert comparable(got, case["masked"]) == [(lab, ts, v) for lab, ts, v in case["expected"]]


def test_value_key_follows_the_total_order():
    keys = [so.total_key(x) for x in TOTAL_ORDER]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    assert so.total_keys(np.array(TOTAL_ORDER)).tolist() == keys
    vals = np.array(TOTAL_ORDER)[::-1].copy()  # reversed, one row
    ok = np.ones((1, vals.size), bool)
    assert so.value_order(vals, ok, False).tolist() == list(range(vals.size))[::-1]
    assert so.value_order(vals, ok, True).tolist() == list(range(vals.size))


def test_ties_keep_row_major_order_in_both_directions():
    vals = np.array([[2.0, 1.0, 2.0], [1.0, 2.0, 1.0]])
    ok = np.ones((2, 3), bool)
    assert so.value_order(vals, ok, False).tolist() == [1, 3, 5, 0, 2, 4]
    assert so.value_order(vals, ok, True).tolist() == [0, 2, 4, 1, 3, 5]
    ok[0, 1] = False
    assert so.value_order(vals, ok, False).tolist() == [3, 5, 0, 2, 4]


def test_label_order_is_bytes_with_null_last():
    rows = [(0.0, {"a": v}, i) for i, v in enumerate(["b", None, "", "ä", "B", "", None, "b"])]
    asc = [r[2] for r in so.sort_rows("sort_by_label", rows, ["a"])]
    desc = [r[2] for r in so.sort_rows("sort_by_label_desc", rows, ["a"])]
    assert asc == [2, 5, 4, 0, 7, 3, 1, 6]   # "" < "B" < "b" < "ä" (0xC3 0xA4), then NULL in row order
    assert desc == [3, 0, 7, 4, 2, 5, 1, 6]  # reversed strings, ties in row order, NULL still last
    # a label the rows lack reads as NULL: every row ties, the order is the rows'
    assert [r[2] for r in so.sort_rows("sort_by_label", rows, ["zz"])] == list(range(8))
