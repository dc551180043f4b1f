"""CPU restatement of PromQL sort / sort_desc / sort_by_label / sort_by_label_desc as the reference plans them (test
infrastructure only).

The reference (src/query/src/promql/planner.rs:1060-1089, 2743-2772) plans
  Projection(time index, value, tags..) -> Filter(value IS NOT NULL) -> Sort(keys)
over the child, with keys
  * sort:               value ASC NULLS FIRST
  * sort_desc:          value DESC NULLS FIRST
  * sort_by_label:      the listed labels ASC NULLS LAST
  * sort_by_label_desc: the listed labels DESC NULLS LAST
Values compare in arrow's f64 total order (-NaN < -inf < .. < -0.0 < +0.0 < .. < +inf < +NaN; descending is the exact
reverse); labels compare as arrow's Utf8, byte-wise, NULL after every string in both directions.  Ties keep the child's
row-major order (row, then step), which a stable sort of the child's rows gives.

Two forms:
  * `value_order`: the dense form K14 computes, the valid cells of a [rows x T] grid as cell indices r * T + k;
  * `sort_rows`: over exported rows (value, {tag: label}, ts) in the child's row-major order.
"""
import struct

import numpy as np

FUNCTIONS = ("sort", "sort_desc", "sort_by_label", "sort_by_label_desc")


def total_key(x: float) -> int:
    """f64::total_cmp's key: the bit pattern as i64, the low 63 bits flipped for negative values."""
    b = struct.unpack("<q", struct.pack("<d", float(x)))[0]
    return b ^ (0x7FFFFFFFFFFFFFFF if b < 0 else 0)


def total_keys(vals) -> np.ndarray:
    """total_key of every element, as int64"""
    b = np.ascontiguousarray(vals, np.float64).view(np.int64)
    return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


def value_order(vals, ok, desc: bool) -> np.ndarray:
    """the valid cells (ok [rows, T] bool) of vals [rows, T] as cell indices in value order, ties in row-major order"""
    cells = np.flatnonzero(np.asarray(ok, bool).reshape(-1))
    keys = total_keys(np.asarray(vals, np.float64).reshape(-1)[cells])
    if desc:
        keys = ~keys  # strictly decreasing in the key: the exact reverse order, and the stable sort keeps ties in place
    return cells[np.argsort(keys, kind="stable")].astype(np.uint64)


def label_order(labels_of, n: int, labels, desc: bool) -> list:
    """positions 0..n-1 ranked by the listed labels (labels_of(i, l): a str or None), byte order, NULL last, stable"""
    order = list(range(n))
    for l in reversed(list(labels)):  # least significant label first; each pass is stable
        present = [i for i in order if labels_of(i, l) is not None]
        nulls = [i for i in order if labels_of(i, l) is None]
        present.sort(key=lambda i: labels_of(i, l).encode(), reverse=desc)  # (reverse keeps ties in order)
        order = present + nulls
    return order


def sort_rows(function: str, rows, labels=()):
    """rows: [(value, {tag: label}, ts)] in the child's row-major order -> the same rows in the function's order"""
    if function not in FUNCTIONS:
        raise ValueError(function)
    desc = function.endswith("_desc")
    if function.startswith("sort_by_label"):
        order = label_order(lambda i, l: rows[i][1].get(l), len(rows), labels, desc)
    else:
        order = value_order(np.array([v for v, _, _ in rows], np.float64), np.ones(len(rows), bool), desc)
    return [rows[int(i)] for i in order]
