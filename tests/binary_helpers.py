"""Shared by the binary-operator tests: the golden tables, node results computed by the CPU oracle, and the conversion
between dense [rows x T] grids and the reference's (labels..., ts, value) rows."""
import json
import os

import numpy as np

from oracle import oracle as orc
from tests.helpers import GOLDEN_DIR

LOOKBACK = 300_000  # the reference's default lookback delta


def load_binary():
    with open(os.path.join(GOLDEN_DIR, "reference_binary_vectors.json")) as f:
        return json.load(f)


def sum_rate_table():
    """The `metrics` table of tql/range.result, from reference_sum_rate_vectors.json."""
    with open(os.path.join(GOLDEN_DIR, "reference_sum_rate_vectors.json")) as f:
        g = json.load(f)
    return {"time_index": "ts", "field": "val", "tags": g["tags"], "series": g["series"]}


def table_arrays(table):
    """-> (label tuples per series, ts, val, offsets) with the series in tag order."""
    tags = table["tags"]
    series = sorted(table["series"], key=lambda s: tuple(s[t] for t in tags))
    labels = [tuple(s[t] for t in tags) for s in series]
    ts = np.array([t for s in series for t in s["ts"]], np.int64)
    val = np.array([v for s in series for v in s["val"]], np.float64)
    offsets = np.cumsum([0] + [len(s["ts"]) for s in series]).astype(np.uint64)
    return labels, ts, val, offsets


def oracle_node(table, start, end, interval, fn=None, range_ms=None, agg=None, by=()):
    """A node's result on the CPU: fn(table[range]) or the instant selector, optionally `agg by (by)`.
    -> (tag names, label tuples per row, out [rows x T], valid words, eval ts)"""
    labels, ts, val, offsets = table_arrays(table)
    T = orc.num_steps(start, end, interval)
    eval_ts = start + interval * np.arange(T, dtype=np.int64)
    if fn is None:
        out, valid = orc.instant_query(ts, val, offsets, start, end, interval, LOOKBACK)
    else:
        out, valid = orc.range_query(orc.make_params(fn, start, end, interval, range_ms), ts, val, None, offsets)
    tags = list(table["tags"])
    if agg is None:
        return tags, labels, out, valid, eval_ts
    idx = [tags.index(b) for b in by]
    keys = sorted({tuple(lab[i] for i in idx) for lab in labels})
    gid = np.array([keys.index(tuple(lab[i] for i in idx)) for lab in labels], np.uint32)
    gval, gcnt = orc.group_aggregate(agg, out, valid, gid, len(keys))
    gvalid = np.zeros((len(keys), (T + 31) // 32), np.uint32)
    for k in range(T):
        gvalid[:, k // 32] |= (gcnt[:, k] != 0).astype(np.uint32) << np.uint32(k % 32)
    return list(by), keys, np.where(gcnt != 0, gval, 0.0), gvalid, eval_ts


def dense_rows(tags, labels, out, valid, eval_ts):
    """Dense result -> (tag names, rows [(labels..., ts, value)]) in row order, steps ascending."""
    rows = []
    T = eval_ts.size
    for r, lab in enumerate(labels):
        for k in range(T):
            if (int(valid[r, k // 32]) >> (k % 32)) & 1:
                rows.append(tuple(lab) + (int(eval_ts[k]), float(out[r, k])))
    return list(tags), rows


def count_rows(rows):
    """count(...) without by-labels, row-literal: one row per timestamp with the number of rows there."""
    n = {}
    for r in rows:
        n[r[-2]] = n.get(r[-2], 0) + 1
    return [(ts, float(c)) for ts, c in sorted(n.items())]


def expected_rows(case, tags):
    """A golden case's printed rows as (labels in `tags` order..., ts, value), sorted."""
    return sorted(tuple(lab[t] for t in tags) + (ts, v) for lab, ts, v in case["expected"])
