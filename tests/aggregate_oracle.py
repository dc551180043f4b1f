"""Restatement of the reference's by-label aggregate over any expression (prom_aggr_expr_to_plan, planner.rs:334-452,
create_aggregate_exprs 2808-2897), in two forms:

- row-literal (`aggregate_rows`): rows -> (group tuple, ts) buckets in row order -> the accumulator -> sort by group
  labels, then ts;
- dense (`group_quantile`): what b2p_group_quantile computes per (group, step) over a [rows x T] grid.

The seven aggregators K3 already runs go through oracle.group_aggregate, quantile through oracle.quantile (the
restatement of quantile.rs:201-225 pinned in oracle/), group is 1.0 (planner.rs:2836-2838, `max(1.0)`).
"""
import numpy as np

from oracle import oracle as orc

SEVEN = ("sum", "avg", "count", "min", "max", "stddev", "stdvar")


def group_names(tags, by=None, without=None):
    """agg_modifier_to_col (planner.rs:1400-1480): `by` the listed labels the input has, in the listed order; `without`
    the input's tags not listed, in name order; neither: none."""
    if by is not None:
        return [l for l in by if l in tags]
    if without is not None:
        return sorted(t for t in tags if t not in without)
    return []


def label_order(v):
    """The plan layer's order of label values: "" first, then NULL, then the other strings (DESIGN.md section 2)."""
    return (1, "") if v is None else (0, "") if v == "" else (2, v)


def accumulate(op, values, param=None):
    """One bucket's value, the values in row order"""
    if op == "group":
        return 1.0
    if op == "quantile":
        return float(orc.quantile(np.array(values, np.float64), param))
    assert op in SEVEN, op
    vals = np.array(values, np.float64).reshape(-1, 1)
    out, cnt = orc.group_aggregate(op, vals, np.ones((len(values), 1), np.uint32), np.zeros(len(values), np.uint32), 1)
    return float(out[0, 0])


def aggregate_rows(rows, tags, op, param=None, by=None, without=None):
    """rows [(value, {tag: label}, ts)] in row order, with tag names `tags` -> ([(value, {group label: label}, ts)] in
    output order, group label names)"""
    names = group_names(tags, by, without)
    buckets = {}
    for v, lab, ts in rows:
        buckets.setdefault((tuple(lab.get(n) for n in names), ts), []).append(v)
    out = [(accumulate(op, vs, param), dict(zip(names, key)), ts) for (key, ts), vs in buckets.items()]
    out.sort(key=lambda r: (tuple(label_order(r[1][n]) for n in names), r[2]))
    return out, names


def group_quantile(phi, vals, valid, gid, n_groups):
    """Dense quantile(phi) per (group, step): vals [rows, T] f64, valid [rows, Tw] u32 words, gid [rows] (>= n_groups:
    no group) -> (out [G, T] f64, cnt [G, T] u32), cnt 0 and value 0.0 where a group has no valid cell."""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    gid = np.asarray(gid, np.int64)
    bits = ((np.asarray(valid, np.uint32)[:, np.arange(T) // 32] >> (np.arange(T) % 32).astype(np.uint32)) & 1).astype(bool)
    out = np.zeros((n_groups, T), np.float64)
    cnt = np.zeros((n_groups, T), np.uint32)
    order = np.argsort(gid, kind="stable")
    bounds = np.searchsorted(gid[order], np.arange(n_groups + 1))
    for g in range(n_groups):
        rows = order[bounds[g]:bounds[g + 1]]
        if rows.size == 0:
            continue
        sub, ok = vals[rows], bits[rows]
        for k in range(T):
            cell = sub[ok[:, k], k]
            cnt[g, k] = cell.size
            if cell.size:
                out[g, k] = orc.quantile(cell, phi)
    return out, cnt
