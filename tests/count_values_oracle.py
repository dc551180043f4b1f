"""Restatement of the reference's count_values (planner.rs:402-445): Aggregate(groupBy = [group labels.., ts, value],
count(value)) -> Projection(count, group labels.., ts, value AS label) -> Sort(group labels, ts, value), in two forms:

- row-literal (`count_values_rows`): rows -> a dict on (group tuple, ts, value bits) -> count, then the reference's
  sort;
- dense (`count_values`): what b2p_count_values computes over a [rows x T] grid grouped by gid.

Two rules come from DataFusion and arrow rather than from the reference's tree, and are restated here:
- DataFusion groups a Float64 column by its bits: -0.0 and +0.0 are two values, and NaNs with different bits are
  different values;
- arrow sorts Float64 in the f64 total order (f64::total_cmp): -NaN < -inf < .. < -0.0 < +0.0 < .. < +inf < +NaN, NaN
  payloads ordered by their bits.
Group labels sort by the plan layer's Labels::less ("" first, then NULL, then the other strings), the known divergence
from the reference's NULLS LAST listed in DESIGN.md section 2.
"""
import struct

import numpy as np

from tests.aggregate_oracle import group_names, label_order


def value_bits(v: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", float(v)))[0]


def total_key(v: float) -> int:
    """f64::total_cmp's key: the bit pattern as i64, the low 63 bits flipped for negative values."""
    b = struct.unpack("<q", struct.pack("<d", float(v)))[0]
    return b ^ (0x7FFFFFFFFFFFFFFF if b < 0 else 0)


def count_values_rows(rows, tags, by=None, without=None):
    """rows [(value, {tag: label}, ts)] with tag names `tags` -> ([(count, {group label: label}, ts, value)] in the
    reference's output order, group label names)"""
    names = group_names(tags, by, without)
    counts = {}
    for v, lab, ts in rows:
        key = (tuple(lab.get(n) for n in names), ts, value_bits(v))
        counts[key] = counts.get(key, 0) + 1
    out = [(n, dict(zip(names, g)), ts, struct.unpack("<d", struct.pack("<Q", b))[0]) for (g, ts, b), n in counts.items()]
    out.sort(key=lambda r: (tuple(label_order(r[1][n]) for n in names), r[2], total_key(r[3])))
    return out, names


def _bits(valid, T):
    valid = np.asarray(valid, np.uint32)
    return ((valid[:, np.arange(T) // 32] >> (np.arange(T) % 32).astype(np.uint32)) & 1).astype(bool)


def member_order(gid, n_groups):
    """The rows of b2p_count_values' output: a stable sort of the rows by gid (rows of gid >= n_groups last), and each
    group's first position."""
    gid = np.asarray(gid, np.int64)
    order = np.argsort(gid, kind="stable")
    return order, np.searchsorted(gid[order], np.arange(n_groups + 1))


def count_values(vals, valid, gid, n_groups):
    """Dense count_values: vals [rows, T] f64, valid [rows, Tw] u32 words, gid [rows] (>= n_groups: no group) ->
    (out [rows, T] f64, cnt [rows, T] u32) in member order: at step k, group g's j-th row (position goff[g] + j) holds
    the j-th smallest distinct value of the group's valid cells in the total order and its multiplicity; cnt 0 and
    value 0.0 past the last distinct value and on the rows of no group."""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    ok = _bits(valid, T)
    out = np.zeros((R, T), np.float64)
    cnt = np.zeros((R, T), np.uint32)
    order, goff = member_order(gid, n_groups)
    keys = vals.view(np.int64) ^ ((vals.view(np.int64) >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))
    for g in range(n_groups):
        rows = order[goff[g]:goff[g + 1]]
        for k in range(T):
            cell = keys[rows[ok[rows, k]], k]
            if cell.size == 0:
                continue
            uniq, n = np.unique(cell, return_counts=True)  # ascending keys = the total order, equal keys = equal bits
            b = uniq ^ ((uniq >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))
            out[goff[g]:goff[g] + uniq.size, k] = b.view(np.float64)
            cnt[goff[g]:goff[g] + uniq.size, k] = n
    return out, cnt


def dense_to_rows(out, cnt, gid, group_keys, names):
    """The dense form as the row-literal one's output: group_keys[g] is group g's label tuple over `names`; groups in
    label order, then ts, then rank (= value order)."""
    order, goff = member_order(gid, len(group_keys))
    T = out.shape[1]
    rows = []
    for g in sorted(range(len(group_keys)), key=lambda g: tuple(label_order(v) for v in group_keys[g])):
        for k in range(T):
            for p in range(goff[g], goff[g + 1]):
                if cnt[p, k]:
                    rows.append((int(cnt[p, k]), dict(zip(names, group_keys[g])), k, float(out[p, k])))
    return rows
