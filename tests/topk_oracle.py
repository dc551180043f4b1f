"""CPU restatement of PromQL topk / bottomk as the reference plans them (test infrastructure only).

The reference (src/query/src/promql/planner.rs:454-541, 2963-3016) builds
  Window(row_number() OVER (PARTITION BY group_exprs ORDER BY value, tags)) -> Filter(row_number <= k)
  -> Sort(group_exprs, row_number) -> Projection(value, tags.., ts)
with
  * group_exprs: `by (l..)` the listed labels the input has, in the listed order; `without (l..)` the input's tags
    minus the listed ones in name order; no modifier: none.  The time index always follows.
  * ORDER BY: the value in the f64 total order (+NaN above +inf, -NaN below -inf, -0.0 < +0.0), then every tag of the
    input in column order; descending for topk, ascending for bottomk; NULL first in both.
  * row_number <= k: the UInt64 row number coerced to Float64 against the Float64 literal k, in the total order.
  * the final sort puts NULLs last.

Two forms:
  * `topk_rows`: row-literal, over rows (value, labels, ts) — partition, sort, filter, sort;
  * `topk_keys` + `topk`: the dense form the library computes — a group id and a distinct tie ordinal per row (the
    plan layer's host part), then per (group, step) the min(kk, valid cells) best cells of the grid (kernel K10).
"""
import functools
import math
import struct

import numpy as np

KMAX = 32  # largest k of the kernel's fast path


def total_key(x: float) -> int:
    """f64::total_cmp's key: the bit pattern as i64, the low 63 bits flipped for negative values."""
    b = struct.unpack("<q", struct.pack("<d", float(x)))[0]
    return b ^ (0x7FFFFFFFFFFFFFFF if b < 0 else 0)


def kept_ranks(k: float, n: int) -> int:
    """How many of n ranks row_number <= k keeps, compared as Float64 in the total order."""
    kk = total_key(k)
    return sum(1 for rn in range(1, n + 1) if total_key(float(rn)) <= kk)


def ranks_of_k(k: float) -> float:
    """The closed form of kept_ranks (an upper bound that is not a count: math.inf)."""
    if math.isnan(k):
        return 0 if math.copysign(1.0, k) < 0 else math.inf
    if k < 1:
        return 0
    return math.inf if math.isinf(k) else math.floor(k)


def group_columns(tags, modifier=None, labels=()):
    """The group labels: `by` the listed ones the input has (listed order), `without` the rest in name order."""
    if modifier == "by":
        return [l for l in labels if l in tags]
    if modifier == "without":
        return sorted(t for t in tags if t not in labels)
    return []


def _label_cmp(a, b, descending):
    """One tag of the window's ORDER BY: NULL first, then the values ascending / descending."""
    if a == b:
        return 0
    if a is None:
        return -1
    if b is None:
        return 1
    c = -1 if a < b else 1
    return -c if descending else c


def _tuple_cmp(a, b, descending):
    for x, y in zip(a, b):
        c = _label_cmp(x, y, descending)
        if c:
            return c
    return 0


def _nulls_last_key(t):
    return tuple((1, "") if v is None else (0, v) for v in t)


def topk_rows(bottom, k, rows, tags, modifier=None, labels=()):
    """rows: [(value, {tag: label or None}, ts)] of a node with tag columns `tags`.  Returns the kept rows in the
    reference's output order, each (value, {tag: label}, ts)."""
    gcols = group_columns(tags, modifier, labels)
    parts = {}
    for i, (v, lab, ts) in enumerate(rows):
        key = tuple(lab.get(c) for c in gcols) + (ts,)
        parts.setdefault(key, []).append(i)
    desc = not bottom

    def cmp(i, j):
        ki, kj = total_key(rows[i][0]), total_key(rows[j][0])
        if ki != kj:
            return (-1 if ki > kj else 1) if desc else (-1 if ki < kj else 1)
        c = _tuple_cmp([rows[i][1].get(t) for t in tags], [rows[j][1].get(t) for t in tags], desc)
        return c if c else (i > j) - (i < j)  # identical tuples: row order (the reference leaves it undefined)

    out = []
    for key in sorted(parts, key=lambda p: (_nulls_last_key(p[:-1]), p[-1])):
        ranked = sorted(parts[key], key=functools.cmp_to_key(cmp))
        n = kept_ranks(k, len(ranked))
        out.extend(rows[i] for i in ranked[:n])
    return out


def topk_keys(bottom, tags, tuples, modifier=None, labels=()):
    """Host part: tuples [rows] of label tuples over `tags`.  Returns (gid uint32 [rows], n_groups, tie uint32 [rows],
    group columns).  Groups are numbered in first-appearance order; tie ranks the rows by their tuple in the direction
    of the op with NULL first (identical tuples: the earlier row first), so that comparing (value, tie) descending for
    topk / ascending for bottomk is the window's order."""
    gcols = group_columns(tags, modifier, labels)
    gidx = [tags.index(c) for c in gcols]
    ids, gid = {}, np.zeros(len(tuples), np.uint32)
    for r, t in enumerate(tuples):
        gid[r] = ids.setdefault(tuple(t[i] for i in gidx), len(ids))
    desc = not bottom
    order = sorted(range(len(tuples)),
                   key=functools.cmp_to_key(lambda i, j: _tuple_cmp(tuples[i], tuples[j], desc) or (i > j) - (i < j)))
    tie = np.zeros(len(tuples), np.uint32)
    n = len(tuples)
    for p, r in enumerate(order):
        tie[r] = (n - 1 - p) if desc else p
    return gid, len(ids), tie, gcols


def _bits(valid_words, T):
    w = np.ascontiguousarray(valid_words, np.uint32)
    return np.unpackbits(w.view(np.uint8).reshape(w.shape[0], -1), axis=1, bitorder="little")[:, :T].astype(bool)


def _words(bits):
    R, T = bits.shape
    Tw = (T + 31) // 32
    pad = np.zeros((R, Tw * 32), np.uint8)
    pad[:, :T] = bits
    return np.packbits(pad, axis=1, bitorder="little").view(np.uint32).reshape(R, Tw)


def total_keys_np(vals):
    b = np.ascontiguousarray(vals, np.float64).view(np.int64)
    return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


def rank_keys(bottom, vals, tie):
    """(hi uint64 [R,T], lo uint32 [R]): larger is better, as the kernel compares them."""
    hi = total_keys_np(vals).view(np.uint64) ^ np.uint64(1 << 63)
    lo = np.asarray(tie, np.uint32)
    if bottom:
        hi, lo = ~hi, ~lo
    return hi, lo


def topk(bottom, k, vals, valid_words, gid, n_groups, tie):
    """K10: validity words [R, Tw] of the cells kept per (group, step); bits at or past T are 0; a row whose group id is
    >= n_groups keeps nothing."""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    valid = _bits(valid_words, T)
    kept = np.zeros((R, T), bool)
    kk = ranks_of_k(k)
    gid = np.asarray(gid, np.int64)
    if kk > 0 and T > 0:
        hi, lo = rank_keys(bottom, vals, tie)
        for g in range(n_groups):
            m = np.nonzero(gid == g)[0]
            if m.size == 0:
                continue
            v = valid[m]
            lo_b = np.broadcast_to(lo[m][:, None], v.shape)
            order = np.lexsort((lo_b, hi[m], v), axis=0)  # ascending; invalid cells first
            n_keep = np.minimum(v.sum(axis=0), kk)  # [T]
            pos = np.empty_like(order)
            np.put_along_axis(pos, order, np.arange(m.size)[:, None].repeat(T, axis=1), axis=0)
            kept[m] = pos >= (m.size - n_keep)[None, :]
            kept[m] &= v
    return _words(kept)


def export_rows(bottom, vals, kept_words, tags, tuples, ts, gcols, tie):
    """The kept cells of the dense form in the reference's output order: group labels (NULLs last), ts, rank."""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    kept = _bits(kept_words, T)
    hi, lo = rank_keys(bottom, vals, tie)
    gidx = [tags.index(c) for c in gcols]
    cells = []
    for r, k in zip(*np.nonzero(kept)):
        g = tuple(tuples[r][i] for i in gidx)
        cells.append(((_nulls_last_key(g), int(ts[k]), -int(hi[r, k]), -int(lo[r])), r, k))
    cells.sort(key=lambda c: c[0])
    return [(float(vals[r, k]), dict(zip(tags, tuples[r])), int(ts[k])) for _, r, k in cells]
