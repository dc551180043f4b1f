"""CPU restatement of the PromQL set operators `and`, `or`, `unless` (test infrastructure; the product never imports it).

planner.rs:3549-3703 (and / unless: left.distinct() LeftSemi / LeftAnti joined on (key columns, ts)), planner.rs:3707-3906
and union_distinct_on.rs:338-577 (or).  Labels are strings or None (NULL); NULL equals NULL and no string.

Two forms, as for the binary operators (tests/binary_oracle.py):
  * row-literal — `setop_rows` works on (labels..., ts, value) rows with dicts on (key, ts), as the reference's joins do;
  * dense — `setop_pairs` gives every row a dense key id (what the plan layer does on the host), `distinct_cells` is the
    plan layer's host pass for `distinct()`, and `setop` is the per-cell pass over the grids (what K8 does).
"""
import numpy as np

from tests.binary_oracle import _bits, _words

SET_OPS = {"and": 0, "or": 1, "unless": 2}
NO_KEY = 0xFFFFFFFF


def _narrow(tags, on=None, ignoring=None):
    return [t for t in tags if (on is None or t in on) and (ignoring is None or t not in ignoring)]


def setop_key_columns(op, lhs_tags, rhs_tags, on=None, ignoring=None):
    """Match columns.  and / unless: each side's tags narrowed by on / ignoring, which must agree (else the planner's
    CombineTableColumnMismatch, raised here as KeyError).  or: the `on` labels (one that neither side has fails, as
    UnionDistinctOnExec's "Column not found" does), or the union of both sides' tags without `ignoring`.
    -> (match columns, output tag columns)"""
    if op != "or":
        ln, rn = _narrow(lhs_tags, on, ignoring), _narrow(rhs_tags, on, ignoring)
        if sorted(ln) != sorted(rn):
            raise KeyError(f"set operator {op}: key columns differ: {ln} vs {rn}")
        return sorted(ln), list(lhs_tags)
    union = sorted(set(lhs_tags) | set(rhs_tags))
    if on is not None:
        for label in on:
            if label not in union:
                raise KeyError(f"Column {label} not found")
        return sorted(on), union
    return _narrow(union, None, ignoring), union


def _label(tags, row, name):
    return row[tags.index(name)] if name in tags else None


def _fbits(v):
    return np.array([v], np.float64).view(np.uint64)[0]


def setop_rows(lhs, rhs, op, on=None, ignoring=None):
    """Row-literal `lhs op rhs`.  lhs / rhs: (tag names, rows [(tag values..., ts, value)]).
    and / unless: left.distinct() (a row equal to an earlier one in labels, ts and value bits goes), then a dict on
    (key, ts) of the rhs rows for the semi / anti join; the output has the lhs columns.
    or: every lhs row, then each rhs row whose (key, ts) no lhs row and no earlier rhs row has (HashedData::new keeps
    the first row per key; update_map removes the keys the lhs has); the output tags are the union of both sides'.
    -> (tag names, rows)"""
    (ltags, lrows), (rtags, rrows) = lhs, rhs
    keys, out_tags = setop_key_columns(op, ltags, rtags, on, ignoring)
    key = lambda tags, r: (tuple(_label(tags, r, k) for k in keys), r[-2])
    if op != "or":
        seen, distinct = set(), []
        for r in lrows:
            d = tuple(r[:-1]) + (_fbits(r[-1]),)
            if d not in seen:
                seen.add(d)
                distinct.append(r)
        right = {key(rtags, r) for r in rrows}
        return list(ltags), [r for r in distinct if (key(ltags, r) in right) == (op == "and")]
    widen = lambda tags, r: tuple(_label(tags, r, t) for t in out_tags) + tuple(r[-2:])
    out = [widen(ltags, r) for r in lrows]
    left = {key(ltags, r) for r in lrows}
    first = set()
    for r in rrows:
        k = key(rtags, r)
        if k in left or k in first:
            continue
        first.add(k)
        out.append(widen(rtags, r))
    return out_tags, out


def setop_pairs(op, lhs_tags, lhs_labels, rhs_tags, rhs_labels, on=None, ignoring=None):
    """Dense key ids of both sides' rows (what the plan layer computes on the host).  and / unless: ids of the rhs
    key tuples in row order, NO_KEY for an lhs row whose tuple the rhs lacks; or: ids over the lhs rows, then the rhs.
    -> (lhs_key, rhs_key uint32 arrays, n_keys, output tag names)"""
    keys, out_tags = setop_key_columns(op, lhs_tags, rhs_tags, on, ignoring)
    ids = {}
    tup = lambda tags, lab: tuple(_label(tags, lab, k) for k in keys)

    def add(tags, lab):
        return ids.setdefault(tup(tags, lab), len(ids))

    if op == "or":
        lk = [add(lhs_tags, lab) for lab in lhs_labels]
        rk = [add(rhs_tags, lab) for lab in rhs_labels]
    else:
        rk = [add(rhs_tags, lab) for lab in rhs_labels]
        lk = [ids.get(tup(lhs_tags, lab), NO_KEY) for lab in lhs_labels]
    return np.array(lk, np.uint32), np.array(rk, np.uint32), len(ids), out_tags


def distinct_cells(labels, vals, valid):
    """left.distinct() on a dense grid: a cell equal in labels, step and value bits to a valid cell of an earlier row
    is cleared.  -> (vals, valid) copies."""
    vals, T = np.array(vals, np.float64), np.asarray(vals).shape[1]
    ok = _bits(np.asarray(valid, np.uint32), T)
    b = vals.view(np.uint64)
    first = {}
    for r, lab in enumerate(labels):
        first.setdefault(tuple(lab), []).append(r)
    for rows in first.values():
        for i, q in enumerate(rows):
            for p in rows[:i]:
                ok[q] &= ~(ok[p] & (b[p] == b[q]))
    return np.where(ok, vals, 0.0), _words(ok)


def setop(op, lhs, lhs_valid, lhs_key, rhs, rhs_valid, rhs_key, n_keys):
    """Dense restatement of b2p_setop: -> (out, valid words); [L x T] for and / unless, [(L + R) x T] for or."""
    op = op if isinstance(op, str) else {v: k for k, v in SET_OPS.items()}[int(op)]
    lhs, rhs = np.asarray(lhs, np.float64), np.asarray(rhs, np.float64)
    T = lhs.shape[1] if lhs.ndim == 2 and lhs.shape[0] else rhs.shape[1]
    lhs, rhs = lhs.reshape(-1, T), rhs.reshape(-1, T)
    Tw = (T + 31) // 32
    lok = _bits(np.asarray(lhs_valid, np.uint32).reshape(lhs.shape[0], Tw), T)
    rok = _bits(np.asarray(rhs_valid, np.uint32).reshape(rhs.shape[0], Tw), T)
    lk, rk = np.asarray(lhs_key, np.int64), np.asarray(rhs_key, np.int64)

    def mask(ok, keys):
        m = np.zeros((n_keys, T), bool)
        for r, k in enumerate(keys):
            if k < n_keys:
                m[k] |= ok[r]
        return m

    if op != "or":
        m = mask(rok, rk)
        out = np.zeros_like(lok)
        for r, k in enumerate(lk):
            if k == NO_KEY:
                out[r] = lok[r] if op == "unless" else False
            elif k < n_keys:
                out[r] = lok[r] & (m[k] if op == "and" else ~m[k])
        return np.where(out, lhs, 0.0), _words(out)
    running = mask(lok, lk)
    lout = lok & ((lk < n_keys) | (lk == NO_KEY))[:, None]
    rout = np.zeros_like(rok)
    for r, k in enumerate(rk):
        if k == NO_KEY:
            rout[r] = rok[r]
        elif k < n_keys:
            rout[r] = rok[r] & ~running[k]
            running[k] |= rok[r]
    ok = np.concatenate([lout, rout])
    return np.where(ok, np.concatenate([lhs, rhs]), 0.0), _words(ok)
