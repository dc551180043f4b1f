"""CPU restatement of the plan layer over nodes with several field columns, built from the single-field oracles.

GreptimeDB's planner carries a node's field columns through every operator above a multi-field selector
(src/query/src/promql/planner.rs; F is a node's field count):
  - instant functions, `node op scalar` and `bool` comparisons are projected once per field (2416, 3930-3960);
  - a vector-vector arithmetic or `bool` operator zips the fields pairwise, field i with field i, min(F_l, F_r) of them
    (align_binary_field_columns, 3401-3414); a filtering comparison decides on its one pair and keeps the lhs side's
    fields (712-777);
  - sum avg count min max stddev stdvar quantile fold every field (2824-2866);
  - sort / sort_desc order by every field in turn, each ASC or DESC NULLS FIRST (1066-1071, 2743-2749);
  - a subquery applies its function per field, then keeps a cell where every field's result is (292-332);
  - the rest refuse F >= 2 (REFUSALS, the reference's error texts).
Grids are dense: a node's values [F, rows, T] under one validity [rows, Tw], as the plan layer holds them.
"""
import numpy as np

from oracle import oracle as orc
from tests import aggregate_oracle as ag
from tests import binary_oracle as bo
from tests import instant_fn_oracle as ifo
from tests import select_keys as sk
from tests import subquery_oracle as sq

FILTER = "Unsupported expr type: filter on multi-value input"
REFUSALS = {
    "filter": FILTER,
    "topk": "Unsupported expr type: topk or bottomk on multi-value input",
    "count_values": "Unsupported expr type: count_values on multi-value input",
    "group": "Multi fields calculation is not supported in group()",
    "scalar": "Multi fields calculation is not supported in scalar",
    "and": "Multi fields calculation is not supported in AND operator",
    "unless": "Multi fields calculation is not supported in AND operator",
    "or": "Multi fields calculation is not supported in OR operator",
}
COMPARISONS = ("==", "!=", ">", "<", ">=", "<=")


class Refused(ValueError):
    pass


def is_filter(op, return_bool):
    return op in COMPARISONS and not return_bool


def leaf_names(function, time_index, fields):
    """the value column of each field: prom_fn(<ti>_range,<field>) for a range function, the field for an instant one"""
    return [f"{function}({time_index}_range,{f})" if function else f for f in fields]


def instant_fn(fn, vals, valid, arg0=0.0, arg1=0.0):
    """a function once per field -> (vals [F, R, T], valid): a function keeps every bit"""
    res = [ifo.instant_fn(fn, v, valid, arg0, arg1) for v in vals]
    for _, w in res:
        assert np.array_equal(w, valid)
    return np.stack([o for o, _ in res]), valid


def scalar_op(op, scalar, vals, valid, scalar_on_left=False, return_bool=False):
    """`node op scalar` once per field; a filtering comparison is refused for F >= 2"""
    if is_filter(op, return_bool) and len(vals) > 1:
        raise Refused(FILTER)
    res = [bo.scalar_op(op, scalar, v, valid, scalar_on_left, return_bool) for v in vals]
    if len(vals) > 1:
        for _, w in res:
            assert np.array_equal(w, res[0][1])
    return np.stack([o for o, _ in res]), res[0][1]


def binary_op(op, lhs, lhs_valid, lhs_row, rhs, rhs_valid, rhs_row, return_bool=False):
    """`lhs op rhs` over matched pairs -> (vals [F', P, T], valid [P, Tw]): F' = min(F_l, F_r) zipped fields for
    arithmetic and `bool`; a filtering comparison needs exactly one pair, which decides, and keeps all F_l lhs fields"""
    pairs = min(len(lhs), len(rhs))
    lr = np.asarray(lhs_row, np.int64)
    if is_filter(op, return_bool):
        if pairs > 1:
            raise Refused(FILTER)
        out0, ov = bo.binary_op(op, lhs[0], lhs_valid, lhs_row, rhs[0], rhs_valid, rhs_row, False)
        ok = orc.valid_to_bool(ov, lhs[0].shape[1])
        outs = [out0] + [np.where(ok, np.asarray(v, np.float64)[lr], 0.0) for v in lhs[1:]]
        return np.stack(outs), ov
    res = [bo.binary_op(op, lhs[f], lhs_valid, lhs_row, rhs[f], rhs_valid, rhs_row, return_bool) for f in range(pairs)]
    for _, w in res:
        assert np.array_equal(w, res[0][1])
    return np.stack([o for o, _ in res]), res[0][1]


def binary_names(op, lhs_names, rhs_names, return_bool=False):
    if is_filter(op, return_bool):
        return list(lhs_names)
    return [f"{a} {op} {b}" for a, b in zip(lhs_names, rhs_names)]


def aggregate(op, vals, valid, gid, n_groups, param=None):
    """op by group, once per field -> (vals [F, G, T], cnt [G, T]); group() is refused for F >= 2"""
    if op == "group" and len(vals) > 1:
        raise Refused(REFUSALS["group"])
    outs, cnt = [], None
    for v in vals:
        if op == "quantile":
            o, c = ag.group_quantile(param, v, valid, gid, n_groups)
        else:
            o, c = orc.group_aggregate("count" if op == "group" else op, v, valid, np.asarray(gid, np.uint32), n_groups)
            if op == "group":
                o = np.where(c != 0, 1.0, 0.0)
        assert cnt is None or np.array_equal(c, cnt)
        cnt = c
        outs.append(o)
    return np.stack(outs), cnt


def subquery(fn, start, end, interval, range_ms, inner_start, inner_interval, vals, valid, param0=0.0, param1=0.0):
    """fn(child[range:step]) once per field, then the conjunction of the fields' validity"""
    res = [sq.subquery(fn, start, end, interval, range_ms, inner_start, inner_interval, v, valid, param0, param1)
           for v in vals]
    ov = res[0][1].copy()
    for _, w in res[1:]:
        ov &= w
    return np.stack([o for o, _ in res]), ov


def sort(desc, vals, ok):
    """the valid cells as indices r * T + k, ordered lexicographically by the fields' total-order keys (field 0 first;
    every key inverted for sort_desc), equal tuples in row-major order: a stable numpy.lexsort"""
    cells = np.flatnonzero(np.asarray(ok, bool).reshape(-1))
    keys = [sk.keys_of_values(np.asarray(v, np.float64).reshape(-1)[cells]) for v in vals]
    if desc:
        keys = [~k for k in keys]
    return cells[np.lexsort(tuple(reversed(keys)))].astype(np.uint64)
