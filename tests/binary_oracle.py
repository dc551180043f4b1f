"""CPU restatement of the PromQL binary operators (test infrastructure; the product never imports it).

src/query/src/promql/planner.rs:556-777, 779-838, 3320-3546, 3915-3990: both operands are Float64; `/` is IEEE, `%` is
Rust's `%` on f64 (fmod), `^` is `f64::powf` and `atan2(lhs, rhs)` is `lhs.atan2(rhs)` — glibc's pow / atan2 / fmod,
which is what the reference calls on Linux, bound here through ctypes.  Comparisons are arrow-rs cmp kernels, which order
f64 by the IEEE 754 totalOrder predicate (`f64::total_cmp`): NaN == NaN, -0.0 < +0.0, -NaN below -inf.  A comparison
without `bool` filters: the cell stays only when it holds, with the vector operand's value (the lhs of a pair); with
`bool` it is 1.0 / 0.0.  A cell is valid iff both operands are (and, filtering, the comparison holds); invalid cells are
0.0, like every dense result of the library.

Two forms of the vector-vector operator:
  * dense — `binary_pairs` matches series on their key tuples (what the plan layer does on the host), `binary_op` is
    the element-wise pass over the pairs (what the kernel does);
  * row-literal — `binary_rows` inner-joins (labels..., ts, value) rows on (key columns, ts) through a dict, then
    projects or filters, as the reference's HashJoinExec + ProjectionExec / FilterExec do.
"""
import ctypes as C

import numpy as np

BIN_OPS = {"+": 0, "-": 1, "*": 2, "/": 3, "%": 4, "^": 5, "atan2": 6,
           "==": 7, "!=": 8, ">": 9, "<": 10, ">=": 11, "<=": 12}
_EQ = BIN_OPS["=="]

_libm = C.CDLL("libm.so.6")
_LIBM = {}
for _name in ("pow", "atan2", "fmod"):
    _f = getattr(_libm, _name)
    _f.restype = C.c_double
    _f.argtypes = [C.c_double, C.c_double]
    _LIBM[_name] = np.frompyfunc(_f, 2, 1)


def _op_id(op):
    return BIN_OPS[op] if isinstance(op, str) else int(op)


def _libm_call(name, a, b):
    a, b = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64))
    if a.size == 0:
        return np.zeros(a.shape, np.float64)
    return _LIBM[name](a, b).astype(np.float64)


def total_key(x):
    """f64::total_cmp's key: the bit pattern as i64, the low 63 bits flipped for negative values."""
    b = np.ascontiguousarray(x, np.float64).view(np.int64)
    return b ^ ((b >> 63).view(np.uint64) >> np.uint64(1)).view(np.int64)


def _arith(op, a, b):
    with np.errstate(all="ignore"):
        if op == 0:
            return a + b
        if op == 1:
            return a - b
        if op == 2:
            return a * b
        if op == 3:
            return a / b
    return _libm_call(("fmod", "pow", "atan2")[op - 4], a, b)


def _cmp(op, a, b):
    ka, kb = total_key(a), total_key(b)
    return {7: ka == kb, 8: ka != kb, 9: ka > kb, 10: ka < kb, 11: ka >= kb, 12: ka <= kb}[op]


def _bits(valid_words, T):
    if T == 0:
        return np.zeros((valid_words.shape[0], 0), bool)
    b = np.unpackbits(np.ascontiguousarray(valid_words, np.uint32).view(np.uint8), axis=1, bitorder="little")
    return b[:, :T].astype(bool)


def _words(ok):
    rows, T = ok.shape
    Tw = (T + 31) // 32
    padded = np.zeros((rows, Tw * 32), np.uint8)
    padded[:, :T] = ok
    return np.packbits(padded, axis=1, bitorder="little").view(np.uint32).reshape(rows, Tw).copy()


def _cells(op, return_bool, x, y, vec, ok):
    """x op y on cells of joint validity ok; vec = the vector operand (what a filter keeps)."""
    op = _op_id(op)
    if op < _EQ:
        out = _arith(op, x, y)
        keep = ok
    else:
        c = _cmp(op, x, y)
        if return_bool:
            out, keep = np.where(c, 1.0, 0.0), ok
        else:
            out, keep = vec, ok & c
    return np.where(keep, out, 0.0), _words(keep)


def binary_op(op, lhs, lhs_valid, lhs_row, rhs, rhs_valid, rhs_row, return_bool=False):
    """Dense: lhs[lhs_row[p]] op rhs[rhs_row[p]] -> (out [P x T], valid words [P x Tw])."""
    lhs, rhs = np.asarray(lhs, np.float64), np.asarray(rhs, np.float64)
    lr, rr = np.asarray(lhs_row, np.int64), np.asarray(rhs_row, np.int64)
    T = lhs.shape[1]
    x, y = lhs[lr].reshape(lr.size, T), rhs[rr].reshape(rr.size, T)
    Tw = (T + 31) // 32
    ok = _bits(np.asarray(lhs_valid, np.uint32)[lr].reshape(lr.size, Tw), T) & \
        _bits(np.asarray(rhs_valid, np.uint32)[rr].reshape(rr.size, Tw), T)
    return _cells(op, return_bool, x, y, x, ok)


def scalar_op(op, scalar, vals, valid, scalar_on_left=False, return_bool=False):
    """Dense: `vals op scalar` (or `scalar op vals`) -> (out [S x T], valid words [S x Tw])."""
    vals = np.asarray(vals, np.float64)
    s = np.full(vals.shape, float(scalar))
    ok = _bits(np.asarray(valid, np.uint32), vals.shape[1])
    x, y = (s, vals) if scalar_on_left else (vals, s)
    return _cells(op, return_bool, x, y, vals, ok)


def binary_value(op, a, b, return_bool=False):
    """One cell `a op b` -> value, or None when a filtering comparison drops it."""
    out, ov = scalar_op(op, b, np.array([[a]], np.float64), np.array([[1]], np.uint32), return_bool=return_bool)
    return float(out[0, 0]) if ov[0, 0] & 1 else None


def binary_key_columns(lhs_tags, rhs_tags, on=None, ignoring=None):
    """Join key of a vector-vector operator (planner.rs:696-729): the rhs context's tag columns, intersected with `on` /
    without `ignoring`; none when either side has no tags.  A key column the lhs lacks is a planning error."""
    if not lhs_tags or not rhs_tags:
        return []
    keys = [t for t in rhs_tags if (on is None or t in on) and (ignoring is None or t not in ignoring)]
    for k in keys:
        if k not in lhs_tags:
            raise KeyError(f"No field named {k}")
    return keys


def binary_rows(lhs, rhs, op, return_bool=False, on=None, ignoring=None, label_side="rhs"):
    """Row-literal `lhs op rhs`.  lhs / rhs: (tag names, rows) with rows [(tag values..., ts, value)].
    -> (tag names, rows) in lhs row order, then the order of the matching rhs rows.  Output tags: label_side's for a
    projection, the lhs's for a filter."""
    (ltags, lrows), (rtags, rrows) = lhs, rhs
    keys = binary_key_columns(ltags, rtags, on, ignoring)
    li = [ltags.index(k) for k in keys]
    ri = [rtags.index(k) for k in keys]
    table = {}
    for r in rrows:
        table.setdefault((tuple(r[i] for i in ri), r[-2]), []).append(r)
    is_filter = _op_id(op) >= _EQ and not return_bool
    from_lhs = is_filter or label_side == "lhs"
    out = []
    for l in lrows:
        for r in table.get((tuple(l[i] for i in li), l[-2]), []):
            v = binary_value(op, l[-1], r[-1], return_bool)
            if v is None:
                continue
            side = l if from_lhs else r
            out.append(tuple(side[:-2]) + (l[-2], v))
    return (list(ltags) if from_lhs else list(rtags)), out


def scalar_value(op, scalar, v, scalar_on_left=False, return_bool=False):
    """One cell `v op scalar` (or `scalar op v`) -> value, or None when a filtering comparison drops it; a filter keeps
    the vector's value on either side."""
    out, ov = scalar_op(op, scalar, np.array([[v]], np.float64), np.array([[1]], np.uint32), scalar_on_left, return_bool)
    return float(out[0, 0]) if ov[0, 0] & 1 else None


def scalar_rows(rows, op, scalar, scalar_on_left=False, return_bool=False):
    """Row-literal `rows op scalar` (or `scalar op rows`): a projection, or a filter keeping the vector's value."""
    out = []
    for r in rows:
        v = scalar_value(op, scalar, r[-1], scalar_on_left, return_bool)
        if v is not None:
            out.append(tuple(r[:-1]) + (v,))
    return out


def binary_pairs(lhs_tags, lhs_labels, rhs_tags, rhs_labels, on=None, ignoring=None):
    """Series matched on the key tuple.  lhs_labels / rhs_labels: one label tuple per series.
    -> (lhs_row, rhs_row) uint32 arrays, lhs series order then rhs series order."""
    keys = binary_key_columns(lhs_tags, rhs_tags, on, ignoring)
    li = [lhs_tags.index(k) for k in keys]
    ri = [rhs_tags.index(k) for k in keys]
    table = {}
    for s, lab in enumerate(rhs_labels):
        table.setdefault(tuple(lab[i] for i in ri), []).append(s)
    lrow, rrow = [], []
    for s, lab in enumerate(lhs_labels):
        for m in table.get(tuple(lab[i] for i in li), []):
            lrow.append(s)
            rrow.append(m)
    return np.array(lrow, np.uint32), np.array(rrow, np.uint32)
