"""CPU restatement of the PromQL instant-vector math functions and scalar() (test infrastructure; the product never
imports it).

Functions (src/query/src/promql/planner.rs:2368-2413, then `Filter(value IS NOT NULL)` at :1063): element-wise over the
value column; a function of a non-null f64 is never null, so validity is unchanged and invalid cells hold 0.0, like
every dense result of the library.
  * abs ceil floor sqrt: Rust's f64 methods (IEEE, exact); numpy computes the same.
  * exp ln log2 log10 and the trigonometric / hyperbolic functions: Rust's std calls glibc's libm on Linux, bound here
    through ctypes (numpy's own exp / sin are not glibc's).  asinh / acosh / atanh are the exception: Rust's std
    (library/std/src/f64.rs) does not call libm for them but composes ln_1p / ln / sqrt / hypot (acosh:
    `(x + (x - 1).sqrt() * (x + 1).sqrt()).ln()`, NaN below 1; atanh: `0.5 * ((2x) / (1 - x)).ln_1p()`), which can
    differ from glibc's in the last bits.  The restatement here is glibc's for all sixteen, and the device's ulp bound
    is stated against it (DESIGN.md section 2).
  * round(v, n): prom_round, src/promql/src/functions/round.rs:52-105: `n == 0 ? v.round() : (v / n).round() * n`,
    round half away from zero.
  * deg / rad: one multiplication by the f64 constant 180/π (Rust's to_degrees) / π/180 (to_radians).
  * sgn: DataFusion's signum: 0.0 for ±0, NaN for NaN, else ±1.0.
  * clamp(v, lo, hi): `v < lo ? lo : v > hi ? hi : v` (clamp.rs:75-224); clamp_min(v, lo) takes hi = f64::MAX,
    clamp_max(v, hi) takes lo = -f64::MAX (ScalarValue::max / min of Float64); lo > hi is an error.

scalar(v) (ScalarCalculateStream, src/promql/src/extension_plan/scalar_calculate.rs:532-637) in two forms:
  * `scalar_calculate_rows` — row-literal: batches of (labels..., ts, value) rows through update_batch / poll_next,
    NULL labels as None, including the way a NULL label is compared (as None against the "" recorded for it);
  * `scalar_calculate` — dense: one series key per grid row (NO_KEY for a tuple with a NULL), what the kernels do.
"""
import ctypes as C
import sys

import numpy as np

IFNS = {"abs": 0, "ceil": 1, "floor": 2, "sqrt": 3, "exp": 4, "ln": 5, "log2": 6, "log10": 7, "sin": 8, "cos": 9,
        "tan": 10, "asin": 11, "acos": 12, "atan": 13, "sinh": 14, "cosh": 15, "tanh": 16, "asinh": 17, "acosh": 18,
        "atanh": 19, "round": 20, "deg": 21, "rad": 22, "sgn": 23, "clamp": 24, "clamp_min": 25, "clamp_max": 26}
# the functions computed by libm (the rest are exact)
TRANSCENDENTAL = ("exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh", "tanh",
                  "asinh", "acosh", "atanh")
NO_KEY = 0xFFFFFFFF
F64_MAX = sys.float_info.max
DEG = 57.29577951308232      # 180.0 / π in f64
RAD = 0.017453292519943295   # π / 180.0 in f64

_libm = C.CDLL("libm.so.6")
_LIBM = {}
for _fn, _c in {"exp": "exp", "ln": "log", "log2": "log2", "log10": "log10", "sin": "sin", "cos": "cos", "tan": "tan",
                "asin": "asin", "acos": "acos", "atan": "atan", "sinh": "sinh", "cosh": "cosh", "tanh": "tanh",
                "asinh": "asinh", "acosh": "acosh", "atanh": "atanh"}.items():
    _f = getattr(_libm, _c)
    _f.restype = C.c_double
    _f.argtypes = [C.c_double]
    _LIBM[_fn] = np.frompyfunc(_f, 1, 1)


def fn_name(fn):
    if isinstance(fn, str):
        return fn
    return {v: k for k, v in IFNS.items()}[int(fn)]


def round_half_away(x):
    """f64::round: half away from zero, -0.0 and ±inf / NaN kept."""
    x = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        r = np.trunc(x)
        up = np.abs(x - r) >= 0.5
    return np.where(up, r + np.copysign(1.0, x), r)


def clamp_bounds(fn, arg0=0.0, arg1=0.0):
    """(lo, hi) of clamp / clamp_min / clamp_max; ValueError like the reference's `min '..' > max '..'`."""
    fn = fn_name(fn)
    lo, hi = {"clamp": (arg0, arg1), "clamp_min": (arg0, F64_MAX), "clamp_max": (-F64_MAX, arg0)}[fn]
    if lo > hi:
        raise ValueError(f"min '{lo}' > max '{hi}'")
    return lo, hi


def apply(fn, x, arg0=0.0, arg1=0.0):
    """fn over an array of values (every cell valid)."""
    fn = fn_name(fn)
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        if fn == "abs":
            return np.abs(x)
        if fn == "ceil":
            return np.ceil(x)
        if fn == "floor":
            return np.floor(x)
        if fn == "sqrt":
            return np.sqrt(x)
        if fn in _LIBM:
            return _LIBM[fn](x).astype(np.float64) if x.size else np.zeros(x.shape)
        if fn == "round":
            return round_half_away(x) if arg0 == 0.0 else round_half_away(x / arg0) * arg0
        if fn == "deg":
            return x * DEG
        if fn == "rad":
            return x * RAD
        if fn == "sgn":
            return np.where(x == 0.0, 0.0, np.where(np.isnan(x), x, np.where(x < 0.0, -1.0, 1.0)))
        lo, hi = clamp_bounds(fn, arg0, arg1)
        return np.where(x < lo, lo, np.where(x > hi, hi, x))


def _bits(valid_words, T):
    w = np.ascontiguousarray(valid_words, np.uint32).reshape(-1, (T + 31) // 32) if T else np.zeros((0, 0), np.uint32)
    return np.unpackbits(w.view(np.uint8), axis=1, bitorder="little")[:, :T].astype(bool)


def _words(ok):
    ok = np.asarray(ok, bool)
    rows, T = ok.shape
    pad = np.zeros((rows, ((T + 31) // 32) * 32), np.uint8)
    pad[:, :T] = ok
    return np.packbits(pad, axis=1, bitorder="little").view(np.uint32).reshape(rows, (T + 31) // 32)


def instant_fn(fn, vals, valid_words, arg0=0.0, arg1=0.0):
    """Dense form: (out [rows x T], valid words unchanged); fn(v) where valid, 0.0 elsewhere."""
    vals = np.asarray(vals, np.float64)
    ok = _bits(valid_words, vals.shape[1])
    out = np.where(ok, apply(fn, vals, arg0, arg1), 0.0)
    return out, np.array(valid_words, np.uint32, copy=True)


# ---- scalar() ------------------------------------------------------------------------------------------------------
def scalar_calculate_rows(batches, n_tags, start, end, interval):
    """Row-literal ScalarCalculateStream.  `batches`: lists of rows (labels[n_tags]..., ts, value) as the input stream
    delivers them, a NULL label as None.  -> [(ts, value)] of the output batch."""
    have_multi, kept, tag_value = False, [], None
    for batch in batches:
        if have_multi or not batch:
            continue
        if n_tags == 0:
            kept.extend(batch)
            continue
        cols = [[row[i] for row in batch] for i in range(n_tags)]

        def all_same(val, array):
            if val is not None:
                return all(s == val for s in array)
            # array.value(0) of a NULL slot is "" (the empty string its offsets describe)
            v0 = array[0] if array[0] is not None else ""
            return all(s == v0 for s in array[1:])

        if tag_value is not None:
            same = all(all_same(v, col) for v, col in zip(tag_value, cols))
        else:
            tag_value = [col[0] if col[0] is not None else "" for col in cols]
            same = all([all_same(None, col) for col in cols])
        if same:
            kept.extend(batch)
        else:
            have_multi = True
    if kept and not have_multi:
        return [(int(r[-2]), r[-1]) for r in kept]
    return [(int(t), float("nan")) for t in range(start, end + 1, interval)]


def scalar_calculate(vals, valid_words, row_key):
    """Dense scalar(): (out [T], words [Tw]).  One series when every live row carries one key (a NO_KEY row: only with
    a single cell); NaN at every step otherwise.  ValueError for two rows of the key at one step."""
    vals = np.asarray(vals, np.float64)
    T = vals.shape[1]
    ok = _bits(valid_words, T)
    key = np.asarray(row_key, np.uint32)
    live = ok.any(axis=1)
    keys = set(key[live].tolist())
    null_cells = int(ok[live & (key == NO_KEY)].sum())
    one = len(keys) == 1 and (NO_KEY not in keys or null_cells == 1)
    if not one:
        return np.full(T, np.nan), _words(np.ones((1, T), bool))[0]
    rows = np.flatnonzero(live)
    if (ok[rows].sum(axis=0) > 1).any():
        raise ValueError("two rows of one series have a cell at the same step")
    cell = ok[rows].any(axis=0)
    out = np.zeros(T)
    for r in rows:
        out = np.where(ok[r], vals[r], out)
    return np.where(cell, out, 0.0), _words(cell[None, :])[0]
