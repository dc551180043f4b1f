"""Layout edge cases of the dense-grid kernels and plain references of each, written from the kernel headers' contracts
(test infrastructure; the product never imports it).

The kernels read a dense [rows x T] grid of Float64 cells and its validity words (bit k % 32 of word k / 32 of a row)
and write a grid back: K7 binary_op / count_valid (b2p_binary.cuh), K8 set operators (b2p_setop.cuh), K9 instant_fn,
scalar() and i64_to_f64 (b2p_instant.cuh), K13 the subquery count / scatter (b2p_subquery.cuh), K15 absent()
(b2p_absent.cuh), K18 the multi-field validity conjunction (b2p_fields.cuh) and K19 the step functions (b2p_time.cuh).
What can go wrong there is the work decomposition, not the arithmetic, so the cases here are layouts:
  * T around the 32-step words and the 64-step units of the 128-bit (VEC) variants: T mod 64 in {0, 2, 30, 32, 34, 62},
    T mod 32 of every kind for the scalar route;
  * validity words all, none, holes, one step only, the last step only, and junk bits past T in every row's last word
    (undefined by contract: every kernel but K9 must ignore them);
  * invalid cells holding NaN payloads of both signs and ±inf (a kept cell is a bit copy, an invalid one reads 0.0).
Each case records the classes its data actually hit (`classes`), so the tests can assert that every class ran.

The calendar reference `calendar` does not restate the kernel's civil-from-days algorithm: it asks Python's datetime
for years 1 to 9999 and walks 400-year cycles and then year and month lengths from 0001-01-01 for the rest of the
+-262143-year range.
"""
import ctypes as C
import datetime
from fractions import Fraction

import numpy as np

T_LIST = [1, 2, 31, 32, 33, 62, 63, 64, 65, 66, 94, 95, 96, 97, 98, 126, 128, 130, 255, 256, 257, 1000]
PATTERNS = ["all", "none", "holes", "one", "last"]
NO_KEY = 0xFFFFFFFF
MAX_YEAR = 262143
MS_PER_DAY = 86_400_000

# what invalid cells hold: quiet NaNs with payloads of both signs, a signalling-pattern NaN, and both infinities
INVALID_FILL = np.array([0x7FF8000000000001, 0xFFF8DEADBEEF0000, 0x7FF0000000000123, 0xFFF4000000000000,
                         0x7FF0000000000000, 0xFFF0000000000000], np.uint64).view(np.float64)
# what valid cells hold: signed zeros, subnormals, ±inf, NaN payloads of both signs and ordinary numbers
VALID_FILL = np.concatenate([
    np.array([0x8000000000000000, 0x0000000000000000, 0x0000000000000001, 0x800FFFFFFFFFFFFF, 0x7FF0000000000000,
              0xFFF0000000000000, 0x7FF8000000000456, 0xFFF8000000000789], np.uint64).view(np.float64),
    np.array([1.0, -1.0, 2.5, -3.75, 0.1, 1e300, -1e-300, 123456.789, 2.0 ** 53 + 2, -7.0])])

_libm = C.CDLL("libm.so.6")
_LIBM = {}
for _name in ("pow", "atan2", "fmod"):
    _f = getattr(_libm, _name)
    _f.restype, _f.argtypes = C.c_double, [C.c_double, C.c_double]
    _LIBM[_name] = np.frompyfunc(_f, 2, 1)


# ---- validity words ----------------------------------------------------------------------------------------------------
def words_of(ok):
    """bool [rows, T] -> u32 words [rows, Tw], bits past T zero"""
    ok = np.asarray(ok, bool)
    rows, T = ok.shape
    Tw = (T + 31) // 32
    pad = np.zeros((rows, Tw * 32), np.uint8)
    pad[:, :T] = ok
    return np.packbits(pad, axis=1, bitorder="little").view(np.uint32).reshape(rows, Tw).copy()


def ok_of(words, T):
    """u32 words [rows, Tw] -> bool [rows, T] (bits past T dropped)"""
    w = np.ascontiguousarray(words, np.uint32).reshape(-1, (T + 31) // 32)
    return np.unpackbits(w.view(np.uint8), axis=1, bitorder="little")[:, :T].astype(bool)


def past_t_mask(T):
    """the bits of a row's last word that are not steps (0 when T is a multiple of 32)"""
    tail = T % 32
    return 0 if tail == 0 else (0xFFFFFFFF ^ ((1 << tail) - 1))


def add_junk(words, T, rng):
    """sets random bits past T, at least one, in every row's last word (a no-op when T is a multiple of 32)"""
    words = np.array(words, np.uint32, copy=True)
    m = past_t_mask(T)
    if m and words.size:
        junk = rng.integers(0, 2 ** 32, words.shape[0], dtype=np.uint64).astype(np.uint32) & np.uint32(m)
        junk |= np.uint32(1 << 31)
        words[:, -1] |= junk
    return words


def pattern_ok(rng, rows, T, pattern):
    ok = np.zeros((rows, T), bool)
    if pattern == "all":
        ok[:] = True
    elif pattern == "holes":
        ok = rng.random((rows, T)) < 0.55
        ok[:, 0], ok[:, -1] = True, False  # (a hole at the last step, whatever the draw)
        if T > 2:
            ok[:, T // 2] = False
    elif pattern == "one":
        ok[np.arange(rows), rng.integers(0, T, rows)] = True
    elif pattern == "last":
        ok[:, T - 1] = True
    return ok


def grid(rng, rows, T, pattern, junk=True):
    """A grid case: vals [rows, T], ok [rows, T], valid words (with junk past T when asked) and the classes it hit."""
    ok = pattern_ok(rng, rows, T, pattern)
    vals = VALID_FILL[rng.integers(0, VALID_FILL.size, (rows, T))]
    bad = INVALID_FILL[np.arange(rows * T).reshape(rows, T) % INVALID_FILL.size]
    vals = np.where(ok, vals, bad)
    valid = words_of(ok)
    if junk:
        valid = add_junk(valid, T, rng)
    return {"vals": vals, "ok": ok, "valid": valid, "T": T, "rows": rows, "pattern": pattern,
            "classes": data_classes(vals, ok, valid, T)}


def data_classes(vals, ok, valid, T):
    """the classes a grid's data actually hits"""
    c = set()
    rows = ok.shape[0]
    if rows == 0:
        return c
    if ok.all():
        c.add("valid:all")
    if not ok.any():
        c.add("valid:none")
    if ok.any() and not ok.all() and (ok.sum(axis=1) > 1).any():
        c.add("valid:holes")
    if (ok.sum(axis=1) == 1).all():
        c.add("valid:one")
        if ok[:, T - 1].all():
            c.add("valid:last")
    m = past_t_mask(T)
    if m and (np.asarray(valid, np.uint32)[:, -1] & np.uint32(m)).all():
        c.add("junk_past_T")
    b = np.ascontiguousarray(vals).view(np.uint64)[~ok]
    nan = (b & np.uint64(0x7FF0000000000000)) == np.uint64(0x7FF0000000000000)
    frac = b & np.uint64(0x000FFFFFFFFFFFFF)
    sign = b >> np.uint64(63)
    if (nan & (frac != 0) & (sign == 0)).any() and (nan & (frac != 0) & (sign == 1)).any():
        c.add("invalid:nan_both_signs")
    if (nan & (frac == 0) & (sign == 0)).any() and (nan & (frac == 0) & (sign == 1)).any():
        c.add("invalid:inf_both_signs")
    c.add(f"T={T}")
    return c


def route(T, aligned=True):
    """the route a K7 / K8 / K9 call takes: the 128-bit variant needs T even and 16-byte aligned pointers"""
    return "vec" if T % 2 == 0 and aligned else ("scalar_odd" if T % 2 else "scalar_even_unaligned")


# ---- grid-stride sizes ---------------------------------------------------------------------------------------------------
def capped_ctas(sms, units, per_block, per_sm):
    """capped_grid (b2p_runtime.cuh)"""
    return min(-(-units // per_block), sms * per_sm)


def rows_past_warp_grid(sms, T, steps):
    """rows at which K7 / K8's copy / K9 (8 warps per CTA, 16 CTAs per SM) have more (row, tile) units than warps"""
    return sms * 16 * 8 // (-(-T // steps)) + 3


def step_fn_geometry(sms, T, rows):
    """K19's launch (step_fn_run): W, rows per pass, gx, gy and whether the blockIdx.y loop takes a second pass"""
    W = 256 if T >= 256 else (max(T, 1) if T < 32 else -(-T // 32) * 32)
    rpp = 256 // W
    gx = -(-T // W)
    cap = max(1, sms * 16 // gx)
    gy = min(-(-rows // rpp), cap, 65535)
    return {"W": W, "rpp": rpp, "gx": gx, "gy": gy, "second_pass": rows > gy * rpp, "idle": 256 - rpp * W}


def step_fn_classes(sms, T, rows):
    g = step_fn_geometry(sms, T, rows)
    c = set()
    if T < 32 and g["rpp"] > 1 and rows > 1:
        c.add("k19:rows_per_warp")
    if 32 <= T < 256 and g["W"] in (96, 160, 192, 224):
        c.add(f"k19:W={g['W']}")
    if g["second_pass"]:
        c.add("k19:second_y_pass")
    return c


def absent_regime(sms, rows, T):
    """K15's OR pass (absent_run / absent_or_kernel): 'shared' (Tw < 256), 'rows' (256 <= Tw <= P) or 'columns'
    (Tw > P, the per-thread column walk), with P the grid's threads"""
    Tw = (T + 31) // 32
    P = 256 * max(1, capped_ctas(sms, rows * Tw, 256 * 4, 8))
    if Tw < 256:
        return "shared"
    return "rows" if Tw <= P else "columns"


# ---- references -----------------------------------------------------------------------------------------------------------
def total_key(x):
    b = np.ascontiguousarray(x, np.float64).view(np.int64)
    return b ^ ((b >> 63).view(np.uint64) >> np.uint64(1)).view(np.int64)


ARITH = {"+": np.add, "-": np.subtract, "*": np.multiply, "/": np.divide}
CMP = {"==": np.equal, "!=": np.not_equal, ">": np.greater, "<": np.less, ">=": np.greater_equal, "<=": np.less_equal}


def binary_ref(op, x, y, ok, vec, return_bool=False):
    """K7 on operand grids x (lhs) / y (rhs) of joint validity ok; vec is the vector operand (what a filter keeps).
    -> (out, words): arithmetic and bool keep ok, a filter keeps ok & (x op y) on the f64 total order; invalid cells
    hold 0.0 and no bit past T is set."""
    x, y = np.broadcast_arrays(np.asarray(x, np.float64), np.asarray(y, np.float64))
    with np.errstate(all="ignore"):
        if op in ARITH:
            val, keep = ARITH[op](x, y), ok
        elif op in ("%", "^", "atan2"):
            f = _LIBM[{"%": "fmod", "^": "pow", "atan2": "atan2"}[op]]
            val = f(x, y).astype(np.float64) if x.size else np.zeros(x.shape)
            keep = ok
        else:
            c = CMP[op](total_key(x), total_key(y))
            val, keep = (np.where(c, 1.0, 0.0), ok) if return_bool else (np.asarray(vec, np.float64), ok & c)
    return np.where(keep, val, 0.0), words_of(keep)


def setop_ref(op, lhs, lok, lkey, rhs, rok, rkey, n_keys):
    """K8 from b2p_setop.cuh's contract: and = lv & mask_rhs[key] (no key: nothing); unless = lv & ~mask_rhs[key] (no
    key: lv); or = the lhs rows, then each rhs row's rv & ~(mask_lhs[key] | the rv of earlier rhs rows of its key).  A
    key out of range (other than NO_KEY) gives an invalid row.  Values are bit copies; invalid cells 0.0."""
    T = lok.shape[1]

    def mask(ok, keys):
        m = np.zeros((n_keys, T), bool)
        for r, k in enumerate(keys):
            if k < n_keys:
                m[k] |= ok[r]
        return m

    def rows_ok(ok, keys, f):
        out = np.zeros_like(ok)
        for r, k in enumerate(keys):
            out[r] = f(r, int(k))
        return out

    if op in ("and", "unless"):
        m = mask(rok, rkey)
        out = rows_ok(lok, lkey, lambda r, k: (lok[r] if op == "unless" else False) if k == NO_KEY else
                      (False if k >= n_keys else lok[r] & (m[k] if op == "and" else ~m[k])))
        return np.where(out, lhs, 0.0), words_of(out)
    running = mask(lok, lkey)
    lout = rows_ok(lok, lkey, lambda r, k: lok[r] if (k == NO_KEY or k < n_keys) else False)
    rout = np.zeros_like(rok)
    for r, k in enumerate(rkey):
        k = int(k)
        if k == NO_KEY:
            rout[r] = rok[r]
        elif k < n_keys:
            rout[r] = rok[r] & ~running[k]
            running[k] |= rok[r]
    ok = np.concatenate([lout, rout])
    return np.where(ok, np.concatenate([lhs, rhs]), 0.0), words_of(ok)


# K9's exact functions (b2p_instant.cuh): value -> value, NaN handling as documented there
def _neg(x):
    return (np.ascontiguousarray(x, np.float64).view(np.uint64) ^ np.uint64(1 << 63)).view(np.float64)


def _sgn(x):
    with np.errstate(invalid="ignore"):
        return np.where(x == 0.0, 0.0, np.where(np.isnan(x), x, np.where(x < 0.0, -1.0, 1.0)))


def _clamp(x, lo, hi):
    with np.errstate(invalid="ignore"):
        return np.where(x < lo, lo, np.where(x > hi, hi, x))


INSTANT_FNS = {  # name -> (arg0, arg1, value function, whether a NaN keeps its bits)
    "neg": (0.0, 0.0, _neg, True),
    "abs": (0.0, 0.0, lambda x: (np.ascontiguousarray(x).view(np.uint64) & np.uint64((1 << 63) - 1)).view(np.float64),
            True),
    "sgn": (0.0, 0.0, _sgn, True),
    "clamp": (-2.0, 3.0, lambda x: _clamp(x, -2.0, 3.0), True),
    "floor": (0.0, 0.0, np.floor, False),
}


def instant_fn_ref(fn, vals, ok):
    """K9: fn at valid cells, 0.0 elsewhere; validity words unchanged (bits past T included: copied, undefined)"""
    _, _, f, _ = INSTANT_FNS[fn]
    with np.errstate(all="ignore"):
        return np.where(ok, f(np.asarray(vals, np.float64)), 0.0)


def scalar_ref(vals, ok, key):
    """scalar() from b2p_instant.cuh's contract: live rows (a cell at a step < T) of one key -> that series' cells;
    a NO_KEY row counts as a series only while all NO_KEY rows hold one cell together; else NaN at every step.
    -> (out [T], words [Tw], overlap): overlap = two live rows of the one key at one step (B2P_E_INVALID)."""
    T = ok.shape[1]
    live = ok.any(axis=1)
    keys = {int(k) for k in np.asarray(key)[live]}
    one = len(keys) == 1 and (NO_KEY not in keys or int(ok[live].sum()) == 1)
    if not one:
        return np.full(T, np.nan), words_of(np.ones((1, T), bool))[0], False
    rows = np.flatnonzero(live)
    overlap = bool((ok[rows].sum(axis=0) > 1).any())
    out, cell = np.zeros(T), np.zeros(T, bool)
    for r in rows:
        out = np.where(ok[r] & ~cell, vals[r], out)
        cell |= ok[r]
    return out, words_of(cell[None, :])[0], overlap


def absent_ref(ok):
    """K15: 1.0 and a set bit at the steps where no row has a cell, 0.0 and a clear bit elsewhere"""
    gone = ~np.asarray(ok, bool).any(axis=0)
    return np.where(gone, 1.0, 0.0), words_of(gone[None, :])[0]


def count_valid_ref(cnt):
    """count_valid_kernel: bit k of a row iff cnt != 0, no bit past T"""
    return words_of(np.asarray(cnt) != 0)


def subquery_rows(vals, ok, start, step):
    """K13's contract: the sample rows of a child grid on the inner steps start + k * step — every valid cell k < T
    of a row, in step order, as (ts, value bits) — with row offsets.  -> (ts i64, val f64, offsets u64)"""
    rows, T = ok.shape
    k = np.broadcast_to(np.arange(T, dtype=np.int64), (rows, T))
    ts = (start + k * step)[ok]
    val = np.ascontiguousarray(vals, np.float64)[ok]
    offsets = np.concatenate([[0], np.cumsum(ok.sum(axis=1))]).astype(np.uint64)
    return ts.astype(np.int64), val, offsets


def i64_to_f64_ref(v):
    """(double)i64 rounded to nearest, ties to even: Python's float(int) is correctly rounded"""
    return np.array([float(int(x)) for x in np.asarray(v, np.int64)], np.float64)


I64_EDGES = np.array([2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 3, -(2 ** 53 + 1), 2 ** 54 + 1, 2 ** 54 + 2,
                      2 ** 54 + 3, 2 ** 54 + 6, 2 ** 54 + 10, -(2 ** 54 + 2), -(2 ** 54 + 6), 2 ** 63 - 1, -(2 ** 63),
                      -(2 ** 63) + 1, 2 ** 62 + 2 ** 9, 2 ** 62 + 3 * 2 ** 9, 0, -1, 1], np.int64)


# ---- calendar ----------------------------------------------------------------------------------------------------------
def _leap(y):
    return y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)


_MONTH_DAYS = [31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]
_ORDINAL_1970 = datetime.date(1970, 1, 1).toordinal()  # 0001-01-01 is ordinal 1


def civil_walk(ordinal):
    """(year, month, day, day of year) of a proleptic Gregorian day number (0001-01-01 = 1), by 400-year cycles of
    146097 days and then year and month lengths: no closed-form era arithmetic"""
    y, o = 1, ordinal
    if o < 1:
        n = (-o) // 146097 + 1
        y, o = y - 400 * n, o + 146097 * n
    if o > 146097:
        n = (o - 1) // 146097
        y, o = y + 400 * n, o - 146097 * n
    while o > (366 if _leap(y) else 365):
        o -= 366 if _leap(y) else 365
        y += 1
    doy, m = o, 1
    for m0, n in enumerate(_MONTH_DAYS):
        n += 1 if (m0 == 1 and _leap(y)) else 0
        if o <= n:
            m = m0 + 1
            break
        o -= n
    return y, m, o, doy


def civil_date(ordinal):
    """datetime for years 1 to 9999, the walk for the rest"""
    if 1 <= ordinal <= datetime.date.max.toordinal():
        d = datetime.date.fromordinal(ordinal)
        return d.year, d.month, d.day, d.timetuple().tm_yday
    return civil_walk(ordinal)


def calendar(part, ts):
    """K19's value of one step: time() is (double)ts / 1000.0; the calendar parts of the UTC millisecond timestamp
    ts, or None when its year is outside [-262143, 262143] (the kernel refuses it)"""
    ts = int(ts)
    if part == "time":
        return float(ts) / 1000.0
    days, ms = divmod(ts, MS_PER_DAY)
    ordinal = days + _ORDINAL_1970
    y, m, d, doy = civil_date(ordinal)
    if not -MAX_YEAR <= y <= MAX_YEAR:
        return None
    v = {"minute": ms // 60_000 % 60, "hour": ms // 3_600_000, "day_of_month": d, "day_of_week": ordinal % 7,
         "day_of_year": doy, "month": m, "year": y,
         "days_in_month": _MONTH_DAYS[m - 1] + (1 if m == 2 and _leap(y) else 0)}[part]
    return float(v)


def ms_of(y, m, d):
    """milliseconds since the epoch of midnight (UTC) of the proleptic Gregorian date (y, m, d), any year"""
    days = sum(366 if _leap(x) else 365 for x in range(1, y)) if 1 <= y <= 9999 else None
    if days is None:  # the walk's inverse over whole 400-year cycles
        n = (y - 1) // 400
        yy = y - 400 * n
        days = n * 146097 + sum(366 if _leap(x) else 365 for x in range(1, yy))
    days += sum(_MONTH_DAYS[:m - 1]) + (1 if m > 2 and _leap(y) else 0) + d - 1
    return (days + 1 - _ORDINAL_1970) * MS_PER_DAY


def calendar_steps():
    """K19's eval timestamps: the last millisecond before and the first after every midnight that ends a month of a
    year, 29 February of leap years 2000, 2400 and -400 (with 1 March of 1900 and 2100, which have none), both ends of
    the year range, and the epoch.  -> int64 [n]"""
    ts = [0, -1, 1]
    for y in (1970, 2000, 2023, 2024, -1, 0, 1, 9999, -262143, 262143):
        for m in range(1, 13):
            nm, ny = (m % 12) + 1, y + (m == 12)
            t = ms_of(ny, nm, 1)
            ts += [t - 1, t]
    for y in (1900, 2000, 2100, 2400, -400, -100, -4):
        feb28 = ms_of(y, 2, 28)
        ts += [feb28 + MS_PER_DAY - 1, feb28 + MS_PER_DAY, feb28 + 2 * MS_PER_DAY - 1]
    ts += [ms_of(-MAX_YEAR, 1, 1), ms_of(MAX_YEAR + 1, 1, 1) - 1]
    return np.array(sorted(t for t in set(ts) if calendar("year", t) is not None), np.int64)


def calendar_edge_steps():
    """the first millisecond past each end of the year range (refused) and the last inside it"""
    lo, hi = ms_of(-MAX_YEAR, 1, 1), ms_of(MAX_YEAR + 1, 1, 1)
    return {"in": np.array([lo, hi - 1], np.int64), "out": np.array([lo - 1, hi], np.int64)}


TIME_EDGES = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, np.iinfo(np.int64).min + 1,
                       np.iinfo(np.int64).max - 1, 2 ** 53 + 1, -(2 ** 53) - 1, 1, -1, 999, -999], np.int64)


def time_correctly_rounded(ts):
    """(double)ts / 1000.0 as one round-to-nearest conversion and one correctly rounded division, checked exactly"""
    x = float(int(ts))
    want = float(Fraction(x) / 1000)
    return want == x / 1000.0


# ---- cases ---------------------------------------------------------------------------------------------------------------
def grid_cases(seed=0x6D1D, rows=4):
    """one grid per (T, pattern), every one with junk past T"""
    rng = np.random.default_rng(seed)
    return [grid(rng, rows, T, p) for T in T_LIST for p in PATTERNS]


def scalar_cases(seed=0x5CA1, T_list=(1, 33, 64, 97, 1000)):
    """scalar() layouts over four rows (keys are below the row count, as the kernel requires):
    -> [(name, vals, ok, valid, key, expect_overlap)]"""
    rng = np.random.default_rng(seed)
    out = []
    for T in T_list:
        base = VALID_FILL[rng.integers(0, VALID_FILL.size, (4, T))]
        ok = np.zeros((4, T), bool)
        ok[0, 0::3], ok[1, 1::3], ok[2, 2::3] = True, True, True  # one key over three rows at disjoint steps
        out.append(("one_key_disjoint", base, ok.copy(), np.array([1, 1, 1, 3], np.uint32), False))
        if T > 1:
            ok2 = ok.copy()
            ok2[1, 0] = True  # two rows of the key at step 0
            out.append(("one_key_overlap", base, ok2, np.array([1, 1, 1, 3], np.uint32), True))
        one = np.zeros((4, T), bool)
        one[2, T - 1] = True
        out.append(("no_key_one_cell", base, one, np.array([2, 2, NO_KEY, 3], np.uint32), False))
        two = one.copy()
        two[2, 0] = True
        if T > 1:
            out.append(("no_key_two_cells", base, two, np.array([2, 2, NO_KEY, 3], np.uint32), False))
        out.append(("two_keys", base, ok.copy(), np.array([1, 1, 2, 3], np.uint32), False))
    res = []
    for name, vals, ok, key, ov in out:
        bad = INVALID_FILL[np.arange(ok.size).reshape(ok.shape) % INVALID_FILL.size]
        v = np.where(ok, vals, bad)
        res.append((name, v, ok, add_junk(words_of(ok), ok.shape[1], rng), key, ov))
    return res


def all_classes(sms):
    """every class the GPU file runs, with the grid-stride and geometry classes computed for `sms` SMs"""
    c = set()
    for g in grid_cases():
        c |= g["classes"]
    for T in T_LIST:
        c.add(f"route:{route(T)}")
        if T % 2 == 0:
            c.add("route:scalar_even_unaligned")
    c |= {"inplace", "outofplace"}
    for T, rows in K19_SHAPES(sms):
        c |= step_fn_classes(sms, T, rows)
    for rows, T in ABSENT_SHAPES:
        c.add(f"k15:{absent_regime(sms, rows, T)}")
    c.add("k15:T=1_over_2^20_rows")
    for name, *_ in scalar_cases():
        c.add(f"scalar:{name}")
    return c


def K19_SHAPES(sms):
    """(T, rows): T < 32 with several rows per warp, W of 96, 160, 192 and 224, and row counts past gy x rows per
    pass so that the blockIdx.y loop takes a second pass"""
    shapes = [(1, 7), (5, 53), (31, 9), (65, 5), (129, 5), (161, 3), (193, 3), (255, 2)]
    for T in (1, 3, 96, 1000):
        g = step_fn_geometry(sms, T, 1)
        rows = min(max(1, sms * 16 // g["gx"]), 65535) * g["rpp"] + 3
        shapes.append((T, rows))
    return shapes


# (rows, T) of the K15 regimes: Tw < 256; Tw >= 256 read as whole rows; 1 to 3 rows with Tw above the grid's threads
ABSENT_SHAPES = [(5, 33), (4, 8190), (1, 64_000), (2, 96_001), (3, 200_000)]
