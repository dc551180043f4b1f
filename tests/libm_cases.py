"""Operands by class for the results this library takes from CUDA's libm — K9's transcendental functions (`exp ln log2
log10 sin cos tan asin acos atan sinh cosh tanh asinh acosh atanh`) and K7's `^` (pow) and `atan2` — and a correctly
rounded reference for them (test infrastructure only; the product never imports mpmath).

Uniformly drawn operands almost never land where a libm goes wrong, so every class here aims at one such place and
states a property that `tests/test_libm_cases.py` checks.  Every threshold and neighbour is derived with mpmath, none is
typed in.  A class is one of three kinds:
  exact      glibc is exact and the printed value is an integer or a short decimal: log2(2^k), log10(10^k), ln(1),
             exp(0), exp(±tiny), 2^k, 10^k, 3^k, x^2, x^0.5, x^1, x^-1.  `value` holds the exact result.
  threshold  ±3 ulps around an edge of the result's range: the largest finite exp / sinh / cosh / pow, the smallest
             normal and the smallest subnormal result of exp / pow.  The window straddles the edge, so the result's
             outcome (zero, subnormal, normal, inf) changes inside it.
  ill        an ill-conditioned region: logarithms near 1 and at subnormals, trigonometric arguments nearest kπ/2
             (and the worst case of the whole double range), tan near π/2, asin / acos / atanh near ±1, acosh near 1,
             odd functions below 2^-26, the switch points of tanh / sinh / asin / acos / atan, pow with a base within
             ulps of 1, a negative base or a subnormal base, and atan2's overflowing, underflowing, equal, signed-zero,
             subnormal and huge operand pairs.

`cases(seed)` -> a tuple of `Case`; the same seed gives the same operands.  `correctly_rounded(fn, x[, y])` is mpmath at
PREC (or more) bits, rounded to f64 by hand: to the nearest multiple of the quantum of the result's binade (2^-1074 for
subnormals, where `float(mpf)` would round twice), ties to even, and ±inf from f64::MAX + half an ulp up.  A binary
case's `x` is K7's lhs and `y` its rhs: pow(x, y), atan2(x, y) with x the ordinate, as `lhs atan2 rhs` is in PromQL.
"""
import functools
import math
from dataclasses import dataclass

import mpmath as mp
import numpy as np

PREC = 192
UNARY = ("exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh", "tanh", "asinh",
         "acosh", "atanh")
BINARY = ("pow", "atan2")
ODD = ("sin", "tan", "asin", "atan", "sinh", "tanh", "asinh", "atanh")
F64_MAX = np.finfo(np.float64).max
TINY = 2.0 ** -1074          # the smallest subnormal
MIN_NORMAL = 2.0 ** -1022


@dataclass(frozen=True)
class Case:
    fn: str                   # one of UNARY or BINARY
    cls: str                  # the class's name, unique per fn
    kind: str                 # "exact", "threshold" or "ill"
    x: np.ndarray             # the operand (binary: the lhs)
    y: np.ndarray = None      # binary: the rhs
    value: np.ndarray = None  # exact: the exact result
    edge: str = None          # threshold: "overflow", "normal" or "subnormal"


# ---- f64 neighbours and the correctly rounded reference -----------------------------------------------------------
def step(x, k):
    """The double k representable steps above x (below for k < 0), across zero and binades."""
    i = np.asarray(x, np.float64).view(np.int64)
    with np.errstate(over="ignore"):
        o = np.where(i < 0, np.int64(-0x8000000000000000) - i, i) + np.int64(k)
        return np.where(o < 0, np.int64(-0x8000000000000000) - o, o).view(np.float64)


def around(x, k=3):
    """x and its k neighbours on either side (2k + 1 doubles)."""
    return step(np.full(2 * k + 1, x), np.arange(-k, k + 1))


def _mpf(x):
    return mp.mpf(float(x))


def to_f64(v):
    """mpf -> the nearest double, ties to even; subnormals rounded once, to a multiple of 2^-1074; ±inf from
    f64::MAX + half an ulp up; an exact zero keeps no sign (+0.0)."""
    if mp.isnan(v):
        return math.nan
    if mp.isinf(v):
        return math.inf if v > 0 else -math.inf
    if v == 0:
        return 0.0
    a = abs(v)
    if a >= mp.mpf(2) ** 1024 - mp.mpf(2) ** 970:
        return math.copysign(math.inf, v)
    _, e = mp.frexp(a)            # a = m 2^e, 1/2 <= m < 1: the leading bit is 2^(e - 1)
    q = max(int(e) - 53, -1074)   # the quantum of a's binade (53 significant bits), or the subnormal quantum
    n = int(mp.nint(mp.ldexp(a, -q)))
    r = math.ldexp(float(n), q)   # n <= 2^53: exact
    return r if v > 0 else -r


def _cr1(fn, x):
    if math.isnan(x):
        return math.nan
    if x == 0 and fn in ODD:
        return x                  # ±0 kept
    if math.isinf(x):
        return None
    a = _mpf(x)
    extra = max(0, math.frexp(x)[1]) if fn in ("sin", "cos", "tan") else 0   # argument reduction of huge arguments
    with mp.workprec(PREC + extra):
        if fn == "exp":
            v = mp.exp(a)
        elif fn in ("ln", "log2", "log10"):
            if a < 0:
                return math.nan
            if a == 0:
                return -math.inf
            v = mp.log(a) if fn == "ln" else mp.log(a, 2) if fn == "log2" else mp.log10(a)
        elif fn in ("asin", "acos", "atanh"):
            if abs(a) > 1:
                return math.nan
            if fn == "atanh" and abs(a) == 1:
                return math.copysign(math.inf, x)
            v = getattr(mp, fn)(a)
        elif fn == "acosh":
            if a < 1:
                return math.nan
            v = mp.acosh(a)
        else:
            v = getattr(mp, fn)(a)
        r = to_f64(v)
    return -0.0 if r == 0 and x < 0 and fn in ODD else r


def _cr2(fn, x, y):
    if math.isnan(x) or math.isnan(y) or math.isinf(x) or math.isinf(y):
        return None
    a, b = _mpf(x), _mpf(y)
    with mp.workprec(PREC):
        if fn == "atan2":
            if x == 0:
                return math.copysign(0.0 if math.copysign(1, y) > 0 else math.pi, x)
            return to_f64(mp.atan2(a, b))
        if y == 0:
            return 1.0
        if x == 0:
            odd = y == int(y) and int(y) % 2 == 1
            zero_sign = math.copysign(1, x) if odd else 1.0
            return math.copysign(0.0 if y > 0 else math.inf, zero_sign)
        if x < 0:
            if y != int(y):
                return math.nan
            v = mp.power(-a, b) * (-1 if int(y) % 2 else 1)
        else:
            v = mp.power(a, b)
        r = to_f64(v)
    return -0.0 if r == 0 and v < 0 else r


def correctly_rounded(fn, x, y=None):
    """fn over arrays of finite operands (and the zeros, NaNs and domain errors these classes contain), correctly
    rounded to f64.  An operand this reference does not cover (±inf) gives NaN, so no class may hold one."""
    x = np.asarray(x, np.float64)
    if fn in BINARY:
        out = [_cr2(fn, float(a), float(b)) for a, b in zip(x.ravel(), np.broadcast_to(y, x.shape).ravel())]
    else:
        out = [_cr1(fn, float(a)) for a in x.ravel()]
    return np.array([math.nan if v is None else v for v in out], np.float64).reshape(x.shape)


def outcome(v):
    """'zero', 'subnormal', 'normal', 'inf' or 'nan' per value."""
    v = np.asarray(v, np.float64)
    a = np.abs(v)
    return np.where(np.isnan(v), "nan", np.where(np.isinf(v), "inf", np.where(a == 0, "zero",
                    np.where(a < MIN_NORMAL, "subnormal", "normal"))))


def nearest_below(v):
    """The largest double <= the mpf v."""
    r = to_f64(v)
    return float(step(r, -1)) if _mpf(r) > v else r


# ---- the classes ---------------------------------------------------------------------------------------------------
def _ks(rng, top=1 << 20, n=48):
    """ulp counts: 1..16, every power of two up to `top` and its neighbours, and n random ones below `top`."""
    ks = set(range(1, 17)) | {1 << j for j in range(top.bit_length())} | {(1 << j) + 1 for j in range(top.bit_length() - 1)}
    ks |= {(1 << j) - 1 for j in range(2, top.bit_length())}
    ks |= set(rng.integers(1, top + 1, n).tolist())
    return np.array(sorted(k for k in ks if k <= top), np.int64)


def _subnormals(rng, n=32):
    u = rng.integers(1, 1 << 52, n, dtype=np.int64)
    return np.concatenate([np.array([1, 2, 3, (1 << 52) - 1, 1 << 51], np.int64), u]).view(np.float64)


def _f(a):
    return np.asarray(a, np.float64)


def _signed(x):
    return np.concatenate([_f(x), -_f(x)])


def _exact():
    out = []
    k = np.arange(-1074, 1024)
    p2 = np.ldexp(1.0, k)
    out.append(Case("log2", "powers of two", "exact", p2, value=k.astype(np.float64)))
    k10 = np.arange(0, 23)
    out.append(Case("log10", "powers of ten", "exact", _f([10.0 ** int(i) for i in k10]), value=k10.astype(np.float64)))
    out.append(Case("ln", "one", "exact", _f([1.0]), value=_f([0.0])))
    tiny = np.concatenate([[0.0, -0.0, TINY, -TINY], _signed(np.ldexp(1.0, np.arange(-1074, -54, 7)))])
    out.append(Case("exp", "zero and tiny", "exact", tiny, value=np.ones(tiny.size)))
    out.append(Case("pow", "2^k", "exact", np.full(k.size, 2.0), _f(k), value=p2))
    out.append(Case("pow", "10^k", "exact", np.full(k10.size, 10.0), _f(k10), value=_f([10.0 ** int(i) for i in k10])))
    k3 = np.arange(0, 34)   # 3^33 < 2^53 < 3^34
    out.append(Case("pow", "3^k", "exact", np.full(k3.size, 3.0), _f(k3), value=_f([3.0 ** int(i) for i in k3])))
    n = np.concatenate([np.arange(0, 1025), np.arange(1025, 1 << 26, 65537), [(1 << 26) - 1, 1 << 26]]).astype(np.float64)
    out.append(Case("pow", "x^2", "exact", n, np.full(n.size, 2.0), value=n * n))
    out.append(Case("pow", "x^0.5 of squares", "exact", n * n, np.full(n.size, 0.5), value=n))
    p = _signed(p2)
    out.append(Case("pow", "x^1 of powers of two", "exact", p, np.ones(p.size), value=p))
    kr = np.arange(-1023, 1024)
    p = _signed(np.ldexp(1.0, kr))
    out.append(Case("pow", "x^-1 of powers of two", "exact", p, np.full(p.size, -1.0), value=1.0 / p))
    return out


def _thresholds():
    big = mp.mpf(2) ** 1024 - mp.mpf(2) ** 970   # the least real that rounds to +inf
    normal, sub = mp.mpf(2) ** -1022, mp.mpf(2) ** -1075   # a result below 2^-1075 rounds to zero
    out = []
    with mp.workprec(PREC):
        for fn, inv in (("exp", mp.log), ("sinh", mp.asinh), ("cosh", mp.acosh)):
            out.append(Case(fn, "largest finite", "threshold", around(nearest_below(inv(big))), edge="overflow"))
        out.append(Case("exp", "smallest normal", "threshold", around(to_f64(mp.log(normal))), edge="normal"))
        out.append(Case("exp", "smallest subnormal", "threshold", around(to_f64(mp.log(sub))), edge="subnormal"))
        for edge, t in (("overflow", big), ("normal", normal), ("subnormal", sub)):
            # routes to each edge: 2^y, 10^y, 0.5^y and x^2
            for base in (2.0, 10.0, 0.5):
                y = around(to_f64(mp.log(t) / mp.log(base)))
                out.append(Case("pow", f"{edge} by {base:g}^y", "threshold", np.full(y.size, base), y, edge=edge))
            x = around(to_f64(mp.sqrt(t)))
            out.append(Case("pow", f"{edge} by x^2", "threshold", x, np.full(x.size, 2.0), edge=edge))
    return out


def _ill(rng):
    out = []
    ks = _ks(rng)
    near1 = np.concatenate([1.0 + ks * 2.0 ** -52, 1.0 - ks * 2.0 ** -53])
    for fn in ("ln", "log2", "log10"):
        out.append(Case(fn, "1 ± k ulps", "ill", near1))
        out.append(Case(fn, "subnormal", "ill", _subnormals(rng)))
    # trigonometric arguments: the doubles nearest kπ/2, |k| <= 2^20, and the hardest argument reduction of the range
    kk = np.unique(np.concatenate([np.arange(1, 65), rng.integers(65, (1 << 20) + 1, 192), [1 << 20]]))
    with mp.workprec(PREC):
        half_pi = mp.pi / 2
        xs = _signed([to_f64(int(k) * half_pi) for k in kk])
    worst = math.ldexp(6381956970095103.0, 797)
    for fn in ("sin", "cos", "tan"):
        out.append(Case(fn, "nearest kπ/2", "ill", xs))
        out.append(Case(fn, "worst reduction", "ill", _signed([worst])))
    with mp.workprec(PREC):
        out.append(Case("tan", "π/2 ± k ulps", "ill", _signed(around(to_f64(mp.pi / 2), 8))))
    one_minus = _signed(1.0 - ks * 2.0 ** -53)
    for fn in ("asin", "acos", "atanh"):
        out.append(Case(fn, "±(1 - k ulps)", "ill", one_minus))
    out.append(Case("acosh", "1 + k ulps", "ill", 1.0 + ks * 2.0 ** -52))
    small = np.concatenate([np.ldexp(1.0, np.arange(-1074, -26)), np.ldexp(1.5, np.arange(-1074, -27)),
                            step(2.0 ** -26, -np.arange(1, 4)), _subnormals(rng),
                            np.ldexp(rng.random(64) + 1.0, rng.integers(-1022, -27, 64))])
    for fn in ODD:
        out.append(Case(fn, "|x| < 2^-26", "ill", np.concatenate([[0.0, -0.0], _signed(small)])))
    for fn, points in (("tanh", (0.5, 1.0, 22.0)), ("sinh", (0.5, 1.0, 22.0)), ("asin", (0.5,)), ("acos", (0.5,)),
                       ("atan", (1.0,))):
        for p in points:
            out.append(Case(fn, f"switch at {p:g}", "ill", _signed(around(p, 8))))
    # pow: a base within k ulps of 1 and |y| up to 2^60; a negative base with an integer y near 2^53; a subnormal base
    base = np.concatenate([1.0 + np.arange(1, 9) * 2.0 ** -52, 1.0 - np.arange(1, 9) * 2.0 ** -53,
                           1.0 + ks[ks <= 1 << 12] * 2.0 ** -52])
    ys = _signed(np.concatenate([np.ldexp(1.0, np.arange(0, 61)), np.ldexp(1.0, np.arange(10, 61)) * 0.75,
                                 rng.uniform(1, 2, 16) * np.ldexp(1.0, rng.integers(20, 60, 16))]))
    b, e = np.meshgrid(base, ys, indexing="ij")
    out.append(Case("pow", "base 1 ± k ulps", "ill", b.ravel(), e.ravel()))
    n53 = 2.0 ** 53
    ys = _signed([n53 - 1, n53 - 3, n53 - 2, n53 - 4, n53, n53 + 2])   # odd below 2^53, even from it
    nb = -np.concatenate([1.0 + np.arange(0, 5) * 2.0 ** -52, 1.0 - np.arange(1, 5) * 2.0 ** -53])
    b, e = np.meshgrid(nb, ys, indexing="ij")
    out.append(Case("pow", "negative base, integer y near 2^53", "ill", b.ravel(), e.ravel()))
    sb = _signed(_subnormals(rng, 16))
    ys = _f([0.5, 1.0, 2.0, 3.0, -1.0, -0.5, 0.25, 1.0 / 3.0, -0.125, 1e-3, 0.9990234375, 1.0009765625])
    b, e = np.meshgrid(sb, ys, indexing="ij")
    out.append(Case("pow", "subnormal base", "ill", b.ravel(), e.ravel()))
    # atan2(y, x)
    r = lambda n, lo, hi: np.ldexp(rng.random(n) + 1.0, rng.integers(lo, hi, n))
    big, tiny = r(32, 900, 1023), r(32, -1022, -900)
    sg = lambda a: a * np.where(rng.random(a.size) < 0.5, -1.0, 1.0)
    out.append(Case("atan2", "|y/x| subnormal", "ill", sg(np.concatenate([tiny, _subnormals(rng, 27)])),
                    sg(np.concatenate([big, r(32, 60, 1023)]))))
    out.append(Case("atan2", "|y/x| above f64::MAX", "ill", sg(np.concatenate([big, r(32, 60, 1023)])),
                    sg(np.concatenate([tiny, _subnormals(rng, 27)]))))
    v = np.concatenate([r(48, -1074 + 52, 1023), _subnormals(rng, 8), [1.0, F64_MAX, TINY]])
    out.append(Case("atan2", "x = ±y", "ill", np.concatenate([v, v, -v, -v]), np.concatenate([v, -v, v, -v])))
    neg = -np.concatenate([r(24, -1022, 1023), _subnormals(rng, 4), [F64_MAX, 1.0]])
    out.append(Case("atan2", "y = ±0, x < 0", "ill", np.concatenate([np.zeros(neg.size), np.full(neg.size, -0.0)]),
                    np.concatenate([neg, neg])))
    out.append(Case("atan2", "both subnormal", "ill", sg(_subnormals(rng, 48)), sg(_subnormals(rng, 48))))
    hi = step(np.full(48, F64_MAX), -rng.integers(0, 1 << 40, 48))
    out.append(Case("atan2", "both near f64::MAX", "ill", sg(hi), sg(hi[::-1].copy())))
    return out


@functools.lru_cache(maxsize=4)
def cases(seed=0x11BB):
    """Every class, for every function: exact cases, thresholds, ill-conditioned regions."""
    rng = np.random.default_rng(seed)
    return tuple(_exact() + _thresholds() + _ill(rng))


def glibc(fn, x, y=None):
    """What the reference computes: glibc's libm through ctypes (the oracles' bindings)."""
    from tests import binary_oracle as bor
    from tests import instant_fn_oracle as ifo
    return bor._libm_call(fn, x, y) if fn in BINARY else ifo.apply(fn, x)
