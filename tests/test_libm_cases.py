"""CPU: the operand classes of tests/libm_cases.py have the properties they state, the hand rounding of the correctly
rounded reference is right at its edges, glibc is exact on every exact case, and glibc's distance from the correctly
rounded result is what GLIBC_CR_ULPS records."""
import math

import mpmath as mp
import numpy as np
import pytest

from tests import libm_cases as lc
from tests.ulp_bounds import ulp_distance

CASES = lc.cases()
# glibc's largest distance from the correctly rounded result over these classes, per function (0 where not listed).
# A device result held "within n ulps of glibc" can be up to n + this far from the correctly rounded one.  The 8 and 14
# are glibc's cos / tan at 6381956970095103 * 2^797, the double nearest a multiple of π/2.
GLIBC_CR_ULPS = {"log10": 1, "sinh": 1, "cosh": 1, "tanh": 1, "asinh": 1, "acosh": 1, "atanh": 1, "pow": 1,
                 "cos": 8, "tan": 14}


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


def _id(c):
    return f"{c.fn}-{c.cls}"


@pytest.fixture(scope="module")
def reference():
    """(correctly rounded, glibc) per class."""
    return {_id(c): (lc.correctly_rounded(c.fn, c.x, c.y), lc.glibc(c.fn, c.x, c.y)) for c in CASES}


def test_every_function_has_every_kind_it_should():
    fns = {c.fn for c in CASES}
    assert fns == set(lc.UNARY) | set(lc.BINARY)
    ids = [_id(c) for c in CASES]
    assert len(ids) == len(set(ids))
    kinds = {(c.fn, c.kind) for c in CASES}
    for fn in ("log2", "log10", "ln", "exp", "pow"):
        assert (fn, "exact") in kinds
    for fn in ("exp", "sinh", "cosh", "pow"):
        assert (fn, "threshold") in kinds
    assert {c.edge for c in CASES if c.fn == "pow"} >= {"overflow", "normal", "subnormal"}
    for c in CASES:
        assert np.isfinite(c.x).all() and (c.y is None or np.isfinite(c.y).all()), _id(c)
        assert c.y is None or c.y.shape == c.x.shape, _id(c)


def test_the_same_seed_gives_the_same_operands():
    a, b = lc.cases(7), lc.cases.__wrapped__(7)
    assert [_id(c) for c in a] == [_id(c) for c in b]
    for c, d in zip(a, b):
        assert (bits(c.x) == bits(d.x)).all() and (c.y is None or (bits(c.y) == bits(d.y)).all())
    other = lc.cases.__wrapped__(8)
    assert any(c.x.shape != d.x.shape or (bits(c.x) != bits(d.x)).any() for c, d in zip(a, other))


def test_rounding_by_hand():
    """to_f64 rounds subnormals once, ties to even, and overflows at f64::MAX + half an ulp."""
    with mp.workprec(400):
        q = mp.mpf(2) ** -1074
        assert lc.to_f64(q * mp.mpf(1.5)) == 2 * lc.TINY                       # a tie: to the even multiple
        assert lc.to_f64(q * mp.mpf(2.5)) == 2 * lc.TINY
        assert lc.to_f64(q * (mp.mpf(2.5) + mp.mpf(2) ** -200)) == 3 * lc.TINY   # just above the tie
        assert lc.to_f64(q * mp.mpf(0.5)) == 0.0 and lc.to_f64(-q * mp.mpf(0.75)) == -lc.TINY
        m = mp.mpf(lc.F64_MAX)
        half = mp.mpf(2) ** 970
        assert lc.to_f64(m + half) == math.inf and lc.to_f64(-(m + half)) == -math.inf
        assert lc.to_f64(m + half - mp.mpf(2) ** 900) == lc.F64_MAX
        assert lc.to_f64(mp.mpf(1) + mp.mpf(2) ** -53) == 1.0                  # a tie at 1: even
        assert lc.to_f64(mp.mpf(1) + 3 * mp.mpf(2) ** -53) == 1.0 + 2.0 ** -51
        assert lc.to_f64(mp.mpf(2) ** -1022 - q / 2) == 2.0 ** -1022            # a tie below the smallest normal
    assert (bits(lc.step(np.array([0.0, -0.0, lc.F64_MAX]), 1)) == bits(np.array([lc.TINY, lc.TINY, math.inf]))).all()
    assert lc.step(np.array([0.0]), -1)[0] == -lc.TINY


@pytest.mark.parametrize("c", [c for c in CASES if c.kind == "exact"], ids=_id)
def test_exact_cases(reference, c):
    """The stated value is exact, the correctly rounded reference gives it, and so does glibc, bit for bit."""
    cr, g = reference[_id(c)]
    assert (bits(cr) == bits(c.value)).all(), c.x[bits(cr) != bits(c.value)][:5]
    assert (bits(g) == bits(c.value)).all(), c.x[bits(g) != bits(c.value)][:5]
    assert np.isfinite(c.value).all()
    if c.fn in ("log2", "log10") or c.cls in ("10^k", "3^k", "x^2", "x^0.5 of squares"):
        assert (c.value == np.round(c.value)).all()   # printed as an integer


EDGE_PAIR = {"overflow": {"normal", "inf"}, "normal": {"subnormal", "normal"}, "subnormal": {"zero", "subnormal"}}


@pytest.mark.parametrize("c", [c for c in CASES if c.kind == "threshold"], ids=_id)
def test_threshold_windows_straddle_their_edge(reference, c):
    """±3 ulps around the edge: the correctly rounded outcome changes exactly once inside the window, between the two
    outcomes of the edge; for exp / sinh / cosh the centre is the largest operand with a finite result."""
    cr, g = reference[_id(c)]
    out = lc.outcome(cr)
    assert set(out.tolist()) == EDGE_PAIR[c.edge], out
    assert (out[1:] != out[:-1]).sum() == 1, out
    if c.cls == "largest finite":
        assert np.isfinite(cr[:4]).all() and np.isinf(cr[4:]).all()
    assert (lc.outcome(g) == out).all(), (lc.outcome(g), out)   # glibc crosses the edge where the exact result does
    assert (np.signbit(g) == np.signbit(cr)).all()


def _mp_dist_to_half_pi_multiple(x):
    with mp.workprec(1200 + max(0, math.frexp(x)[1])):
        a = mp.mpf(x)
        k = mp.nint(a / (mp.pi / 2))
        return abs(a - k * mp.pi / 2), int(k)


def _within_ulps_of(x, p, k):
    d = ulp_distance(x, np.full(np.shape(x), p))
    return (d <= k).all()


def _check_property(c):
    x, y = np.asarray(c.x), c.y
    ax = np.abs(x)
    n = c.cls
    if n == "1 ± k ulps":
        return (x != 1).all() and _within_ulps_of(x, 1.0, 1 << 21) and (x > 1).any() and (x < 1).any()
    if n == "subnormal":
        return ((ax > 0) & (ax < lc.MIN_NORMAL)).all()
    if n == "nearest kπ/2":
        for v in x:
            d, k = _mp_dist_to_half_pi_multiple(v)
            lo, _ = _mp_dist_to_half_pi_multiple(float(lc.step(v, -1)))
            hi, _ = _mp_dist_to_half_pi_multiple(float(lc.step(v, 1)))
            if not (0 < abs(k) <= 1 << 20 and d <= lo and d <= hi):
                return False
        return True
    if n == "worst reduction":
        return all(_mp_dist_to_half_pi_multiple(v)[0] < mp.mpf(2) ** -60 for v in x)
    if n == "π/2 ± k ulps":
        with mp.workprec(lc.PREC):
            return _within_ulps_of(ax, lc.to_f64(mp.pi / 2), 8)
    if n == "±(1 - k ulps)":
        return (ax < 1).all() and _within_ulps_of(ax, 1.0, 1 << 21) and (x < 0).any()
    if n == "1 + k ulps":
        return (x > 1).all() and _within_ulps_of(x, 1.0, 1 << 20)
    if n == "|x| < 2^-26":
        sub = (ax > 0) & (ax < lc.MIN_NORMAL)
        return ((ax < 2.0 ** -26).all() and (sub & (x < 0)).any() and (sub & (x > 0)).any()
                and (bits(x) == bits(-0.0)).any() and (bits(x) == 0).any())
    if n.startswith("switch at "):
        p = float(n.split()[-1])
        return _within_ulps_of(ax, p, 8) and (x < 0).any() and (x > 0).any()
    if n == "base 1 ± k ulps":
        return (x != 1).all() and _within_ulps_of(x, 1.0, 1 << 13) and np.abs(y).max() == 2.0 ** 60
    if n == "negative base, integer y near 2^53":
        odd = np.array([int(v) % 2 == 1 for v in y])
        return ((x < 0).all() and (y == np.round(y)).all() and (np.abs(np.abs(y) - 2.0 ** 53) <= 4).all()
                and odd.any() and (~odd).any())
    if n == "subnormal base":
        return ((ax > 0) & (ax < lc.MIN_NORMAL)).all()
    with mp.workprec(lc.PREC):
        q = [abs(mp.mpf(a) / mp.mpf(b)) for a, b in zip(x, y)]
    if n == "|y/x| subnormal":
        return all(v < lc.MIN_NORMAL for v in q)
    if n == "|y/x| above f64::MAX":
        return all(v > lc.F64_MAX for v in q)
    if n == "x = ±y":
        return (ax == np.abs(y)).all() and {(a > 0, b > 0) for a, b in zip(x, y)} == {(1, 1), (1, 0), (0, 1), (0, 0)}
    if n == "y = ±0, x < 0":
        return (x == 0).all() and np.signbit(x).any() and (~np.signbit(x)).any() and (y < 0).all()
    if n == "both subnormal":
        return ((ax > 0) & (ax < lc.MIN_NORMAL) & (np.abs(y) > 0) & (np.abs(y) < lc.MIN_NORMAL)).all()
    if n == "both near f64::MAX":
        return (ax >= lc.F64_MAX * (1 - 2.0 ** -11)).all() and (np.abs(y) >= lc.F64_MAX * (1 - 2.0 ** -11)).all()
    raise AssertionError(f"no property stated for class {n!r}")


@pytest.mark.parametrize("c", [c for c in CASES if c.kind == "ill"], ids=_id)
def test_ill_conditioned_classes_have_their_property(c):
    assert _check_property(c)


def test_glibc_distance_from_correctly_rounded(reference):
    """Per function, glibc is at most GLIBC_CR_ULPS from the correctly rounded result over every class."""
    worst = {}
    for c in CASES:
        cr, g = reference[_id(c)]
        assert (np.isnan(cr) == np.isnan(g)).all(), _id(c)
        d = float(ulp_distance(g, cr).max(initial=0))
        worst[c.fn] = max(worst.get(c.fn, 0.0), d)
    for fn, d in worst.items():
        assert d <= GLIBC_CR_ULPS.get(fn, 0), (fn, d)
