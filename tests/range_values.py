"""Seeded value classes for the range-function tests: the samples where a range kernel's arithmetic, ordering and
special-value handling can go wrong (non-finite, signed zero, huge, subnormal, constant, tied, NaN with payloads).

`series_values(cls, n, rng)` returns n float64 samples of one class.  The classes are chosen so that the oracle's
expression-by-expression restatement and a kernel that reorders, drops or re-associates a single operation give
different bits on at least some windows."""
import numpy as np

F64_MAX = np.finfo(np.float64).max
SUBNORMAL = np.float64(5e-324)

VALUE_CLASSES = ("counter", "gauge", "offset", "huge", "inf", "zeros", "subnormal", "const", "ties", "nan")


def nan_with_payload(rng, n):
    """NaNs of both signs with random non-zero payloads (quiet and signalling bit patterns)."""
    payload = rng.integers(1, 1 << 51, n, dtype=np.int64).astype(np.uint64)
    quiet = rng.random(n) < 0.5
    sign = rng.random(n) < 0.5
    bits = np.uint64(0x7FF0000000000000) | payload | np.where(quiet, np.uint64(1 << 51), np.uint64(0))
    bits = bits | np.where(sign, np.uint64(1 << 63), np.uint64(0))
    return bits.view(np.float64)


def series_values(cls, n, rng):
    if cls == "counter":            # monotone counter with the odd reset
        v = np.cumsum(rng.random(n) * 10)
        for i in np.flatnonzero(rng.random(n) < 0.04):
            v[i:] -= v[i] * rng.random()
        return v
    if cls == "gauge":
        return rng.normal(size=n) * 100
    if cls == "offset":             # large offset, small noise: summation order and compensation terms show
        return 1e12 + rng.random(n)
    if cls == "huge":               # near +-f64::MAX: sums, products and differences overflow
        return rng.choice([-1.0, 1.0], n) * F64_MAX * (0.5 + 0.5 * rng.random(n))
    if cls == "inf":                # gauges with sprinkled +-inf
        v = rng.normal(size=n) * 100
        m = rng.random(n) < 0.1
        v[m] = rng.choice([-np.inf, np.inf], int(m.sum()))
        return v
    if cls == "zeros":              # +0.0 and -0.0 only
        return np.where(rng.random(n) < 0.5, 0.0, -0.0)
    if cls == "subnormal":
        k = rng.integers(0, 1 << 20, n).astype(np.float64)
        return rng.choice([-1.0, 1.0], n) * k * SUBNORMAL
    if cls == "const":              # one value for the whole series, infinities and zeros included
        c = rng.choice([3.5, np.inf, -np.inf, -0.0, 0.0, -7.25])
        return np.full(n, c)
    if cls == "ties":               # few distinct values: ranking ties, equal neighbours
        return rng.integers(0, 3, n).astype(np.float64) - 1.0
    if cls == "nan":                # gauges with NaNs of both signs and random payloads
        v = rng.normal(size=n) * 100
        m = rng.random(n) < 0.1
        v[m] = nan_with_payload(rng, int(m.sum()))
        return v
    raise ValueError(cls)
