"""CPU-only: the host mirror's fold of one (histogram, step) (distributed._fold_cells, what K5 computes over the present
buckets) against the reference's evaluate_row (oracle.histogram_evaluate_row) behind the safe mode's checks: fewer than
two buckets or a last bound other than +Inf is NaN.  Bounds come ordered as the fold index orders them (ascending, NaN
last); the shapes include NaN and duplicate bounds, more than 64 buckets, non-finite, decreasing and negative counters,
and quantiles outside [0, 1]."""
import math

import numpy as np
import pytest

from greptimedb_b200.distributed import _fold_cells
from oracle.oracle import histogram_evaluate_row

PHIS = [-0.5, 0.0, 0.25, 0.5, 0.9, 0.99, 1.0, 1.5, math.nan]


def expected(phi, bounds, counters):
    if len(bounds) < 2 or not (math.isinf(bounds[-1]) and bounds[-1] > 0):
        return math.nan
    v, err = histogram_evaluate_row(phi, np.array(bounds), np.array(counters))
    return math.nan if err else v


def shapes(rng):
    yield [0.1, 0.5, 1.0, math.inf], [1.0, 2.0, 3.0, 4.0]
    yield [1.0, 1.0, 1.0, math.inf], [0.0, 5.0, 5.0, 9.0]                       # duplicate bounds ("1" and "1.0")
    yield [0.5, 1.0, math.inf, math.nan], [1.0, 2.0, 3.0, 4.0]                  # a NaN bound last: no +Inf last
    yield [0.5, math.inf], [-3.0, -1.0]                                         # negative counters
    yield [0.5, 1.0, math.inf], [-5.0, -4.0, -4.5]                              # negative and decreasing
    yield [0.5, 1.0, math.inf], [math.nan, math.inf, 2.0]                       # non-finite counters
    yield [math.inf], [3.0]                                                     # one bucket
    yield [-2.0, -1.0, math.inf], [1.0, 1.0, 1.0]                               # flat counters, negative bounds
    yield [0.25, 4.0], [1.0, 2.0]                                               # no +Inf bound
    for n in (65, 70, 100):                                                     # more than 64 buckets
        b = sorted(rng.random(n - 1).round(2).tolist()) + [math.inf]
        c = np.cumsum(rng.random(n) * 2).tolist()
        c[int(rng.integers(n))] = math.nan
        yield b, c
    for _ in range(40):
        n = int(rng.integers(2, 12))
        b = sorted(rng.choice([0.1, 0.5, 1.0, 2.5, 10.0], n - 1).tolist()) + [math.inf]
        yield b, (rng.random(n) * 10 - 2).tolist()


@pytest.mark.parametrize("phi", PHIS)
def test_fold_cells_equals_evaluate_row(phi):
    for bounds, counters in shapes(np.random.default_rng(4)):
        got, want = _fold_cells(phi, bounds, counters), expected(phi, bounds, counters)
        assert got is not None
        assert (math.isnan(got) and math.isnan(want)) or got == want, (phi, bounds, counters, got, want)


def test_no_bucket_present_is_no_row():
    assert _fold_cells(0.5, [], []) is None
