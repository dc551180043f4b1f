"""CPU: the instant-function / scalar() oracle reproduces every printed golden value exactly, pins the unit vectors of
round.rs and clamp.rs and the special cases of each function, and the dense scalar() agrees with the row-literal one on
random label sets (NULL labels, batch splits, empty and tagless inputs)."""
import math
import zlib

import numpy as np
import pytest

from tests import instant_fn_oracle as ifo
from tests.instant_fn_helpers import G, check_rows, oracle_rows

CASES = [c for c in G["cases"] if "oracle" in c["layers"]]


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_tables(case):
    tags, rows = oracle_rows(case["expr"], case)
    check_rows(case, tags, rows)


def test_clamp_error_message():
    e = G["errors"][0]
    with pytest.raises(ValueError) as ei:
        oracle_rows(e["expr"], e)
    assert str(ei.value) == "min '12.0' > max '0.0'"   # Python's repr; the library writes Rust's Display: '12', '0'


def test_round_unit_vectors():
    for v, n, want in G["units"]["round"]:
        assert ifo.apply("round", [v], n)[0] == want


def test_clamp_unit_vectors():
    u = G["units"]
    for c in u["clamp"]:
        ok = np.array([x is not None for x in c["in"]])
        vals = np.array([0.0 if x is None else x for x in c["in"]])[None, :]
        out, words = ifo.instant_fn("clamp", vals, ifo._words(ok[None, :]), c["min"], c["max"])
        assert (ifo._bits(words, ok.size)[0] == ok).all()
        assert [x if k else None for x, k in zip(out[0].tolist(), ok)] == c["out"]
    for c in u["clamp_min"]:
        assert ifo.apply("clamp_min", c["in"], c["min"]).tolist() == c["out"]
    for c in u["clamp_max"]:
        assert ifo.apply("clamp_max", c["in"], c["max"]).tolist() == c["out"]
    for c in u["clamp_invalid"]:
        with pytest.raises(ValueError):
            ifo.apply("clamp", c["in"], c["min"], c["max"])


def _b(x):
    return np.float64(x).view(np.uint64)


def test_special_cases():
    inf, nan = math.inf, math.nan
    assert ifo.apply("ln", [0.0])[0] == -inf and math.isnan(ifo.apply("ln", [-1.0])[0])
    assert ifo.apply("atanh", [1.0])[0] == inf and ifo.apply("atanh", [-1.0])[0] == -inf
    assert _b(ifo.apply("acos", [1.0])[0]) == _b(0.0)
    # round is half away from zero and keeps -0.0; not Prometheus's floor(x + 0.5)
    assert ifo.apply("round", [2.5, -2.5, 0.49999999999999994, -0.3]).tolist() == [3.0, -3.0, 0.0, -0.0]
    assert _b(ifo.apply("round", [-0.3])[0]) == _b(-0.0)
    # deg is one multiplication by the constant 180/π: math.result:121 prints 90.00021045914971
    assert ifo.apply("deg", [1.5708])[0] == 90.00021045914971 != 1.5708 * 180 / math.pi
    # sgn: 0.0 for ±0 (positive zero), NaN stays NaN
    s = ifo.apply("sgn", [-0.0, 0.0, -3.0, 1e-310, nan, -inf])
    assert _b(s[0]) == _b(0.0) and s[1] == 0.0 and s[2] == -1.0 and s[3] == 1.0 and math.isnan(s[4]) and s[5] == -1.0
    # clamp: a NaN value passes with its bits, a NaN bound never binds; clamp_min / clamp_max meet ±f64::MAX
    payload = np.array([0x7FF8000000000123], np.uint64).view(np.float64)
    assert ifo.apply("clamp", payload, 0.0, 1.0).view(np.uint64)[0] == 0x7FF8000000000123
    assert ifo.apply("clamp", [5.0], nan, 1.0)[0] == 1.0 and ifo.apply("clamp", [-5.0], 0.0, nan)[0] == 0.0
    assert ifo.apply("clamp_min", [inf], 0.0)[0] == 1.7976931348623157e308
    assert ifo.apply("clamp_max", [-inf], 0.0)[0] == -1.7976931348623157e308
    with pytest.raises(ValueError):
        ifo.apply("clamp_min", [1.0], inf)
    with pytest.raises(ValueError):
        ifo.apply("clamp_max", [1.0], -inf)


def _random_labelled_grid(rng, n_series, T, null_rate, n_tags):
    """n_series distinct label tuples (some with NULL labels), each a dense row with random cells."""
    tuples = set()
    while len(tuples) < n_series:
        tuples.add(tuple(None if rng.random() < null_rate else f"v{rng.integers(0, 4)}" for _ in range(n_tags)))
    tuples = sorted(tuples, key=lambda t: tuple((x is not None, x or "") for x in t))
    ok = rng.random((n_series, T)) < rng.choice([0.02, 0.3, 0.9])
    vals = rng.normal(size=(n_series, T))
    return tuples, vals, ok


def _dense_keys(tuples):
    ids, key = {}, []
    for t in tuples:
        key.append(ifo.NO_KEY if None in t else ids.setdefault(t, len(ids)))
    return np.array(key, np.uint32)


def test_dense_scalar_matches_row_literal_on_random_label_sets():
    start, interval = 1000, 500
    for seed in range(400):
        rng = np.random.default_rng(zlib.crc32(f"scalar {seed}".encode()))
        T = int(rng.choice([1, 5, 33, 70]))
        n_tags = int(rng.integers(0, 3))
        n_series = 1 if n_tags == 0 else int(rng.integers(0, 4))
        tuples, vals, ok = _random_labelled_grid(rng, n_series, T, 0.3, n_tags)
        rows = [t + (start + k * interval, float(vals[r, k])) for r, t in enumerate(tuples) for k in range(T) if ok[r, k]]
        cuts = sorted(rng.choice(len(rows) + 1, size=int(rng.integers(0, 4)), replace=True).tolist()) if rows else []
        batches = [rows[a:b] for a, b in zip([0] + cuts, cuts + [len(rows)])]   # (empty batches included)
        lit = dict(ifo.scalar_calculate_rows(batches, n_tags, start, start + (T - 1) * interval, interval))
        out, words = ifo.scalar_calculate(vals, ifo._words(ok), _dense_keys(tuples))
        cell = ifo._bits(words[None, :], T)[0]
        dense = {start + k * interval: float(out[k]) for k in range(T) if cell[k]}
        assert dense.keys() == lit.keys(), (seed, tuples)
        for t in dense:
            assert (math.isnan(dense[t]) and math.isnan(lit[t])) or dense[t] == lit[t], (seed, t)


def test_scalar_null_label_quirk():
    """A series with a NULL label counts as one series with one row, as several with two or more."""
    T = 4
    one = ifo.scalar_calculate_rows([[(None, 0, 7.0)]], 1, 0, 3, 1)
    two = ifo.scalar_calculate_rows([[(None, 0, 7.0), (None, 1, 8.0)]], 1, 0, 3, 1)
    assert one == [(0, 7.0)] and len(two) == T and all(math.isnan(v) for _, v in two)
    split = ifo.scalar_calculate_rows([[(None, 0, 7.0)], [(None, 1, 8.0)]], 1, 0, 3, 1)
    assert all(math.isnan(v) for _, v in split)
    ok = np.zeros((1, T), bool)
    ok[0, 0] = True
    out, _ = ifo.scalar_calculate(np.full((1, T), 7.0), ifo._words(ok), [ifo.NO_KEY])
    assert out[0] == 7.0
    ok[0, 1] = True
    out, _ = ifo.scalar_calculate(np.full((1, T), 7.0), ifo._words(ok), [ifo.NO_KEY])
    assert np.isnan(out).all()
