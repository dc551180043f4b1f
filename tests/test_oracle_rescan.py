"""The oracle's whole-query rescan switch (CPU only): orc.range_query(..., rescan=True) is the per-series pipeline
SeriesNormalize -> calculate_range -> orc.range_udf(..., rescan=True), scattered onto the grid, in both drivers.  It
differs from the default (sliding) grid only where the reference's sliding counter correction rounds differently
(extrapolate_rate.rs:216-238), i.e. for rate and increase."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests.range_values import VALUE_CLASSES, series_values

ALL_FNS = list(orc.FN_IDS)
PARAMS = {"predict_linear": (600.0, 0.0), "quantile_over_time": (0.9, 0.0), "holt_winters": (0.3, 0.1)}
QUERIES = [  # (start, end, interval, range, offset)
    (1_000_000, 4_000_000, 15_000, 300_000, 0),
    (999_001, 6_000_000, 60_000, 90_000, 0),
    (0, 5_000_000, 7_000, 20_000, 123_000),
    (1_000_000, 4_000_000, 15_000, 15_000, 0),
]


def irregular(seed, n_series, classes=("counter", "gauge")):
    rng = np.random.default_rng(seed)
    ts_l, val_l, offs = [], [], [0]
    for s in range(n_series):
        n = int(rng.integers(0, 300)) if s % 5 else int(rng.integers(0, 4))
        kind = s % 3
        if kind == 0:
            t = 1_000_000 + np.arange(n) * 15_000
        elif kind == 1:
            t = 1_000_000 + np.arange(n) * 15_000 + rng.integers(0, 5_000, n)
        else:
            t = 900_000 + np.cumsum(rng.integers(1, 40_000, n))
        v = series_values(classes[s % len(classes)], n, rng)
        if n:
            v[rng.random(n) < 0.04] = np.nan
        ts_l.append(t.astype(np.int64))
        val_l.append(v)
        offs.append(offs[-1] + n)
    return np.concatenate(ts_l), np.concatenate(val_l), np.array(offs, np.uint64)


def per_series_rescan(fn, q, ts, val, offsets, filter_nan, p0, p1):
    """The rescan grid assembled from the oracle's per-window primitives."""
    start, end, interval, rng_ms, offset = q
    S, T = offsets.size - 1, orc.num_steps(start, end, interval)
    out, valid = np.zeros((S, T)), np.zeros((S, T), bool)
    for s in range(S):
        o0, o1 = int(offsets[s]), int(offsets[s + 1])
        nts, nval = orc.normalize(ts[o0:o1], val[o0:o1], offset, filter_nan)
        off, ln, s2, _ = orc.calculate_range(nts, start, end, interval, rng_ms)
        if off.size == 0 or not ln.any():
            continue  # every window empty: the series yields no rows (range_manipulate.rs:641-643)
        ets = s2 + np.arange(off.size, dtype=np.int64) * interval
        r, v = orc.range_udf(fn, nts, nval, np.stack([off, ln], 1), ets, rng_ms, p0, p1, rescan=True)
        k = (ets - start) // interval
        keep = v & (k >= 0) & (k < T)
        out[s, k[keep]] = r[keep]
        valid[s, k[keep]] = True
    return out, valid


@pytest.mark.parametrize("mode", ["flat", "faithful"])
@pytest.mark.parametrize("fn", ALL_FNS)
def test_rescan_grid_is_the_per_series_rescan_udf(fn, mode):
    ts, val, offsets = irregular(31, 60)
    p0, p1 = PARAMS.get(fn, (0.0, 0.0))
    for q in QUERIES:
        for filter_nan in (True, False):
            p = orc.make_params(fn, *q[:4], offset=q[4], filter_nan=filter_nan, param0=p0, param1=p1)
            out, vw = orc.range_query(p, ts, val, None, offsets, mode=mode, threads=3, rescan=True)
            T = out.shape[1]
            e_out, e_valid = per_series_rescan(fn, q, ts, val, offsets, filter_nan, p0, p1)
            assert (orc.valid_to_bool(vw, T) == e_valid).all(), (fn, q, filter_nan)
            assert (out.view(np.uint64) == e_out.view(np.uint64)).all(), (fn, q, filter_nan)
            # the sliding grid: the same bits except for the counter correction of rate / increase
            s_out, s_vw = orc.range_query(p, ts, val, None, offsets, mode=mode, threads=3)
            assert (s_vw == vw).all()
            if fn in ("rate", "increase"):
                g, e = out[e_valid], s_out[e_valid]
                both_nan = np.isnan(g) & np.isnan(e)
                with np.errstate(invalid="ignore"):
                    ok = both_nan | (g == e) | (np.abs(g - e) <= 1e-9 * np.maximum(np.abs(g), np.abs(e)))
                assert ok.all(), (fn, q, filter_nan, g[~ok][:3], e[~ok][:3])
            else:
                assert (s_out.view(np.uint64) == out.view(np.uint64)).all(), (fn, q, filter_nan)


@pytest.mark.parametrize("fn", ALL_FNS)
def test_rescan_grid_on_special_values(fn):
    """Every value class (non-finite, signed zero, huge, subnormal, NaN payloads) through both drivers: the rescan grid
    is still the per-series rescan UDF, bit for bit, NaN payloads included."""
    ts, val, offsets = irregular(57, 2 * len(VALUE_CLASSES), classes=VALUE_CLASSES)
    p0, p1 = PARAMS.get(fn, (0.0, 0.0))
    q = QUERIES[0]
    for filter_nan in (True, False):
        p = orc.make_params(fn, *q[:4], offset=q[4], filter_nan=filter_nan, param0=p0, param1=p1)
        e_out, e_valid = per_series_rescan(fn, q, ts, val, offsets, filter_nan, p0, p1)
        for mode in ("flat", "faithful"):
            out, vw = orc.range_query(p, ts, val, None, offsets, mode=mode, threads=2, rescan=True)
            assert (orc.valid_to_bool(vw, out.shape[1]) == e_valid).all(), (fn, mode, filter_nan)
            assert (out.view(np.uint64) == e_out.view(np.uint64)).all(), (fn, mode, filter_nan)


def test_rescan_switch_keeps_the_default_call():
    """range_query's positional form (the benchmark's call) still selects the sliding restatement."""
    ts, val, offsets = irregular(5, 30, classes=("counter",))
    p = orc.make_params("rate", *QUERIES[0][:4])
    a = orc.range_query(p, ts, val, None, offsets, "faithful", 2)
    b = orc.range_query(p, ts, val, None, offsets, mode="faithful", threads=2, rescan=False)
    assert all((x == y).all() for x, y in zip(a, b))
