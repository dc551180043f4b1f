"""GPU parity tests (run on an H100 with -m gpu): the CUDA path, called through the C ABI,
against (1) the reference's own golden vectors and (2) the CPU oracle on seeded inputs.

What is compared: validity bitmaps bit for bit everywhere, and null slots hold 0.0.  The per-function, int64,
big-ring, long-window, outstanding-call and fuzz tests compare every value with the oracle's *rescan* restatement
(orc.range_query(..., rescan=True)) bit for bit (the library is compiled with -fmad=false and uses IEEE div/sqrt); a
NaN only has to be a NaN there.  Where the comparison is with the reference's *sliding* restatement (the thread tier's
arms, and the tests that predate the rescan grid: lean hand-off, uniform cadence, pipelined host path, bench shape)
rate / increase / delta values are held to 1e-9 relative, because the two reference code paths differ in the last ulps
(extrapolate_rate.rs:216-238), and the functions in BIT_EXACT bit for bit.  The fused sum by tests hold group sums of
the rescan grid to the error bound of recursive summation (tests/sum_by_check.py).  tests/test_gpu_range_tiers.py
holds every tier to the rescan oracle on special values and at the kernels' window-length boundaries.
"""
import math

import numpy as np
import pytest

from oracle import oracle as orc
from tests import sum_by_check as sbc
from tests.helpers import (check_expected, farr, fnum, load_sqlness, load_unit, pack_series, promql_series,
                           udf_case_inputs)

pytestmark = pytest.mark.gpu

UNIT = load_unit()
SQL = load_sqlness()
REL = 1e-9

ALL_FNS = ["rate", "increase", "delta", "irate", "idelta", "resets", "changes", "count_over_time", "sum_over_time",
           "avg_over_time", "min_over_time", "max_over_time", "last_over_time", "present_over_time",
           "absent_over_time", "stdvar_over_time", "stddev_over_time", "deriv", "predict_linear",
           "quantile_over_time", "holt_winters"]
FN_PARAMS = {"predict_linear": (600.0, 0.0), "quantile_over_time": (0.9, 0.0), "holt_winters": (0.3, 0.1)}
BIT_EXACT = {"resets", "changes", "count_over_time", "present_over_time", "absent_over_time", "last_over_time",
             "min_over_time", "max_over_time", "idelta"}


@pytest.fixture(scope="module")
def ctx():
    """The default context, with the adaptive back-off of the lean tier pinned off so that every test below runs the
    tier it means to run (a reset-heavy call would otherwise make the next 32 calls skip K2L)."""
    import os
    from greptimedb_b200 import Context
    os.environ["B2P_LEAN_ADAPTIVE"] = "0"
    try:
        c = Context(0)
    finally:
        del os.environ["B2P_LEAN_ADAPTIVE"]
    yield c
    c.close()


def assert_close(got, exp, gv, ev, what, bit_exact=False):
    assert (gv == ev).all(), f"{what}: validity differs at {np.argwhere(gv != ev)[:5].tolist()}"
    g, e = got[ev], exp[ev]
    nan_g, nan_e = np.isnan(g), np.isnan(e)
    assert (nan_g == nan_e).all(), f"{what}: NaN pattern differs"
    g, e = g[~nan_e], e[~nan_e]
    if bit_exact:
        bad = g.view(np.uint64) != e.view(np.uint64)   # -0.0 != +0.0
    else:
        with np.errstate(invalid="ignore"):
            bad = ~((g == e) | (np.abs(g - e) <= REL * np.maximum(np.abs(g), np.abs(e))))
    assert not bad.any(), f"{what}: {int(bad.sum())} mismatches, first {g[bad][:3]} vs {e[bad][:3]}"
    assert (got[~ev] == 0.0).all(), f"{what}: null slots must hold 0.0"


# ---------------------------------------------------------------------------------------------------
# 1. the reference's unit-test vectors, through the UDF-level entry point (b2p_range_udf)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", UNIT["range_udf"], ids=lambda c: c["name"])
def test_udf_reference_goldens(ctx, case):
    ts, val, ranges = udf_case_inputs(case, UNIT)
    out, valid = ctx.range_udf(case["fn"], ts, val, ranges, eval_ts=case.get("eval_ts"),
                               range_length=case.get("range_length", 0), param0=case.get("param0", 0.0),
                               param1=case.get("param1", 0.0))
    check_expected(out, valid, case["expected"], case["tol"], case["name"])
    o_out, o_valid = orc.range_udf(case["fn"], ts, val, ranges, eval_ts=case.get("eval_ts"),
                                   range_length=case.get("range_length", 0), param0=case.get("param0", 0.0),
                                   param1=case.get("param1", 0.0), rescan=True)
    assert (valid == o_valid).all() and (out.view(np.uint64) == o_out.view(np.uint64)).all(), "bit-exact vs oracle"


def test_udf_holt_winters_trends(ctx):
    for spec, expected in UNIT["holt_winters_trends"]["cases"]:
        v = promql_series(spec)
        ts = np.arange(v.size, dtype=np.int64)
        out, valid = ctx.range_udf("holt_winters", ts, v, [[0, 801]], param0=0.01, param1=0.1)
        assert valid[0] and abs(out[0] - expected) < 1e-4, (spec, out[0])


def test_udf_quantile_and_edge_values(ctx):
    for c in UNIT["quantile_impl"]["cases"]:
        v = farr(c["values"])
        ts = np.arange(max(v.size, 1), dtype=np.int64)
        vv = v if v.size else np.zeros(1)
        out, valid = ctx.range_udf("quantile_over_time", ts, vv, [[0, v.size]], param0=fnum(c["q"]))
        e = fnum(c["expected"])
        assert valid[0] and ((math.isnan(e) and math.isnan(out[0])) or out[0] == e), c
    for c in UNIT["holt_winters_impl"]["cases"]:
        v = farr(c["values"])
        ts = np.arange(max(v.size, 1), dtype=np.int64)
        vv = v if v.size else np.zeros(1)
        out, valid = ctx.range_udf("holt_winters", ts, vv, [[0, v.size]], param0=fnum(c["sf"]), param1=fnum(c["tf"]))
        e = fnum(c["expected"])
        assert valid[0] and ((math.isnan(e) and math.isnan(out[0])) or out[0] == e), c


# ---------------------------------------------------------------------------------------------------
# 2. the reference's operator-level vectors through the fused sub-plan entry point (b2p_range_eval)
# ---------------------------------------------------------------------------------------------------
def test_range_manipulate_goldens_via_count(ctx):
    """count_over_time exposes the window lengths RangeManipulate computed (range_manipulate.rs:995-1049)."""
    g = UNIT["range_manipulate"]
    ts = np.array(g["ts"], np.int64)
    val = np.ones(ts.size)
    for c in g["cases"]:
        p = ctx_params("count_over_time", c)
        out, valid, ets = ctx.range_eval(p, ts, val, offsets=[0, ts.size])
        T = ets.size
        vb = orc.valid_to_bool(valid, T)[0]
        exp = {t: r[1] for t, r in zip(c["eval_ts"], c["ranges"]) if r[1] > 0}
        got = {int(ets[k]): out[0, k] for k in range(T) if vb[k]}
        assert got == {t: float(l) for t, l in exp.items()}, c["name"]
        # last_over_time pins the window END, sum over ts-as-values pins the START
        p2 = ctx_params("min_over_time", c)
        out2, valid2, _ = ctx.range_eval(p2, ts, ts.astype(np.float64), offsets=[0, ts.size])
        first = {int(ets[k]): out2[0, k] for k in range(T) if orc.valid_to_bool(valid2, T)[0][k]}
        assert first == {t: float(ts[r[0]]) for t, r in zip(c["eval_ts"], c["ranges"]) if r[1] > 0}, c["name"]


def ctx_params(fn, c, **kw):
    from greptimedb_b200 import make_params
    return make_params(fn, c["start"], c["end"], c["interval"], c["range"], offset=c.get("offset", 0),
                       param0=c.get("param0", 0.0), **kw)


@pytest.mark.parametrize("case", SQL["range_cases"], ids=lambda c: c["name"])
def test_sqlness_range_cases(ctx, case):
    series = case["series"] if "series" in case else SQL["series_sets"][case["series_ref"]]
    names, ts, val, sid, offsets = pack_series(series)
    p = ctx_params(case["fn"], case)
    out, valid, ets = ctx.range_eval_n(p, ts, val, sid, None, len(names))
    T = ets.size
    vb = orc.valid_to_bool(valid, T)
    got = {(names[s], int(ets[k])): out[s, k] for s in range(len(names)) for k in range(T) if vb[s, k]}
    exp = {(n, t): fnum(v) for n, t, v in case["expected"]}
    assert set(got) == set(exp), (case["name"], got)
    for key, e in exp.items():
        assert got[key] == e, (case["name"], key, got[key], e)


@pytest.mark.parametrize("case", SQL["instant_cases"], ids=lambda c: c["name"])
def test_sqlness_instant_cases(ctx, case):
    names, ts, val, sid, offsets = pack_series(case["series"])
    out, valid = ctx.instant_select(ts, val, case["start"], case["end"], case["interval"], case["lookback"],
                                    case["offset"], offsets=offsets)
    T = orc.num_steps(case["start"], case["end"], case["interval"])
    vb = orc.valid_to_bool(valid, T)
    got = {(names[s], case["start"] + k * case["interval"]): out[s, k]
           for s in range(len(names)) for k in range(T) if vb[s, k]}
    assert got == {(n, t): fnum(v) for n, t, v in case["expected"]}


def test_instant_manipulate_goldens(ctx):
    g = UNIT["instant_manipulate"]
    for c in g["cases"]:
        if c["name"] == "ultra_large_range":
            continue  # 1.8e11-step grid: the host must trim to the data extent first (B2P_E_TOO_LARGE, below)
        d = g["data_nan"] if c["nan"] else g["data"]
        ts, val = np.array(d["ts"], np.int64), farr(d["val"])
        out, valid = ctx.instant_select(ts, val, c["start"], c["end"], c["interval"], c["lookback"], 0,
                                        offsets=[0, ts.size])
        T = orc.num_steps(c["start"], c["end"], c["interval"])
        vb = orc.valid_to_bool(valid, T)[0]
        got_ts = [c["start"] + k * c["interval"] for k in range(T) if vb[k]]
        assert got_ts == c["out_ts"], c["name"]
        if "out_val" in c:
            assert [out[0, k] for k in range(T) if vb[k]] == c["out_val"], c["name"]


def test_too_large_grid_is_an_error_not_a_hang(ctx):
    from greptimedb_b200 import B2PError
    with pytest.raises(B2PError):
        ctx.instant_select(np.array([0], np.int64), np.array([1.0]), -899999999999999, 900000000000000, 10000, 10000, 0,
                           offsets=[0, 1])


@pytest.mark.parametrize("case", SQL["histogram_cases"], ids=lambda c: c["name"])
def test_sqlness_histogram_cases(ctx, case):
    B = len(case["le"])
    series = {f"b{b}": {"ts": case["bucket_ts"], "val": case["bucket_val"][b]} for b in range(B)}
    names, ts, val, sid, offsets = pack_series(series)
    p = ctx_params(case["fn"], case)
    rates, valid, ets = ctx.range_eval_n(p, ts, val, sid, None, B)
    # sum by (le, s): one series per group -> identity, but exercise the kernel anyway
    gsum, gcnt = ctx.group_aggregate("sum", rates, valid, np.arange(B, dtype=np.uint32), B)
    T = ets.size
    Tw = (T + 31) // 32
    gvalid = np.zeros((B, Tw), np.uint32)
    for b in range(B):
        for k in range(T):
            if gcnt[b, k]:
                gvalid[b, k >> 5] |= np.uint32(1 << (k & 31))
    for q, expected in case["quantiles"]:
        out, ov = ctx.histogram_quantile(q, farr(case["le"]), gsum, gvalid)
        vb = orc.valid_to_bool(ov, T)
        exp = expected if isinstance(expected, list) else [expected]
        assert [out[0, k] for k in range(T) if vb[0, k]] == exp, (case["name"], q)


def test_histogram_evaluate_row_goldens(ctx):
    for c in UNIT["histogram_evaluate_row"]["cases"]:
        le, counters = farr(c["bucket"]), farr(c["counters"])
        B = le.size
        rates = counters.reshape(B, 1)
        valid = np.ones((B, 1), np.uint32)
        out, ov = ctx.histogram_quantile(c["q"], le, rates, valid)
        assert ov[0, 0] & 1
        if c["expected"] == "err":
            assert math.isnan(out[0, 0])  # Err -> unwrap_or(NaN), histogram_fold.rs:806
            continue
        e = fnum(c["expected"])
        if math.isnan(e):
            assert math.isnan(out[0, 0]), c
        elif "tol" in c:
            assert abs(out[0, 0] - e) < c["tol"], c
        else:
            assert repr(float(out[0, 0])) == repr(e), (c, out[0, 0])


# ---------------------------------------------------------------------------------------------------
# 3. seeded parity against the oracle on synthetic series (every function)
# ---------------------------------------------------------------------------------------------------
def make_irregular(seed, n_series, with_nan=True):
    rng = np.random.default_rng(seed)
    ts_l, val_l, offs = [], [], [0]
    for s in range(n_series):
        kind = s % 6
        n = int(rng.integers(0, 400)) if kind else int(rng.integers(0, 4))
        if kind == 1:      # regular scrape
            t = 1_000_000 + np.arange(n) * 15_000
        elif kind == 2:    # jittered
            t = 1_000_000 + np.arange(n) * 15_000 + rng.integers(0, 5_000, n)
        elif kind == 3:    # gaps
            t = 1_000_000 + np.cumsum(rng.choice([15_000, 15_000, 15_000, 400_000], n))
        elif kind == 4:    # dense bursts + duplicates-free random increments
            t = 900_000 + np.cumsum(rng.integers(1, 40_000, n))
        else:
            t = 1_200_000 + np.cumsum(rng.integers(1, 3_000, n))
        v = np.cumsum(rng.random(n) * 10)
        resets = rng.random(n) < 0.05
        for i in np.flatnonzero(resets):
            v[i:] -= v[i] * rng.random()
        if kind == 4:
            v = rng.normal(size=n) * 100
        if with_nan and n:
            v[rng.random(n) < 0.04] = np.nan
        ts_l.append(t.astype(np.int64))
        val_l.append(v.astype(np.float64))
        offs.append(offs[-1] + n)
    return (np.concatenate(ts_l) if ts_l else np.zeros(0, np.int64),
            np.concatenate(val_l) if val_l else np.zeros(0), np.array(offs, np.uint64))


QUERY_SHAPES = [
    dict(start=1_000_000, end=4_000_000, interval=15_000, range=300_000, offset=0),
    dict(start=999_001, end=7_000_000, interval=60_000, range=90_000, offset=0),       # unaligned start
    dict(start=0, end=8_000_000, interval=7_000, range=20_000, offset=123_000),          # offset, short windows
    dict(start=2_000_000, end=2_000_000, interval=1_000, range=600_000, offset=0),       # instant query
    dict(start=1_000_000, end=9_000_000, interval=300_000, range=3_600_000, offset=0),   # long windows, sparse steps
]


@pytest.mark.parametrize("fn", ALL_FNS)
def test_every_function_matches_oracle_on_irregular_series(ctx, fn):
    from greptimedb_b200 import make_params
    ts, val, offsets = make_irregular(1234, 96)
    p0, p1 = FN_PARAMS.get(fn, (0.0, 0.0))
    for qi, q in enumerate(QUERY_SHAPES):
        p = make_params(fn, q["start"], q["end"], q["interval"], q["range"], offset=q["offset"], param0=p0, param1=p1)
        out, valid, ets = ctx.range_eval(p, ts, val, offsets=offsets)
        T = ets.size
        op = orc.make_params(fn, q["start"], q["end"], q["interval"], q["range"], offset=q["offset"], param0=p0, param1=p1)
        e_out, e_valid = orc.range_query(op, ts, val, None, offsets, mode="flat", rescan=True)
        gv, ev = orc.valid_to_bool(valid, T), orc.valid_to_bool(e_valid, T)
        assert_close(out, e_out, gv, ev, f"{fn} shape {qi}", bit_exact=True)


def test_int64_ring_path_on_spans_over_24_days(ctx):
    """end - start + range >= 2^31 ms selects the int64 ring variant of the fused kernel."""
    from greptimedb_b200 import make_params
    rng = np.random.default_rng(99)
    day = 86_400_000
    ts_l, val_l, offs = [], [], [0]
    for s in range(40):
        n = int(rng.integers(0, 300))
        t = 1_700_000_000_000 + np.sort(rng.integers(0, 40 * day, n)).astype(np.int64)
        t = np.unique(t)
        v = np.cumsum(rng.random(t.size) * 5)
        v[rng.random(t.size) < 0.05] = np.nan
        ts_l.append(t)
        val_l.append(v)
        offs.append(offs[-1] + t.size)
    ts, val, offsets = np.concatenate(ts_l), np.concatenate(val_l), np.array(offs, np.uint64)
    for fn in ("rate", "avg_over_time", "resets", "deriv", "irate"):
        p = make_params(fn, 1_700_000_000_000, 1_700_000_000_000 + 40 * day, 3_600_000, 2 * day)
        out, valid, ets = ctx.range_eval(p, ts, val, offsets=offsets)
        op = orc.make_params(fn, 1_700_000_000_000, 1_700_000_000_000 + 40 * day, 3_600_000, 2 * day)
        e_out, e_valid = orc.range_query(op, ts, val, None, offsets, rescan=True)
        assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size),
                     f"ts64 {fn}", bit_exact=True)


@pytest.fixture(scope="module")
def ctx_thread_tier():
    """A context with the opt-in thread-per-series tier (K2T) switched on for rate / increase / delta."""
    import os
    from greptimedb_b200 import Context
    os.environ["B2P_ENABLE_THREAD_TIER"] = "1"
    try:
        c = Context(0)
    finally:
        del os.environ["B2P_ENABLE_THREAD_TIER"]
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_no_lean():
    """A context with the lean first tier (K2L) switched off: rate / increase / delta go straight to K2."""
    import os
    from greptimedb_b200 import Context
    os.environ["B2P_DISABLE_LEAN_TIER"] = "1"
    try:
        c = Context(0)
    finally:
        del os.environ["B2P_DISABLE_LEAN_TIER"]
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_lean_flags():
    """A context whose lean tier always runs the bit-word variant for rate / increase (the one the adaptive policy
    switches to after a reset-heavy call), with the adaptive policy itself pinned off."""
    import os
    from greptimedb_b200 import Context
    os.environ["B2P_LEAN_FORCE_FLAGS"] = "1"
    os.environ["B2P_LEAN_ADAPTIVE"] = "0"
    try:
        c = Context(0)
    finally:
        del os.environ["B2P_LEAN_FORCE_FLAGS"]
        del os.environ["B2P_LEAN_ADAPTIVE"]
    yield c
    c.close()


RATE_EXACT_SHAPES = ((1000, 1, 300_000), (0, 0, 300_000), (977, 1, 77_777), (1000, 0, 1_000_000))


@pytest.mark.parametrize("lean", [True, False, "flags"])
def test_rate_warp_tier_is_bit_exact_against_the_rescan_oracle(ctx, ctx_no_lean, ctx_lean_flags, lean):
    """Warp-per-series kernels (lean tier + K2, or K2 alone): the two-FMA divisions (by window length, by range
    seconds) must round exactly like IEEE division, and the bitmask reset correction must add exactly what the
    reference's rescan adds."""
    from greptimedb_b200 import make_params
    ctx = ctx_lean_flags if lean == "flags" else (ctx if lean else ctx_no_lean)
    S, N, T0 = 256, 1000, 1_700_000_000_000
    for jitter, resets, rng_ms in RATE_EXACT_SHAPES:
        ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, jitter, resets, 0x5EED)
        p = make_params("rate", T0, T0 + 999 * 15_000, 15_000, rng_ms)
        out, valid, ets = ctx.range_eval_n(p, ts, val, sid, None, S)
        vb = orc.valid_to_bool(valid, ets.size)
        for s in range(0, S, 37):
            o = s * N
            off, ln, s2, e2 = orc.calculate_range(ts[o:o + N], T0, T0 + 999 * 15_000, 15_000, rng_ms)
            ets_s = np.arange(s2, e2 + 1, 15_000)
            e, ev = orc.range_udf("rate", ts[o:o + N], val[o:o + N], np.stack([off, ln], 1), ets_s, rng_ms, rescan=True)
            k0 = (s2 - T0) // 15_000
            got = out[s, k0:k0 + e.size]
            assert (vb[s, k0:k0 + e.size] == ev).all()
            assert (got.view(np.uint64)[ev] == e.view(np.uint64)[ev]).all(), (jitter, resets, rng_ms, s)


def test_rate_thread_tier_is_bit_exact_against_the_reference_sliding_path(ctx_thread_tier):
    ctx = ctx_thread_tier
    """Thread-per-series kernel: visits the steps in order and maintains counter_correction exactly like
    ExtrapolatedRate::calc (slide when the window slides by one sample, rescan otherwise), so whole series must be
    bit-identical to the oracle's default (sliding) restatement — for rate, increase and delta."""
    from greptimedb_b200 import make_params
    S, N, T0 = 256, 1000, 1_700_000_000_000
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    for fn in ("rate", "increase", "delta"):
        for jitter, resets, rng_ms in RATE_EXACT_SHAPES:
            ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, jitter, resets, 0x5EED)
            for interval in (15_000, 45_000, 7_000):
                p = make_params(fn, T0 + 5, T0 + 999 * 15_000 + 40_000, interval, rng_ms)
                out, valid, ets = ctx.range_eval_n(p, ts, val, sid, None, S)
                op = orc.make_params(fn, T0 + 5, T0 + 999 * 15_000 + 40_000, interval, rng_ms)
                e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=4)
                assert (valid == e_valid).all(), (fn, jitter, resets, rng_ms, interval)
                assert (out.view(np.uint64) == e_out.view(np.uint64)).all(), (fn, jitter, resets, rng_ms, interval)
                assert ctx.last_slow_series() == 0


def test_lean_tier_keeps_regular_series_and_hands_off_the_rest(ctx, ctx_no_lean):
    """K2L evaluates every series of the BASELINE shape itself (no hand-off) and is bit-identical to K2 alone; series
    with counter resets or NaN samples, sparse step grids and windows longer than its ring go to K2 and still match."""
    from greptimedb_b200 import make_params
    S, N, T0 = 512, 1000, 1_700_000_000_000
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    for fn in ("rate", "increase", "delta"):
        for jitter, resets, start, end, interval, rng_ms, all_lean in (
                (1000, 0, T0, T0 + 999 * 15_000, 15_000, 300_000, True),          # BASELINE config 2
                (0, 0, T0 + 7, T0 + 999 * 15_000 + 100_000, 15_000, 300_000, True),  # steps off the scrape grid, past the data
                (1000, 0, T0 - 600_000, T0 + 500 * 15_000, 5_000, 60_000, True),   # leading empty windows, 3 steps per sample
                (1000, 0, T0 + 3_000_000, T0 + 6_000_000, 45_000, 300_000, True),  # history before the query: clamped samples
                (1000, 1, T0, T0 + 999 * 15_000, 15_000, 300_000, fn == "delta"),  # counter resets: hand-off (not for delta)
                (1000, 0, T0, T0 + 999 * 15_000, 300_000, 300_000, False),         # 20 samples per step: ring pressure
                (1000, 0, T0, T0 + 999 * 15_000, 15_000, 6_000_000, False)):       # 400-sample windows
            ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, jitter, resets, 0x5EED)
            p = make_params(fn, start, end, interval, rng_ms)
            out, valid, ets = ctx.range_eval_n(p, ts, val, sid, None, S)
            handed = ctx.last_warp_tier_series()
            out2, valid2, _ = ctx_no_lean.range_eval_n(p, ts, val, sid, None, S)
            vb, vb2 = orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(valid2, ets.size)
            tag = (fn, jitter, resets, start - T0, interval, rng_ms)
            assert (vb == vb2).all(), tag
            assert (out.view(np.uint64)[vb] == out2.view(np.uint64)[vb]).all(), tag
            op = orc.make_params(fn, start, end, interval, rng_ms)
            e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=4)
            assert_close(out, e_out, vb, orc.valid_to_bool(e_valid, ets.size), f"lean tier {tag}")
            if all_lean:
                # a sample exactly on an eval step next to the series' end can make calculate_range's cursor
                # overshoot (DESIGN.md C-13); those few series rightly go on to K2 and the exact slow kernel
                assert handed <= S // 64, (tag, handed)
            else:
                assert handed > 0, tag
    # NaN samples (SeriesNormalize drops them): those series leave the tier, the others stay
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 0, 0x5EED)
    val = val.copy()
    val.reshape(S, N)[::4, 500] = np.nan
    p = make_params("rate", T0, T0 + 999 * 15_000, 15_000, 300_000)
    out, valid, ets = ctx.range_eval_n(p, ts, val, sid, None, S)
    assert S // 4 <= ctx.last_warp_tier_series() <= S // 4 + S // 64
    op = orc.make_params("rate", T0, T0 + 999 * 15_000, 15_000, 300_000)
    e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=4)
    assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size), "lean tier NaN hand-off")


def make_uniform_cadence(seed, n_series, scrape=15_000, t0=1_700_000_000_000):
    """Ragged series sampled exactly every `scrape` ms (the layout of aligned scrapes): different lengths and start
    phases; every 7th series carries a defect: a NaN sample or a counter reset (the series has to leave the first
    tier), one late scrape or a missing scrape (the run of equally spaced samples restarts behind it).
    -> ts, val, offsets, defect kind per series (-1 none, 0 NaN, 1 reset, 2 late, 3 gap)"""
    rng = np.random.default_rng(seed)
    ts_l, val_l, offs, defect = [], [], [0], []
    for s in range(n_series):
        n = int(rng.integers(1, 700)) if s % 5 else int(rng.integers(1, 30))
        first = t0 + int(rng.integers(-40, 200)) * scrape + (int(rng.integers(0, scrape)) if s % 3 == 0 else 0)
        t = first + np.arange(n, dtype=np.int64) * scrape
        v = np.cumsum(rng.random(n) * 10) + (0.0 if s % 4 else 1e6)
        kind = s % 7 if n > 8 else 1
        if kind == 0:
            j = int(rng.integers(1, n - 1))
            which = (s // 7) % 4
            if which == 0:
                v[j] = np.nan
            elif which == 1:
                v[j:] -= v[j] * 0.9
            elif which == 2:
                t[j] += 1
            else:
                t[j:] += scrape
        defect.append((s // 7) % 4 if kind == 0 else -1)
        ts_l.append(t)
        val_l.append(v.astype(np.float64))
        offs.append(offs[-1] + n)
    return np.concatenate(ts_l), np.concatenate(val_l), np.array(offs, np.uint64), np.array(defect)


@pytest.mark.parametrize("fn", ["rate", "increase", "delta"])
def test_uniform_cadence_tier_matches_oracle_and_the_general_tiers(ctx, ctx_no_lean, fn):
    """The uniform-cadence variant of K2L (series sampled exactly at the eval interval): window edges without
    verification reads, one extrapolation factor per window shape.  Bit-identical to the general kernels and equal to
    the oracle on ragged regular series — windows cut by either end of a series, history before the query, queries
    ending after the data, the offset modifier, range == interval, timestamps off the grid in the middle of a series
    — and the series with a NaN sample or a counter reset leave the tier as they do on the general variant."""
    import os
    from greptimedb_b200 import Context, make_params
    T0, SC = 1_700_000_000_000, 15_000
    ts, val, offsets, defect = make_uniform_cadence(77, 420)
    S = offsets.size - 1
    os.environ["B2P_LEAN_ADAPTIVE"] = "0"
    os.environ["B2P_UNIFORM"] = "1"   # (the probe would pick it as well: most series are regular)
    try:
        forced = Context(0)
    finally:
        del os.environ["B2P_LEAN_ADAPTIVE"], os.environ["B2P_UNIFORM"]
    try:
        for start, end, rng_ms, offset in (
                (T0, T0 + 999 * SC, 300_000, 0),                    # BASELINE geometry
                (T0 + 7, T0 + 400 * SC + 7, 300_000, 0),             # steps off the scrape grid
                (T0 - 100 * SC, T0 + 900 * SC, 15_000, 0),           # range == interval: one-sample windows are null
                (T0 + 300 * SC + 14_999, T0 + 1200 * SC, 77_777, 0),  # history before the query, steps past the data
                (T0 + 500 * SC, T0 + 520 * SC, 1_000_000, 0),        # late start: the cursor-start quirk on short series
                (T0 + 50 * SC, T0 + 800 * SC, 600_000, 45_000)):     # offset modifier
            p = make_params(fn, start, end, SC, rng_ms, offset=offset)
            out, valid, ets = forced.range_eval(p, ts, val, offsets=offsets)
            handed = forced.last_warp_tier_series()
            out2, valid2, _ = ctx_no_lean.range_eval(p, ts, val, offsets=offsets)
            tag = (fn, start - T0, rng_ms, offset)
            vb, vb2 = orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(valid2, ets.size)
            assert (vb == vb2).all(), tag
            assert (out.view(np.uint64)[vb] == out2.view(np.uint64)[vb]).all(), tag
            op = orc.make_params(fn, start, end, SC, rng_ms, offset=offset)
            e_out, e_valid = orc.range_query(op, ts, val, None, offsets, mode="faithful", threads=4)
            assert_close(out, e_out, vb, orc.valid_to_bool(e_valid, ets.size), f"uniform tier {tag}")
            # NaN samples and (for counters) resets send a series on; the other series stay unless the quirk applies
            must = int((defect == 0).sum()) + (0 if fn == "delta" else int((defect == 1).sum()))
            if end >= T0 + 900 * SC and start <= T0:   # (a reset behind the last window of a short query is never reached)
                assert handed >= must, (tag, handed, must)
            assert handed <= S // 2, (tag, handed)
        # the device probe picks the tier by itself: same bits on regular data, and jittered data takes the other kernel
        p = make_params(fn, T0, T0 + 999 * SC, SC, 300_000)
        out_a, valid_a, _ = ctx.range_eval(p, ts, val, offsets=offsets)
        out_f, valid_f, _ = forced.range_eval(p, ts, val, offsets=offsets)
        assert (valid_a == valid_f).all() and (out_a.view(np.uint64) == out_f.view(np.uint64)).all()
    finally:
        forced.close()


def test_lean_tier_backs_off_after_a_call_it_mostly_declined(ctx_no_lean):
    """Adaptive tiering (default on): a call in which K2L hands more than half of the series to K2 makes the following
    calls skip K2L; results are the same either way."""
    from greptimedb_b200 import Context, make_params
    S, N, T0 = 256, 1000, 1_700_000_000_000
    p = make_params("rate", T0, T0 + 999 * 15_000, 15_000, 300_000)
    c = Context(0)
    try:
        ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 0x5EED)   # every series has counter resets
        out1, valid1, _ = c.range_eval_n(p, ts, val, sid, None, S)
        assert c.last_warp_tier_series() == S                                # K2L ran and declined all of them
        out2, valid2, _ = c.range_eval_n(p, ts, val, sid, None, S)
        assert c.last_warp_tier_series() == 0                                # skipped: K2 took the whole batch
        ref, rvalid, ets = ctx_no_lean.range_eval_n(p, ts, val, sid, None, S)
        for o, v in ((out1, valid1), (out2, valid2)):
            assert (v == rvalid).all()
            vb = orc.valid_to_bool(v, ets.size)
            assert (o.view(np.uint64)[vb] == ref.view(np.uint64)[vb]).all()
    finally:
        c.close()


def test_thread_tier_hands_off_what_it_cannot_do(ctx_thread_tier):
    """NaN series, long windows, the overshoot quirk and dense bursts leave K2T for K2 / the slow kernel; results
    still match the oracle on the irregular suite."""
    from greptimedb_b200 import make_params
    ts, val, offsets = make_irregular(1234, 96)
    for fn in ("rate", "increase", "delta"):
        for qi, q in enumerate(QUERY_SHAPES):
            p = make_params(fn, q["start"], q["end"], q["interval"], q["range"], offset=q["offset"])
            out, valid, ets = ctx_thread_tier.range_eval(p, ts, val, offsets=offsets)
            op = orc.make_params(fn, q["start"], q["end"], q["interval"], q["range"], offset=q["offset"])
            e_out, e_valid = orc.range_query(op, ts, val, None, offsets)
            assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size),
                         f"thread tier {fn} shape {qi}")
    assert ctx_thread_tier.last_warp_tier_series() > 0


def test_nan_filter_off_passes_nan_through(ctx):
    from greptimedb_b200 import make_params
    ts, val, offsets = make_irregular(77, 24)
    for fn in ("last_over_time", "count_over_time", "changes"):
        p = make_params(fn, 1_000_000, 4_000_000, 15_000, 300_000, filter_nan=False)
        out, valid, ets = ctx.range_eval(p, ts, val, offsets=offsets)
        op = orc.make_params(fn, 1_000_000, 4_000_000, 15_000, 300_000, filter_nan=False)
        e_out, e_valid = orc.range_query(op, ts, val, None, offsets)
        assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size), fn,
                     bit_exact=True)


def test_cursor_overshoot_quirk_is_reproduced(ctx):
    """DESIGN.md C-13: the reference reports an empty window when its cursor overshoots; so do we."""
    from greptimedb_b200 import make_params
    ts = np.array([0, 1, 2, 3, 4, 100, 149, 150], np.int64)
    val = np.arange(8, dtype=np.float64)
    p = make_params("count_over_time", 0, 150, 50, 10)
    out, valid, ets = ctx.range_eval(p, ts, val, offsets=[0, 8])
    vb = orc.valid_to_bool(valid, ets.size)[0]
    assert ets.tolist() == [0, 50, 100, 150]
    assert vb.tolist() == [True, False, True, False]          # the reference drops t=150 although {149,150} match
    assert out[0].tolist() == [1.0, 0.0, 1.0, 0.0]
    assert ctx.last_slow_series() == 1                         # decided by the exact slow path


def test_long_windows_overflow_the_ring_and_still_match(ctx):
    from greptimedb_b200 import make_params
    n = 5000
    ts = (np.arange(n) * 1000).astype(np.int64)
    val = np.cumsum(np.ones(n))
    val[::97] = 1.0
    offsets = np.array([0, n, 2 * n], np.uint64)
    ts2, val2 = np.concatenate([ts, ts]), np.concatenate([val, val * 2])
    for fn in ("rate", "sum_over_time", "resets"):
        p = make_params(fn, 0, n * 1000, 10_000, 2_000_000)     # 2000-sample windows >> 256-sample ring
        out, valid, ets = ctx.range_eval(p, ts2, val2, offsets=offsets)
        assert ctx.last_slow_series() == 2
        op = orc.make_params(fn, 0, n * 1000, 10_000, 2_000_000)
        e_out, e_valid = orc.range_query(op, ts2, val2, None, offsets, rescan=True)
        assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size), fn,
                     bit_exact=True)


def test_hour_long_windows_take_the_big_ring_not_the_slow_path(ctx):
    """rate(x[1h]) at a 15 s scrape holds 240 samples per window: too many for the 256-sample ring next to a 64-row
    block, so the warp-per-series kernel hands the series to its 1024-sample instantiation (ADVICE r1: only the
    cursor-overshoot quirk and windows beyond that ring should reach the serial slow kernel)."""
    from greptimedb_b200 import make_params
    S, N, T0 = 64, 1500, 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 7)
    val[5::211] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    for fn in ("rate", "sum_over_time", "resets", "quantile_over_time", "deriv"):
        p0, p1 = FN_PARAMS.get(fn, (0.0, 0.0))
        p = make_params(fn, T0, T0 + (N - 1) * 15_000, 60_000, 3_600_000, param0=p0, param1=p1)
        out, valid, ets = ctx.range_eval(p, ts, val, offsets=offsets)
        assert ctx.last_slow_series() == 0, fn
        op = orc.make_params(fn, T0, T0 + (N - 1) * 15_000, 60_000, 3_600_000, param0=p0, param1=p1)
        e_out, e_valid = orc.range_query(op, ts, val, None, offsets, threads=4, rescan=True)
        assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size), fn,
                     bit_exact=True)


def test_several_outstanding_range_calls_each_keep_their_slow_path_verdict(ctx):
    """ADVICE r1 (medium): *_dev range calls are asynchronous and several may be outstanding; a call whose slow path
    ran out of arena must not be forgotten when the next call starts.  Three calls, the first and the last with
    windows far longer than any ring (slow path; the series do not fit a warp's arena region), one b2p_sync at the end."""
    import torch
    from greptimedb_b200 import Context, make_params
    dev = torch.device("cuda:0")
    c = Context(0)   # a fresh context: default 1 M-row arena
    try:
        S, N, T0 = 200, 4000, 1_700_000_000_000   # 4000-row series > one warp's region of the default arena
        ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 0, 3)
        offsets = np.arange(S + 1, dtype=np.uint64) * N
        d_ts, d_val = torch.from_numpy(ts).to(dev), torch.from_numpy(val).to(dev)
        d_off = torch.from_numpy(offsets.astype(np.int64)).to(dev)
        queries = [("sum_over_time", 1_500_000, 6_000_000 * 4), ("rate", 15_000, 300_000), ("avg_over_time", 750_000, 6_000_000 * 4)]
        outs = []
        c.use_own_stream()
        torch.cuda.synchronize()
        for fn, step, rng in queries:
            p = make_params(fn, T0, T0 + (N - 1) * 15_000, step, rng)
            T = ((N - 1) * 15_000) // step + 1
            out = torch.full((S * T,), -1.0, dtype=torch.float64, device=dev)
            valid = torch.full((S * ((T + 31) // 32),), -1, dtype=torch.int32, device=dev)
            c.range_eval_dev(p, d_ts, d_val, d_off, S * N, S, out, valid)
            outs.append((fn, step, rng, T, out, valid))
        c.sync()
        assert c.last_slow_series() == S   # the last call: every series took the slow path
        for fn, step, rng, T, out, valid in outs:
            op = orc.make_params(fn, T0, T0 + (N - 1) * 15_000, step, rng)
            e_out, e_valid = orc.range_query(op, ts, val, None, offsets, threads=8, rescan=True)
            g_out = out.cpu().numpy().reshape(S, T)
            g_valid = valid.cpu().numpy().view(np.uint32).reshape(S, (T + 31) // 32)
            assert_close(g_out, e_out, orc.valid_to_bool(g_valid, T), orc.valid_to_bool(e_valid, T), f"outstanding {fn}",
                         bit_exact=True)
    finally:
        c.close()


def test_series_offsets_from_sid_and_unsorted_error(ctx):
    from greptimedb_b200 import B2PError, make_params
    ts, val, offsets = make_irregular(5, 40, with_nan=False)
    sid = np.repeat(np.arange(40, dtype=np.uint32), np.diff(offsets).astype(np.int64))
    p = make_params("rate", 1_000_000, 4_000_000, 15_000, 300_000)
    a = ctx.range_eval_n(p, ts, val, sid, None, 40)
    b = ctx.range_eval(p, ts, val, offsets=offsets)
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
    bad = sid.copy()
    bad[[3, 4]] = bad[[4, 3]] if bad[3] != bad[4] else bad[[3, 4]]
    bad[10:20] = bad[10:20][::-1]
    if (np.diff(bad.astype(np.int64)) < 0).any():
        with pytest.raises(B2PError) as ei:
            ctx.range_eval_n(p, ts, val, bad, None, 40)
        assert ei.value.code == -3


def test_bench_shape_matches_oracle_both_variants(ctx):
    """The BASELINE config-2 shape at a size the oracle finishes in seconds; jitter and reset variants."""
    from greptimedb_b200 import make_params
    S, N, T0 = 512, 1000, 1_700_000_000_000
    for jitter, resets in ((0, 0), (1000, 0), (1000, 1)):
        ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, jitter, resets, 0x5EED)
        offsets = np.arange(S + 1, dtype=np.uint64) * N
        p = make_params("rate", T0, T0 + 999 * 15_000, 15_000, 300_000)
        out, valid, ets = ctx.range_eval_n(p, ts, val, sid, None, S)
        assert ctx.last_slow_series() == 0
        op = orc.make_params("rate", T0, T0 + 999 * 15_000, 15_000, 300_000)
        e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, mode="faithful", threads=4)
        gv, ev = orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size)
        assert_close(out, e_out, gv, ev, f"bench jitter={jitter} resets={resets}")
        assert gv.sum() > 0.97 * S * 1000


def test_pipelined_host_path_matches_oracle(ctx):
    """> 6 M rows makes b2p_range_eval split the series into double-buffered chunks (H2D | kernels | D2H overlap)."""
    from greptimedb_b200 import make_params
    S, N, T0 = 9000, 1000, 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 0x5EED)
    val[::1013] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    p = make_params("rate", T0, T0 + 999 * 15_000, 60_000, 300_000)
    op = orc.make_params("rate", T0, T0 + 999 * 15_000, 60_000, 300_000)
    e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=8)
    for use_sid in (True, False):
        out, valid, ets = ctx.range_eval_n(p, ts, val, sid if use_sid else None, None if use_sid else offsets, S)
        assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size),
                     f"pipelined sid={use_sid}")
    # windows far longer than the ring: every series goes to the slow path and overflows its default arena,
    # so each chunk is redone alone after the arena has grown
    p2 = make_params("sum_over_time", T0, T0 + 999 * 15_000, 1_500_000, 6_000_000)
    op2 = orc.make_params("sum_over_time", T0, T0 + 999 * 15_000, 1_500_000, 6_000_000)
    e_out, e_valid = orc.range_query(op2, ts, val, sid, offsets, threads=8)
    out, valid, ets = ctx.range_eval_n(p2, ts, val, sid, None, S)
    assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size), "pipelined slow path")


def test_pipelined_host_path_sends_descriptors_for_equally_spaced_chunks(ctx):
    """b2p_range_eval scans every chunk on the host; where all series of a chunk are equally spaced it sends (offsets,
    first timestamp, cadence) instead of the timestamp and id columns and the device rebuilds the column
    (ts_expand_kernel).  Regular chunks, a chunk with one timestamp off the cadence (ordinary route) and ragged series
    lengths, through the id column and through offsets; B2P_HOST_TS_SCAN=0 gives the same bits."""
    import os
    from greptimedb_b200 import Context, make_params
    T0, SC = 1_700_000_000_000, 15_000
    rng = np.random.default_rng(21)
    S = 9000
    lens = rng.integers(900, 1001, S)
    lens[::97] = 0
    lens[5::211] = 1
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    n = int(offsets[-1])
    sid = np.repeat(np.arange(S, dtype=np.uint32), lens)
    idx = np.arange(n) - np.repeat(offsets[:-1].astype(np.int64), lens)
    phase = np.repeat(rng.integers(0, 4, S) * 7, lens)          # a few start phases; cadence = scrape for all
    ts = (T0 + phase + idx * SC).astype(np.int64)
    val = np.cumsum(rng.random(n)) + 1.0
    val[::4099] = np.nan
    ts_broken = ts.copy()
    ts_broken[int(offsets[5000]) + 17] += 3                      # one row off the cadence in the second chunk
    os.environ["B2P_HOST_TS_SCAN"] = "0"
    try:
        plain = Context(0)
    finally:
        del os.environ["B2P_HOST_TS_SCAN"]
    try:
        for tsx, tag in ((ts, "regular"), (ts_broken, "one chunk irregular")):
            for fn, interval in (("rate", SC), ("avg_over_time", 60_000)):
                p = make_params(fn, T0, T0 + 999 * SC, interval, 300_000)
                op = orc.make_params(fn, T0, T0 + 999 * SC, interval, 300_000)
                e_out, e_valid = orc.range_query(op, tsx, val, None, offsets, threads=8)
                ref = None
                for c, use_sid in ((ctx, True), (ctx, False), (plain, True)):
                    out, valid, ets = c.range_eval_n(p, tsx, val, sid if use_sid else None, None if use_sid else offsets, S)
                    assert_close(out, e_out, orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size),
                                 f"host scan {tag} {fn} sid={use_sid}")
                    if ref is None:
                        ref = (out, valid)
                    else:
                        vb = orc.valid_to_bool(valid, ets.size)
                        assert (valid == ref[1]).all() and (out.view(np.uint64)[vb] == ref[0].view(np.uint64)[vb]).all()
    finally:
        plain.close()


def test_group_aggregate_matches_oracle(ctx):
    rng = np.random.default_rng(3)
    S, T, G = 700, 77, 13
    vals = rng.normal(size=(S, T))
    vb = rng.random((S, T)) > 0.2
    valid = np.packbits(np.pad(vb, ((0, 0), (0, (-T) % 32))), axis=1, bitorder="little").view(np.uint32)
    vals = np.where(vb, vals, 0.0)
    gid = rng.integers(0, G + 2, S).astype(np.uint32)   # ids >= G are dropped
    for op in ("sum", "avg", "count", "min", "max", "stddev", "stdvar"):
        g_out, g_cnt = ctx.group_aggregate(op, vals, valid, gid, G)
        e_out, e_cnt = orc.group_aggregate(op, vals, valid, gid, G)
        assert (g_cnt == e_cnt).all(), op
        assert (g_out.view(np.uint64) == e_out.view(np.uint64)).all(), f"{op}: sequential series order is bit-exact"


def test_instant_select_matches_oracle_on_irregular_series(ctx):
    ts, val, offsets = make_irregular(4242, 80)
    for (start, end, interval, lookback, offset) in ((1_000_000, 4_000_000, 15_000, 300_000, 0),
                                                     (999_001, 6_000_000, 60_000, 90_000, 0),
                                                     (0, 8_000_000, 7_000, 20_000, 123_000),
                                                     (1_500_000, 1_500_000, 1_000, 300_000, -60_000),
                                                     (1_000_000, 3_000_000, 5_000, 0, 0)):
        out, valid = ctx.instant_select(ts, val, start, end, interval, lookback, offset, offsets=offsets)
        e_out, e_valid = orc.instant_query(ts, val, offsets, start, end, interval, lookback, offset)
        T = orc.num_steps(start, end, interval)
        assert_close(out, e_out, orc.valid_to_bool(valid, T), orc.valid_to_bool(e_valid, T),
                     f"instant lookback={lookback} offset={offset}", bit_exact=True)


def test_instant_select_takes_the_first_of_rows_that_share_the_eval_timestamp(ctx):
    """Duplicate timestamps (ADVICE r1): InstantManipulate's cursor stops at the FIRST row whose timestamp equals the
    eval timestamp (instant_manipulate.rs:523-541) — also when that row is NaN (stale: no output) and a later duplicate
    is not; between two timestamps it takes the LAST row at or before (the row in front of the cursor)."""
    rng = np.random.default_rng(99)
    ts_l, val_l, offs = [], [], [0]
    for s in range(40):
        n = int(rng.integers(1, 300))
        t = 1_000_000 + np.cumsum(rng.integers(0, 2, n)) * 15_000 + (0 if s % 2 else 7)   # runs of equal timestamps
        v = rng.normal(size=n) * 10
        v[rng.random(n) < 0.1] = np.nan
        ts_l.append(t.astype(np.int64)); val_l.append(v); offs.append(offs[-1] + n)
    ts, val, offsets = np.concatenate(ts_l), np.concatenate(val_l), np.array(offs, np.uint64)
    for (start, end, interval, lookback, offset) in ((1_000_000, 3_000_000, 15_000, 300_000, 0),
                                                     (1_000_000, 3_000_000, 15_000, 0, 0),
                                                     (1_000_007, 2_500_000, 5_000, 40_000, 0),
                                                     (940_000, 2_000_000, 15_000, 20_000, -60_000)):
        out, valid = ctx.instant_select(ts, val, start, end, interval, lookback, offset, offsets=offsets)
        e_out, e_valid = orc.instant_query(ts, val, offsets, start, end, interval, lookback, offset)
        T = orc.num_steps(start, end, interval)
        assert_close(out, e_out, orc.valid_to_bool(valid, T), orc.valid_to_bool(e_valid, T),
                     f"instant with duplicate timestamps lookback={lookback} offset={offset}", bit_exact=True)


def test_device_api_sum_by_partials_and_finalize(ctx):
    """config 3 shape, small: per-shard range_group_sum partials chained into one buffer, then avg finalize."""
    import torch
    from greptimedb_b200 import make_params
    dev = torch.device("cuda:0")
    S, N, G, T0 = 300, 400, 11, 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 99)
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    gid = (np.arange(S) * 7 % G).astype(np.uint32)
    p = make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    T = N
    gsum = torch.zeros(G * T, dtype=torch.float64, device=dev)
    gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev)
    ctx.use_own_stream()
    for lo, hi in ((0, 120), (120, 300)):   # two "shards" accumulate into the same partial buffers
        r0, r1 = lo * N, hi * N
        d_ts = torch.from_numpy(ts[r0:r1]).to(dev)
        d_val = torch.from_numpy(val[r0:r1]).to(dev)
        d_off = torch.from_numpy((offsets[lo:hi + 1] - offsets[lo]).astype(np.int64)).to(dev)
        d_gid = torch.from_numpy(gid[lo:hi].astype(np.int32)).to(dev)
        torch.cuda.synchronize()
        ctx.range_group_sum_dev(p, d_ts, d_val, d_off, r1 - r0, hi - lo, d_gid, G, gsum, gcnt)
        ctx.sync()
    ctx.group_finalize_dev("avg", gsum, gcnt, G * T)
    ctx.sync()
    op = orc.make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    e_out, e_valid = orc.range_query(op, ts, val, sid, offsets)
    e_avg, e_cnt = orc.group_aggregate("avg", e_out, e_valid, gid, G)
    got = gsum.cpu().numpy().reshape(G, T)
    cnt = gcnt.cpu().numpy().view(np.uint32).reshape(G, T)
    assert (cnt == e_cnt).all()
    rel = np.abs(got - e_avg) / np.maximum(np.abs(e_avg), 1e-300)
    assert rel[e_cnt > 0].max() <= 1e-9


def _sum_by_case(S, N, G, resets, nan_every, seed, gid_mode="hash", jitter=1000):
    T0 = 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, jitter, resets, seed)
    if nan_every:
        val[nan_every // 2::nan_every] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    if gid_mode == "hash":
        from greptimedb_b200 import distributed as D
        gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
    else:  # one huge group and many tiny ones
        gid = np.where(np.arange(S) % 3 == 0, 0, 1 + np.arange(S) % (G - 1)).astype(np.uint32)
    return T0, ts, val, sid, offsets, gid


def _sum_by_values(val, values):
    """Special value classes for the fused sum by: "inf" sprinkles +-inf over the samples, "huge" scales the counters so
    that the largest sample is close to f64::MAX (rates near 1e305, group sums that overflow)."""
    from tests.range_values import F64_MAX
    val = val.copy()
    if values == "inf":
        rng = np.random.default_rng(23)
        m = rng.random(val.size) < 0.003
        val[m] = rng.choice([-np.inf, np.inf], int(m.sum()))
    elif values == "huge":
        val = val / np.nanmax(val) * (0.999 * F64_MAX)
    return val


@pytest.mark.parametrize("fn,resets,nan_every,jitter,values", [pytest.param(*c, id="-".join(str(x) for x in c if x is not None)) for c in [
    ("rate", 0, 0, 1000, None), ("rate", 1, 0, 1000, None), ("rate", 0, 9973, 1000, None),
    ("increase", 1, 7919, 1000, None), ("delta", 0, 0, 1000, None), ("delta", 1, 4099, 1000, None),
    # scrapes on the schedule: the uniform-cadence variant of the fused tier
    ("rate", 0, 0, 0, None), ("rate", 0, 9973, 0, None), ("increase", 1, 7919, 0, None), ("delta", 1, 4099, 0, None),
    # special values: +-inf samples, samples near f64::MAX
    ("rate", 1, 0, 1000, "inf"), ("delta", 0, 4099, 0, "inf"), ("increase", 0, 0, 0, "inf"),
    ("rate", 1, 0, 1000, "huge"), ("increase", 0, 9973, 0, "huge"), ("delta", 1, 0, 1000, "huge")]])
def test_fused_sum_by_matches_oracle_and_two_pass(ctx, ctx_lean_flags, fn, resets, nan_every, jitter, values):
    """sum by (..)(rate(..)) without the [S x T] intermediate (b2p_range_group_sum_indexed_dev): the first tier adds
    group by group, series it hands on (counter resets on the plain variant, NaN samples) are added by the later tiers
    from the step where the first tier stopped.  Checked against the two-pass composition on the same context (range
    eval into [S x T], then the by-label kernel's sum): counts bit for bit, and sums bit for bit where no series leaves
    the first tier (series handed on are added after the first tier's, a different order: both within the bound then); and
    against the oracle's rescan rate + group aggregate: counts bit-exact, sums within the error bound of recursive
    summation (tests/sum_by_check.py), and with +-inf samples the same non-finite entries."""
    import torch
    from greptimedb_b200 import make_params
    dev = torch.device("cuda:0")
    S, N, G = 1500, 700, 97
    T0, ts, val, sid, offsets, gid = _sum_by_case(S, N, G, resets, nan_every, 11, jitter=jitter)
    if values is not None:
        val = _sum_by_values(val, values)
    p = make_params(fn, T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    T = N
    op = orc.make_params(fn, T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=8, rescan=True)
    e_sum, e_cnt = orc.group_aggregate("sum", e_out, e_valid, gid, G)
    ref = sbc.reference(e_out, e_valid, gid, G)
    d_ts, d_val = torch.from_numpy(ts).to(dev), torch.from_numpy(val).to(dev)
    d_off = torch.from_numpy(offsets.astype(np.int64)).to(dev)
    d_gid = torch.from_numpy(gid.astype(np.int32)).to(dev)
    for c in (ctx, ctx_lean_flags):
        c.use_own_stream()
        torch.cuda.synchronize()
        ix = c.group_index_create_dev(d_gid, S, G)
        try:
            assert c.range_group_sum_fused(p, ix)
            gsum = torch.zeros(G * T, dtype=torch.float64, device=dev)
            gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev)
            # two group ranges chained into the same buffers, like tiles
            c.range_group_sum_indexed_dev(p, d_ts, d_val, d_off, S * N, S, ix, 0, 40, gsum, gcnt)
            c.range_group_sum_indexed_dev(p, d_ts, d_val, d_off, S * N, S, ix, 40, G, gsum, gcnt)
            c.sync()
            got = gsum.cpu().numpy().reshape(G, T)
            cnt = gcnt.cpu().numpy().view(np.uint32).reshape(G, T)
            assert (cnt == e_cnt).all(), f"counts differ at {np.argwhere(cnt != e_cnt)[:4].tolist()}"
            sbc.check(ref, got, cnt, "bound", "fused vs oracle")
            if not (values == "huge" and fn == "delta"):
                # (delta's signed rates near f64::MAX make partial sums overflow, and whether one does depends on the
                # order of the addends; rate / increase rates are positive and their group sums stay finite)
                assert (np.isnan(got) == np.isnan(e_sum)).all() and (np.isinf(got) == np.isinf(e_sum)).all()
            assert (got[e_cnt == 0] == 0.0).all()
            # the two-pass composition on the same context: the same bits
            r_out, r_valid, _ = c.range_eval_n(p, ts, val, sid, None, S)
            t_sum, t_cnt = c.group_aggregate("sum", r_out, r_valid, gid, G)
            assert (t_cnt == cnt).all()
            # NaN samples, and counter resets on the plain variant, send series on to the later tiers
            # (a sample after a +inf is a counter reset)
            stays = nan_every == 0 and (fn == "delta" or c is ctx_lean_flags or (resets == 0 and values != "inf"))
            if stays:
                diff = np.argwhere(t_sum.view(np.uint64) != got.view(np.uint64))
                assert not diff.size, (f"fused sum by differs from range eval + sum at {diff[:4].tolist()}: "
                                       f"{got[tuple(diff[0])]} vs {t_sum[tuple(diff[0])]}")
            else:
                sbc.check_pair((got, cnt), (t_sum, t_cnt), ref, "fused vs two-pass")
        finally:
            c.group_index_destroy(ix)


def test_fused_sum_by_falls_back_on_unbalanced_groups_and_other_functions(ctx):
    """One group holding a third of all series would serialise on one warp: the call takes the two-pass route (and says
    so); so do functions without a fused first tier.  Results still match the oracle."""
    import torch
    from greptimedb_b200 import make_params
    dev = torch.device("cuda:0")
    S, N, G = 6000, 300, 50
    T0, ts, val, sid, offsets, gid = _sum_by_case(S, N, G, 0, 0, 5, gid_mode="skewed")
    T = N
    d_ts, d_val = torch.from_numpy(ts).to(dev), torch.from_numpy(val).to(dev)
    d_off = torch.from_numpy(offsets.astype(np.int64)).to(dev)
    d_gid = torch.from_numpy(gid.astype(np.int32)).to(dev)
    ctx.use_own_stream()
    torch.cuda.synchronize()
    ix = ctx.group_index_create_dev(d_gid, S, G)
    try:
        for fn in ("rate", "avg_over_time"):
            p = make_params(fn, T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
            assert not ctx.range_group_sum_fused(p, ix)
            gsum = torch.zeros(G * T, dtype=torch.float64, device=dev)
            gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev)
            ctx.range_group_sum_indexed_dev(p, d_ts, d_val, d_off, S * N, S, ix, 0, G, gsum, gcnt)
            ctx.sync()
            op = orc.make_params(fn, T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
            e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=8, rescan=True)
            got = gsum.cpu().numpy().reshape(G, T)
            cnt = gcnt.cpu().numpy().view(np.uint32).reshape(G, T)
            sbc.check(sbc.reference(e_out, e_valid, gid, G), got, cnt, "bound", f"{fn} two-pass fallback")
    finally:
        ctx.group_index_destroy(ix)


def test_fused_sum_by_long_windows_and_quirk_series_add_exactly_once(ctx):
    """Series that leave the first tier for the long-window ring (1 h windows) or the exact slow kernel (windows beyond
    any ring; the cursor-overshoot quirk) must contribute every step exactly once."""
    import torch
    from greptimedb_b200 import make_params
    dev = torch.device("cuda:0")
    T0 = 1_700_000_000_000
    S, N, G = 96, 1200, 7
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 0, 21)
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    gid = (np.arange(S) % G).astype(np.uint32)
    d_ts, d_val = torch.from_numpy(ts).to(dev), torch.from_numpy(val).to(dev)
    d_off = torch.from_numpy(offsets.astype(np.int64)).to(dev)
    d_gid = torch.from_numpy(gid.astype(np.int32)).to(dev)
    ctx.use_own_stream()
    torch.cuda.synchronize()
    ix = ctx.group_index_create_dev(d_gid, S, G)
    try:
        for rng, step in ((3_600_000, 60_000), (24_000_000, 600_000)):
            p = make_params("rate", T0, T0 + (N - 1) * 15_000, step, rng)
            T = ((N - 1) * 15_000) // step + 1
            gsum = torch.zeros(G * T, dtype=torch.float64, device=dev)
            gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev)
            ctx.range_group_sum_indexed_dev(p, d_ts, d_val, d_off, S * N, S, ix, 0, G, gsum, gcnt)
            ctx.sync()
            op = orc.make_params("rate", T0, T0 + (N - 1) * 15_000, step, rng)
            e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=8, rescan=True)
            got = gsum.cpu().numpy().reshape(G, T)
            cnt = gcnt.cpu().numpy().view(np.uint32).reshape(G, T)
            sbc.check(sbc.reference(e_out, e_valid, gid, G), got, cnt, "bound", f"range {rng}")
    finally:
        ctx.group_index_destroy(ix)


def test_column_reduce_config5_shape(ctx):
    """avg_over_time over a wide table (config 5, small): per-column (sum, count), NaN rows skipped."""
    import torch
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(11)
    n_rows, n_cols = 200_003, 32
    data = rng.normal(size=(n_cols, n_rows)) * 1e3
    data[rng.random((n_cols, n_rows)) < 0.01] = np.nan
    cols = [torch.from_numpy(data[c]).to(dev) for c in range(n_cols)]
    ptrs = torch.tensor([c.data_ptr() for c in cols], dtype=torch.int64, device=dev)
    out_sum = torch.zeros(n_cols, dtype=torch.float64, device=dev)
    out_cnt = torch.zeros(n_cols, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    ctx.use_own_stream()
    for _ in range(2):   # accumulates: two passes double everything
        ctx.column_reduce_dev(ptrs, n_cols, n_rows, out_sum, out_cnt)
    ctx.sync()
    s, c = out_sum.cpu().numpy(), out_cnt.cpu().numpy()
    assert (c == 2 * (~np.isnan(data)).sum(1)).all()
    assert np.allclose(s, 2 * np.nansum(data, 1), rtol=1e-11, atol=0)
    avg = s / c
    assert np.allclose(avg, np.nanmean(data, 1), rtol=1e-11)


def _fuzz_series(rng, n_series):
    """Random series zoo: regular / jittered / gappy / bursty / duplicate timestamps / NaN runs / tiny / empty."""
    ts_l, val_l, offs = [], [], [0]
    t_base = int(rng.integers(-5_000_000, 5_000_000))
    for _ in range(n_series):
        kind = int(rng.integers(0, 8))
        n = int(rng.integers(0, 260)) if kind else int(rng.integers(0, 3))
        scrape = int(rng.choice([1_000, 5_000, 15_000, 60_000]))
        if kind in (1, 2):
            t = t_base + np.arange(n) * scrape + (rng.integers(0, max(scrape // 3, 1), n) if kind == 2 else 0)
        elif kind == 3:
            t = t_base + np.cumsum(rng.choice([scrape, scrape, 20 * scrape], n))
        elif kind == 4:
            t = t_base + np.cumsum(rng.integers(1, 200, n))                  # dense burst: many samples per step
        elif kind == 5:
            t = t_base + np.cumsum(rng.integers(0, 2, n) * scrape)           # duplicate timestamps
        else:
            t = t_base + np.sort(rng.integers(0, 3_000_000, n))
        v = np.cumsum(rng.random(n) * rng.choice([0.0, 1.0, 100.0]))
        if n and rng.random() < 0.5:
            for i in np.flatnonzero(rng.random(n) < 0.06):
                v[i:] -= v[i] * rng.random()
        if n and rng.random() < 0.4:
            v[rng.random(n) < 0.1] = np.nan
        if n and rng.random() < 0.1:
            v[:] = np.nan
        ts_l.append(np.asarray(t, np.int64))
        val_l.append(np.asarray(v, np.float64))
        offs.append(offs[-1] + n)
    return np.concatenate(ts_l), np.concatenate(val_l), np.array(offs, np.uint64), t_base


@pytest.mark.parametrize("seed", range(24))
def test_fuzz_random_queries_match_oracle(ctx, ctx_thread_tier, ctx_no_lean, ctx_lean_flags, seed):
    """Random series zoo x random (start, end, interval, range, offset): validity and values bit-exact against the rescan
    oracle; the thread tier (sliding counter correction) against the sliding oracle, values <= 1e-9 rel."""
    from greptimedb_b200 import make_params
    rng = np.random.default_rng(1000 + seed)
    ts, val, offsets, t_base = _fuzz_series(rng, 40)
    fns = ["rate", "increase", "delta", "irate", "resets", "changes", "count_over_time", "avg_over_time", "max_over_time",
           "last_over_time", "stddev_over_time", "deriv", "quantile_over_time", "absent_over_time"]
    for _ in range(5):
        interval = int(rng.choice([1_000, 7_000, 15_000, 60_000, 300_000]))
        rng_ms = int(rng.choice([1, 999, 5_000, 60_000, 300_000, 900_000]))
        start = t_base + int(rng.integers(-400_000, 1_000_000))
        end = start + int(rng.integers(0, 400)) * interval + int(rng.integers(0, interval))
        offset = int(rng.choice([0, 0, 30_000, -45_000]))
        for fn in rng.choice(fns, 4, replace=False):
            fn = str(fn)
            p = make_params(fn, start, end, interval, rng_ms, offset=offset, param0=0.75)
            op = orc.make_params(fn, start, end, interval, rng_ms, offset=offset, param0=0.75)
            e_out, e_valid = orc.range_query(op, ts, val, None, offsets, rescan=True)
            s_out, s_valid = orc.range_query(op, ts, val, None, offsets)
            for c in ((ctx, ctx_thread_tier, ctx_no_lean, ctx_lean_flags) if fn in ("rate", "increase", "delta") else (ctx,)):
                out, valid, ets = c.range_eval(p, ts, val, offsets=offsets)
                sliding = c is ctx_thread_tier
                assert_close(out, s_out if sliding else e_out, orc.valid_to_bool(valid, ets.size),
                             orc.valid_to_bool(s_valid if sliding else e_valid, ets.size),
                             f"fuzz seed={seed} {fn} start={start} end={end} int={interval} rng={rng_ms} off={offset}",
                             bit_exact=not sliding or fn in BIT_EXACT)


def test_full_size_chunk_properties_and_tier_equivalence(ctx, ctx_no_lean):
    """BASELINE config 2 at the full per-GPU chunk size (1.25 M series x 1000 samples, device-resident, through the
    _dev C ABI): size-independent properties instead of an oracle pass over 1.25e9 samples.

      * tier equivalence: K2L + K2 and K2 alone write bit-identical values and validity words;
      * linearity: increase(x[5m]) == rate(x[5m]) * 300 to the last bits (one extra rounding: <= 2 ulp);
      * validity: every step of every series whose window holds >= 2 samples is valid (a closed-form count for the
        synthetic shape), and the same series re-evaluated alone (a 4096-series slice) gives the same bits — the
        result of a series cannot depend on what else is in the batch;
      * a sample of series against the oracle."""
    import torch
    from greptimedb_b200 import make_params
    S, N, T0 = 1_250_000, 1000, 1_700_000_000_000
    T, Tw = 1000, 32
    dev = torch.device("cuda:0")
    ts = torch.empty(S * N, dtype=torch.int64, device=dev)
    val = torch.empty(S * N, dtype=torch.float64, device=dev)
    sid = torch.empty(S * N, dtype=torch.int32, device=dev)
    off = torch.empty(S + 1, dtype=torch.int64, device=dev)
    outs = {}
    for name, c in (("lean", ctx), ("k2", ctx_no_lean)):
        c.synth_fill_dev(0, S, N, T0, 15_000, 1000, 0, 0x5EED, ts, val, sid)
        c.series_offsets_dev(sid, S * N, S, off)
        for fn in (("rate", "increase") if name == "lean" else ("rate",)):
            out = torch.empty(S * T, dtype=torch.float64, device=dev)
            valid = torch.empty(S * Tw, dtype=torch.int32, device=dev)
            c.range_eval_dev(make_params(fn, T0, T0 + 999 * 15_000, 15_000, 300_000), ts, val, off, S * N, S, out, valid)
            c.sync()
            outs[(name, fn)] = (out, valid)
        if name == "lean":
            assert c.last_warp_tier_series() <= S // 64
    r_lean, v_lean = outs[("lean", "rate")]
    r_k2, v_k2 = outs.pop(("k2", "rate"))
    assert torch.equal(v_lean, v_k2)
    assert torch.equal(r_lean.view(torch.int64), r_k2.view(torch.int64))
    del r_k2, v_k2  # 80 GB hold the inputs and three [S x T] outputs, not the temporaries below on top of them
    # validity: steps 1 .. 999 have >= 2 samples in (t - 5m, t] unless a zero-jitter sample sits on an edge; step 0 never
    bits = v_lean.view(S, Tw)
    popc = sum(((bits >> b) & 1).sum(dtype=torch.int64) for b in range(32))
    n_valid = int(popc.item())
    assert S * 997 <= n_valid <= S * 999, n_valid
    # linearity of increase against rate (every valid step, taken in slices of series)
    inc, v_inc = outs[("lean", "increase")]
    assert torch.equal(v_inc, v_lean)
    lanes = torch.arange(32, device=dev, dtype=torch.int32)
    rel = 0.0
    for a in range(0, S, 125_000):
        b = min(S, a + 125_000)
        mask = ((bits[a:b].unsqueeze(-1) >> lanes) & 1).bool().reshape(b - a, Tw * 32)[:, :T].reshape(-1)
        i_, r_ = inc[a * T:b * T][mask], r_lean[a * T:b * T][mask]
        rel = max(rel, ((i_ - r_ * 300.0).abs() / i_.abs().clamp_min(1e-300)).max().item())
    assert rel <= 1e-15, rel
    # a slice evaluated alone gives the same bits
    s0, ns = 777_216, 4096
    off2 = (off[s0:s0 + ns + 1] - off[s0]).contiguous()
    torch.cuda.synchronize()  # off2 was produced on torch's stream, the context runs on its own
    out2 = torch.empty(ns * T, dtype=torch.float64, device=dev)
    valid2 = torch.empty(ns * Tw, dtype=torch.int32, device=dev)
    r0 = s0 * N
    ctx.range_eval_dev(make_params("rate", T0, T0 + 999 * 15_000, 15_000, 300_000), ts[r0:r0 + ns * N], val[r0:r0 + ns * N],
                       off2, ns * N, ns, out2, valid2)
    ctx.sync()
    assert torch.equal(valid2, v_lean[s0 * Tw:(s0 + ns) * Tw])
    assert torch.equal(out2.view(torch.int64), r_lean[s0 * T:(s0 + ns) * T].view(torch.int64))
    # a sample of series against the oracle
    pick = np.array([0, 1, 4095, 65_537, 777_216, 1_249_999])
    h_ts = np.concatenate([ts[s * N:(s + 1) * N].cpu().numpy() for s in pick])
    h_val = np.concatenate([val[s * N:(s + 1) * N].cpu().numpy() for s in pick])
    offsets = np.arange(pick.size + 1, dtype=np.uint64) * N
    op = orc.make_params("rate", T0, T0 + 999 * 15_000, 15_000, 300_000)
    e_out, e_valid = orc.range_query(op, h_ts, h_val, None, offsets)
    got = np.stack([r_lean[s * T:(s + 1) * T].cpu().numpy() for s in pick])
    gv = np.stack([v_lean[s * Tw:(s + 1) * Tw].cpu().numpy().view(np.uint32) for s in pick])
    assert_close(got, e_out, orc.valid_to_bool(gv, T), orc.valid_to_bool(e_valid, T), "full-size chunk sample vs oracle")


# ---------------------------------------------------------------------------------------------------
# HistogramFold on the device: the reference's operator tests (histogram_fold.rs:1452-1630), mixed bucket layouts,
# the 64-bucket config-4 shape
# ---------------------------------------------------------------------------------------------------
def _fold_golden():
    import json
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "reference_histogram_fold_vectors.json")) as f:
        return json.load(f)


FOLD = _fold_golden()


def _dense_from_rows(case):
    """rows (group, ts, le, val) -> the dense form the device fold takes: one series per (group, le), steps = the
    distinct (ts | explicit step) values in order, validity = a row exists."""
    rows = case["rows"]
    steps = case.get("step_of_row")
    if steps is None:
        ts_sorted = sorted({r[1] for r in rows})
        steps = [ts_sorted.index(r[1]) for r in rows]
    T = max(steps) + 1
    groups = []
    for r in rows:
        if r[0] not in groups:
            groups.append(r[0])
    series = []          # (group index, le label)
    for r in rows:
        key = (groups.index(r[0]), r[2])
        if key not in series:
            series.append(key)
    S = len(series)
    rates = np.zeros((S, T))
    valid = np.zeros((S, 1), np.uint32)
    for r, k in zip(rows, steps):
        s = series.index((groups.index(r[0]), r[2]))
        rates[s, k] = r[3]
        valid[s, 0] |= np.uint32(1 << k)
    les = np.array([orc.parse_f64_rust(le) for _, le in series])
    order = sorted(range(S), key=lambda s: (series[s][0], np.isnan(les[s]), les[s] if not np.isnan(les[s]) else 0.0))
    hist_off = np.zeros(len(groups) + 1, np.uint32)
    for s in order:
        hist_off[series[s][0] + 1] += 1
    hist_off = np.cumsum(hist_off).astype(np.uint32)
    return groups, T, rates, valid, np.array(order, np.uint32), les[order].copy(), hist_off


@pytest.mark.parametrize("case", FOLD["cases"], ids=lambda c: c["name"])
def test_histogram_fold_operator_goldens_on_the_device(ctx, case):
    import torch
    dev = torch.device("cuda:0")
    groups, T, rates, valid, bucket_series, bucket_le, hist_off = _dense_from_rows(case)
    H = len(groups)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = torch.zeros(H * T, dtype=torch.float64, device=dev)
    ov = torch.zeros(H * 1, dtype=torch.int32, device=dev)
    ctx.use_own_stream()
    torch.cuda.synchronize()
    ctx.histogram_fold_dev(case["phi"], d(hist_off.astype(np.int32)), d(bucket_series.astype(np.int32)), d(bucket_le), H,
                           d(rates), d(valid.astype(np.int32)), T, out, ov)
    ctx.sync()
    got, gv = out.cpu().numpy().reshape(H, T), ov.cpu().numpy().view(np.uint32).reshape(H, 1)
    flat = [(groups[h], float(got[h, k])) for h in range(H) for k in range(T) if (gv[h, 0] >> k) & 1]
    assert len(flat) == len(case["expected"]), (flat, case["expected"])
    for (g, v), (eg, ev) in zip(flat, case["expected"]):
        assert g == eg
        if ev == "NaN":
            assert np.isnan(v)
        else:
            assert abs(v - float(ev)) <= max(case["tol"], 0.0) * max(abs(float(ev)), 1.0) or v == float(ev), (case["name"], v, ev)


def test_histogram_fold_64_buckets_and_missing_buckets_match_the_row_literal_fold(ctx):
    """The config-4 shape (64 buckets per histogram) with holes: some bucket series have no sample at some steps, some
    histograms lack the +Inf bucket or have fewer buckets.  The dense device fold must equal the row-literal restatement
    of fold_buf / safe mode on the same rows."""
    import torch
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(4)
    H, T = 23, 70
    rows, series, les, hist_of = [], [], [], []
    for h in range(H):
        B = [64, 64, 64, 17, 2, 1][h % 6]
        bounds = list(np.round(0.005 * 1.3 ** np.arange(B - 1), 6)) + [np.inf]
        if h % 7 == 3:
            bounds[-1] = 1e9            # no +Inf bucket at all
        for b in range(B):
            series.append((h, b))
            les.append(bounds[b])
            hist_of.append(h)
    S = len(series)
    Tw = (T + 31) // 32
    rates = np.zeros((S, T))
    valid = np.zeros((S, Tw), np.uint32)
    base = np.cumsum(rng.random((S, T)), axis=0)            # cumulative over buckets within the flat order (good enough)
    for s, (h, b) in enumerate(series):
        for k in range(T):
            if rng.random() < 0.04:
                continue                                    # hole: this bucket has no sample at this step
            v = base[s, k] - base[[i for i, x in enumerate(series) if x[0] == h][0], k] + 1.0
            if rng.random() < 0.01:
                v = np.nan
            rates[s, k] = v
            valid[s, k >> 5] |= np.uint32(1 << (k & 31))
    phi = 0.99
    # row-literal fold on the same data: rows sorted by (histogram, step, le)
    lit = []
    for h in range(H):
        sidx = [i for i, x in enumerate(series) if x[0] == h]
        for k in range(T):
            rr = [((h,), k, ("+Inf" if np.isinf(les[i]) else repr(float(les[i]))), rates[i, k]) for i in sidx
                  if (valid[i, k >> 5] >> (k & 31)) & 1]
            lit += rr
    exp = {(t[0], k): v for t, k, v in orc.histogram_fold_rows(lit, phi)}
    hist_off = np.zeros(H + 1, np.int32)
    for h in hist_of:
        hist_off[h + 1] += 1
    hist_off = np.cumsum(hist_off).astype(np.int32)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = torch.zeros(H * T, dtype=torch.float64, device=dev)
    ov = torch.zeros(H * Tw, dtype=torch.int32, device=dev)
    ctx.use_own_stream()
    torch.cuda.synchronize()
    ctx.histogram_fold_dev(phi, d(hist_off), d(np.arange(S, dtype=np.int32)), d(np.array(les)), H, d(rates),
                           d(valid.astype(np.int32)), T, out, ov)
    ctx.sync()
    got, gv = out.cpu().numpy().reshape(H, T), ov.cpu().numpy().view(np.uint32).reshape(H, Tw)
    n_rows = 0
    for h in range(H):
        for k in range(T):
            has = bool((gv[h, k >> 5] >> (k & 31)) & 1)
            assert has == ((h, k) in exp), (h, k)
            if has:
                n_rows += 1
                e, g = exp[(h, k)], got[h, k]
                assert (np.isnan(e) and np.isnan(g)) or e == g or abs(e - g) <= 1e-12 * abs(e), (h, k, e, g)
    assert n_rows > H * T // 2
