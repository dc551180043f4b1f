"""Every range function on every range tier, bit for bit against the oracle's rescan restatement (run with -m gpu).

The tiers compute the same 21 functions through one eval_window<FN> (b2p_window.cuh) but reach it through different
rings, time domains, edge searches and hand-offs.  Each test below picks a route with the library's existing switches
only, asserts from the counters (or from the construction of the query) that the route was taken, and compares the
grid with orc.range_query(..., rescan=True):

  * validity bitmaps are equal and null slots hold +0.0;
  * every non-NaN value has the oracle's bits (so -0.0 != +0.0);
  * a NaN is matched as a NaN (the default NaN of a GPU operation and of the CPU differ and are not pinned), except for
    last / min / max_over_time, which copy a sample: their NaNs must carry the sample's bits;
  * the route's grid has the same bits as the default context's grid of the same call, NaNs included for the functions
    that copy a sample (a NaN computed from two NaN operands may carry either payload, depending on the kernel).

Inputs: one seeded series per (value class, shape), tests/range_values.py — counters, gauges, 1e12 + U(0,1), values
near +-f64::MAX, sprinkled +-inf, +-0.0 only, subnormals, constant series (+-inf and +-0 included), ties and NaNs of
both signs with payloads.  Samples are regular (jittered by less than a quarter scrape for some series) and the eval
grid sits half a scrape off the samples, so no sample lies on an eval step and a window of range = l >= 1 scrapes holds
exactly l samples of every series.  For l = 0 (range just below half a scrape) the windows of the regular series are
empty; a jittered sample more than 1 ms after its scrape slot still falls into one, so those hold 0 or 1.
"""
import functools
import os

import numpy as np
import pytest

from oracle import oracle as orc
from tests.range_values import VALUE_CLASSES, series_values

pytestmark = pytest.mark.gpu

ALL_FNS = list(orc.FN_IDS)
NOT_LEAN = {"absent_over_time", "quantile_over_time", "holt_winters"}   # no K2L variant: K2 is their first tier
LEAN_FNS = [f for f in ALL_FNS if f not in NOT_LEAN]
FLAGS_FNS = ["rate", "increase", "resets", "changes"]                  # K2L's bit-word variant
UNI_FNS = ["rate", "increase", "delta"]                                # K2L's uniform-cadence variant
COPY_FNS = {"last_over_time", "min_over_time", "max_over_time"}        # results are samples: NaN bits are pinned
PARAMS = {"predict_linear": (600.0, 0.0), "quantile_over_time": (0.9, 0.0), "holt_winters": (0.3, 0.1)}
THREADS = max(1, min(16, os.cpu_count() or 1))

SC = 15_000              # scrape interval (ms)
T0 = 10_000_000          # first sample of the 32-bit-domain sets
LENGTHS = [0, 1, 2, 3, 7, 8, 9, 63, 64, 65, 255, 256, 257]


def _context(**env):
    from greptimedb_b200 import Context
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def ctxs():
    """default: the library as shipped.  k2l: the lean first tier, general variant.  k2l_flags: its bit-word variant
    for rate / increase.  k2l_uni: its uniform-cadence variant, forced.  k2: the lean tier off (K2, its big ring and the
    slow kernel).  k2t: the thread tier in front of K2 for rate / increase / delta."""
    c = {
        "default": _context(),
        "k2l": _context(B2P_LEAN_ADAPTIVE="0", B2P_UNIFORM="0"),
        "k2l_flags": _context(B2P_LEAN_ADAPTIVE="0", B2P_UNIFORM="0", B2P_LEAN_FORCE_FLAGS="1"),
        "k2l_uni": _context(B2P_LEAN_ADAPTIVE="0", B2P_UNIFORM="1"),
        "k2": _context(B2P_DISABLE_LEAN_TIER="1"),
        "k2t": _context(B2P_ENABLE_THREAD_TIER="1"),
    }
    yield c
    for x in c.values():
        x.close()


# ---------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------
def build_set(seed, n, per_class, t0=T0, sc=SC, marker_gap=0):
    """per_class series of every value class, about n samples each: three of four on the scrape grid (different start
    phases), the fourth jittered by less than sc/4.  marker_gap > 0 adds one gauge series whose samples stop for
    marker_gap ms in the middle (windows empty between non-empty ones) and one empty series, which K2L always hands on
    to K2: a non-zero hand-off count proves that K2L ran."""
    rng = np.random.default_rng(seed)
    ts_l, val_l = [], []
    for cls in VALUE_CLASSES:
        for i in range(per_class):
            m = n - int(rng.integers(0, 6))
            t = t0 + (np.arange(m, dtype=np.int64) + int(rng.integers(0, 4))) * sc
            if i % 4 == 3:
                t = t + rng.integers(0, sc // 4, m)
            ts_l.append(t)
            val_l.append(series_values(cls, m, rng))
    if marker_gap:
        h = n // 2
        t = t0 + np.arange(n, dtype=np.int64) * sc
        t[h:] += marker_gap
        ts_l.append(t)
        val_l.append(rng.normal(size=n) * 10)
        ts_l.append(np.zeros(0, np.int64))
        val_l.append(np.zeros(0))
    offsets = np.concatenate([[0], np.cumsum([x.size for x in ts_l])]).astype(np.uint64)
    return np.concatenate(ts_l), np.concatenate(val_l), offsets


def window_range(l, sc=SC):
    """range (ms) for which a window of the half-phase grid holds exactly l samples (l = 0: of the regular series)"""
    return l * sc if l else sc // 2 - 1


@functools.lru_cache(maxsize=None)
def set_small():
    return build_set(1, 420, 12, marker_gap=300 * SC)


@functools.lru_cache(maxsize=None)
def set_big():
    return build_set(2, 1050, 3)


@functools.lru_cache(maxsize=None)
def set_slow():
    return build_set(3, 1750, 3)


@functools.lru_cache(maxsize=None)
def set_domain(domain):
    """-> (scrape, first sample, data) of the time-domain tests"""
    if domain == "negative_start":
        return SC, -40_000_000, build_set(4, 300, 6, t0=-40_000_000, sc=SC, marker_gap=80 * SC)
    sc = 10_000_000   # ~2.8 h scrapes: 230 samples span fits_ts32's threshold
    return sc, 1_000_000_000_000, build_set(5, 230, 6, t0=1_000_000_000_000, sc=sc, marker_gap=80 * sc)


# ---------------------------------------------------------------------------------------------------
# the bar
# ---------------------------------------------------------------------------------------------------
def check_values(got, gv, exp, ev, fn, what):
    """gv / ev: bool validity of the same shape as got / exp."""
    bad = np.argwhere(gv != ev)
    assert not bad.size, f"{what}: validity differs at {bad[:5].tolist()} (got {gv[tuple(bad[0])]})"
    nz = np.argwhere(~gv & (got.view(np.uint64) != 0))
    assert not nz.size, f"{what}: null slots must hold +0.0, {nz[:3].tolist()}"
    g, e = got[ev], exp[ev]
    gb, eb = g.view(np.uint64), e.view(np.uint64)
    ok = (gb == eb) if fn in COPY_FNS else np.where(np.isnan(e), np.isnan(g), gb == eb)
    if not ok.all():
        i = np.flatnonzero(~ok)[:4]
        idx = np.argwhere(ev)[i].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} values differ; at {idx}: got {g[i].tolist()} "
                             f"({[hex(x) for x in gb[i]]}) expected {e[i].tolist()} ({[hex(x) for x in eb[i]]})")


def oracle_grid(p, data, rescan=True):
    ts, val, offsets = data
    return orc.range_query(p, ts, val, None, offsets, mode="flat", threads=THREADS, rescan=rescan)


def to_orc(p):
    return orc.make_params(p.fn_id, p.start, p.end, p.interval, p.range, offset=p.offset,
                           filter_nan=bool(p.filter_nan), param0=p.param0, param1=p.param1)


def same_grid(out, vw, ref, fn, what):
    """bit equality of two grids, the validity words' padding included.  NaN payloads are compared for the functions
    that copy a sample; a NaN an operation computes from two NaN operands carries one of their payloads, and which one
    depends on the operand order the compiler chose in that kernel (IEEE 754 leaves it open), so there it is NaN as
    NaN."""
    w = np.argwhere(vw != ref[1])
    assert not w.size, f"{what}: validity words differ from the default context's at {w[:3].tolist()}: " \
                       f"{[hex(vw[tuple(i)]) for i in w[:3]]} vs {[hex(ref[1][tuple(i)]) for i in w[:3]]}"
    diff = out.view(np.uint64) != ref[0].view(np.uint64)
    if fn not in COPY_FNS:
        diff &= ~(np.isnan(out) & np.isnan(ref[0]))
    d = np.argwhere(diff)
    assert not d.size, f"{what}: {len(d)} values differ from the default context's grid at {d[:3].tolist()}: " \
                       f"{[hex(out.view(np.uint64)[tuple(i)]) for i in d[:3]]} vs " \
                       f"{[hex(ref[0].view(np.uint64)[tuple(i)]) for i in d[:3]]}"


def run_route(ctx, p, data, exp, ref, fn, what):
    """One range_eval call on one context, checked against the oracle grid `exp` and (unless None) the default
    context's grid `ref`.  -> (out, valid words, series K2L handed on, series on the slow kernel)"""
    ts, val, offsets = data
    out, vw, ets = ctx.range_eval(p, ts, val, offsets=offsets)
    T = ets.size
    check_values(out, orc.valid_to_bool(vw, T), exp[0], orc.valid_to_bool(exp[1], T), fn, what)
    if ref is not None:
        same_grid(out, vw, ref, fn, what)
    return out, vw, ctx.last_warp_tier_series(), ctx.last_slow_series()


def k2t_keeps(p, data, l):
    """The series K2T must evaluate itself: windows of at most 9 samples (well inside its 64-row ring), no NaN sample
    when the NaN filter is on, and no window where calculate_range's cursor overshoots (C-13: calculate_range and the
    definitional windows differ).  Every other series may be handed on to K2 / the slow kernel."""
    ts, val, offsets = data
    S = offsets.size - 1
    keep = np.zeros(S, bool)
    if l > 9:
        return keep
    for s in range(S):
        o0, o1 = int(offsets[s]), int(offsets[s + 1])
        if p.filter_nan and np.isnan(val[o0:o1]).any():
            continue
        t, _ = orc.normalize(ts[o0:o1], val[o0:o1], p.offset, bool(p.filter_nan))
        a = orc.calculate_range(t, p.start, p.end, p.interval, p.range)
        d = orc.calculate_range(t, p.start, p.end, p.interval, p.range, definitional=True)
        keep[s] = a[2:] == d[2:] and (a[1] == d[1]).all() and (a[0][a[1] > 0] == d[0][d[1] > 0]).all()
    return keep


def k2t_route(ctx, p, data, exp, ref, fn, what, l):
    """K2T keeps the reference's sliding counter correction; the series it hands on are evaluated by K2 with the rescan
    one.  So every series has all its values from one of the two restatements (NaN as NaN), and the series K2T must keep
    (k2t_keeps) have the sliding restatement's."""
    ts, val, offsets = data
    out, vw, ets = ctx.range_eval(p, ts, val, offsets=offsets)
    T = ets.size
    sl = oracle_grid(to_orc(p), data, rescan=False)
    gv, ev = orc.valid_to_bool(vw, T), orc.valid_to_bool(exp[1], T)
    assert (vw == sl[1]).all()
    check_values(np.where(gv, 0.0, out), gv, np.zeros_like(out), ev, "count_over_time", what)  # validity, null slots
    keep = k2t_keeps(p, data, l)
    assert l > 9 or keep.sum() > (offsets.size - 1) // 2, f"{what}: too few series certain to stay on K2T"
    for s in range(offsets.size - 1):
        g = out[s, ev[s]]
        gb = g.view(np.uint64)
        same = [bool(((np.isnan(g) & np.isnan(e)) | (gb == e.view(np.uint64))).all())
                for e in (sl[0][s, ev[s]], exp[0][s, ev[s]])]
        if keep[s]:
            assert same[0], f"{what}: series {s} stays on K2T but does not have the sliding restatement's values"
        else:
            assert same[0] or same[1], f"{what}: series {s} has values of neither restatement"
    if ref is not None:
        same_grid(out, vw, ref, fn, what)


_WINDOWS = {}


def oracle_windows(p, data):
    """SeriesNormalize + calculate_range of every series, concatenated: (ts, val, [(offset, len)], eval ts).  `data` is
    always one of the lru-cached sets, which live as long as the module, so its id names it."""
    key = (id(data), p.start, p.end, p.interval, p.range, p.offset, p.filter_nan)
    if key not in _WINDOWS:
        ts, val, offsets = data
        n_ts, n_val, ranges, ets = [], [], [], []
        base = 0
        for s in range(offsets.size - 1):
            o0, o1 = int(offsets[s]), int(offsets[s + 1])
            t, v = orc.normalize(ts[o0:o1], val[o0:o1], p.offset, bool(p.filter_nan))
            off, ln, s2, _ = orc.calculate_range(t, p.start, p.end, p.interval, p.range)
            n_ts.append(t)
            n_val.append(v)
            ranges.append(np.stack([off.astype(np.int64) + base, ln.astype(np.int64)], 1))
            ets.append(s2 + np.arange(off.size, dtype=np.int64) * p.interval)
            base += t.size
        _WINDOWS.clear()
        _WINDOWS[key] = (np.concatenate(n_ts), np.concatenate(n_val), np.concatenate(ranges), np.concatenate(ets))
    return _WINDOWS[key]


def udf_route(ctx, fn, p, data, what):
    """range_udf_kernel over the oracle's own windows, all series in one call, against orc.range_udf(..., rescan=True)
    on the same windows."""
    n_ts, n_val, ranges, ets = oracle_windows(p, data)
    if not ranges.shape[0]:
        return
    out, valid = ctx.range_udf(fn, n_ts, n_val, ranges, eval_ts=ets, range_length=p.range, param0=p.param0,
                               param1=p.param1)
    e, ev = orc.range_udf(fn, n_ts, n_val, ranges, ets, p.range, p.param0, p.param1, rescan=True)
    check_values(out, valid, e, ev, fn, what)


def params(fn, start, end, interval, rng_ms, filter_nan, p0=None, p1=None):
    from greptimedb_b200 import make_params
    d0, d1 = PARAMS.get(fn, (0.0, 0.0))
    return make_params(fn, start, end, interval, rng_ms, filter_nan=filter_nan,
                       param0=d0 if p0 is None else p0, param1=d1 if p1 is None else p1)


# ---------------------------------------------------------------------------------------------------
# 1. windows of 0 .. 257 samples: K2L (general, bit words, uniform cadence), K2 (256 ring / big ring), the default
#    context, the UDF kernel and the thread tier, with and without the NaN filter
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("filter_nan", [1, 0], ids=["filter_nan", "keep_nan"])
@pytest.mark.parametrize("l", LENGTHS)
def test_every_function_on_every_first_and_second_tier_route(ctxs, l, filter_nan):
    data = set_small()
    S = data[2].size - 1
    n = 420
    start = T0 + SC // 2
    end = start + (n + 4) * SC
    rng_ms = window_range(l)
    lean_geometry = rng_ms >= SC    # K2L needs range >= interval
    for fn in ALL_FNS:
        p = params(fn, start, end, SC, rng_ms, filter_nan)
        exp = oracle_grid(to_orc(p), data)
        tag = f"{fn} l={l} filter_nan={filter_nan}"
        d_out, d_vw, handed, _ = run_route(ctxs["default"], p, data, exp, None, fn, f"default {tag}")
        if fn in NOT_LEAN:
            assert handed == 0, f"default {tag}: no K2L variant, K2 is the first tier"
        ref = (d_out, d_vw)
        _, _, handed, _ = run_route(ctxs["k2"], p, data, exp, ref, fn, f"k2 {tag}")
        assert handed == 0, f"k2 {tag}: the lean tier is off, nothing can be handed on from it"
        routes = (["k2l"] if fn in LEAN_FNS else []) + (["k2l_flags"] if fn in FLAGS_FNS else []) + \
            (["k2l_uni"] if fn in UNI_FNS else [])
        for r in routes:
            _, _, handed, _ = run_route(ctxs[r], p, data, exp, ref, fn, f"{r} {tag}")
            if lean_geometry:
                # the empty series always leaves K2L; windows that do not fit its ring (l > 192) send every series on
                assert handed >= 1 and (handed < S or l > 192), f"{r} {tag}: K2L must run ({handed} of {S} handed on)"
            else:
                assert handed == 0, f"{r} {tag}: range < interval never takes K2L"
        udf_route(ctxs["default"], fn, p, data, f"udf {tag}")
        if fn in UNI_FNS:
            k2t_route(ctxs["k2t"], p, data, exp, ref if fn == "delta" else None, fn, f"k2t {tag}", l)
            if filter_nan:
                handed = ctxs["k2t"].last_warp_tier_series()
                assert handed >= 1, f"k2t {tag}: K2T must run and hand on the series with NaN samples"


# ---------------------------------------------------------------------------------------------------
# 2. long windows: K2's 1024-sample ring (no series reaches the slow kernel) and the exact slow kernel (every series)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("filter_nan", [1, 0], ids=["filter_nan", "keep_nan"])
@pytest.mark.parametrize("route,l", [("big_ring", 300), ("big_ring", 600), ("big_ring", 900),
                                     ("slow", 1300), ("slow", 1600)])
def test_every_function_on_the_long_window_tiers(ctxs, route, l, filter_nan):
    data = set_big() if route == "big_ring" else set_slow()
    S = data[2].size - 1
    n = 1050 if route == "big_ring" else 1750
    step = SC * (8 if route == "big_ring" else 16)
    start = T0 + SC // 2
    end = start + (n + 4) * SC
    for fn in ALL_FNS:
        p = params(fn, start, end, step, window_range(l), filter_nan)
        exp = oracle_grid(to_orc(p), data)
        tag = f"{fn} {route} l={l} filter_nan={filter_nan}"
        want = 0 if route == "big_ring" else S
        d_out, d_vw, _, slow = run_route(ctxs["default"], p, data, exp, None, fn, f"default {tag}")
        assert slow == want, f"default {tag}: {slow} of {S} series on the slow kernel"
        for r in ["k2"] + (["k2l"] if fn in LEAN_FNS else []):
            _, _, _, slow = run_route(ctxs[r], p, data, exp, (d_out, d_vw), fn, f"{r} {tag}")
            assert slow == want, f"{r} {tag}: {slow} of {S} series on the slow kernel"
        udf_route(ctxs["default"], fn, p, data, f"udf {tag}")


# ---------------------------------------------------------------------------------------------------
# 3. time domains: spans just under and just over fits_ts32's threshold (32-bit ring vs int64 ring), a negative start
# ---------------------------------------------------------------------------------------------------
TS32_LIMIT = 2_147_483_000   # fits_ts32: end - start + range below this many ms


@pytest.mark.parametrize("filter_nan", [1, 0], ids=["filter_nan", "keep_nan"])
@pytest.mark.parametrize("domain", ["ts32_just_under", "int64_just_over", "negative_start"])
def test_every_function_across_the_time_domains(ctxs, domain, filter_nan):
    sc, t0, data = set_domain(domain)
    S = data[2].size - 1
    start = t0 + sc // 2
    for l in (1, 2, 3, 8, 9, 64, 65):
        rng_ms = window_range(l, sc)
        if domain == "negative_start":
            end = start + 304 * sc
        else:
            end = start + TS32_LIMIT + (-1 if domain == "ts32_just_under" else 1) - rng_ms
        span = end - start + rng_ms
        assert (span < TS32_LIMIT) == (domain == "ts32_just_under") or domain == "negative_start"
        for fn in ALL_FNS:
            p = params(fn, start, end, sc, rng_ms, filter_nan)
            exp = oracle_grid(to_orc(p), data)
            tag = f"{fn} {domain} l={l} filter_nan={filter_nan}"
            d_out, d_vw, _, _ = run_route(ctxs["default"], p, data, exp, None, fn, f"default {tag}")
            run_route(ctxs["k2"], p, data, exp, (d_out, d_vw), fn, f"k2 {tag}")
            if fn in LEAN_FNS:
                _, _, handed, _ = run_route(ctxs["k2l"], p, data, exp, (d_out, d_vw), fn, f"k2l {tag}")
                if domain == "ts32_just_under":
                    assert handed >= 1, f"k2l {tag}: the 32-bit domain takes K2L first"
                else:
                    assert handed == 0, f"k2l {tag}: K2L runs only in the 32-bit domain with start >= 0"
            if l in (2, 9):
                udf_route(ctxs["default"], fn, p, data, f"udf {tag}")


# ---------------------------------------------------------------------------------------------------
# 4. parameters: quantile_over_time's phi, holt_winters' (sf, tf), predict_linear's seconds
# ---------------------------------------------------------------------------------------------------
PARAM_CASES = ([("quantile_over_time", q, 0.0) for q in (0.0, 0.5, 0.9, 1.0, -0.1, 1.1, float("nan"))]
               + [("holt_winters", sf, tf) for sf, tf in ((0.0, 0.0), (1.0, 1.0), (0.0, 1.0), (1.0, 0.5), (0.5, 0.0),
                                                          (-0.1, 0.5), (0.5, 1.1), (float("nan"), 0.5), (0.5, float("nan")))]
               + [("predict_linear", t, 0.0) for t in (0.0, 37.5, -120.7, -3600.0)])


@pytest.mark.parametrize("filter_nan", [1, 0], ids=["filter_nan", "keep_nan"])
@pytest.mark.parametrize("fn,p0,p1", PARAM_CASES)
def test_function_parameters_on_every_route(ctxs, fn, p0, p1, filter_nan):
    data = set_small()
    start = T0 + SC // 2
    end = start + 424 * SC
    for l in (0, 1, 2, 3, 9, 64, 65):
        p = params(fn, start, end, SC, window_range(l), filter_nan, p0, p1)
        exp = oracle_grid(to_orc(p), data)
        tag = f"{fn}({p0}, {p1}) l={l} filter_nan={filter_nan}"
        d_out, d_vw, _, _ = run_route(ctxs["default"], p, data, exp, None, fn, f"default {tag}")
        for r in ["k2"] + (["k2l"] if fn in LEAN_FNS else []):
            run_route(ctxs[r], p, data, exp, (d_out, d_vw), fn, f"{r} {tag}")
        udf_route(ctxs["default"], fn, p, data, f"udf {tag}")
