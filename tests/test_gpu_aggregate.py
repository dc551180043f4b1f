"""GPU tests of the kernels above the range functions, at their edges (run on an H100 with -m gpu):

  K3 group_aggregate_kernel    by-label aggregate, through its three entry points, partial states + finalize, and the
                               cross-rank merge (two shards on one GPU; a one-rank NCCL communicator)
  K5 histogram_fold_kernel     the shared-validity, compacted and wide (> 64 buckets) paths
  K6 column_reduce_stage1/2    per-column sum / count
  sum(rate()) tables of tql/range.result through the device routes

The reference is the CPU oracle (orc.group_aggregate, orc.histogram_fold_rows), which is pinned on the reference's own
tables.  Where the inputs are finite an independent exact computation sits beside it (math.fsum, fractions.Fraction),
so that the oracle is not the only judge of new inputs.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as orc
from tests.helpers import total_order_case
from tests.ranks import one_rank_comm

pytestmark = pytest.mark.gpu

AGGS = ("sum", "avg", "count", "min", "max", "stddev", "stdvar")
EPS = 2.0 ** -53


@pytest.fixture(scope="module")
def ctx():
    """Own context; the lean tier's adaptive back-off is pinned off so that the fused sum-by route is the one asked for.
    The library enqueues on torch's current stream, so it runs after the fills and copies that set up its buffers."""
    import os
    from greptimedb_b200 import Context
    os.environ["B2P_LEAN_ADAPTIVE"] = "0"
    try:
        c = Context(0)
    finally:
        del os.environ["B2P_LEAN_ADAPTIVE"]
    c.use_torch_stream()
    yield c
    c.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _words(vb):
    """[S x T] bool -> [S x Tw] uint32 validity words (bit k & 31 of word k >> 5)."""
    T = vb.shape[1]
    return np.packbits(np.pad(vb, ((0, 0), (0, (-T) % 32))), axis=1, bitorder="little").view(np.uint32).reshape(vb.shape[0], -1)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def assert_same_values(got, exp, agg, what):
    """Bit for bit.  The one allowed difference: a NaN produced by arithmetic (sum / avg / stddev / stdvar of inf - inf
    or of a NaN member) may differ in sign and payload — IEEE 754 leaves them to the hardware (x86 returns the negative
    default NaN, the GPU a positive one).  min / max select a member, so there even NaN payloads must be the same."""
    g, e = np.ascontiguousarray(got).ravel(), np.ascontiguousarray(exp).ravel()
    same = _bits(g) == _bits(e)
    if agg not in ("min", "max"):
        same |= np.isnan(g) & np.isnan(e)
    if not same.all():
        i = int(np.flatnonzero(~same)[0])
        raise AssertionError(f"{what}: {int((~same).sum())} cells differ, first at flat index {i}: "
                             f"{g[i]!r} ({_bits(g)[i]:#x}) vs {e[i]!r} ({_bits(e)[i]:#x})")


# ---------------------------------------------------------------------------------------------------------------------
# 1. K3 by-label aggregate: all three entry points, all seven aggregators
# ---------------------------------------------------------------------------------------------------------------------
# Group sizes hit the batch-of-32 member fetch (31 / 32 / 33, 128 / 129) and the four-ahead value loads (3 / 4 / 5); an
# empty group reads cnt 0 / value 0.0.  Every size comes with every validity mode.
GROUP_SIZES = (0, 1, 3, 4, 5, 31, 32, 33, 128, 129)
VALIDITY = ("all", "none", "holes", "one_step")
BIG_GROUP = 4100
VALUE_MODES = ("normal", "inf", "nan", "zeros", "huge", "cancel", "subnormal")
FINITE_MODES = ("normal", "zeros", "cancel", "subnormal")
K3_T = (1, 31, 32, 33, 64, 65, 200)


def _values(rng, mode, shape):
    n = int(np.prod(shape))
    if mode == "normal":
        v = rng.normal(size=n) * 100.0
    elif mode == "inf":
        v = rng.normal(size=n)
        v[rng.random(n) < 0.05] = np.inf
        v[rng.random(n) < 0.05] = -np.inf
    elif mode == "nan":
        v = rng.normal(size=n)
        specials = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF800000000BEEF, 0xFFF0000000000001,
                             0x7FF0000000000000, 0xFFF0000000000000, 0x8000000000000000], np.uint64).view(np.float64)
        pick = rng.random(n) < 0.08
        v[pick] = specials[rng.integers(0, specials.size, int(pick.sum()))]
    elif mode == "zeros":
        v = np.where(rng.random(n) < 0.5, -0.0, 0.0)
        pick = rng.random(n) < 0.05
        v[pick] = rng.choice([1.0, -1.0, 0.5], int(pick.sum()))
    elif mode == "huge":   # the sum overflows to +-inf part-way
        v = rng.choice([1e308, 1.5e308, -1e308, 0.5], n, p=[0.45, 0.2, 0.3, 0.05])
    elif mode == "cancel":  # Welford on 1e9 + small: the mean cancels catastrophically in a naive formula
        v = 1e9 + rng.normal(size=n) * 1e-3
    else:                   # subnormals, down to the smallest one
        v = rng.normal(size=n) * 1e-310
        v[rng.random(n) < 0.2] = 5e-324
    return v.reshape(shape)


def make_k3_case(T, mode, seed):
    """-> (vals [S x T], valid words, gid [S], G).  Series of one group are interleaved with the others' (random
    series order); some series carry ids >= G, which the aggregate must drop."""
    rng = np.random.default_rng(seed)
    spec = [(n, v) for n in GROUP_SIZES for v in VALIDITY] + [(BIG_GROUP, "holes")]
    G = len(spec)
    gid = np.concatenate([np.full(n, g, np.uint32) for g, (n, _) in enumerate(spec)] +
                         [np.array([G, G + 1, 0xFFFFFFFF] * 5, np.uint32)])
    S = gid.size
    perm = rng.permutation(S)
    gid = gid[perm]
    mode_of = np.array([VALIDITY.index(spec[g][1]) if g < G else 2 for g in gid.astype(np.int64).clip(0, G)])
    vb = np.zeros((S, T), bool)
    vb[mode_of == 0] = True
    holes = mode_of == 2
    vb[holes] = rng.random((int(holes.sum()), T)) > 0.2
    one = np.flatnonzero(mode_of == 3)
    vb[one, rng.integers(0, T, one.size)] = True
    vals = _values(rng, mode, (S, T))
    vals[~vb] = 0.0
    return vals, _words(vb), gid, G


def _members(vals, valid, gid, g, k):
    bits = (valid[:, k >> 5] >> np.uint32(k & 31)) & 1
    return vals[(gid == g) & (bits == 1), k]


def check_k3_against_exact(vals, valid, gid, G, agg, got, cnt, n_var_samples=40, seed=0):
    """Independent of the oracle, finite inputs only: sums and means against math.fsum within n * 2^-53 * sum|x|;
    stdvar against an exact two-pass Fraction computation on a sample of cells."""
    T = vals.shape[1]
    if agg in ("sum", "avg"):
        for g in range(G):
            for k in range(T):
                x = _members(vals, valid, gid, g, k)
                n = x.size
                assert cnt[g, k] == n
                if n == 0:
                    continue
                exact = math.fsum(x)
                bound = n * EPS * float(np.abs(x).sum())
                if agg == "avg":   # plus half the smallest subnormal: a subnormal quotient rounds absolutely
                    exact, bound = exact / n, (n + 1) * EPS * float(np.abs(x).sum()) / n + 5e-324
                assert abs(got[g, k] - exact) <= bound, (agg, g, k, n, got[g, k], exact, bound)
    elif agg in ("stdvar", "stddev"):
        rng = np.random.default_rng(seed)
        cells = [(g, k) for g in range(G) for k in range(T) if cnt[g, k] > 0]
        for i in rng.permutation(len(cells))[:n_var_samples]:
            g, k = cells[i]
            x = _members(vals, valid, gid, g, k)
            n = x.size
            fx = [Fraction(float(v)) for v in x]
            m = sum(fx) / n
            var = float(sum((v - m) ** 2 for v in fx) / n)
            # Welford's error grows with n and with the mean's size against the spread (cancellation)
            bound = 8 * n * EPS * (var + math.sqrt(var) * float(np.abs(x).max())) + 8 * n * 5e-324
            v = got[g, k] if agg == "stdvar" else got[g, k] ** 2
            assert abs(v - var) <= bound + (4 * EPS * var if agg == "stddev" else 0.0), (agg, g, k, n, v, var, bound)


@pytest.mark.parametrize("mode", VALUE_MODES)
@pytest.mark.parametrize("T", K3_T)
def test_group_aggregate_entry_points_match_the_oracle(ctx, T, mode):
    """b2p_group_aggregate (host), b2p_group_aggregate_dev (gid) and b2p_group_aggregate_indexed_dev (group index) for
    every aggregator: counts exact, values bit for bit against the oracle (both fold in series order), empty cells 0.0,
    and the three entry points bit for bit equal to each other.  Outputs start out as garbage: they are overwritten."""
    import torch
    vals, valid, gid, G = make_k3_case(T, mode, seed=T * 31 + VALUE_MODES.index(mode))
    S = gid.size
    d_vals, d_valid, d_gid = _dev(vals), _dev(valid.view(np.int32)), _dev(gid.view(np.int32))
    torch.cuda.synchronize()
    ix = ctx.group_index_create_dev(d_gid, S, G)
    try:
        for agg in AGGS:
            e_val, e_cnt = orc.group_aggregate(agg, vals, valid, gid, G)
            h_val, h_cnt = ctx.group_aggregate(agg, vals, valid, gid, G)
            outs = []
            for route in ("gid", "index"):
                ov = torch.full((G * T,), 7.25, dtype=torch.float64, device="cuda:0")
                oc = torch.full((G * T,), 99, dtype=torch.int32, device="cuda:0")
                if route == "gid":
                    ctx.group_aggregate_dev(agg, d_vals, d_valid, d_gid, S, G, T, ov, oc)
                else:
                    ctx.group_aggregate_indexed_dev(agg, d_vals, d_valid, ix, T, ov, oc)
                ctx.sync()
                outs.append((ov.cpu().numpy().reshape(G, T), oc.cpu().numpy().view(np.uint32).reshape(G, T)))
            what = f"{agg} T={T} {mode}"
            assert (h_cnt == e_cnt).all(), f"{what}: counts differ at {np.argwhere(h_cnt != e_cnt)[:4].tolist()}"
            assert_same_values(h_val, e_val, agg, what)
            assert (_bits(h_val[e_cnt == 0]) == 0).all(), f"{what}: empty cells must hold +0.0"
            for route, (v, c) in zip(("gid", "index"), outs):
                assert (c == h_cnt).all(), f"{what}: {route} counts differ from the host entry point"
                assert (_bits(v) == _bits(h_val)).all(), f"{what}: {route} values differ from the host entry point"
            if mode in FINITE_MODES:
                check_k3_against_exact(vals, valid, gid, G, agg, h_val, h_cnt, seed=T)
    finally:
        ctx.group_index_destroy(ix)


def test_group_aggregate_without_series_writes_empty_groups(ctx):
    """n_series = 0: every (group, step) is absent — cnt 0, value 0.0 — on all three entry points."""
    import torch
    G, T = 5, 40
    for agg in AGGS:
        h_val, h_cnt = ctx.group_aggregate(agg, np.zeros((0, T)), np.zeros((0, 2), np.uint32), np.zeros(0, np.uint32), G)
        assert (h_cnt == 0).all() and (_bits(h_val) == 0).all(), agg
        empty_v = torch.zeros(1, dtype=torch.float64, device="cuda:0")
        empty_w = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        ix = ctx.group_index_create_dev(empty_w, 0, G)
        try:
            for route in ("gid", "index"):
                ov = torch.full((G * T,), 7.25, dtype=torch.float64, device="cuda:0")
                oc = torch.full((G * T,), 99, dtype=torch.int32, device="cuda:0")
                if route == "gid":
                    ctx.group_aggregate_dev(agg, empty_v, empty_w, empty_w, 0, G, T, ov, oc)
                else:
                    ctx.group_aggregate_indexed_dev(agg, empty_v, empty_w, ix, T, ov, oc)
                ctx.sync()
                assert (oc.cpu().numpy() == 0).all() and (_bits(ov.cpu().numpy()) == 0).all(), (agg, route)
        finally:
            ctx.group_index_destroy(ix)


# ---------------------------------------------------------------------------------------------------------------------
# 2. Partial states, finalize and the cross-rank merge on one GPU
# ---------------------------------------------------------------------------------------------------------------------
def _partial(ctx, agg, vals, valid, gid, G):
    """b2p_group_aggregate_partial_dev -> (val, cnt, mean or None) as numpy [G x T]."""
    import torch
    S, T = vals.shape
    pv = torch.full((G * T,), 7.25, dtype=torch.float64, device="cuda:0")
    pc = torch.full((G * T,), 99, dtype=torch.int32, device="cuda:0")
    var = agg in ("stddev", "stdvar")
    pm = torch.full((G * T,), 7.25, dtype=torch.float64, device="cuda:0") if var else None
    d_vals = _dev(vals if S else np.zeros((1, T)))
    d_valid = _dev((valid if S else np.zeros((1, 1), np.uint32)).view(np.int32))
    d_gid = _dev((gid if S else np.zeros(1, np.uint32)).view(np.int32))
    ctx.group_aggregate_partial_dev(agg, d_vals, d_valid, d_gid, S, G, T, pv, pc, pm)
    ctx.sync()
    return (pv.cpu().numpy().reshape(G, T), pc.cpu().numpy().view(np.uint32).reshape(G, T),
            pm.cpu().numpy().reshape(G, T) if var else None)


def _total_key(v):
    b = np.ascontiguousarray(v).view(np.int64)
    return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


def merge_host(agg, parts):
    """The merge_partials arithmetic in numpy, over the partial states of every shard -> finished values and counts."""
    cnts = [p[1].astype(np.int64) for p in parts]
    cnt = sum(cnts)
    if agg in ("min", "max"):
        big = np.iinfo(np.int64).max if agg == "min" else np.iinfo(np.int64).min
        keys = [np.where(c > 0, _total_key(p[0]), big) for p, c in zip(parts, cnts)]
        key = np.minimum.reduce(keys) if agg == "min" else np.maximum.reduce(keys)
        val = _total_key(key).view(np.float64).copy()
    elif agg in ("stddev", "stdvar"):
        wsum = sum(c.astype(np.float64) * p[2] for p, c in zip(parts, cnts))
        mg = np.where(cnt > 0, wsum / np.maximum(cnt, 1), 0.0)
        m2 = sum(np.where(c > 0, p[0] + c * (p[2] - mg) ** 2, 0.0) for p, c in zip(parts, cnts))
        val = m2 / np.maximum(cnt, 1)
        if agg == "stddev":
            val = np.sqrt(val)
    else:
        val = sum(p[0] for p in parts)
        if agg == "avg":
            val = val / np.maximum(cnt, 1)
        elif agg == "count":
            val = cnt.astype(np.float64)
    val[cnt == 0] = 0.0
    return val, cnt


def _mixed_case(seed, T=70):
    """Finite normal data with 20 % holes over 23 groups, some series with the dropped id 23."""
    rng = np.random.default_rng(seed)
    S1, G1 = 600, 23
    vals1 = rng.normal(size=(S1, T)) * 10 + 3
    vb1 = rng.random((S1, T)) > 0.2
    vals1[~vb1] = 0.0
    gid1 = rng.integers(0, G1 + 1, S1).astype(np.uint32)   # id G1 is dropped
    return vals1, _words(vb1), gid1, G1


def test_partial_then_finalize_equals_the_single_pass(ctx):
    """group_aggregate_partial_dev then group_finalize_dev == the oracle's single pass, bit for bit (finalize performs
    the division and sqrt of K3); the stddev / stdvar state (cnt, mean, M2) == distributed.partial_state_host."""
    from greptimedb_b200 import distributed as D
    for vals, valid, gid, G in (_mixed_case(5), make_k3_case(33, "nan", 8), make_k3_case(65, "cancel", 9)):
        T = vals.shape[1]
        for agg in AGGS:
            e_val, e_cnt = orc.group_aggregate(agg, vals, valid, gid, G)
            pv, pc, pm = _partial(ctx, agg, vals, valid, gid, G)
            assert (pc == e_cnt).all(), agg
            if pm is not None:
                m2, hc, hmean = D.partial_state_host(agg, vals, valid, gid, G)
                assert (hc == pc).all(), agg
                assert_same_values(pv, m2, agg, f"{agg} partial M2")
                assert_same_values(pm, hmean, agg, f"{agg} partial mean")
            d_v, d_c = _dev(pv.ravel()), _dev(pc.ravel().view(np.int32))
            ctx.group_finalize_dev(agg, d_v, d_c, G * T)
            ctx.sync()
            assert_same_values(d_v.cpu().numpy().reshape(G, T), e_val, agg, f"{agg} partial + finalize")


def test_two_shards_on_one_gpu_merge_to_the_single_pass(ctx):
    """Device partials of two disjoint halves of the series, merged with the merge_partials arithmetic: min / max and
    counts exact (NaN and +-0 members on either half), sum / avg / stddev / stdvar within 1e-9 relative or 1e-9 of the
    data scale (the halves add in another order than the single pass)."""
    cases = [_mixed_case(6)]
    tv, tvalid, tgid, TG = total_order_case()
    cases.append((tv, tvalid, tgid, TG))
    for vals, valid, gid, G in cases:
        S = vals.shape[0]
        halves = [slice(0, S // 2), slice(S // 2, S)]
        scale = float(np.abs(vals[np.isfinite(vals)]).max())
        for agg in AGGS:
            e_val, e_cnt = orc.group_aggregate(agg, vals, valid, gid, G)
            parts = [_partial(ctx, agg, vals[h], valid[h], gid[h], G) for h in halves]
            got, cnt = merge_host(agg, parts)
            assert (cnt == e_cnt).all(), agg
            if agg in ("min", "max", "count"):
                assert (_bits(got) == _bits(e_val)).all(), f"two-shard {agg}: not bit for bit"
            else:
                fin = np.isfinite(e_val)
                assert (np.isnan(got) == np.isnan(e_val)).all(), agg
                assert (got[~fin & ~np.isnan(e_val)] == e_val[~fin & ~np.isnan(e_val)]).all(), agg
                err = np.abs(got[fin] - e_val[fin])
                bad = (err > 1e-9 * np.abs(e_val[fin])) & (err > 1e-9 * scale)
                assert not bad.any(), (agg, got[fin][bad][:3], e_val[fin][bad][:3])


def test_single_rank_communicator_round_trips_the_partials():
    """Over a one-rank communicator, allreduce_partials_dev: min / max partials (NaN payloads, -0.0, absent groups) come back
    bit for bit, absent groups as 0.0 whatever they held; variance states within 1e-12 relative or 1e-12 of the data
    scale (the one-rank mean cnt * mean / cnt may be an ulp off).  On one GPU this is the only run of the merge kernels
    and their total-order key conversion."""
    import torch
    from greptimedb_b200 import Context
    c = Context(0)
    try:
        c.use_torch_stream()
        with one_rank_comm(c):
            tv, tvalid, tgid, TG = total_order_case()
            for vals, valid, gid, G in ((tv, tvalid, tgid, TG), _mixed_case(7)):
                T = vals.shape[1]
                scale = float(np.abs(vals[np.isfinite(vals)]).max())
                for agg in ("min", "max", "stddev", "stdvar"):
                    pv, pc, pm = _partial(c, agg, vals, valid, gid, G)
                    sent = pv.copy()
                    sent[pc == 0] = 5.5                      # absent groups: whatever they hold reads 0.0 afterwards
                    d_v, d_c = _dev(sent.ravel()), _dev(pc.ravel().view(np.int32))
                    d_m = _dev(pm.ravel()) if pm is not None else None
                    torch.cuda.synchronize()
                    c.allreduce_partials_dev(agg, d_v, d_c, d_m, G * T)
                    c.sync()
                    got = d_v.cpu().numpy().reshape(G, T)
                    assert (d_c.cpu().numpy().view(np.uint32).reshape(G, T) == pc).all(), agg
                    if pm is None:
                        assert_same_values(got, pv, agg, f"one-rank {agg}")
                        continue
                    for g_, e_ in ((got, pv), (d_m.cpu().numpy().reshape(G, T), pm)):
                        assert (np.isnan(g_) == np.isnan(e_)).all(), agg
                        ok = ~np.isnan(e_)
                        err = np.abs(g_[ok] - e_[ok])
                        assert not ((err > 1e-12 * np.abs(e_[ok])) & (err > 1e-12 * scale ** 2)).any(), agg
                    assert (got[pc == 0] == 0.0).all(), agg
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. K5 HistogramFold: shared-validity path, compacted path, wide path (> 64 buckets)
# ---------------------------------------------------------------------------------------------------------------------
PHIS = (-0.1, 0.0, 0.25, 0.5, 0.99, 1.0, 1.5, float("nan"))
HIST_T = (1, 31, 32, 33, 70)
BOUND_KINDS = ("inf", "noinf", "dup", "nan_end", "unsorted")
COUNTER_KINDS = ("mono", "decreasing", "nonfinite", "equal", "zero")
VALID_KINDS = ("full", "holes", "tile_split", "absent_steps")


def _bounds(kind, B, rng):
    b = list(np.round(0.01 * 1.25 ** np.arange(B), 9))
    if B == 1:
        return [np.inf] if kind != "noinf" else [1.0]
    b[-1] = np.inf
    if kind == "noinf":
        b[-1] = 1e9
    elif kind == "dup":
        for i in rng.choice(np.arange(B - 1), max(1, B // 5), replace=False):
            if i > 0:
                b[i] = b[i - 1]
    elif kind == "nan_end":   # labels that do not parse sort last, behind +Inf
        nn = max(1, B // 10)
        b = b[:B - nn - 1] + [np.inf] + [np.nan] * nn if B > 2 else [np.inf, np.nan]
    elif kind == "unsorted" and B > 2:
        i = int(rng.integers(0, B - 2))
        b[i], b[i + 1] = b[i + 1], b[i]
    return b


def _counters(kind, B, T, rng):
    c = np.cumsum(rng.random((B, T)) * 5, axis=0)
    if kind == "decreasing":
        drop = rng.random((B, T)) < 0.2
        c[drop] -= rng.random(int(drop.sum())) * 10
    elif kind == "nonfinite":
        pick = rng.random((B, T)) < 0.15
        c[pick] = rng.choice([np.nan, np.inf, -np.inf], int(pick.sum()))
    elif kind == "equal":   # adjacent counters equal or within 1e-11: the `< 1e-10` branch answers NaN
        c = np.repeat(np.cumsum(rng.integers(0, 2, (B + 1) // 2 + 1))[:, None] * 1.0, T, axis=1)
        c = np.repeat(c, 2, axis=0)[:B] + (rng.random((B, T)) < 0.3) * 1e-11
    elif kind == "zero":
        c = np.zeros((B, T))
    return c


def _validity(kind, B, T, rng):
    if kind == "full":
        return np.ones((B, T), bool)
    if kind == "holes":
        return rng.random((B, T)) > 0.1
    if kind == "tile_split":          # shared validity in the first 32-step tile, holes from the second on
        v = np.ones((B, T), bool)
        v[:, 32:] = rng.random((B, max(T - 32, 0))) > 0.1
        return v
    steps = rng.random(T) > 0.3       # the whole histogram is absent at some steps: still shared validity
    return np.repeat(steps[None, :], B, axis=0)


def make_hist_case(T, seed):
    """A zoo of histograms in one index: every bucket count (1, 2, 5, 17, 64 on the shared-memory paths; 65, 100, 300 on
    the wide path) with every counter kind, bound kinds and validity kinds rotating.
    -> (specs, hist_off, les [n_buckets], rates [S x T], valid words)"""
    rng = np.random.default_rng(seed)
    specs, les, rates, vb = [], [], [], []
    i = 0
    for B in (1, 2, 5, 17, 64, 65, 100, 300):
        for ck in COUNTER_KINDS:
            bk, vk = BOUND_KINDS[i % len(BOUND_KINDS)], VALID_KINDS[(i // 2) % len(VALID_KINDS)]
            i += 1
            specs.append((B, bk, ck, vk))
            les += _bounds(bk, B, rng)
            rates.append(_counters(ck, B, T, rng))
            vb.append(_validity(vk, B, T, rng))
    hist_off = np.concatenate([[0], np.cumsum([s[0] for s in specs])]).astype(np.uint32)
    rates, vb = np.concatenate(rates), np.concatenate(vb)
    rates[~vb] = 0.0
    return specs, hist_off, np.array(les), rates, _words(vb)


def _le_label(x):
    if np.isnan(x):
        return "NaN"
    return "+Inf" if np.isinf(x) else repr(float(x))


def fold_rows(hist_off, les, rates, valid):
    """The rows the device folds, in scan order: per (histogram, step) the buckets with a sample, in index order.
    A leading one-bucket row group sends the literal fold into safe mode from the first row: the device folds every
    (histogram, step) on its own, which is safe mode's grouping (where the optimistic mode applies it gives the same
    values; test_histogram_fold_64_buckets_and_missing_buckets_match_the_row_literal_fold pins that)."""
    H, T = hist_off.size - 1, rates.shape[1]
    labels = [_le_label(x) for x in les]
    rows = [(("lead",), 0, "1", 1.0)]
    bits = ((valid[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(valid.shape[0], -1)[:, :T].astype(bool)
    for h in range(H):
        b0, b1 = int(hist_off[h]), int(hist_off[h + 1])
        present = bits[b0:b1].T.tolist()
        vals = rates[b0:b1].T.tolist()
        for k in range(T):
            rows += [((h,), k, labels[b0 + i], vals[k][i]) for i, p in enumerate(present[k]) if p]
    return rows


def literal_fold(rows, phi):
    """orc.histogram_fold_rows -> {(h, step): value}"""
    out = {}
    for tags, k, v in orc.histogram_fold_rows(rows, phi):
        if tags == ("lead",):
            continue
        assert (tags[0], k) not in out, "one output row per (histogram, step)"
        out[(tags[0], k)] = v
    return out


def assert_fold_matches(got, gv, exp, what):
    H, T = got.shape
    n_rows = 0
    for h in range(H):
        for k in range(T):
            has = bool((gv[h, k >> 5] >> (k & 31)) & 1)
            assert has == ((h, k) in exp), f"{what}: presence differs at histogram {h} step {k}"
            if not has:
                assert _bits(got[h, k:k + 1])[0] == 0, f"{what}: null slot ({h}, {k}) must hold 0.0"
                continue
            n_rows += 1
            e, g = exp[(h, k)], got[h, k]
            assert (np.isnan(e) and np.isnan(g)) or e == g or abs(e - g) <= 1e-12 * abs(e), (what, h, k, e, g)
    return n_rows


@pytest.mark.parametrize("T", HIST_T)
def test_histogram_fold_paths_match_the_row_literal_fold(ctx, T):
    """b2p_histogram_fold_dev with every layout of the zoo in one call, for every phi (< 0, 0, inside, 1, > 1, NaN):
    presence of every (histogram, step) exact, values NaN for NaN or within 1e-12 relative, null slots 0.0."""
    import torch
    specs, hist_off, les, rates, valid = make_hist_case(T, seed=100 + T)
    H, Tw = len(specs), (T + 31) // 32
    d_off, d_bs = _dev(hist_off.view(np.int32)), _dev(np.arange(les.size, dtype=np.int32))
    d_le, d_rates, d_valid = _dev(les), _dev(rates), _dev(valid.view(np.int32))
    rows = fold_rows(hist_off, les, rates, valid)
    for phi in PHIS:
        out = torch.full((H * T,), 7.25, dtype=torch.float64, device="cuda:0")
        ov = torch.full((H * Tw,), -1, dtype=torch.int32, device="cuda:0")
        torch.cuda.synchronize()
        ctx.histogram_fold_dev(phi, d_off, d_bs, d_le, H, d_rates, d_valid, T, out, ov)
        ctx.sync()
        got, gv = out.cpu().numpy().reshape(H, T), ov.cpu().numpy().view(np.uint32).reshape(H, Tw)
        n = assert_fold_matches(got, gv, literal_fold(rows, phi), f"fold T={T} phi={phi}")
        assert n > H * T // 3


@pytest.mark.parametrize("B", (1, 2, 64, 65, 100, 300))
def test_histogram_quantile_uniform_front_end_matches_the_row_literal_fold(ctx, B):
    """b2p_histogram_quantile (every histogram has the same bounds): histograms with each counter kind and validity kind
    (shared-validity, compacted and, above 64 buckets, wide path), bounds with duplicates and NaN labels at the end."""
    rng = np.random.default_rng(B)
    for bk in ("inf", "dup", "nan_end"):
        for T in (1, 33, 70):
            le = np.array(_bounds(bk, B, rng))
            rates, vb = [], []
            for i, ck in enumerate(COUNTER_KINDS):
                rates.append(_counters(ck, B, T, rng))
                vb.append(_validity(VALID_KINDS[(i + T) % len(VALID_KINDS)], B, T, rng))
            rates, vb = np.concatenate(rates), np.concatenate(vb)
            rates[~vb] = 0.0
            valid = _words(vb)
            H = rates.shape[0] // B
            rows = fold_rows((np.arange(H + 1) * B).astype(np.uint32), np.tile(le, H), rates, valid)
            for phi in PHIS:
                got, gv = ctx.histogram_quantile(phi, le, rates, valid)
                assert_fold_matches(got, gv, literal_fold(rows, phi), f"uniform B={B} {bk} T={T} phi={phi}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. K6 column reduce
# ---------------------------------------------------------------------------------------------------------------------
COL_KINDS = ("normal", "holes", "all_nan", "inf", "inf_both", "cancel")


def _column(kind, n, rng):
    if kind == "normal":
        return rng.normal(size=n) * 1e3
    if kind == "holes":
        v = rng.normal(size=n)
        v[rng.random(n) < 0.1] = np.nan
        return v
    if kind == "all_nan":
        return np.full(n, np.nan)
    if kind == "inf":                 # sum +inf
        v = rng.normal(size=n)
        v[rng.integers(0, n)] = np.inf
        return v
    if kind == "inf_both":            # +inf and -inf: the sum is NaN (when n >= 2)
        v = rng.normal(size=n)
        v[0], v[-1] = np.inf, -np.inf
        return v
    v = rng.normal(size=n) * 1e-3     # heavy cancellation: +-1e16 pairs around small values
    big = rng.random(n) < 0.3
    v[big] = 1e16 * np.where(np.arange(int(big.sum())) % 2 == 0, 1.0, -1.0)
    return v


def _ieee_sum(x):
    """The IEEE result a finite-precision sum of x must have, with fsum for the finite part."""
    x = x[~np.isnan(x)]
    pos, neg = bool(np.isposinf(x).any()), bool(np.isneginf(x).any())
    if pos and neg:
        return math.nan
    if pos or neg:
        return math.inf if pos else -math.inf
    return math.fsum(x)


# every (rows, columns) pair but 200 003 x 1 100 (1.8 GB on the host; the one-block-per-column path of 1 100 columns is
# covered by the smaller row counts)
COL_SHAPES = [(r, c) for r in (1, 2, 3, 511, 512, 513, 200_003) for c in (1, 3, 32, 1100) if r * c <= 50_000_000]


@pytest.mark.parametrize("n_rows,n_cols", COL_SHAPES)
def test_column_reduce_edges(ctx, n_rows, n_cols):
    """Per-column (sum, count) with NaN rows skipped, called twice to check that it accumulates: counts exact; sums
    against math.fsum within n * 2^-53 * sum|x| when finite, the IEEE inf / NaN otherwise.  Columns are 16-byte aligned
    (even row stride), as the header requires.  With 1 100 columns every column gets one block."""
    import torch
    rng = np.random.default_rng(n_rows * 7 + n_cols)
    rotations = range(len(COL_KINDS)) if n_cols < len(COL_KINDS) else range(1)
    for rot in rotations:
        kinds = [COL_KINDS[(c + rot) % len(COL_KINDS)] for c in range(n_cols)]
        stride = n_rows + (n_rows & 1)
        data = np.zeros((n_cols, stride))
        for c, kd in enumerate(kinds):
            data[c, :n_rows] = _column(kd, n_rows, rng)
        d = _dev(data)
        ptrs = torch.tensor([d.data_ptr() + c * stride * 8 for c in range(n_cols)], dtype=torch.int64, device="cuda:0")
        out_sum = torch.zeros(n_cols, dtype=torch.float64, device="cuda:0")
        out_cnt = torch.zeros(n_cols, dtype=torch.int64, device="cuda:0")
        torch.cuda.synchronize()
        ctx.column_reduce_dev(ptrs, n_cols, n_rows, out_sum, out_cnt)
        ctx.sync()
        s1, c1 = out_sum.cpu().numpy().copy(), out_cnt.cpu().numpy().copy()
        ctx.column_reduce_dev(ptrs, n_cols, n_rows, out_sum, out_cnt)
        ctx.sync()
        s2, c2 = out_sum.cpu().numpy(), out_cnt.cpu().numpy()
        assert (c2 == 2 * c1).all() and ((_bits(s2) == _bits(s1 + s1)) | (np.isnan(s1) & np.isnan(s2))).all(), \
            "a second call adds the same partials again"
        for c, kd in enumerate(kinds):
            x = data[c, :n_rows]
            n = int((~np.isnan(x)).sum())
            assert c1[c] == n, (kd, c)
            e = _ieee_sum(x)
            what = (kd, c, n_rows, float(s1[c]), e)
            if math.isnan(e):
                assert np.isnan(s1[c]), what
            elif math.isinf(e):
                assert s1[c] == e, what
            else:
                bound = n * EPS * float(np.nansum(np.abs(x)))
                assert abs(s1[c] - e) <= bound, what


# ---------------------------------------------------------------------------------------------------------------------
# 5. sum(rate()) tables of tql/range.result on the device
# ---------------------------------------------------------------------------------------------------------------------
def _sum_rate_cases():
    import json
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "reference_sum_rate_vectors.json")) as f:
        return json.load(f)


SUM_RATE = _sum_rate_cases()


@pytest.mark.parametrize("case", SUM_RATE["cases"], ids=lambda c: c["name"])
def test_sum_rate_reference_tables_on_the_device(ctx, case):
    """Every printed value of range.result, exactly (== like test_sum_rate_reference_tables), through (a) range_eval +
    group_aggregate("sum"), (b) range_group_sum_indexed_dev, fused where the first tier applies, and (c) PromRangeExec
    with aggregate="sum"."""
    import pyarrow as pa
    import torch
    from greptimedb_b200 import make_params
    from greptimedb_b200.plan import PromRangeExec
    scale = case.get("scale", 1.0)
    keep = [s for s in SUM_RATE["series"] if all(s[k] == v for k, v in case["filter"].items())]
    T = orc.num_steps(case["start"], case["end"], case["interval"])
    p = make_params("rate", case["start"], case["end"], case["interval"], case["range"])

    def table(keys, gsum, gcnt):
        return [[dict(zip(case["by"], key)), case["start"] + k * case["interval"], float(gsum[g, k]) * scale]
                for g, key in enumerate(keys) for k in range(T) if gcnt[g, k]]

    if keep:
        ts = np.concatenate([np.array(s["ts"], np.int64) for s in keep])
        val = np.concatenate([np.array(s["val"], np.float64) for s in keep])
        offsets = np.concatenate([[0], np.cumsum([len(s["ts"]) for s in keep])]).astype(np.uint64)
        keys = sorted({tuple(s[t] for t in case["by"]) for s in keep})
        gid = np.array([keys.index(tuple(s[t] for t in case["by"])) for s in keep], np.uint32)
        S, G = len(keep), len(keys)
        # (a) two passes through the host API
        out, valid, _ = ctx.range_eval(p, ts, val, offsets=offsets)
        gsum, gcnt = ctx.group_aggregate("sum", out, valid, gid, G)
        assert table(keys, gsum, gcnt) == case["expected"], "range_eval + group_aggregate"
        # (b) the fused device route
        d_ts, d_val, d_off = _dev(ts), _dev(val), _dev(offsets.view(np.int64))
        d_gid = _dev(gid.view(np.int32))
        torch.cuda.synchronize()
        ix = ctx.group_index_create_dev(d_gid, S, G)
        try:
            # the first tier needs range >= interval (its end trim); the 31 s range at a 60 s step takes the two-pass
            # route of the same entry point
            assert ctx.range_group_sum_fused(p, ix) == (case["range"] >= case["interval"])
            fs = torch.zeros(G * T, dtype=torch.float64, device="cuda:0")
            fc = torch.zeros(G * T, dtype=torch.int32, device="cuda:0")
            ctx.range_group_sum_indexed_dev(p, d_ts, d_val, d_off, ts.size, S, ix, 0, G, fs, fc)
            ctx.sync()
            assert table(keys, fs.cpu().numpy().reshape(G, T), fc.cpu().numpy().reshape(G, T)) == case["expected"], \
                "fused range_group_sum_indexed_dev"
        finally:
            ctx.group_index_destroy(ix)
    # (c) the plan node on a RecordBatch of the matched rows (empty when the matchers select nothing)
    tags = SUM_RATE["tags"]
    cols = {"ts": [], "val": [], **{t: [] for t in tags}}
    for s in keep:
        cols["ts"] += s["ts"]
        cols["val"] += s["val"]
        for t in tags:
            cols[t] += [s[t]] * len(s["ts"])
    batch = pa.record_batch([pa.array(cols["ts"], pa.timestamp("ms")), pa.array(cols["val"], pa.float64())] +
                            [pa.array(cols[t], pa.string()) for t in tags], names=["ts", "val"] + tags)
    ex = PromRangeExec(ctx, "prom_rate", case["start"], case["end"], case["interval"], case["range"], "ts", "val", tags,
                       aggregate="sum", by_columns=case["by"])
    try:
        ex.push(batch)
        res = ex.execute()
    finally:
        ex.close()
    ts_out = res.column("ts").cast(pa.int64()).to_pylist()
    by_vals = [res.column(b).to_pylist() for b in case["by"]]
    got = [[{b: by_vals[j][i] for j, b in enumerate(case["by"])}, ts_out[i], v * scale]
           for i, v in enumerate(res.column(res.num_columns - 1).to_pylist())]
    assert got == case["expected"], "PromRangeExec(aggregate='sum')"
