"""sum by (..)(rate | increase | delta(..)) on one GPU, on every route the library has for it (run with -m gpu):

  * range_group_sum_indexed_dev over [0, G) and over split group ranges;
  * range_group_sum_allreduce_dev (the config-3 entry point) in 1, 2, 3, 7, G and G + 5 tiles, without a communicator
    and with a one-rank NCCL communicator (which all-reduces every tile on the communication stream), also with 16 SMs
    left to the collective and no head start;
  * their fallbacks (range eval + the by-label kernel, then the all-reduce of the partials);

each on contexts that pin the first tier's variant (the probe's choice, uniform cadence on / off, the bit-word variant).
Results are compared with tests/sum_by_check.py's reference over the oracle's rescan grid, which every range tier
reproduces bit for bit:

  * bits: the first tier adds a group's members in series-id order and a series it hands on adds its remaining steps
    after every first-tier member, so when at most one member of a group leaves the tier and it is the group's last
    member, every route gives the series-order sum's bits;
  * bound: otherwise every sum is within gamma(n - 1) * sum |x| of the exact sum, counts bit for bit.

Every test asserts the route it means from range_group_sum_fused(), last_warp_tier_series() and last_slow_series(); a
tiled call's counters cover all of its tiles.
"""
import contextlib
import functools
import os

import numpy as np
import pytest

from oracle import oracle as orc
from tests import sum_by_check as sbc
from tests.ranks import one_rank_comm
from tests.range_values import F64_MAX, SUBNORMAL

pytestmark = pytest.mark.gpu

THREADS = max(1, min(16, os.cpu_count() or 1))
SC = 15_000
T0 = 10_000_000
POSITIONS = (0, 1, 31, 32, 63, 64, 65, -2, -1)   # 64-row blocks, pairs and groups of 32 steps, the tail
B2P_E_INVALID = -1


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
    """One context per first-tier route, the adaptive policy off so that each runs the variant it names.  "comm" and
    "comm16" carry a one-rank communicator (absent when NCCL cannot be loaded); "comm16" leaves 16 SMs to the collective
    while the next tile computes and gives it no head start."""
    off = {"B2P_LEAN_ADAPTIVE": "0"}
    c = {"default": _context(**off), "uniform": _context(B2P_UNIFORM="1", **off),
         "general": _context(B2P_UNIFORM="0", **off), "flags": _context(B2P_LEAN_FORCE_FLAGS="1", **off)}
    with contextlib.ExitStack() as comms:
        for name, env in (("comm", {}), ("comm16", {"B2P_COMM_RESERVE_SMS": "16", "B2P_COMM_HEADSTART_US": "0"})):
            x = _context(**off, **env)
            try:
                comms.enter_context(one_rank_comm(x))
            except pytest.skip.Exception:  # NCCL cannot be loaded: the routes without a communicator still run
                x.close()
                continue
            c[name] = x
        for x in c.values():
            x.use_own_stream()
        yield c
    for x in c.values():
        x.close()


# ---------------------------------------------------------------------------------------------------
# routes
# ---------------------------------------------------------------------------------------------------
class Dev:
    """device copies of one data set and its group ids"""

    def __init__(self, ts, val, offsets, gid):
        import torch
        dev = torch.device("cuda:0")
        self.S = offsets.size - 1
        self.n_rows = int(offsets[-1])
        pad = lambda a: a if a.size else np.zeros(2, a.dtype)   # (an empty column still needs an aligned pointer)
        self.ts = torch.from_numpy(pad(np.ascontiguousarray(ts, np.int64))).to(dev)
        self.val = torch.from_numpy(pad(np.ascontiguousarray(val, np.float64))).to(dev)
        self.off = torch.from_numpy(np.ascontiguousarray(offsets, np.uint64).astype(np.int64)).to(dev)
        self.gid = torch.from_numpy(np.ascontiguousarray(gid, np.uint32).astype(np.int32)).to(dev)
        torch.cuda.synchronize()


def routes(G, fused=True):
    """(name, kind, arg): group ranges of indexed_dev (split ones only where the call runs fused), or the tile count
    of allreduce_dev"""
    r = [("indexed", "indexed", [(0, G)])]
    if fused:
        r.append(("indexed split", "indexed", [(0, 1), (1, G // 2), (G // 2, G)]))
    for n in sorted({1, 2, 3, 7, G, G + 5}):
        r.append((f"allreduce {n} tiles", "allreduce", n))
    return r


def run_route(c, p, d, ix, G, T, kind, arg, init=None):
    """-> (sum [G, T], count [G, T] u32, series handed on by the first tier, series on the slow kernel), the counters
    summed over the calls of a split route"""
    import torch
    dev = torch.device("cuda:0")
    gsum = torch.zeros(G * T, dtype=torch.float64, device=dev) if init is None else \
        torch.from_numpy(init[0].ravel().copy()).to(dev)
    gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev) if init is None else \
        torch.from_numpy(init[1].ravel().astype(np.int32)).to(dev)
    torch.cuda.synchronize()
    handed = slow = 0
    if kind == "indexed":
        for lo, hi in arg:
            c.range_group_sum_indexed_dev(p, d.ts, d.val, d.off, d.n_rows, d.S, ix, lo, hi, gsum, gcnt)
            c.sync()
            handed += c.last_warp_tier_series()
            slow += c.last_slow_series()
    else:
        c.range_group_sum_allreduce_dev(p, d.ts, d.val, d.off, d.n_rows, d.S, ix, arg, gsum, gcnt)
        c.sync()
        handed, slow = c.last_warp_tier_series(), c.last_slow_series()
    torch.cuda.synchronize()
    return (gsum.cpu().numpy().reshape(G, T), gcnt.cpu().numpy().view(np.uint32).reshape(G, T), handed, slow)


def every_route(ctxs, p, d, G, T, fused, names=None):
    """Runs every route on every context (names: a subset) and yields (label, context name, route kind, result);
    asserts range_group_sum_fused() == fused on each context first."""
    for cname, c in ctxs.items():
        if names is not None and cname not in names:
            continue
        ix = c.group_index_create_dev(d.gid, d.S, G)
        try:
            assert c.range_group_sum_fused(p, ix) == fused, f"{cname}: range_group_sum_fused() is not {fused}"
            for rname, kind, arg in routes(G, fused):
                yield f"{cname} {rname}", cname, kind, run_route(c, p, d, ix, G, T, kind, arg)
        finally:
            c.group_index_destroy(ix)


def orc_params(p):
    return orc.make_params(p.fn_id, p.start, p.end, p.interval, p.range, offset=p.offset,
                           filter_nan=bool(p.filter_nan), param0=p.param0, param1=p.param1)


def oracle_grid(p, ts, val, offsets):
    return orc.range_query(orc_params(p), ts, val, None, offsets, threads=THREADS, rescan=True)


def c13_series(p, ts, val, offsets, series):
    """the series among `series` whose reference windows differ from the definitional ones (cursor overshoot, DESIGN
    C-13): only the exact slow kernel reproduces them"""
    out = []
    for s in series:
        o0, o1 = int(offsets[s]), int(offsets[s + 1])
        t, _ = orc.normalize(ts[o0:o1], val[o0:o1], p.offset, bool(p.filter_nan))
        a = orc.calculate_range(t, p.start, p.end, p.interval, p.range)
        e = orc.calculate_range(t, p.start, p.end, p.interval, p.range, definitional=True)
        if not (a[2:] == e[2:] and (a[1] == e[1]).all() and (a[0][a[1] > 0] == e[0][e[1] > 0]).all()):
            out.append(s)
    return out


# ---------------------------------------------------------------------------------------------------
# 2a. one defective last member per group: bit for bit on every route
# ---------------------------------------------------------------------------------------------------
DEFECTS = ("nan", "reset", "late", "missing", "dup", "burst", "dense")


def class_values(cls, n, rng):
    """n non-decreasing samples of a value class (no counter reset anywhere)"""
    if cls == "counter":
        return np.cumsum(1.0 + rng.random(n) * 10)
    if cls == "zeros":
        return rng.choice([0.0, -0.0], n)
    if cls == "subnormal":
        return np.cumsum(rng.integers(1, 1000, n)).astype(np.float64) * SUBNORMAL
    if cls == "huge":
        return F64_MAX * (0.5 + 0.49 * np.sort(rng.random(n)))
    if cls == "inf":
        v = np.cumsum(1.0 + rng.random(n) * 10)
        v[int(rng.integers(n // 2, n)):] = np.inf
        return v
    raise ValueError(cls)


def below(x):
    """a sample that is a counter reset after x"""
    if np.isinf(x):
        return F64_MAX
    return x * 0.5 if x > 0 else -1.0


def plant(kind, i, t, v):
    """series (t, v) with one defect at sample position i"""
    t, v = t.copy(), v.copy()
    if kind == "nan":
        v[i] = np.nan
    elif kind == "reset":
        if i > 0:
            v[i] = below(v[i - 1])
    elif kind == "late":
        t[i] += 1
    elif kind == "missing":
        t, v = np.delete(t, i), np.delete(v, i)
    elif kind == "dup":
        t, v = np.insert(t, i, t[i]), np.insert(v, i, v[i])
    elif kind == "burst":     # 300 samples 1 ms apart after sample i: windows beyond the 256 ring, mostly quirk C-13
        t = np.insert(t, i + 1, t[i] + 1 + np.arange(300))
        v = np.insert(v, i + 1, np.full(300, v[i]))
    elif kind == "dense":     # 300 samples spread over the scrape after sample i: windows beyond the 256 ring
        t = np.insert(t, i + 1, t[i] + 1 + (np.arange(300) * (SC - 2)) // 300)
        v = np.insert(v, i + 1, np.full(300, v[i]))
    else:
        raise ValueError(kind)
    return t, v


@functools.lru_cache(maxsize=None)
def handoff_set(cls, seed=5, n=200, K=4):
    """G groups of K members, group of series s = s % G (members interleaved), the last member (highest series id) of
    each group defective: every kind of DEFECTS at every position of POSITIONS, an empty series, a one-sample series,
    and two groups without a defect.  -> (ts, val, offsets, gid, G, {series: (kind, position)})"""
    rng = np.random.default_rng(seed)
    plan = [(k, i) for k in DEFECTS for i in POSITIONS] + [("empty", 0), ("one", 0), ("clean", 0), ("clean", 0)]
    G = len(plan)
    S = G * K
    ts_l, val_l, kinds = [], [], {}
    for s in range(S):
        g, m = s % G, s // G
        t = T0 + np.arange(n, dtype=np.int64) * SC
        v = class_values(cls, n, rng)
        if m == K - 1:
            kind, i = plan[g]
            kinds[s] = (kind, i)
            if kind == "empty":
                t, v = t[:0], v[:0]
            elif kind == "one":
                t, v = t[n // 2:n // 2 + 1], v[n // 2:n // 2 + 1]
            elif kind != "clean":
                t, v = plant(kind, i % n, t, v)
        ts_l.append(t)
        val_l.append(v)
    offsets = np.concatenate([[0], np.cumsum([x.size for x in ts_l])]).astype(np.uint64)
    gid = (np.arange(S) % G).astype(np.uint32)
    return np.concatenate(ts_l), np.concatenate(val_l), offsets, gid, G, kinds


@pytest.mark.parametrize("fn,cls", [("rate", "counter"), ("increase", "counter"), ("delta", "counter"),
                                    ("rate", "huge"), ("increase", "subnormal"), ("delta", "zeros"),
                                    ("rate", "inf"), ("delta", "huge"), ("delta", "subnormal")])
def test_one_hand_off_per_group_adds_in_member_order_on_every_route(ctxs, fn, cls):
    """At most one member of a group leaves the first tier, and it is the group's last: every route, tile count,
    variant and communicator gives the series-order sum's bits.  The planted series that must leave the tier (a NaN
    sample, a counter reset on the plain variant, windows beyond the 256 ring, quirk C-13, an empty series) are counted
    by last_warp_tier_series(), and no clean member leaves; the series with quirk C-13 reach the slow kernel.  Every
    route reports the same counters as the one-call indexed route."""
    from greptimedb_b200 import make_params
    ts, val, offsets, gid, G, kinds = handoff_set(cls)
    n_ev = 200 + 4
    start = T0 + SC // 2
    p = make_params(fn, start, start + n_ev * SC, SC, 4 * SC)
    T = n_ev + 1
    out, vw = oracle_grid(p, ts, val, offsets)
    ref = sbc.reference(out, vw, gid, G)
    d = Dev(ts, val, offsets, gid)
    planted = len([k for k, _ in kinds.values() if k != "clean"])
    c13 = c13_series(p, ts, val, offsets, kinds)
    assert c13, "the bursts must produce quirk C-13 windows"
    counters = {}
    for label, cname, kind, (got, cnt, handed, slow) in every_route(ctxs, p, d, G, T, True):
        sbc.check(ref, got, cnt, "bits", f"{fn} {cls} {label}")
        plain = fn != "delta" and cname != "flags"
        must = sum(1 for s, (k, i) in kinds.items()
                   if k in ("nan", "burst", "dense", "empty") or (k == "reset" and i != 0 and plain) or s in c13)
        assert must <= handed <= planted, f"{fn} {cls} {label}: {handed} series handed on, {must} .. {planted} expected"
        assert len(c13) <= slow <= planted, f"{fn} {cls} {label}: {slow} on the slow kernel, {len(c13)} have C-13"
        first = counters.setdefault(cname, (handed, slow))
        assert (handed, slow) == first, f"{fn} {cls} {label}: counters {(handed, slow)}, one indexed call {first}"


# ---------------------------------------------------------------------------------------------------
# 2b. many hand-offs per group: the error bound on every route, routes agree, bits where nothing leaves
# ---------------------------------------------------------------------------------------------------
def sum_by_case(S, N, G, resets, nan_every, seed, jitter=1000):
    from greptimedb_b200 import distributed as D
    T0b = 1_700_000_000_000
    ts, val, _ = orc.synth_fill(0, S, N, T0b, SC, jitter, resets, seed)
    if nan_every:
        val[nan_every // 2::nan_every] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
    return T0b, ts, val, offsets, gid


@pytest.mark.parametrize("fn,resets,nan_every,jitter", [
    ("rate", 1, 0, 1000), ("rate", 0, 613, 1000), ("increase", 1, 997, 0), ("delta", 1, 401, 1000),
    ("rate", 0, 0, 0), ("delta", 0, 0, 1000)])
def test_many_hand_offs_per_group_hold_the_bound_on_every_route(ctxs, fn, resets, nan_every, jitter):
    S, N, G = 1200, 500, 37
    T0b, ts, val, offsets, gid = sum_by_case(S, N, G, resets, nan_every, 17, jitter)
    from greptimedb_b200 import make_params
    p = make_params(fn, T0b, T0b + (N - 1) * SC, SC, 300_000)
    T = N
    out, vw = oracle_grid(p, ts, val, offsets)
    ref = sbc.reference(out, vw, gid, G)
    d = Dev(ts, val, offsets, gid)
    results, tiles1 = [], {}
    for label, cname, kind, res in every_route(ctxs, p, d, G, T, True):
        got, cnt, handed, slow = res
        sbc.check(ref, got, cnt, "bound", f"{fn} {label}")
        leaves = nan_every > 0 or (resets and fn != "delta" and cname != "flags")
        if leaves:
            assert handed > 0, f"{fn} {label}: series with NaN samples / resets must leave the first tier"
        else:
            assert handed == 0 and slow == 0, f"{fn} {label}: nothing leaves the first tier ({handed}, {slow})"
            # nothing leaves: every route adds in member order, the same bits as one tile
            if label.endswith("allreduce 1 tiles"):
                tiles1[cname] = got
            elif kind == "allreduce":
                assert (got.view(np.uint64) == tiles1[cname].view(np.uint64)).all(), f"{fn} {label} vs 1 tile"
            sbc.check(ref, got, cnt, "bits", f"{fn} {label}")
        results.append((label, got, cnt))
    a = results[0]
    for b in results[1:]:
        sbc.check_pair((a[1], a[2]), (b[1], b[2]), ref, f"{fn} {a[0]} vs {b[0]}")


# ---------------------------------------------------------------------------------------------------
# 2c. group shapes and gates
# ---------------------------------------------------------------------------------------------------
def two_pass(c, p, d, G, T):
    """range_eval_dev + the by-label kernel's sum (K3) over the same group index"""
    import torch
    dev = torch.device("cuda:0")
    out = torch.zeros(max(d.S, 1) * T, dtype=torch.float64, device=dev)
    vw = torch.zeros(max(d.S, 1) * ((T + 31) // 32), dtype=torch.int32, device=dev)
    gsum = torch.zeros(G * T, dtype=torch.float64, device=dev)
    gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()   # (the context's own stream does not wait for torch's)
    ix = c.group_index_create_dev(d.gid, d.S, G)
    try:
        c.range_eval_dev(p, d.ts, d.val, d.off, d.n_rows, d.S, out, vw)
        c.sync()
        c.group_aggregate_indexed_dev("sum", out, vw, ix, T, gsum, gcnt)
        c.sync()
    finally:
        c.group_index_destroy(ix)
    torch.cuda.synchronize()
    return gsum.cpu().numpy().reshape(G, T), gcnt.cpu().numpy().view(np.uint32).reshape(G, T)


def shapes_set(n=120, seed=3):
    """regular counters; groups: empty ones, groups of one, groups holding only empty series, and series whose group id
    is >= n_groups (they belong to no group).  -> (ts, val, offsets, gid, G)"""
    rng = np.random.default_rng(seed)
    G = 24
    gid = []
    ts_l, val_l = [], []
    layout = [(g, 3) for g in range(0, 8)] + [(g, 1) for g in range(8, 14)] + [(g, -2) for g in range(14, 18)] + \
             [(G, 2), (G + 7, 1)]                 # groups 18 .. 23 stay empty
    for g, m in layout:
        for _ in range(abs(m)):
            empty = m < 0
            k = 0 if empty else n - int(rng.integers(0, 3))
            ts_l.append(T0 + np.arange(k, dtype=np.int64) * SC)
            val_l.append(np.cumsum(1.0 + rng.random(k)))
            gid.append(g)
    order = rng.permutation(len(gid))
    ts_l, val_l = [ts_l[i] for i in order], [val_l[i] for i in order]
    offsets = np.concatenate([[0], np.cumsum([x.size for x in ts_l])]).astype(np.uint64)
    return np.concatenate(ts_l), np.concatenate(val_l), offsets, np.array(gid, np.uint32)[order], G


def test_group_shapes_on_every_route(ctxs):
    """Empty groups, groups of one, groups of empty series only, and group ids >= n_groups (dropped on every route):
    the fused routes give the series-order bits (only the empty series leave, and each is its group's only kind of
    member), the fallback of the same call (avg_over_time has no fused tier) the two-pass route's bits."""
    from greptimedb_b200 import B2PError, make_params
    ts, val, offsets, gid, G = shapes_set()
    d = Dev(ts, val, offsets, gid)
    start = T0 + SC // 2
    n_empty = int(((np.diff(offsets) == 0) & (gid < G)).sum())   # (series of groups >= n_groups are never walked)
    for fn in ("rate", "delta", "avg_over_time"):
        p = make_params(fn, start, start + 124 * SC, SC, 4 * SC)
        T = 125
        out, vw = oracle_grid(p, ts, val, offsets)
        ref = sbc.reference(out, vw, gid, G)
        fused = fn != "avg_over_time"
        for label, cname, kind, (got, cnt, handed, slow) in every_route(ctxs, p, d, G, T, fused,
                                                                        names=("default", "comm")):
            sbc.check(ref, got, cnt, "bits" if fused else "bound", f"{fn} {label}")
            if fused:
                # (the later tiers hand an empty series on to the slow kernel)
                assert handed == n_empty and slow <= n_empty, \
                    f"{fn} {label}: ({handed}, {slow}) handed on / slow, only the {n_empty} empty series leave the first tier"
        if not fused:
            c = ctxs["default"]
            tp = two_pass(c, p, d, G, T)
            ix = c.group_index_create_dev(d.gid, d.S, G)
            try:
                for kind, arg in (("indexed", [(0, G)]), ("allreduce", 1), ("allreduce", 4)):
                    got, cnt, _, _ = run_route(c, p, d, ix, G, T, kind, arg)
                    assert (got.view(np.uint64) == tp[0].view(np.uint64)).all() and (cnt == tp[1]).all(), \
                        f"{fn} {kind} {arg}: the fallback differs from range eval + K3 sum"
                # a group range needs the fused tier
                import torch
                gs = torch.zeros(G * T, dtype=torch.float64, device="cuda:0")
                gc = torch.zeros(G * T, dtype=torch.int32, device="cuda:0")
                with pytest.raises(B2PError) as e:
                    c.range_group_sum_indexed_dev(p, d.ts, d.val, d.off, d.n_rows, d.S, ix, 0, G // 2, gs, gc)
                assert e.value.code == B2P_E_INVALID
            finally:
                c.group_index_destroy(ix)


def test_empty_group_range_and_no_series(ctxs):
    """g_lo == g_hi adds nothing; a call over no series adds nothing on the fused, merged and fallback routes."""
    import torch
    from greptimedb_b200 import make_params
    ts, val, offsets, gid, G = shapes_set()
    d = Dev(ts, val, offsets, gid)
    start = T0 + SC // 2
    T = 125
    c = ctxs["default"]
    ix = c.group_index_create_dev(d.gid, d.S, G)
    try:
        p = make_params("rate", start, start + 124 * SC, SC, 4 * SC)
        for lo in (0, 5, G):
            got, cnt, _, _ = run_route(c, p, d, ix, G, T, "indexed", [(lo, lo)])
            assert not got.any() and not cnt.any(), f"g_lo == g_hi == {lo} added something"
    finally:
        c.group_index_destroy(ix)
    none = Dev(np.zeros(0, np.int64), np.zeros(0), np.zeros(1, np.uint64), np.zeros(0, np.uint32))
    for fn in ("rate", "avg_over_time"):
        p = make_params(fn, start, start + 124 * SC, SC, 4 * SC)
        for cname in ("default", "comm"):
            if cname not in ctxs:
                continue
            c = ctxs[cname]
            ix = c.group_index_create_dev(none.gid, 0, G)
            try:
                for kind, arg in (("indexed", [(0, G)]), ("allreduce", 1), ("allreduce", 3)):
                    init = (np.full((G, T), 2.5), np.full((G, T), 3, np.uint32))
                    got, cnt, _, _ = run_route(c, p, none, ix, G, T, kind, arg, init=init)
                    assert (got == 2.5).all() and (cnt == 3).all(), f"{fn} {cname} {kind} {arg}: no series changed the partials"
            finally:
                c.group_index_destroy(ix)


def test_balance_gate_and_step_gate(ctxs):
    """The fused tier walks a group with one warp: it runs up to max_members = 8 * share + 64 (share from the SM
    count, as fused_group_ok computes it) and falls back one member later; it runs up to T = 8192 steps and falls back
    at 8193.  Both sides of each gate against the reference, fused in bits (nothing leaves), fallback in bits against
    range eval + K3 sum."""
    import torch
    from greptimedb_b200 import make_params
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps = sms * 1 * 24
    rng = np.random.default_rng(9)
    n = 40
    start = T0 + SC // 2
    c = ctxs["default"]
    # balance gate: S series, one big group of 8 * share + 64 (+1) members, the rest in groups of 4
    S = 4000
    share = S // warps + 1
    for big, fused in ((8 * share + 64, True), (8 * share + 65, False)):
        gid = np.concatenate([np.zeros(big, np.uint32), 1 + np.arange(S - big, dtype=np.uint32) // 4])
        gid = gid[rng.permutation(S)]
        G = int(gid.max()) + 1
        ts = np.tile(T0 + np.arange(n, dtype=np.int64) * SC, S)
        val = np.cumsum(1.0 + rng.random((S, n)), axis=1).ravel()
        offsets = np.arange(S + 1, dtype=np.uint64) * n
        d = Dev(ts, val, offsets, gid)
        p = make_params("rate", start, start + (n + 4) * SC, SC, 4 * SC)
        T = n + 5
        out, vw = oracle_grid(p, ts, val, offsets)
        ref = sbc.reference(out, vw, gid, G)
        tp = two_pass(c, p, d, G, T) if not fused else None
        for label, cname, kind, (got, cnt, handed, slow) in every_route(ctxs, p, d, G, T, fused,
                                                                        names=("default", "comm")):
            sbc.check(ref, got, cnt, "bits" if fused else "bound", f"balance {big} {label}")
            if not fused:
                assert (got.view(np.uint64) == tp[0].view(np.uint64)).all(), f"balance {big} {label} vs two-pass"
            assert handed == 0 and slow == 0
    # step gate: T = 8192 (fused) and 8193 (fallback) over a few long series; and short grids
    S, n = 64, 8200
    gid = (np.arange(S) % 5).astype(np.uint32)
    ts = np.tile(T0 + np.arange(n, dtype=np.int64) * SC, S)
    val = np.cumsum(1.0 + rng.random((S, n)), axis=1).ravel()
    offsets = np.arange(S + 1, dtype=np.uint64) * n
    d = Dev(ts, val, offsets, gid)
    for T, fused in ((8192, True), (8193, False), (1, True), (31, True), (32, True), (33, True), (63, True),
                     (64, True), (65, True)):
        p = make_params("increase", start, start + (T - 1) * SC, SC, 4 * SC)
        out, vw = oracle_grid(p, ts, val, offsets)
        ref = sbc.reference(out, vw, gid, 5)
        tp = two_pass(c, p, d, 5, T)
        for cname in ("default", "comm"):
            if cname not in ctxs:
                continue
            cc = ctxs[cname]
            ix = cc.group_index_create_dev(d.gid, d.S, 5)
            try:
                assert cc.range_group_sum_fused(p, ix) == fused, f"T={T}"
                for kind, arg in (("indexed", [(0, 5)]), ("allreduce", 1), ("allreduce", 3)):
                    got, cnt, handed, slow = run_route(cc, p, d, ix, 5, T, kind, arg)
                    what = f"T={T} {cname} {kind} {arg}"
                    sbc.check(ref, got, cnt, "bits", what)
                    assert (got.view(np.uint64) == tp[0].view(np.uint64)).all() and (cnt == tp[1]).all(), what
                    assert handed == 0 and slow == 0, what
            finally:
                cc.group_index_destroy(ix)


def test_int64_time_domain_falls_back(ctxs):
    """A query span beyond the 32-bit time domain has no fused tier: indexed_dev and allreduce_dev (with and without a
    communicator) give range eval + K3 sum's bits."""
    from greptimedb_b200 import make_params
    sc = 10_000_000
    S, n = 48, 230
    rng = np.random.default_rng(4)
    t0 = 1_000_000_000_000
    ts = np.tile(t0 + np.arange(n, dtype=np.int64) * sc, S)
    val = np.cumsum(1.0 + rng.random((S, n)), axis=1).ravel()
    val[::53] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * n
    gid = (np.arange(S) % 7).astype(np.uint32)
    G = 7
    d = Dev(ts, val, offsets, gid)
    p = make_params("rate", t0 + sc // 2, t0 + sc // 2 + (n + 2) * sc, sc, 5 * sc)
    T = n + 3
    out, vw = oracle_grid(p, ts, val, offsets)
    ref = sbc.reference(out, vw, gid, G)
    for cname in ("default", "comm"):
        if cname not in ctxs:
            continue
        c = ctxs[cname]
        tp = two_pass(c, p, d, G, T)
        sbc.check(ref, tp[0], tp[1], "bound", "two-pass")
        ix = c.group_index_create_dev(d.gid, d.S, G)
        try:
            assert not c.range_group_sum_fused(p, ix)
            for kind, arg in (("indexed", [(0, G)]), ("allreduce", 1), ("allreduce", 4)):
                got, cnt, _, _ = run_route(c, p, d, ix, G, T, kind, arg)
                assert (got.view(np.uint64) == tp[0].view(np.uint64)).all() and (cnt == tp[1]).all(), \
                    f"{cname} {kind} {arg}: the int64-domain fallback differs from range eval + K3 sum"
        finally:
            c.group_index_destroy(ix)


def test_calls_add_into_partials_two_shards(ctxs):
    """Output buffers that already hold partials: a call adds into them.  Two shards of the series (the first ids
    below the second's), called one after the other into one buffer, stand in for two ranks: the series-order bits of
    the whole set, on every route."""
    from greptimedb_b200 import make_params
    ts, val, offsets, gid, G, _ = handoff_set("counter")
    S = offsets.size - 1
    cut = S // 2
    start = T0 + SC // 2
    p = make_params("rate", start, start + 204 * SC, SC, 4 * SC)
    T = 205
    out, vw = oracle_grid(p, ts, val, offsets)
    ref = sbc.reference(out, vw, gid, G)
    shards = []
    for lo, hi in ((0, cut), (cut, S)):
        r0, r1 = int(offsets[lo]), int(offsets[hi])
        shards.append(Dev(ts[r0:r1], val[r0:r1], offsets[lo:hi + 1] - offsets[lo], gid[lo:hi]))
    for cname, c in ctxs.items():
        for rname, kind, arg in routes(G):
            acc = None
            for d in shards:
                ix = c.group_index_create_dev(d.gid, d.S, G)
                try:
                    got, cnt, _, _ = run_route(c, p, d, ix, G, T, kind, arg, init=acc)
                finally:
                    c.group_index_destroy(ix)
                acc = (got, cnt)
            # the second shard's defective last members leave after the first shard's members were added: still in
            # series order, because every one of them is its group's last member overall
            sbc.check(ref, acc[0], acc[1], "bits", f"two shards {cname} {rname}")


# ---------------------------------------------------------------------------------------------------
# 2d. config 3 at full size
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("resets", [0, 1], ids=["no_resets", "resets"])
def test_config3_full_size(ctxs, resets):
    """1.25 M series x 1000 samples, 100 k groups (synth_fill_dev, jitter 0): allreduce_dev at 1 and 4 tiles,
    indexed_dev and the two-pass route agree (counts equal, sums within 2 gamma(n - 1) sum |x|, sum |x| from the two-pass
    grid on the device), and 64 seeded groups hold the bound against the oracle over their member series."""
    import torch
    from greptimedb_b200 import distributed as D
    from greptimedb_b200 import make_params
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(0)
    if free < 48 * 2 ** 30:
        pytest.skip(f"needs 48 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    dev = torch.device("cuda:0")
    S, N, G, T0c, seed = 1_250_000, 1000, 100_000, 1_700_000_000_000, 0x5EED + resets
    c = ctxs["comm"] if "comm" in ctxs else ctxs["default"]
    ts = torch.empty(S * N, dtype=torch.int64, device=dev)
    val = torch.empty(S * N, dtype=torch.float64, device=dev)
    sid = torch.empty(S * N, dtype=torch.int32, device=dev)
    c.synth_fill_dev(0, S, N, T0c, SC, 0, resets, seed, ts, val, sid)
    del sid
    off = torch.arange(S + 1, dtype=torch.int64, device=dev) * N
    gid_h = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
    gid = torch.from_numpy(gid_h.astype(np.int32)).to(dev)
    p = make_params("rate", T0c, T0c + (N - 1) * SC, SC, 300_000)
    T = N
    torch.cuda.synchronize()
    ix = c.group_index_create_dev(gid, S, G)
    res = {}
    try:
        assert c.range_group_sum_fused(p, ix)

        class _D:   # the device columns in the shape run_route takes
            pass
        d = _D()
        d.ts, d.val, d.off, d.n_rows, d.S = ts, val, off, S * N, S
        for name, kind, arg in (("allreduce 1", "allreduce", 1), ("allreduce 4", "allreduce", 4),
                                ("indexed", "indexed", [(0, G)])):
            got, cnt, handed, slow = run_route(c, p, d, ix, G, T, kind, arg)
            res[name] = (got, cnt, handed, slow)
        # two-pass, and sum |x| by group on the device from the same grid
        out = torch.empty(S * T, dtype=torch.float64, device=dev)
        vw = torch.empty(S * ((T + 31) // 32), dtype=torch.int32, device=dev)
        c.range_eval_dev(p, ts, val, off, S * N, S, out, vw)
        c.sync()
        gs = torch.zeros(G * T, dtype=torch.float64, device=dev)
        gc = torch.zeros(G * T, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()   # (the context's own stream does not wait for torch's)
        c.group_aggregate_indexed_dev("sum", out, vw, ix, T, gs, gc)
        c.sync()
        tp = (gs.cpu().numpy().reshape(G, T), gc.cpu().numpy().view(np.uint32).reshape(G, T))
        bits = vw.view(torch.uint8).reshape(S, -1)
        shifts = torch.arange(8, device=dev, dtype=torch.uint8)
        valid = ((bits.unsqueeze(-1) >> shifts) & 1).reshape(S, -1)[:, :T].bool()
        del bits
        o = out.view(S, T)
        o.abs_()
        o.masked_fill_(~valid, 0.0)
        del valid
        mag = torch.zeros(G, T, dtype=torch.float64, device=dev)
        mag.index_add_(0, gid.long(), o)
        mag = mag.cpu().numpy()
        del out, o, vw
    finally:
        c.group_index_destroy(ix)
    # 64 seeded groups against the oracle over their member series (their rows copied back from the device)
    rng = np.random.default_rng(64)
    order = np.sort(rng.choice(G, 64, replace=False))
    members = np.flatnonzero(np.isin(gid_h, order))
    rows = torch.from_numpy((members[:, None] * N + np.arange(N)).ravel()).to(dev)
    m_ts, m_val = ts[rows].cpu().numpy(), val[rows].cpu().numpy()
    del ts, val, rows
    torch.cuda.empty_cache()
    o_out, o_vw = oracle_grid(p, m_ts, m_val, np.arange(members.size + 1, dtype=np.uint64) * N)
    ref = sbc.reference(o_out, o_vw, np.searchsorted(order, gid_h[members]).astype(np.uint32), 64)
    res["two-pass"] = tp + (None, None)
    for name, (got, cnt, _, _) in res.items():
        sbc.check(ref, got[order], cnt[order], "bound", f"config 3 {name}, seeded groups")
    # every group: the routes against the two-pass route
    cnt_ref = tp[1]
    bound = 2.0 * sbc.gamma(np.maximum(cnt_ref.astype(np.float64) - 1.0, 0.0)) * mag
    assert res["allreduce 1"][2] == res["allreduce 4"][2] == res["indexed"][2], \
        f"hand-off counters differ between routes: {[(k, v[2], v[3]) for k, v in res.items()]}"
    assert (res["indexed"][2] > 0) == bool(resets), "resets must send series on (plain variant), none without"
    for name, (got, cnt, _, _) in res.items():
        bad = cnt != cnt_ref
        assert not bad.any(), f"{name}: {int(bad.sum())} counts differ from the two-pass route at {np.argwhere(bad)[:4]}" \
                              f": {cnt[bad][:4]} vs {cnt_ref[bad][:4]}"
        bad = np.abs(got - tp[0]) > bound
        assert not bad.any(), f"{name}: {int(bad.sum())} sums beyond 2 gamma(n-1) mag of the two-pass route"


# ---------------------------------------------------------------------------------------------------
# 2e. the counters of a tiled call cover all of its tiles
# ---------------------------------------------------------------------------------------------------
def nan_everywhere(S=2000, n=300, G=50, seed=8, c13_every=0):
    """every series carries one NaN sample; with c13_every, every c13_every-th series also a 300-sample burst (quirk
    C-13, the slow kernel)"""
    rng = np.random.default_rng(seed)
    ts_l, val_l = [], []
    for s in range(S):
        t = T0 + np.arange(n, dtype=np.int64) * SC
        v = np.cumsum(1.0 + rng.random(n))
        v[int(rng.integers(0, n))] = np.nan
        if c13_every and s % c13_every == 0:
            t, v = plant("burst", int(rng.integers(0, 66)), t, v)
        ts_l.append(t)
        val_l.append(v)
    offsets = np.concatenate([[0], np.cumsum([x.size for x in ts_l])]).astype(np.uint64)
    return np.concatenate(ts_l), np.concatenate(val_l), offsets, (np.arange(S) % G).astype(np.uint32), G


def test_tiled_call_counts_every_tile(ctxs):
    """Every series of S carries a NaN sample: last_warp_tier_series() == S for 4 tiles exactly as for one; with
    series of quirk C-13 spread over all tiles, last_slow_series() counts every one of them."""
    from greptimedb_b200 import make_params
    start = T0 + SC // 2
    for c13_every in (0, 7):
        ts, val, offsets, gid, G = nan_everywhere(c13_every=c13_every)
        S = offsets.size - 1
        d = Dev(ts, val, offsets, gid)
        p = make_params("rate", start, start + 304 * SC, SC, 4 * SC)
        T = 305
        out, vw = oracle_grid(p, ts, val, offsets)
        ref = sbc.reference(out, vw, gid, G)
        c13 = c13_series(p, ts, val, offsets, range(0, S, c13_every)) if c13_every else []
        assert not c13_every or len(c13) > 100
        counts = {}
        for cname in ("default", "comm", "comm16"):
            if cname not in ctxs:
                continue
            c = ctxs[cname]
            ix = c.group_index_create_dev(d.gid, S, G)
            try:
                assert c.range_group_sum_fused(p, ix)
                for kind, arg in (("allreduce", 1), ("allreduce", 4), ("indexed", [(0, G)])):
                    got, cnt, handed, slow = run_route(c, p, d, ix, G, T, kind, arg)
                    what = f"{cname} {kind} {arg} c13_every={c13_every}"
                    sbc.check(ref, got, cnt, "bound", what)
                    assert handed == S, f"{what}: {handed} of {S} series counted as handed on"
                    assert slow >= len(c13), f"{what}: {slow} on the slow kernel, {len(c13)} have quirk C-13"
                    one = counts.setdefault(cname, slow)
                    assert slow == one, f"{what}: {slow} on the slow kernel, {one} in one tile"
            finally:
                c.group_index_destroy(ix)


def test_tiled_call_drives_the_adaptive_verdict():
    """With the adaptive policy on, the verdict of a tiled call weighs the hand-offs of all its tiles: a tiled delta
    call that hands on every series makes the next call skip the first tier (range_group_sum_fused() is False); a
    tiled reset-heavy rate call makes the next call run the bit-word variant, which keeps the reset series."""
    import torch
    from greptimedb_b200 import make_params
    c = _context(B2P_LEAN_ADAPTIVE="1")
    try:
        c.use_own_stream()
        start = T0 + SC // 2
        ts, val, offsets, gid, G = nan_everywhere()
        S = offsets.size - 1
        d = Dev(ts, val, offsets, gid)
        p = make_params("delta", start, start + 304 * SC, SC, 4 * SC)
        T = 305
        ix = c.group_index_create_dev(d.gid, S, G)
        try:
            assert c.range_group_sum_fused(p, ix)
            _, _, handed, _ = run_route(c, p, d, ix, G, T, "allreduce", 4)
            assert handed == S
            assert not c.range_group_sum_fused(p, ix), "every series was handed on: the first tier must back off"
        finally:
            c.group_index_destroy(ix)
        # counters with a reset in every series (and no NaN): the plain variant hands every one on
        rng = np.random.default_rng(12)
        n = 300
        v = np.cumsum(1.0 + rng.random((S, n)), axis=1)
        at = rng.integers(1, n, S)
        v[np.arange(S), at] = v[np.arange(S), at - 1] * 0.5
        t = np.tile(T0 + np.arange(n, dtype=np.int64) * SC, S)
        offsets = np.arange(S + 1, dtype=np.uint64) * n
        d = Dev(t, v.ravel(), offsets, gid)
        p = make_params("rate", start, start + 304 * SC, SC, 4 * SC)
        out, vw = oracle_grid(p, t, v.ravel(), offsets)
        ref = sbc.reference(out, vw, gid, G)
        ix = c.group_index_create_dev(d.gid, S, G)
        try:
            got, cnt, handed, _ = run_route(c, p, d, ix, G, T, "allreduce", 4)
            sbc.check(ref, got, cnt, "bound", "reset-heavy rate, 4 tiles")
            assert handed == S, f"the plain variant hands on every reset series ({handed} of {S})"
            assert c.range_group_sum_fused(p, ix)
            got, cnt, handed, _ = run_route(c, p, d, ix, G, T, "allreduce", 4)
            sbc.check(ref, got, cnt, "bound", "rate on the bit-word variant, 4 tiles")
            assert handed <= S // 100, f"the bit-word variant keeps the reset series ({handed} of {S} handed on)"
        finally:
            c.group_index_destroy(ix)
        torch.cuda.synchronize()
    finally:
        c.close()
