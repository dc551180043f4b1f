"""The sum-by checker (tests/sum_by_check.py) has teeth: the series-order sum and a shuffled-order sum of the same grid
pass its bound mode, and the faults a fused group sum could make are rejected — a member's value taken from the
neighbouring step, a member added twice, a one-ulp change (bits mode) and a count off by one.  CPU only."""
import functools

import numpy as np
import pytest

from oracle import oracle as orc
from tests import sum_by_check as sbc

T0, SC = 1_700_000_000_000, 15_000


@functools.lru_cache(maxsize=None)
def grid():
    """rate over 240 counters (resets, jitter, a few NaN samples), 13 groups by hash: (out, valid words, gid, G)"""
    from greptimedb_b200 import distributed as D
    S, N, G = 240, 200, 13
    ts, val, sid = orc.synth_fill(0, S, N, T0, SC, 1000, 1, 7)
    val[50::997] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    p = orc.make_params("rate", T0, T0 + (N - 1) * SC, SC, 120_000)
    out, vw = orc.range_query(p, ts, val, sid, offsets, rescan=True)
    gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
    return out, vw, gid, G


@functools.lru_cache(maxsize=None)
def ref():
    out, vw, gid, G = grid()
    return sbc.reference(out, vw, gid, G)


def members_at(g, k):
    out, vw, gid, _ = grid()
    vb = orc.valid_to_bool(vw, out.shape[1])
    return [s for s in np.flatnonzero(gid == g) if vb[s, k]]


def shuffled_sum(seed):
    """the group sums, every cell's members added in a random order"""
    out, vw, gid, G = grid()
    rng = np.random.default_rng(seed)
    T = out.shape[1]
    vb = orc.valid_to_bool(vw, T)
    res = np.zeros((G, T))
    for g in range(G):
        for k in range(T):
            m = [s for s in np.flatnonzero(gid == g) if vb[s, k]]
            acc = 0.0
            for s in rng.permutation(m):
                acc += out[s, k]
            res[g, k] = acc
    return res


def test_series_order_and_shuffled_sums_pass_the_bound():
    r = ref()
    assert (r.cnt > 10).mean() > 0.9, "the groups must be large enough for the order to matter"
    sbc.check(r, r.seq, r.cnt, "bits", "series order")
    sbc.check(r, r.seq, r.cnt, "bound", "series order")
    sh = shuffled_sum(3)
    assert (sh.view(np.uint64) != r.seq.view(np.uint64)).any(), "a shuffled order must change some bits"
    sbc.check(r, sh, r.cnt, "bound", "shuffled")
    sbc.check_pair((r.seq, r.cnt), (sh, r.cnt), r, "series order vs shuffled")
    with pytest.raises(AssertionError, match="series-order"):
        sbc.check(r, sh, r.cnt, "bits", "shuffled")


def _largest_member_cell(r, want):
    """(g, k, s, delta) of a cell whose change `want(s, k) -> delta` is larger than 16 x the bound there"""
    out, _, _, G = grid()
    T = out.shape[1]
    for g in range(G):
        for k in range(T - 1):
            if r.cnt[g, k] < 4 or r.cls[g, k] != 0.0:
                continue
            bound = sbc.gamma(r.cnt[g, k] - 1) * r.mag[g, k]
            for s in members_at(g, k):
                d = want(s, k)
                if np.isfinite(d) and abs(d) > 16 * bound:
                    return g, k, s, d
    raise AssertionError("no cell to perturb")


def test_neighbouring_step_value_is_rejected():
    r = ref()
    out = grid()[0]
    vb = orc.valid_to_bool(grid()[1], out.shape[1])
    g, k, s, d = _largest_member_cell(r, lambda s, k: out[s, k + 1] - out[s, k] if vb[s, k + 1] else np.nan)
    bad = r.seq.copy()
    bad[g, k] += d              # member s's value of step k + 1 in place of step k, count unchanged
    with pytest.raises(AssertionError, match="error bound"):
        sbc.check(r, bad, r.cnt, "bound", "neighbouring step")


def test_member_added_twice_is_rejected():
    r = ref()
    out = grid()[0]
    g, k, s, d = _largest_member_cell(r, lambda s, k: out[s, k])
    bad = r.seq.copy()
    bad[g, k] += d              # member s added twice, the count as the reference has it
    with pytest.raises(AssertionError, match="error bound"):
        sbc.check(r, bad, r.cnt, "bound", "member twice")
    cnt = r.cnt.copy()
    cnt[g, k] += 1              # ... and with its count moved along: the count is wrong then
    with pytest.raises(AssertionError, match="counts differ"):
        sbc.check(r, bad, cnt, "bound", "member twice, counted")


def test_one_ulp_is_rejected_in_bits_mode_only():
    r = ref()
    g, k = np.argwhere((r.cnt > 4) & (r.cls == 0.0) & (r.seq != 0.0))[0]
    bad = r.seq.copy()
    bad[g, k] = np.nextafter(bad[g, k], np.inf)
    with pytest.raises(AssertionError, match="series-order"):
        sbc.check(r, bad, r.cnt, "bits", "one ulp")
    sbc.check(r, bad, r.cnt, "bound", "one ulp")
    z = r.seq.copy()
    g0, k0 = np.argwhere(r.cnt == 0)[0] if (r.cnt == 0).any() else (g, k)
    if r.cnt[g0, k0] == 0:
        z[g0, k0] = -0.0        # +0.0 and -0.0 differ in bits mode
        with pytest.raises(AssertionError, match="series-order"):
            sbc.check(r, z, r.cnt, "bits", "signed zero")


def test_count_off_by_one_is_rejected():
    r = ref()
    g, k = np.argwhere(r.cnt > 0)[len(np.argwhere(r.cnt > 0)) // 2]
    for delta in (1, -1):
        cnt = r.cnt.astype(np.int64)
        cnt[g, k] += delta
        for mode in ("bits", "bound"):
            with pytest.raises(AssertionError, match="counts differ"):
                sbc.check(r, r.seq, cnt.astype(np.uint32), mode, "count")


def test_non_finite_classes_and_overflow():
    """NaN / +-inf cells must keep their class; a sum of huge members may overflow to inf of exact's sign only."""
    F = sbc.F64_MAX
    out = np.array([[F * 0.75, 1.0, np.inf, np.nan, 1.0, F * 0.9, 1e300],
                    [F * 0.75, 2.0, -np.inf, 1.0, -F, F * 0.9, 1e300],
                    [-F * 0.25, 3.0, 1.0, 2.0, -F, -F * 0.9, -1e300]])
    vw = np.full((3, 1), 0x7F, np.uint32)
    gid = np.zeros(3, np.uint32)
    r = sbc.reference(out, vw, gid, 1)
    assert np.isnan(r.cls[0, 2]) and np.isnan(r.cls[0, 3]) and r.scale[0, 0] < 1.0
    # exact = 1.25 MAX and -2 MAX: inf of that sign; exact = 0.9 MAX with 1.8 MAX of positive members: an order that
    # adds the positive ones first overflows
    got = np.array([[np.inf, 6.0, np.nan, np.nan, -np.inf, np.inf, 1e300]])
    sbc.check(r, got, r.cnt, "bound", "overflowing order")
    got[0, 5] = F * 0.9
    sbc.check(r, got, r.cnt, "bound", "order without overflow")
    for i, wrong in ((0, -np.inf), (2, np.inf), (3, 3.0), (4, np.inf), (5, -np.inf), (6, np.inf)):
        bad = got.copy()
        bad[0, i] = wrong
        with pytest.raises(AssertionError):
            sbc.check(r, bad, r.cnt, "bound", f"cell {i}")
    none = sbc.reference(out, vw, np.full(3, 5, np.uint32), 1)      # gid >= n_groups: no member
    sbc.check(none, np.zeros((1, 7)), np.zeros((1, 7), np.uint32), "bits", "no member")
