"""CPU: the key-space generator of tests/select_keys.py lays out what each class claims, and its plain reference agrees
with the oracles the feature tests use (aggregate_oracle.group_quantile, topk_oracle.topk,
count_values_oracle.count_values, sort_oracle.value_order) on the same grids."""
import math

import numpy as np
import pytest

from tests import aggregate_oracle as ago
from tests import count_values_oracle as cvo
from tests import select_keys as sk
from tests import sort_oracle as so
from tests import topk_oracle as tko

PHIS = [0.0, -0.0, 1.0, 0.5, 1 / 3, 0.25, np.nextafter(0.25, 0.0)]
NS = [1, 2, 3, 7, 64, 65, 257]


@pytest.mark.parametrize("cls", sk.CLASSES)
def test_round_trip_by_bits(cls):
    rng = np.random.default_rng(sk.CLASSES.index(cls))
    for n in NS:
        for phi in (0.5, 1.0, 0.0):
            u = sk.column(cls, n, phi, rng)
            bits = sk.value_of(u)
            assert (sk.key_of(bits) == u).all(), (cls, n)
            assert (sk.value_of(sk.key_of(bits)) == bits).all(), (cls, n)
            v = sk.values_of_keys(u)
            assert (sk.keys_of_values(v) == u).all(), (cls, n)


def test_key_is_the_total_order():
    v = np.array([-np.inf, -1e300, -1.0, -5e-324, -0.0, 0.0, 5e-324, 2.2250738585072014e-308, 1.0, np.inf])
    u = sk.keys_of_values(v)
    assert (np.diff(u.astype(object)) > 0).all()
    assert int(sk.key_of(np.array([0xFFFFFFFFFFFFFFFF], np.uint64))[0]) == 0
    assert int(sk.key_of(np.array([0x7FFFFFFFFFFFFFFF], np.uint64))[0]) == 2 ** 64 - 1
    # the total order's key from an independent restatement
    for b in (0x0, 0x1, 0x7FF0000000000001, 0xFFF8000000000000, 0x8000000000000000, 0xC000000000000000):
        x = np.array([b], np.uint64).view(np.float64)[0]
        assert int(sk.key_of(np.array([b], np.uint64))[0]) == (tko.total_key(x) ^ (1 << 63)) & (2 ** 64 - 1)


def bins_under(s, ref, d):
    """digit d of the keys of s that share ref's first d digits"""
    if d == 0:
        return sk.digit(s, 0)
    shift = np.uint64(64 - 8 * d)
    under = (s >> shift) == (np.uint64(ref) >> shift)
    return sk.digit(s[under], d)


@pytest.mark.parametrize("d", sk.DEPTHS)
@pytest.mark.parametrize("variant", sk.DEPTH_VARIANTS)
def test_depth_classes_differ_first_at_their_digit(d, variant):
    rng = np.random.default_rng(100 * d + len(variant))
    cls = f"depth{d}-{variant}"
    for n in NS[1:]:
        for phi in PHIS:
            s = np.sort(sk.column(cls, n, phi, rng))
            a, b = sk.pair(n, phi)
            assert sk.first_diff_digit(s[a], s[b]) == d, (cls, n, phi)
            assert np.isfinite(sk.values_of_keys(s)).all()
            x, y = int(sk.digit(s[a], d)), int(sk.digit(s[b], d))
            if variant in ("adjacent", "last"):
                assert y == x + 1
            elif variant == "gap":
                assert y >= x + 2
            bins = bins_under(s, s[a], d)
            if variant == "first":  # cum == k: every key below s[a] under the prefix sits in a lower bin
                assert (bins == x).sum() == 1 and (bins < x).sum() == a, (cls, n, phi)
            if variant == "last":  # cum + c == k + 1 with c = a + 1: s[a] ends a full bin
                assert (bins == x).sum() == a + 1 and (bins < x).sum() == 0, (cls, n, phi)


def test_other_classes_have_their_property():
    rng = np.random.default_rng(3)
    for n in NS:
        for phi in (0.0, 0.5, 1.0):
            a, b = sk.pair(n, phi) if n > 1 else (0, 0)
            lo, hi = sk.order_stats(n, phi)
            col = lambda c: np.sort(sk.column(c, n, phi, rng))
            assert len(set(col("equal").tolist())) == 1
            s = col("top")
            assert s[-1] > s[-2] if n > 1 else True
            assert len(set((s >> np.uint64(8)).tolist())) == 1
            s = col("sentinel-lo0")
            assert s[a] == 0 and (n == 1 or s[b] == sk.ALL)
            s = col("sentinel-lomax")
            assert (s[a:] == sk.ALL).all() and s[lo] == sk.ALL
            s = col("sentinel-hi0")
            assert (s[:b + 1] == 0).all() and s[hi] == 0
            assert (col("sentinel-only0") == 0).all() and (col("sentinel-onlymax") == sk.ALL).all()
            v = sk.values_of_keys(col("ulps-zero"))
            assert (np.abs(v) < 1e-322).all()
            s = col("ulps-subnormal")
            v = np.abs(sk.values_of_keys(s))
            assert ((v > 2.2250738585072014e-308 * (1 - 1e-15)) & (v < 2.2250738585072014e-308 * (1 + 1e-15))).all()
            v = sk.values_of_keys(col("ulps-inf"))
            assert (np.abs(v) >= 1.79769313486231e308).all()
            v = sk.values_of_keys(col("signed-zero"))
            assert (v == 0).all()
            v = sk.values_of_keys(col("payloads"))
            assert np.isnan(v).all() and len(set(v.view(np.uint64).tolist())) >= min(n, 2)
    s = sk.values_of_keys(sk.column("signed-zero", 200, 0.5, rng))
    assert {math.copysign(1.0, x) for x in s} == {1.0, -1.0}
    s = sk.values_of_keys(sk.column("payloads", 200, 0.5, rng))
    assert {math.copysign(1.0, x) for x in s} == {1.0, -1.0}


def test_grid_gives_each_lane_of_a_tile_its_own_class():
    rng = np.random.default_rng(4)
    vals, ok, gid, n_groups, names = sk.grid([1, 70], 40, 0.5, rng, drop=0.2, gid_gap=2, stray=3)
    assert n_groups == 4 and (gid == n_groups + 7).sum() == 3
    assert len(set(names[1, :32].tolist())) == 32
    assert ok[gid == 0].all() and not ok[gid == 2].all()  # a group of one member is never thinned
    assert not ok[gid == n_groups + 7].any()


@pytest.mark.parametrize("phi", PHIS + [float("nan"), -0.5, 1.5])
def test_quantile_agrees_with_the_aggregate_oracle(phi):
    rng = np.random.default_rng(5)
    vals, ok, gid, G, _ = sk.grid([1, 2, 5, 64, 65, 130], 33, phi, rng, drop=0.1, gid_gap=2, stray=2)
    out, cnt = sk.quantile(phi, vals, ok, gid, G)
    eout, ecnt = ago.group_quantile(phi, vals, sk.words(ok), gid, G)
    assert (cnt == ecnt).all()
    assert sk.same_or_nan(out, eout)


@pytest.mark.parametrize("bottom", [0, 1])
@pytest.mark.parametrize("kk", [1, 2, 32, 33, 1000])
def test_topk_agrees_with_the_topk_oracle(bottom, kk):
    rng = np.random.default_rng(6 + kk)
    vals, ok, gid, G, _ = sk.grid([1, 2, 40, 34], 35, 0.5, rng, drop=0.2, gid_gap=2, stray=2)
    tie = rng.permutation(gid.size).astype(np.uint32)
    tie[:2] = [0, 0xFFFFFFFF]
    got = sk.topk(bottom, kk, vals, ok, gid, G, tie)
    exp = tko.topk(bottom, float(kk), vals, sk.words(ok), gid, G, tie)
    assert (sk.words(got) == exp).all()


def test_count_values_agrees_with_the_count_values_oracle():
    rng = np.random.default_rng(7)
    vals, ok, gid, G, _ = sk.grid([1, 2, 9, 70], 40, 0.5, rng, drop=0.3, gid_gap=2, stray=2)
    out, cnt = sk.count_values(vals, ok, gid, G)
    eout, ecnt = cvo.count_values(vals, sk.words(ok), gid, G)
    assert (cnt == ecnt).all() and sk.same_bits(out, eout)


@pytest.mark.parametrize("desc", [False, True])
def test_sort_agrees_with_the_sort_oracle(desc):
    rng = np.random.default_rng(8)
    vals, ok, gid, G, _ = sk.grid([3, 9, 70], 40, 0.5, rng, drop=0.3)
    assert (sk.sort(desc, vals, ok) == so.value_order(vals, ok, desc)).all()
