"""CPU: the multi-field plan restatement (tests/multifield_plan_oracle.py) against the single-field oracles it is built
from, its zip and naming rules, the lexicographic sort, and the refusal texts against the reference's goldens."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as orc
from tests import binary_oracle as bo
from tests import multifield_plan_oracle as mp
from tests import select_keys as sk
from tests import subquery_oracle as sq

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_multifield_refusal_vectors.json")


def grid(F, R, T, seed, drop=0.2):
    rng = np.random.default_rng(seed)
    vals = rng.normal(0, 10, (F, R, T))
    ok = rng.random((R, T)) > drop
    return vals, sk.words(ok), ok


def test_one_field_is_each_single_field_oracle():
    vals, valid, ok = grid(1, 6, 40, 1)
    o, w = mp.scalar_op("*", 3.0, vals, valid)
    e, ew = bo.scalar_op("*", 3.0, vals[0], valid)
    assert np.array_equal(o[0], e) and np.array_equal(w, ew)
    o, w = mp.scalar_op(">", 0.0, vals, valid)  # a filter is fine with one field
    e, ew = bo.scalar_op(">", 0.0, vals[0], valid)
    assert np.array_equal(o[0], e) and np.array_equal(w, ew)
    lrow = np.array([0, 1, 2, 5], np.uint32)
    rrow = np.array([3, 3, 4, 0], np.uint32)
    o, w = mp.binary_op("-", vals, valid, lrow, vals, valid, rrow)
    e, ew = bo.binary_op("-", vals[0], valid, lrow, vals[0], valid, rrow)
    assert np.array_equal(o[0], e) and np.array_equal(w, ew)
    gid = np.array([0, 1, 0, 1, 2, 0], np.uint32)
    o, c = mp.aggregate("stddev", vals, valid, gid, 3)
    e, ec = orc.group_aggregate("stddev", vals[0], valid, gid, 3)
    assert np.array_equal(o[0], e) and np.array_equal(c, ec)
    o, c = mp.aggregate("group", vals, valid, gid, 3)
    assert np.array_equal(o[0], np.where(ec != 0, 1.0, 0.0))
    s, step, T_in = sq.inner_grid(1_000_000, 1_340_000, 10_000, 60_000)
    assert T_in == 40
    o, w = mp.subquery("max_over_time", 1_000_000, 1_340_000, 10_000, 60_000, s, step, vals, valid)
    e, ew = sq.subquery("max_over_time", 1_000_000, 1_340_000, 10_000, 60_000, s, step, vals[0], valid)
    assert np.array_equal(o[0], e) and np.array_equal(w, ew)
    assert np.array_equal(mp.sort(True, vals, ok), sk.sort(True, vals[0], ok))
    assert np.array_equal(mp.sort(False, vals, ok), sk.sort(False, vals[0], ok))


@pytest.mark.parametrize("FL,FR", [(2, 2), (3, 2), (2, 3), (1, 3), (3, 1)])
def test_binary_zip(FL, FR):
    L, lv, _ = grid(FL, 4, 35, FL * 10 + FR)
    R, rv, _ = grid(FR, 3, 35, FL * 10 + FR + 1)
    lrow = np.array([0, 1, 3, 3], np.uint32)
    rrow = np.array([2, 0, 1, 2], np.uint32)
    o, w = mp.binary_op("/", L, lv, lrow, R, rv, rrow)
    assert o.shape[0] == min(FL, FR)
    for f in range(min(FL, FR)):
        e, ew = bo.binary_op("/", L[f], lv, lrow, R[f], rv, rrow)
        assert np.array_equal(o[f], e) and np.array_equal(w, ew)
    names = mp.binary_names("/", [f"l{i}" for i in range(FL)], [f"r{i}" for i in range(FR)])
    assert names == [f"l{i} / r{i}" for i in range(min(FL, FR))]
    if min(FL, FR) == 1:  # one pair: the filter decides on it and keeps the lhs fields
        o, w = mp.binary_op(">", L, lv, lrow, R, rv, rrow)
        e, ew = bo.binary_op(">", L[0], lv, lrow, R[0], rv, rrow)
        assert o.shape[0] == FL and np.array_equal(w, ew) and np.array_equal(o[0], e)
        ok = orc.valid_to_bool(w, 35)
        for f in range(1, FL):
            assert np.array_equal(o[f][ok], L[f][lrow.astype(np.int64)][ok])
        assert mp.binary_names(">", ["a"] * FL, ["b"] * FR) == ["a"] * FL
    else:
        with pytest.raises(mp.Refused, match="filter on multi-value input"):
            mp.binary_op(">", L, lv, lrow, R, rv, rrow)
    o, w = mp.binary_op(">", L, lv, lrow, R, rv, rrow, return_bool=True)  # bool zips like arithmetic
    assert o.shape[0] == min(FL, FR)


def test_refusals_of_several_fields():
    vals, valid, _ = grid(2, 3, 10, 3)
    with pytest.raises(mp.Refused, match=mp.FILTER):
        mp.scalar_op("<", 1.0, vals, valid)
    with pytest.raises(mp.Refused, match=r"group\(\)"):
        mp.aggregate("group", vals, valid, np.zeros(3, np.uint32), 1)
    mp.scalar_op("<", 1.0, vals, valid, return_bool=True)


def test_names():
    assert mp.leaf_names("prom_rate", "ts", ["a", "b"]) == ["prom_rate(ts_range,a)", "prom_rate(ts_range,b)"]
    assert mp.leaf_names("", "ts", ["a", "b"]) == ["a", "b"]


def _tie_grid(F, last_differs_at):
    """3 x 4 valid cells whose tuples tie in every field but `last_differs_at`, which takes few distinct keys"""
    rng = np.random.default_rng(F * 7 + last_differs_at)
    vals = np.full((F, 3, 4), 2.5)
    vals[last_differs_at] = rng.choice([-1.0, 0.0, -0.0, 3.0], (3, 4))
    return vals, np.ones((3, 4), bool)


@pytest.mark.parametrize("F", [2, 3, 8])
@pytest.mark.parametrize("desc", [False, True])
def test_sort_is_lexicographic(F, desc):
    for at in (1, F - 1):
        vals, ok = _tie_grid(F, at)
        got = mp.sort(desc, vals, ok)
        assert np.array_equal(got, sk.sort(desc, vals[at], ok))  # every other field ties: field `at` decides
    rng = np.random.default_rng(F)
    vals = rng.choice([np.nan, -np.inf, -0.0, 0.0, 1.0, np.inf], (F, 5, 7))
    vals[:, :, ::3] = -np.nan  # NaN of the other sign
    ok = rng.random((5, 7)) > 0.1
    got = mp.sort(desc, vals, ok)
    cells = np.flatnonzero(ok.reshape(-1))
    tuples = {int(c): tuple(int(sk.keys_of_values(vals[f].reshape(-1)[c:c + 1])[0]) for f in range(F)) for c in cells}
    expect = sorted(cells.tolist(), key=lambda c: tuple((-k if desc else k) for k in tuples[c]) + (c,))
    assert got.tolist() == expect


def test_refusal_texts_are_the_goldens():
    cases = {c["name"]: c for c in json.load(open(GOLDEN))["cases"]}
    assert cases["group_over_multi_field"]["message"] == mp.REFUSALS["group"]
    assert cases["topk_over_multi_field"]["message"] == mp.REFUSALS["topk"]
    for c in cases.values():
        assert c["error"].endswith(c["message"])
