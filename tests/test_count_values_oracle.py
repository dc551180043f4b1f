"""CPU: the count_values restatement (tests/count_values_oracle.py) reproduces the reference's printed tables, and its
dense form agrees with the row-literal one on random label sets."""
import json
import math
import os

import numpy as np
import pytest

from tests import binary_oracle as bor
from tests import count_values_oracle as cvo
from tests.aggregate_oracle import group_names
from tests.helpers import GOLDEN_DIR
from tests.test_aggregate_oracle import instant_rows

with open(os.path.join(GOLDEN_DIR, "reference_count_values_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}
NAN_NEG = -float("nan") if math.copysign(1.0, -float("nan")) < 0 else float("nan")
# NaNs of both signs and three payloads, ±0, ±inf, the smallest subnormal
SPECIAL = np.array([0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0xFFF800000000BEEF, 0x8000000000000000,
                    0x0000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001], np.uint64).view(np.float64)


def bits(v):
    return cvo.value_bits(v)


@pytest.mark.parametrize("name", sorted(c["name"] for c in G["cases"] if "rows" in c["layers"]))
def test_row_literal_reproduces_the_golden_tables(name):
    c = CASES[name]
    rows, tags = instant_rows(G["tables"][c["table"]], c["start"], c["end"], c["interval"], select=c["select"])
    got, names = cvo.count_values_rows(rows, tags, by=c.get("by"), without=c.get("without"))
    assert names == c["columns"][1:-2]
    # (the reference's label column is BIGINT: 200 there, the Float64 200.0 here)
    assert [(lab, ts, n, v) for n, lab, ts, v in got] == [tuple(e) for e in c["expected"]]


def test_value_grouping_is_by_bits_and_order_is_total():
    """-0.0 and +0.0 are two values, NaNs with different bits are different values, the order is f64::total_cmp's."""
    vals = [0.0, -0.0, 0.0, math.nan, NAN_NEG, math.inf, -math.inf, 1.0, float(SPECIAL[1]), float(SPECIAL[1])]
    rows = [(v, {"a": "x"}, 0) for v in vals]
    got, _ = cvo.count_values_rows(rows, ["a"])
    keys = [cvo.total_key(v) for _, _, _, v in got]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    by_bits = {bits(v): n for n, _, _, v in got}
    assert by_bits[bits(0.0)] == 2 and by_bits[bits(-0.0)] == 1
    assert by_bits[bits(math.nan)] == 1 and by_bits[bits(NAN_NEG)] == 1 and by_bits[bits(SPECIAL[1])] == 2
    assert [bits(v) for _, _, _, v in got][0] == bits(NAN_NEG)  # -NaN first, +NaN payloads last
    assert [bits(v) for _, _, _, v in got][-1] == bits(SPECIAL[1])


def random_labelled(rng, sizes, T, values):
    """Rows of groups of the given sizes over labels (job, instance, env); env NULL on some rows; duplicate label tuples;
    values drawn from `values`; some steps and rows without a valid cell."""
    R = int(sum(sizes))
    job = np.concatenate([np.full(s, g) for g, s in enumerate(sizes)])
    rng.shuffle(job)
    vals = rng.choice(values, (R, T))
    ok = rng.random((R, T)) < 0.8
    ok[:, T // 2] = False
    ok[rng.random(R) < 0.05] = False
    labels = [{"job": f"j{job[r]}", "instance": f"i{r % 7}", "env": [None, "a", "b", ""][r % 4]} for r in range(R)]
    return vals, ok, labels


VALUE_SETS = {
    "mixed": np.concatenate([SPECIAL, np.array([1.0, 2.0, -3.0, 2.5, -0.5])]),
    "all_equal": np.array([7.0]),
    "all_distinct": None,  # filled per row and step
}


@pytest.mark.parametrize("values", sorted(VALUE_SETS))
@pytest.mark.parametrize("mod", [(None, None), ("by", ["job"]), ("without", ["instance"]), ("by", ["env", "job"]),
                                 ("by", ["nope"])])
def test_dense_matches_row_literal(values, mod):
    rng = np.random.default_rng(23)
    T = 6
    sizes = [1, 2, 5, 31, 33, 70]
    pool = VALUE_SETS[values]
    vals, ok, labels = random_labelled(rng, sizes, T, pool if pool is not None else np.array([0.0]))
    if pool is None:
        vals = rng.standard_normal(vals.shape)
    tags = ["env", "instance", "job"]
    kw = {mod[0]: mod[1]} if mod[0] else {}
    names = group_names(tags, **kw)
    keys = []
    gid = np.zeros(len(labels), np.uint32)
    for r, lab in enumerate(labels):
        key = tuple(lab[n] for n in names)
        if key not in keys:
            keys.append(key)
        gid[r] = keys.index(key)
    gid[::11] = len(keys) + 3  # rows of no group take part in nothing
    rows = [(vals[r, k], labels[r], k) for r in range(len(labels)) for k in range(T) if ok[r, k] and gid[r] < len(keys)]
    got, _ = cvo.count_values_rows(rows, tags, **kw)
    out, cnt = cvo.count_values(vals, bor._words(ok), gid, len(keys))
    dense = cvo.dense_to_rows(out, cnt, gid, keys, names)
    assert [(n, lab, ts) for n, lab, ts, _ in got] == [(n, lab, ts) for n, lab, ts, _ in dense]
    assert [bits(v) for *_, v in got] == [bits(v) for *_, v in dense]
    assert not cnt[:, T // 2].any()
    order, goff = cvo.member_order(gid, len(keys))
    assert not cnt[goff[-1]:].any()  # rows of no group
    if values == "all_equal":  # one distinct value: only a group's first row holds it
        first = np.zeros(cnt.shape[0], bool)
        first[goff[:-1][np.diff(goff) > 0]] = True
        assert not cnt[~first].any() and cnt[first].any()
    # distinct values never outnumber a group's members, and the counts add up to the valid cells
    for g in range(len(keys)):
        members = order[goff[g]:goff[g + 1]]
        assert (cnt[goff[g]:goff[g + 1]].sum(axis=0) == ok[members].sum(axis=0)).all()


def test_empty_input_and_groups():
    out, cnt = cvo.count_values(np.zeros((0, 3)), np.zeros((0, 1), np.uint32), np.zeros(0, np.uint32), 2)
    assert out.shape == (0, 3) and cnt.shape == (0, 3)
    vals = np.array([[1.0, 2.0], [1.0, 3.0]])
    out, cnt = cvo.count_values(vals, bor._words(np.array([[True, False], [True, False]])), np.array([1, 1], np.uint32), 3)
    assert cnt[:, 0].tolist() == [2, 0] and out[0, 0] == 1.0 and not cnt[:, 1].any()
