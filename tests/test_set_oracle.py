"""CPU: the set operators' restatements (tests/set_oracle.py) against the reference's printed tables, and the dense
restatement (what the plan layer and K8 compute) against the row-literal one on random label sets."""
import itertools

import numpy as np
import pytest

from tests import binary_oracle as bor
from tests import set_oracle as sor
from tests.binary_helpers import count_rows, dense_rows, oracle_node
from tests.set_helpers import CASES, EXPRS, G, MAX_RATIO, MAX_USED, expected_set_rows, oracle_rows, row_key


def test_every_case_is_tagged_and_cited():
    for c in G["cases"]:
        assert c["layers"] and set(c["layers"]) <= {"plan", "device", "oracle"}, c["name"]
        assert ".result:" in c["source"], c["name"]
        if "plan" in c["layers"]:
            assert c["name"] in EXPRS, c["name"]


@pytest.mark.parametrize("name", sorted(EXPRS))
def test_row_literal_reproduces_the_printed_tables(name):
    case = CASES[name]
    tags, rows = oracle_rows(EXPRS[name], case)
    assert sorted(rows, key=row_key) == expected_set_rows(case, tags)


def test_vector1_cases():
    """http_requests AND ON (dummy) / IGNORING (g, instance, job) vector(1): vector(1) is a tagless row at every step."""
    for name, kw in (("and_on_dummy_vector1", {"on": ["dummy"]}), ("and_ignoring_all_vector1", {"ignoring": ["g", "instance", "job"]})):
        case = CASES[name]
        lhs = oracle_rows(("sel", "http_requests", {}, None, ()), case)
        tags, rows = sor.setop_rows(lhs, ([], [(case["start"], 1.0)]), "and", **kw)
        assert sorted(rows, key=row_key) == expected_set_rows(case, tags)


@pytest.mark.parametrize("name,op", [("count_and", "and"), ("count_unless", "unless")])
def test_count_cases(name, op):
    case = CASES[name]
    lhs, rhs = oracle_rows(MAX_USED, case), oracle_rows(MAX_RATIO, case)
    _, rows = sor.setop_rows(lhs, rhs, op)
    assert count_rows(rows) == expected_set_rows(case, [])


def test_sum_by_labels_the_table_lacks():
    """sum by (cloud, tag0, tag1) over a table without tag0 / tag1 groups by cloud alone; `or` with an unknown metric
    (no rows, no tags) on either side keeps the sums (set_operation.result:776, 791, 806)."""
    case = CASES["sum_by_missing_or_unknown"]
    t = G["tables"]["node_network_transmit_bytes_total"]
    sums = dense_rows(*oracle_node(t, case["start"], case["end"], case["interval"], agg="sum", by=("cloud",)))
    unknown = ([], [])
    for name, (tags, rows) in (("sum_by_missing_or_unknown", sor.setop_rows(sums, unknown, "or")),
                               ("unknown_or_unknown_or_sum", sor.setop_rows(sor.setop_rows(unknown, unknown, "or"), sums, "or")),
                               ("sum_or_sum_unknown", sor.setop_rows(sums, (["cloud"], []), "or"))):
        assert sorted(rows, key=row_key) == expected_set_rows(CASES[name], tags), name


def test_plan_errors_in_the_restatement():
    with pytest.raises(KeyError):   # and / unless: key sets must agree (CombineTableColumnMismatch)
        sor.setop_rows((["a", "b"], []), (["a"], []), "and")
    with pytest.raises(KeyError):   # or on(x): x on neither side
        sor.setop_rows((["a"], []), (["b"], []), "or", on=["x"])
    assert sor.setop_rows((["a"], []), (["b"], []), "or", on=["b"])[0] == ["a", "b"]


# ---- dense restatement == row-literal restatement on random label sets ------------------------------------------------
def random_side(rng, tags, n_rows, T, values, null_rate=0.2, dup_rate=0.0, labels_from=None):
    """label tuples (a small alphabet, NULLs, and, with dup_rate, repeated tuples) and a grid with holes"""
    labels = []
    for _ in range(n_rows):
        if labels and rng.random() < dup_rate:
            labels.append(labels[rng.integers(len(labels))])
        elif labels_from and labels_from[1] and rng.random() < 0.5:   # a label tuple of the other side
            src = labels_from[1][rng.integers(len(labels_from[1]))]
            labels.append(tuple(src[labels_from[0].index(t)] if t in labels_from[0] else None for t in tags))
        else:
            labels.append(tuple(None if rng.random() < null_rate else "v%d" % rng.integers(3) for _ in tags))
    vals = values[rng.integers(0, values.size, size=(n_rows, T))]
    ok = rng.random((n_rows, T)) < 0.6
    return labels, np.where(ok, vals, 0.0), bor._words(ok)


def dense_setop(op, ltags, L, rtags, R, on=None, ignoring=None):
    (llab, lv, lw), (rlab, rv, rw) = L, R
    lk, rk, n_keys, out_tags = sor.setop_pairs(op, ltags, llab, rtags, rlab, on, ignoring)
    T = lv.shape[1]
    if op != "or":
        lv, lw = sor.distinct_cells(llab, lv, lw)
    out, ow = sor.setop(op, lv, lw, lk, rv, rw, rk, n_keys)
    if op != "or":
        labels = llab
    else:
        widen = lambda tags, lab: tuple(lab[tags.index(t)] if t in tags else None for t in out_tags)
        labels = [widen(ltags, x) for x in llab] + [widen(rtags, x) for x in rlab]
    return dense_rows(out_tags, labels, out, ow, np.arange(T) * 1000)


VALUES = np.concatenate([np.array([0x7FF8000000000001, 0x8000000000000000], np.uint64).view(np.float64),
                         np.array([0.0, 1.0, 2.0, -3.5])])
TAG_SETS = [((), ()), (("a",), ("a",)), (("a", "b"), ("a", "b")), (("a", "b"), ("b", "c")), (("a",), ()), ((), ("a", "b"))]
MODIFIERS = [{}, {"on": []}, {"on": ["a"]}, {"on": ["b", "a"]}, {"ignoring": ["b"]}, {"ignoring": ["a", "c"]}]


def same(dense, literal):
    dt, dr = dense
    lt, lr = literal
    assert dt == lt
    bits = lambda rows: sorted((r[:-1] + (int(np.array([r[-1]]).view(np.uint64)[0]),) for r in rows), key=row_key)
    assert bits(dr) == bits(lr)


@pytest.mark.parametrize("op", ["and", "or", "unless"])
def test_dense_equals_row_literal_on_random_label_sets(op):
    rng = np.random.default_rng({"and": 1, "or": 2, "unless": 3}[op])
    checked = 0
    for (ltags, rtags), mod, sizes in itertools.product(TAG_SETS, MODIFIERS, [(0, 3), (3, 0), (6, 9), (12, 4)]):
        ltags, rtags = list(ltags), list(rtags)
        for T in (1, 5, 33):
            L = random_side(rng, ltags, sizes[0], T, VALUES, dup_rate=0.3)
            R = random_side(rng, rtags, sizes[1], T, VALUES, dup_rate=0.3, labels_from=(ltags, L[0]))
            try:
                literal = sor.setop_rows(dense_rows(ltags, L[0], L[1], L[2], np.arange(T) * 1000),
                                         dense_rows(rtags, R[0], R[1], R[2], np.arange(T) * 1000), op, **mod)
            except KeyError:
                with pytest.raises(KeyError):
                    sor.setop_pairs(op, ltags, L[0], rtags, R[0], **mod)
                continue
            same(dense_setop(op, ltags, L, rtags, R, **mod), literal)
            checked += 1
    assert checked > 100


def test_nested_or_dense_equals_row_literal():
    rng = np.random.default_rng(9)
    T = 7
    for _ in range(20):
        A = random_side(rng, ["a"], 4, T, VALUES)
        B = random_side(rng, ["a", "b"], 5, T, VALUES, labels_from=(["a"], A[0]))
        C = random_side(rng, ["c"], 3, T, VALUES)
        ts = np.arange(T) * 1000
        ab_tags, ab = dense_setop("or", ["a"], A, ["a", "b"], B)
        lit_ab = sor.setop_rows(dense_rows(["a"], *A, ts), dense_rows(["a", "b"], *B, ts), "or")
        same((ab_tags, ab), lit_ab)
        same(sor.setop_rows((ab_tags, ab), dense_rows(["c"], *C, ts), "or", on=["a"]),
             sor.setop_rows(lit_ab, dense_rows(["c"], *C, ts), "or", on=["a"]))


def test_distinct_drops_only_equal_cells():
    nan_a = np.array([0x7FF8000000000001], np.uint64).view(np.float64)[0]
    nan_b = np.array([0x7FF8000000000002], np.uint64).view(np.float64)[0]
    vals = np.array([[1.0, nan_a, 0.0, 2.0], [1.0, nan_a, -0.0, 3.0], [1.0, nan_b, 0.0, 2.0]])
    words = bor._words(np.ones((3, 4), bool))
    out, ow = sor.distinct_cells([("x",), ("x",), ("y",)], vals, words)
    assert ow[:, 0].tolist() == [0b1111, 0b1100, 0b1111]   # row 1 repeats row 0 at steps 0 and 1 (same bits)
    assert (out[1, :2] == 0).all()
