"""CPU: the topk / bottomk restatement (tests/topk_oracle.py) reproduces the reference's printed tables, and its dense
form (group ids and tie ordinals, then the per-(group, step) selection K10 computes) agrees with the row-literal one."""
import json
import math
import os

import numpy as np
import pytest

from tests import topk_oracle as tko
from tests.helpers import GOLDEN_DIR

with open(os.path.join(GOLDEN_DIR, "reference_topk_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}
NAN_NEG = -float("nan") if math.copysign(1.0, -float("nan")) < 0 else float("nan")
KS = [-1.0, 0.0, 0.5, 1.0, 2.5, tko.KMAX - 1, tko.KMAX, tko.KMAX + 1, "largest", math.inf, math.nan, NAN_NEG]


def golden_input(case):
    """The topk input of a golden case as rows (value, labels, ts) and its tag columns."""
    if "rows_input" in case:
        rows = [(v, lab, ts) for lab, ts, v in case["rows_input"]]
        return rows, list(case["rows_input"][0][0])
    t = G["tables"][case["input"]["table"]]
    steps = range(case["start"], case["end"] + 1, case["interval"])
    # every series has a sample exactly at every step: the instant selector reads it
    rows = [(s["val"][s["ts"].index(ts)], {tag: s[tag] for tag in t["tags"]}, ts) for s in t["series"] for ts in steps]
    if case["input"].get("aggregate") != "sum":
        return rows, list(t["tags"])
    by = case["input"]["by"]
    acc = {}
    for v, lab, ts in rows:
        key = tuple(lab[b] for b in by) + (ts,)
        acc[key] = acc.get(key, 0.0) + v
    return [(v, dict(zip(by, k[:-1])), k[-1]) for k, v in acc.items()], list(by)


ROW_CASES = sorted(c["name"] for c in G["cases"] if "rows" in c["layers"])


def test_every_printed_table_is_a_case():
    assert len(ROW_CASES) == 13 and CASES["topk_multi_value_error"]["layers"] == []


@pytest.mark.parametrize("name", ROW_CASES)
def test_rows_reproduce_the_golden(name):
    case = CASES[name]
    rows, tags = golden_input(case)
    got = tko.topk_rows(case["op"] == "bottomk", case["k"], rows, tags)
    exp = [(v, lab, ts) for lab, ts, v in case["expected"]]
    assert [(v, {t: lab[t] for t in exp[0][1]}, ts) for v, lab, ts in got] == exp


def test_k_to_ranks_follows_the_total_order():
    for k, n in [(-1.0, 0), (0.0, 0), (-0.0, 0), (0.5, 0), (1.0, 1), (2.5, 2), (3.0, 3), (math.inf, 5), (-math.inf, 0),
                 (math.nan, 5), (NAN_NEG, 0), (1e300, 5)]:
        assert tko.kept_ranks(k, 5) == n, k
        assert min(tko.ranks_of_k(k), 5) == n, k


def test_total_key_order():
    xs = [NAN_NEG, -math.inf, -1.0, -0.0, 0.0, 1e-300, 1.0, math.inf, math.nan]
    assert [tko.total_key(x) for x in xs] == sorted(tko.total_key(x) for x in xs)
    assert len({tko.total_key(x) for x in xs}) == len(xs)


VALUES = [math.nan, NAN_NEG, math.inf, -math.inf, 0.0, -0.0, 1.0, 1.0, 2.0, -3.5]
LABEL_VALUES = [None, "", "a", "b", "ab"]


def random_node(rng, n_rows, T, tags):
    tuples = [tuple(LABEL_VALUES[i] for i in rng.integers(0, len(LABEL_VALUES), len(tags))) for _ in range(n_rows)]
    if n_rows > 2:
        tuples[1] = tuples[0]   # a duplicate label tuple
    vals = np.array(VALUES)[rng.integers(0, len(VALUES), (n_rows, T))]
    ok = rng.random((n_rows, T)) < 0.7
    return tuples, vals, ok


def rows_of(tags, tuples, vals, ok, ts):
    return [(float(vals[r, k]), dict(zip(tags, tuples[r])), int(ts[k]))
            for r in range(len(tuples)) for k in range(len(ts)) if ok[r, k]]


def same_rows(a, b):
    key = lambda r: (struct_bits(r[0]), tuple(sorted((k, v is None, v or "") for k, v in r[1].items())), r[2])
    return [key(r) for r in a] == [key(r) for r in b]


def struct_bits(x):
    return np.float64(x).view(np.uint64).item()


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("modifier", [None, ("by", ["b", "zz"]), ("by", ["c", "a"]), ("without", ["a"]),
                                      ("without", [])])
def test_dense_form_agrees_with_the_rows(seed, modifier):
    rng = np.random.default_rng(1000 + seed)
    tags = ["c", "a", "b"]
    T = 5
    ts = 1000 * np.arange(T)
    tuples, vals, ok = random_node(rng, 40 + seed * 7, T, tags)
    mod, labels = modifier if modifier else (None, ())
    rows = rows_of(tags, tuples, vals, ok, ts)
    for bottom in (False, True):
        gid, n_groups, tie, gcols = tko.topk_keys(bottom, tags, tuples, mod, labels)
        largest = int(np.bincount(gid).max())
        for k in KS:
            k = float(largest) if k == "largest" else float(k)
            exp = tko.topk_rows(bottom, k, rows, tags, mod, labels)
            words = tko.topk(bottom, k, vals, tko._words(ok), gid, n_groups, tie)
            got = tko.export_rows(bottom, vals, words, tags, tuples, ts, gcols, tie)
            assert same_rows(got, exp), (bottom, k, modifier)


def test_dense_form_drops_rows_without_a_group_and_masks_the_tail():
    vals = np.array([[1.0, 2.0, 3.0], [3.0, 2.0, 1.0]])
    valid = np.array([[0xFFFFFFFF], [0xFFFFFFFF]], np.uint32)
    words = tko.topk(False, 1, vals, valid, np.array([0, 5], np.uint32), 1, np.array([0, 1], np.uint32))
    assert words.tolist() == [[0b111], [0]]
