"""The plan-tree interpreter (tests/plan_tree_oracle.py) on the CPU: the set-operator goldens rebuilt as trees, every
one-node tree against its single-node oracle, and the seeded generator's reproducibility."""
import math

import numpy as np
import pytest

from tests import aggregate_oracle as ago
from tests import binary_oracle as bor
from tests import instant_fn_oracle as ifo
from tests import plan_tree_oracle as pto
from tests import set_helpers as sh
from tests import sort_oracle as soo
from tests import topk_oracle as tko


def _tree(expr, tables):
    """a set-golden expression (tests/set_helpers.py) as a tree; a selector with matchers gets a table of its own"""
    kind = expr[0]
    if kind == "sel":
        _, table, match, agg, by = expr
        name = table + "".join(f"|{k}={v}" for k, v in sorted(match.items()))
        tables[name] = sh.select(sh.G["tables"][table], match)
        node = pto.leaf(name)
        return pto.aggregate(agg, node, by=list(by)) if agg else node
    if kind == "scalar":
        return pto.scalar_op(_tree(expr[1], tables), expr[2], expr[3])
    lhs, rhs = _tree(expr[2], tables), _tree(expr[3], tables)
    make = pto.binary if kind == "bin" else pto.setop
    return make(expr[1], lhs, rhs, **expr[4])


def _canon(rows):
    return sorted(((tuple(sorted((k, (v is None, v or "")) for k, v in lab.items())), ts, v) for v, lab, ts in rows),
                  key=repr)


@pytest.mark.parametrize("name", sorted(sh.EXPRS))
def test_set_goldens(name):
    c = sh.CASES[name]
    tables = {}
    tree = _tree(sh.EXPRS[name], tables)
    res = pto.evaluate(tree, tables, (c["start"], c["end"], c["interval"]))
    got = [(r.value, {k: v for k, v in r.labels.items() if v is not None}, r.ts) for r in res.export]
    exp = [(v, {k: x for k, x in lab.items() if x is not None}, ts) for lab, ts, v in c["expected"]]
    assert _canon(got) == _canon(exp)
    assert all(r.pin == pto.BITS and not r.maybe for r in res.export)


def _rows(res):
    return [(r.value, r.labels, r.ts) for r in res.rows]


def _same(a, b):
    return len(a) == len(b) and all(x[1:] == y[1:] and (pto.bits(x[0]) == pto.bits(y[0]) or
                                                        (math.isnan(x[0]) and math.isnan(y[0]))) for x, y in zip(a, b))


def _one_node_trees(rng, tags):
    """one tree per node kind over a leaf of table m2, with seeded arguments"""
    leaf = lambda: pto.leaf("m2")
    by = list(rng.permutation(tags)[:2])
    yield pto.scalar_op(leaf(), str(rng.choice(pto.ARITH + pto.CMP)), 2.0, on_left=bool(rng.random() < 0.5))
    yield pto.function(leaf(), "clamp", -1.0, 1.0)
    yield pto.binary(str(rng.choice(pto.ARITH + pto.CMP)), leaf(), pto.leaf("m1"), on=["host", "job"])
    yield pto.setop(str(rng.choice(["and", "or", "unless"])), leaf(), pto.leaf("m1"), on=["job"])
    yield pto.aggregate(str(rng.choice(pto.AGG_OPS[:-2])), leaf(), by=by)
    yield pto.aggregate("quantile", leaf(), param=0.9, without=by)
    yield pto.topk(str(rng.choice(["topk", "bottomk"])), 2, leaf(), by=by)
    yield pto.sort(str(rng.choice(soo.FUNCTIONS[:2])), leaf())
    yield pto.sort("sort_by_label_desc", leaf(), by)
    yield pto.label_join(leaf(), "dst", "-", *by)


def _single_node_oracle(tree, child, tables, grid):
    """the rows the existing single-node oracle gives for a one-node tree over child's rows"""
    a, rows, tags = tree.args, _rows(child), child.tags
    if tree.kind == "scalar_op":   # the dense form of tests/binary_oracle.py over the child's values
        vals = np.array([[v for v, _, _ in rows]], np.float64)
        out, ok = bor.scalar_op(a["op"], a["s"], vals, bor._words(np.ones(vals.shape, bool)), a["on_left"], a["bool"])
        keep = bor._bits(ok, vals.shape[1])[0]
        return [(float(x), lab, ts) for x, k, (_, lab, ts) in zip(out[0], keep, rows) if k]
    if tree.kind == "function":   # the dense form of tests/instant_fn_oracle.py over the child's values
        vals = np.array([[v for v, _, _ in rows]], np.float64)
        out, _ = ifo.instant_fn(pto.EXACT_FNS[a["name"]], vals, ifo._words(np.ones(vals.shape, bool)), *a["args"])
        return [(float(x), lab, ts) for x, (_, lab, ts) in zip(out[0], rows)]
    if tree.kind in ("binary", "setop"):
        rhs = pto.evaluate(tree.children[1], tables, grid)
        side = lambda res: (res.tags, [tuple(r.labels[t] for t in res.tags) + (r.ts, r.value) for r in res.rows])
        f = (lambda l, r: bor.binary_rows(l, r, a["op"], a["bool"], a["on"], a["ignoring"], a["label_side"])) \
            if tree.kind == "binary" else (lambda l, r: sh.sor.setop_rows(l, r, a["op"], a["on"], a["ignoring"]))
        out_tags, out = f(side(child), side(rhs))
        return [(r[-1], dict(zip(out_tags, r[:-2])), r[-2]) for r in out]
    if tree.kind == "aggregate":
        return ago.aggregate_rows(rows, tags, a["op"], a["param"], a["by"], a["without"])[0]
    if tree.kind == "topk":
        mod = ("by", a["by"]) if a["by"] is not None else ("without", a["without"]) if a["without"] else (None, ())
        return tko.topk_rows(a["op"] == "bottomk", a["k"], rows, tags, *mod)
    if tree.kind == "sort":
        return soo.sort_rows(a["function"], rows, a["labels"])
    if tree.kind == "label_join":
        return [(v, dict(lab, dst="-".join(lab[s] for s in a["srcs"] if lab[s] is not None)), ts)
                for v, lab, ts in rows]
    raise ValueError(tree.kind)


def _key(row):
    return repr((sorted((k, (v is None, v or "")) for k, v in row[1].items()), row[2]))


@pytest.mark.parametrize("seed", range(8))
def test_one_node_trees_are_the_single_node_oracles(seed):
    rng = np.random.default_rng(seed)
    grid = pto.make_grid(rng)
    tables = pto.make_tables(rng, grid)
    if not tables["m2"]["series"]:
        tables["m2"] = dict(tables["m1"], tags=["host", "job", "zone"],
                            series=[dict(s, zone=None) for s in tables["m1"]["series"]])
    for tree in _one_node_trees(rng, ["host", "job", "zone"]):
        child = pto.evaluate(tree.children[0], tables, grid)
        got = [(r.value, r.labels, r.ts) for r in pto.evaluate(tree, tables, grid).export]
        exp = _single_node_oracle(tree, child, tables, grid)
        if tree.kind == "topk" and any(any(v is None for v in lab.values()) for _, lab, _ in exp):
            got, exp = sorted(got, key=_key), sorted(exp, key=_key)   # (NULL group labels: the plan layer's order)
        if tree.kind in ("binary", "setop", "scalar_op", "function", "label_join"):
            got, exp = sorted(got, key=_key), sorted(exp, key=_key)   # (row-major grid order against the join's)
        assert _same(got, exp), pto.promql(tree)


@pytest.mark.parametrize("seed", [0, 7, 123])
def test_the_same_seed_draws_the_same_case(seed):
    t1, tab1, g1 = pto.draw_case(seed)
    t2, tab2, g2 = pto.draw_case(seed)
    assert g1 == g2 and pto.promql(t1) == pto.promql(t2)
    assert repr(tab1) == repr(tab2)
    assert t1.depth() <= 4 and t1.size() <= 8


def test_the_generator_covers_every_node_kind():
    kinds, steps = set(), set()
    for seed in range(60):
        tree, _, grid = pto.draw_case(seed)
        kinds |= {n.kind for n in tree.subtrees()}
        steps.add(len(pto.grid_steps(grid)))
    assert kinds == {"leaf", "vector", "time", "binary", "setop", "aggregate", "topk", "sort", "label_join",
                     "label_replace", "scalar_op", "function", "subquery"}
    assert steps == set(pto.STEPS)


def test_unpinned_cells():
    """a computed NaN is unpinned; an order comparison that reads one leaves its row open, an equality does not; max
    over one is open"""
    tables = {"t": {"time_index": "ts", "field": "val", "tags": ["host"],
                    "series": [{"host": "a", "ts": [0], "val": [-1.0]}, {"host": "b", "ts": [0], "val": [4.0]}]}}
    grid = (0, 0, 1000)
    root = lambda: pto.function(pto.leaf("t"), "sqrt")
    sq = pto.evaluate(root(), tables, grid).export
    assert [(r.pin, r.maybe) for r in sq] == [(pto.NAN, False), (pto.BITS, False)]
    gt = pto.evaluate(pto.scalar_op(root(), ">", 0.0), tables, grid).export
    assert [r.maybe for r in gt] == [True, False]
    ne = pto.evaluate(pto.scalar_op(root(), "!=", 0.0), tables, grid).export
    assert [r.maybe for r in ne] == [False, False]
    assert [r.pin for r in pto.evaluate(pto.aggregate("max", root()), tables, grid).export] == [pto.ANY]
    assert [r.pin for r in pto.evaluate(pto.aggregate("count", root()), tables, grid).export] == [pto.BITS]


def test_a_filter_with_the_scalar_on_the_left_keeps_the_vector_value():
    """`1 <= v` keeps v's value, as `v >= 1` does (the row-literal scalar oracle once kept the scalar)"""
    assert bor.scalar_rows([("a", 0, 3.0)], "<=", 1.0, scalar_on_left=True) == [("a", 0, 3.0)]
    assert bor.scalar_rows([("a", 0, 3.0)], ">", 1.0, scalar_on_left=True) == []
