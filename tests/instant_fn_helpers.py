"""Shared by the instant-function tests: the golden cases of reference_instant_fn_vectors.json as expression trees, their
row-literal evaluation on the CPU oracle, and their comparison with the printed tables.

Expression trees (JSON lists):
  ["sel", table, {label: value}]           instant selector over the series of `table` that match
  ["fn", name, [args], expr]               name(expr, args...), name as the reference's projection shows it
  ["op", op, number, on_left, expr]        expr op number (number op expr when on_left)
  ["scalar", expr]                         scalar(expr)
  ["bin", op, lhs, rhs, {label_side}]      vector-vector operator (a tagless side pairs with every row)
  ["agg_by", agg, [labels], expr]           agg(expr) by (labels), agg in count / sum / avg / stddev
  ["count", expr]                          count(expr)
"""
import json
import math
import os

from tests import binary_oracle as bor
from tests import instant_fn_oracle as ifo
from tests.binary_helpers import count_rows, dense_rows, oracle_node
from tests.helpers import GOLDEN_DIR

# the reference's projection name -> the oracle's function name
ORACLE_FN = {"radians": "rad", "degrees": "deg", "signum": "sgn", "prom_round": "round"}


def load_instant_fn():
    with open(os.path.join(GOLDEN_DIR, "reference_instant_fn_vectors.json")) as f:
        return json.load(f)


G = load_instant_fn()


def select(table, match):
    t = dict(G["tables"][table])
    t["series"] = [s for s in t["series"] if all(s.get(k) == v for k, v in match.items())]
    return t


def oracle_rows(expr, case):
    """Row-literal evaluation -> (tag names, rows [(labels..., ts, value)])."""
    kind = expr[0]
    if kind == "sel":
        t = select(expr[1], expr[2])
        if not t["series"]:
            return list(t["tags"]), []
        return dense_rows(*oracle_node(t, case["start"], case["end"], case["interval"]))
    if kind == "fn":
        tags, rows = oracle_rows(expr[3], case)
        name, args = ORACLE_FN.get(expr[1], expr[1]), list(expr[2]) + [0.0, 0.0]
        return tags, [r[:-1] + (float(ifo.apply(name, [r[-1]], args[0], args[1])[0]),) for r in rows]
    if kind == "op":
        tags, rows = oracle_rows(expr[4], case)
        return tags, bor.scalar_rows(rows, expr[1], expr[2], scalar_on_left=expr[3])
    if kind == "scalar":
        tags, rows = oracle_rows(expr[1], case)
        return [], [(ts, v) for ts, v in
                    ifo.scalar_calculate_rows([rows], len(tags), case["start"], case["end"], case["interval"])]
    if kind == "bin":
        lhs, rhs = oracle_rows(expr[2], case), oracle_rows(expr[3], case)
        return bor.binary_rows(lhs, rhs, expr[1], **expr[4])
    if kind == "agg_by":
        tags, rows = oracle_rows(expr[3], case)
        idx = [tags.index(b) for b in expr[2]]
        groups = {}
        for r in rows:
            groups.setdefault(tuple(r[i] for i in idx) + (r[-2],), []).append(r[-1])
        agg = {"count": lambda v: float(len(v)), "sum": math.fsum, "avg": lambda v: math.fsum(v) / len(v),
               "stddev": lambda v: math.sqrt(math.fsum((x - math.fsum(v) / len(v)) ** 2 for x in v) / len(v))}[expr[1]]
        return list(expr[2]), [k + (agg(v),) for k, v in sorted(groups.items())]
    tags, rows = oracle_rows(expr[1], case)   # count
    return [], count_rows(rows)


def expected_rows(case, tags):
    """The printed rows as (labels in `tags` order..., ts, printed value), sorted."""
    return sorted(tuple(lab[t] for t in tags) + (ts, v) for lab, ts, v in case["expected"])


def same_value(printed, x):
    """A printed value (shortest round-trip digits, or NaN) against a computed f64: exact."""
    if printed == "NaN":
        return math.isnan(x)
    return float(printed) == x and not math.isnan(x)


def check_rows(case, tags, rows):
    want = expected_rows(case, tags)
    got = sorted((tuple(r[:-2]) + (int(r[-2]), r[-1]) for r in rows), key=lambda r: r[:-1])
    assert [w[:-1] for w in want] == [g[:-1] for g in got], f"{case['name']}: rows differ"
    for w, g in zip(want, got):
        assert same_value(w[-1], g[-1]), f"{case['name']}: {g} != printed {w}"
