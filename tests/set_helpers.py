"""Shared by the set-operator tests: the golden cases of reference_set_vectors.json written as expression trees, and the
row-literal evaluation of such a tree on the CPU oracle.  The GPU tests evaluate the same trees through the plan layer.

Expression trees:
  ("sel", table, {label: value}, aggregate, by)   instant selector over the series of `table` that match, with an
                                                  optional by-label aggregate
  ("scalar", expr, op, number)                    expr op number
  ("bin", op, lhs, rhs, {on | ignoring | label_side})
  ("set", op, lhs, rhs, {on | ignoring})
"""
import json
import os

from tests import binary_oracle as bor
from tests import set_oracle as sor
from tests.binary_helpers import dense_rows, oracle_node
from tests.helpers import GOLDEN_DIR


def load_set():
    with open(os.path.join(GOLDEN_DIR, "reference_set_vectors.json")) as f:
        return json.load(f)


G = load_set()
CASES = {c["name"]: c for c in G["cases"]}


def sel(table, agg=None, by=(), **match):
    return ("sel", table, match, agg, tuple(by))


HTTP_CANARY_PLUS_1 = ("scalar", sel("http_requests", g="canary"), "+", 1.0)
NESTED = ("set", "or", ("set", "or", sel("http_requests"), sel("cpu_count"), {}), sel("vector_matching_a"), {})
MAX_USED = sel("stats_used_bytes", agg="max", by=("namespace",))
MAX_RATIO = ("scalar", ("bin", "/", MAX_USED, sel("stats_capacity_bytes", agg="max", by=("namespace",)), {}), ">=", 80 / 100)
HIT, MISS = sel("cache_hit_with_null_label"), sel("cache_miss_with_null_label")
WEB1 = ("scalar", sel("http_requests_env", job="web", instance="1", env="production"), "*", 5.0)
API5 = ("scalar", sel("http_requests_env", job="api", instance="0", env="production"), "+", 5.0)

EXPRS = {
    "and_selectors": ("set", "and", sel("http_requests", g="canary"), sel("http_requests", instance="0"), {}),
    "and_plus1": ("set", "and", HTTP_CANARY_PLUS_1, sel("http_requests", instance="0"), {}),
    "and_on_instance_job": ("set", "and", HTTP_CANARY_PLUS_1, sel("http_requests", instance="0", g="production"),
                            {"on": ["instance", "job"]}),
    "and_on_instance": ("set", "and", HTTP_CANARY_PLUS_1, sel("http_requests", instance="0", g="production"),
                        {"on": ["instance"]}),
    "and_ignoring_g": ("set", "and", HTTP_CANARY_PLUS_1, sel("http_requests", instance="0", g="production"),
                       {"ignoring": ["g"]}),
    "and_ignoring_g_job": ("set", "and", HTTP_CANARY_PLUS_1, sel("http_requests", instance="0", g="production"),
                           {"ignoring": ["g", "job"]}),
    "or_canary_production": ("set", "or", sel("http_requests", g="canary"), sel("http_requests", g="production"), {}),
    "or_plus1_instance1": ("set", "or", HTTP_CANARY_PLUS_1, sel("http_requests", instance="1"), {}),
    "or_on_instance_nested": ("set", "or", HTTP_CANARY_PLUS_1, NESTED, {"on": ["instance"]}),
    "or_ignoring_nested": ("set", "or", HTTP_CANARY_PLUS_1, NESTED, {"ignoring": ["l", "g", "job"]}),
    "unless_selectors": ("set", "unless", sel("http_requests", g="canary"), sel("http_requests", instance="0"), {}),
    "unless_on_job": ("set", "unless", sel("http_requests", g="canary"), sel("http_requests", instance="0"),
                      {"on": ["job"]}),
    "unless_on_job_instance": ("set", "unless", sel("http_requests", g="canary"), sel("http_requests", instance="0"),
                               {"on": ["job", "instance"]}),
    "unless_ignoring_g_instance": ("set", "unless", sel("http_requests", g="canary"), sel("http_requests", instance="0"),
                                   {"ignoring": ["g", "instance"]}),
    "unless_ignoring_g": ("set", "unless", sel("http_requests", g="canary"), sel("http_requests", instance="0"),
                          {"ignoring": ["g"]}),
    "t1_or_t2": ("set", "or", sel("t1"), sel("t2"), {}),
    "t1_or_on_empty_t2": ("set", "or", sel("t1"), sel("t2"), {"on": []}),
    "t1_or_on_job_t2": ("set", "or", sel("t1"), sel("t2"), {"on": ["job"]}),
    "t2_or_t1": ("set", "or", sel("t2"), sel("t1"), {}),
    "t2_or_on_empty_t1": ("set", "or", sel("t2"), sel("t1"), {"on": []}),
    "t2_or_on_job_t1": ("set", "or", sel("t2"), sel("t1"), {"on": ["job"]}),
    "and_max_ratio": ("set", "and", MAX_USED, MAX_RATIO, {}),
    "null_label_div": ("bin", "/", HIT, ("bin", "+", MISS, HIT, {}), {}),
    "null_label_div_ignoring": ("bin", "/", HIT, ("bin", "+", MISS, HIT, {"ignoring": ["null_label"]}),
                                {"ignoring": ["null_label"]}),
    "null_label_div_on_job": ("bin", "/", HIT, ("bin", "+", MISS, HIT, {"on": ["job"]}), {"on": ["job"]}),
    "unknown_or_metric": ("set", "or", sel("unknown_metric"), sel("node_network_transmit_bytes_total"), {}),
    "or_empty_times5_or_plus5": ("set", "or", WEB1, API5, {}),
    "or_plus5_or_empty_times5": ("set", "or", API5, WEB1, {}),
    "or_three_way": ("set", "or", ("set", "or", WEB1,
                                   ("scalar", sel("http_requests_env", job="web", instance="2", env="production"), "*", 3.0),
                                   {}), API5, {}),
    "filter_or_fill": ("set", "or", ("set", "or", ("bin", ">", sel("a"), sel("b"), {}), sel("b"), {}), sel("a"), {}),
}


def select(table, match):
    """The table with only the series whose labels match."""
    t = dict(table)
    t["series"] = [s for s in table["series"] if all(s.get(k) == v for k, v in match.items())]
    return t


def oracle_rows(expr, case):
    """Row-literal evaluation of an expression tree -> (tag names, rows [(labels..., ts, value)])."""
    kind = expr[0]
    if kind == "sel":
        _, table, match, agg, by = expr
        t = select(G["tables"][table], match)
        if not t["series"]:
            return (list(by) if agg else list(t["tags"])), []
        return dense_rows(*oracle_node(t, case["start"], case["end"], case["interval"], agg=agg, by=by))
    if kind == "scalar":
        tags, rows = oracle_rows(expr[1], case)
        return tags, bor.scalar_rows(rows, expr[2], expr[3])
    lhs, rhs = oracle_rows(expr[2], case), oracle_rows(expr[3], case)
    if kind == "bin":
        return bor.binary_rows(lhs, rhs, expr[1], **expr[4])
    return sor.setop_rows(lhs, rhs, expr[1], **expr[4])


def row_key(row):
    """sort key of a row whose labels may be None (NULL sorts first, as in the printed tables)"""
    return tuple((0, "") if x is None else (1, x) for x in row)


def expected_set_rows(case, tags):
    return sorted((tuple(lab.get(t) for t in tags) + (ts, v) for lab, ts, v in case["expected"]), key=row_key)

