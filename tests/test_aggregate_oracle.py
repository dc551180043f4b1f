"""CPU: the aggregate restatement (tests/aggregate_oracle.py) reproduces the reference's printed tables — quantile and
group, and the goldens other layers could not build before (`scalar(count(count by (host)(host)))`, the ratio repro's
counts, the aggregator tables) — and its dense quantile agrees with the row-literal one on random label sets."""
import json
import math
import os

import numpy as np
import pytest

from oracle import oracle as orc
from tests import aggregate_oracle as ago
from tests import binary_oracle as bor
from tests.binary_helpers import dense_rows, oracle_node, table_arrays
from tests.helpers import GOLDEN_DIR


def _load(name):
    with open(os.path.join(GOLDEN_DIR, name)) as f:
        return json.load(f)


G = _load("reference_aggregate_vectors.json")
CASES = {c["name"]: c for c in G["cases"]}
NAN_NEG = -float("nan") if math.copysign(1.0, -float("nan")) < 0 else float("nan")
PHIS = [-0.5, -0.0, 0.0, 1.0 / 3.0, 0.5, 0.99, 1.0, 1.5, math.nan]


def instant_rows(table, start, end, interval, lookback=300_000, select=None):
    """The instant selector over `table` (series restricted to `select`) as rows [(value, {tag: label}, ts)] in row
    order: series in tag order, steps ascending."""
    series = [s for s in table["series"] if all(s[k] == v for k, v in (select or {}).items())]
    table = dict(table, series=series)
    labels, ts, val, offsets = table_arrays(table)
    out, valid = orc.instant_query(ts, val, offsets, start, end, interval, lookback)
    tags = list(table["tags"])
    _, rows = dense_rows(tags, labels, out, valid, start + interval * np.arange(out.shape[1], dtype=np.int64))
    return [(r[-1], dict(zip(tags, r[:-2])), r[-2]) for r in rows], tags


def apply_ops(rows, tags, ops):
    for o in ops:
        rows, tags = ago.aggregate_rows(rows, tags, o["op"], o.get("param"), by=o.get("by"), without=o.get("without"))
    return rows, tags


ROW_CASES = sorted(c["name"] for c in G["cases"] if "rows" in c["layers"])


@pytest.mark.parametrize("name", ROW_CASES)
def test_row_literal_reproduces_the_golden_tables(name):
    c = CASES[name]
    rows, tags = instant_rows(G["tables"][c["table"]], c["start"], c["end"], c["interval"], select=c["select"])
    rows, _ = apply_ops(rows, tags, c["ops"])
    assert [(lab, ts, v) for v, lab, ts in rows] == [tuple(e) for e in c["expected"]]


@pytest.mark.parametrize("u", G["units"], ids=[u["name"] for u in G["units"]])
def test_accumulator_unit_vectors(u):
    values = [0.0 if v is None else v for v in u["values"]]  # evaluate()'s unwrap_or(0.0)
    got = ago.accumulate("quantile", values, u["phi"])
    if u["expected"] == "NaN":  # quantile_with_scratch over no values
        assert math.isnan(got)
    else:
        assert got == u["expected"]


def test_inf_times_zero_is_nan():
    """s[lo] (1 - w) + s[hi] w is evaluated as written: with w = 0 the term +inf * 0 is NaN."""
    assert math.isnan(orc.quantile(np.array([1.0, math.inf]), 0.0))
    assert math.isnan(orc.quantile(np.array([1.0, math.inf]), 1.0))
    assert orc.quantile(np.array([1.0, 2.0]), 0.0) == 1.0


def test_scalar_count_of_an_aggregate():
    """scalar.result:128-164: scalar(count(<op>(host) by (host))), now buildable by the aggregate node."""
    g = _load("reference_instant_fn_vectors.json")
    for name in ("scalar:128", "scalar:140", "scalar:152", "scalar:164"):
        c = next(c for c in g["cases"] if c["name"] == name)
        _, (_, inner_op, by, sel) = c["expr"][1]
        rows, tags = instant_rows(g["tables"][sel[1]], c["start"], c["end"], c["interval"], select=sel[2])
        rows, tags = apply_ops(rows, tags, [{"op": inner_op, "by": by}, {"op": "count"}])
        # scalar() of a tagless node with one row per step is that row's value
        assert [({}, ts, v) for v, _, ts in rows] == [(e[0], e[1], float(e[2])) for e in c["expected"]], name


def test_ratio_repro_counts():
    """anon_promql_ratio_repro.result:60,87: count((rate(a) / on(l3,l4) group_left b) > 0.5) and that count over
    count(rate(a)), times 100."""
    g = _load("reference_binary_vectors.json")
    cases = {c["name"]: c for c in g["cases"]}
    c = cases["ratio_filtered_count"]
    kw = dict(start=c["start"], end=c["end"], interval=c["interval"])
    ra = dense_rows(*oracle_node(g["tables"]["metric_a"], fn="rate", range_ms=c["range"], **kw))
    rb = dense_rows(*oracle_node(g["tables"]["metric_b"], **kw))
    tags, joined = bor.binary_rows(ra, rb, "/", on=["l3", "l4"], label_side="rhs")
    kept = [(r[-1], dict(zip(tags, r[:-2])), r[-2]) for r in bor.scalar_rows(joined, ">", 0.5)]
    counted, _ = ago.aggregate_rows(kept, tags, "count")
    assert [(lab, ts, v) for v, lab, ts in counted] == [tuple(e) for e in c["expected"]]
    rate_rows = [(r[-1], dict(zip(ra[0], r[:-2])), r[-2]) for r in ra[1]]
    total, _ = ago.aggregate_rows(rate_rows, ra[0], "count")
    pct = [({}, ts, bor.binary_value("*", bor.binary_value("/", a, b), 100.0)) for (a, _, ts), (b, _, _) in zip(counted, total)]
    assert pct == [tuple(e) for e in cases["ratio_times_100"]["expected"]]


def test_aggregator_tables():
    """promql_test.rs:343-665 (reference_aggregator_vectors.json) through the row-literal aggregate."""
    g = _load("reference_aggregator_vectors.json")
    table = {"time_index": "ts", "field": "val", "tags": g["tags"], "series": g["series"]}
    for c in g["cases"]:
        rows, tags = instant_rows(table, g["start"], g["end"], g["interval"], g["lookback"], select=c["filter"])
        got, _ = ago.aggregate_rows(rows, tags, c["agg"], by=c["by"])
        exp = sorted((tuple(sorted(lab.items())), ts, v) for lab, ts, v in c["expected"])
        got = sorted((tuple(sorted(lab.items())), ts, v) for v, lab, ts in got)
        assert [r[:2] for r in got] == [r[:2] for r in exp], c["name"]
        for (_, _, a), (_, _, b) in zip(got, exp):
            assert a == pytest.approx(b, rel=c.get("rel_tol", 0.0), abs=0.0), c["name"]


# ---- dense quantile against the row-literal form -------------------------------------------------------------------
SPECIAL = np.array([0x7FF8000000000001, 0xFFF800000000BEEF, 0x8000000000000000, 0x0000000000000000,
                    0x7FF0000000000000, 0xFFF0000000000000], np.uint64).view(np.float64)


def random_labelled(rng, sizes, T):
    """Rows of groups of the given sizes over labels (job, instance, env), with NaNs of both signs, ±0, ±inf and
    duplicate values; some steps have no valid cell."""
    R = int(sum(sizes))
    job = np.concatenate([np.full(s, g) for g, s in enumerate(sizes)])
    rng.shuffle(job)
    vals = rng.choice(np.array([1.0, 2.0, -3.0]), (R, T))
    spread = rng.random((R, T)) < 0.6
    vals[spread] = rng.standard_normal(int(spread.sum()))
    special = rng.random((R, T)) < 0.1
    vals[special] = SPECIAL[rng.integers(0, SPECIAL.size, int(special.sum()))]
    ok = rng.random((R, T)) < 0.8
    ok[:, T // 2] = False
    labels = [{"job": f"j{job[r]}", "instance": f"i{r % 7}", "env": ["a", "b"][r % 2]} for r in range(R)]
    return vals, ok, labels


def bits_equal(a, b):
    return (np.isnan(a) & np.isnan(b)) | (np.asarray(a, np.float64).view(np.uint64) == np.asarray(b, np.float64).view(np.uint64))


@pytest.mark.parametrize("phi", PHIS)
@pytest.mark.parametrize("mod", [("by", ["job"]), ("without", ["instance", "env"]), ("by", ["env", "job"])])
def test_dense_quantile_matches_row_literal(phi, mod):
    rng = np.random.default_rng(17)
    T = 5
    sizes = [1, 2, 5, 31, 33, 70, 5000] if phi in (0.5, math.nan) else [1, 2, 5, 31, 33, 70]
    vals, ok, labels = random_labelled(rng, sizes, T)
    tags = ["env", "instance", "job"]
    rows = [(vals[r, k], labels[r], k) for r in range(len(labels)) for k in range(T) if ok[r, k]]
    kw = {mod[0]: mod[1]}
    got_rows, names = ago.aggregate_rows(rows, tags, "quantile", phi, **kw)
    # the dense form: group ids over the group labels, then per (group, step)
    keys = sorted({tuple(lab[n] for n in names) for lab in labels})
    gid = np.array([keys.index(tuple(lab[n] for n in names)) for lab in labels], np.uint32)
    out, cnt = ago.group_quantile(phi, vals, bor._words(ok), gid, len(keys))
    dense = [(out[g, k], dict(zip(names, key)), k) for g, key in enumerate(keys) for k in range(T) if cnt[g, k]]
    assert [(lab, ts) for _, lab, ts in got_rows] == [(lab, ts) for _, lab, ts in dense]
    assert bits_equal(np.array([v for v, _, _ in got_rows]), np.array([v for v, _, _ in dense])).all()
    assert not cnt[:, T // 2].any()
