"""Shared by the metric-engine tests: golden tables as metric-engine batches (series divided on a UInt64 `__tsid`, a
hash of the label tuple, with the Utf8 label columns beside it, sorted by (__tsid, ts)) or as Utf8-keyed batches
(sorted by (labels, ts)), and the golden plans of reference_metric_engine_vectors.json."""
import hashlib
import json
import math
import os

from tests.helpers import GOLDEN_DIR


def load_metric_engine():
    with open(os.path.join(GOLDEN_DIR, "reference_metric_engine_vectors.json")) as f:
        return json.load(f)


def tsid_of(labels):
    """The series id of a label tuple (name, value) pairs: the first 8 bytes of its BLAKE2b hash (NULL hashes apart from
    every string), like the metric engine's hash of the label set"""
    h = hashlib.blake2b(digest_size=8)
    for name, value in labels:
        h.update(name.encode() + b"\x00" + (b"\x01" + value.encode() if value is not None else b"\x00") + b"\x00")
    return int.from_bytes(h.digest(), "little")


def series_rows(table):
    """-> [(label tuple, tsid, ts list, val list)] of the table's series; a series may give its own `__tsid`"""
    tags = table["tags"]
    out = []
    for s in table["series"]:
        lab = tuple(s.get(t) for t in tags)
        out.append((lab, s.get("__tsid", tsid_of(list(zip(tags, lab)))), list(s["ts"]), list(s["val"])))
    return out


def _null_first(v):
    return (v is not None, v or "")


def table_batches(table, metric_engine, splits=1):
    """The table as pyarrow batches: metric-engine (`ts, val, labels.., __tsid` sorted by tsid, ts) or Utf8-keyed
    (sorted by the label tuple, ts); `splits` cuts the rows into that many batches, so series continue across them.
    A table without rows gives no batch."""
    import pyarrow as pa
    tags = table["tags"]
    rows = series_rows(table)
    rows.sort(key=(lambda r: r[1]) if metric_engine else (lambda r: tuple(_null_first(v) for v in r[0])))
    flat = [(lab, tsid, t, v) for lab, tsid, ts, vals in rows for t, v in zip(ts, vals)]
    cols = {table["time_index"]: pa.array([r[2] for r in flat], pa.timestamp("ms")),
            table["field"]: pa.array([r[3] for r in flat], pa.float64())}
    for i, t in enumerate(tags):
        cols[t] = pa.array([r[0][i] for r in flat], pa.string())
    if metric_engine:
        cols["__tsid"] = pa.array([r[1] for r in flat], pa.uint64())
    batch = pa.RecordBatch.from_pydict(cols)
    n = batch.num_rows
    cuts = sorted({0, n} | {n * i // splits for i in range(1, splits)})
    return [batch.slice(a, b - a) for a, b in zip(cuts, cuts[1:])]


def leaf(ctx, table, metric_engine, start, end, interval, fn=None, range_ms=0, lookback=None, splits=1, **kw):
    """A range leaf (fn) or instant leaf (lookback) over the table, fed its batches.  A table without labels (a metric
    that does not exist) has no __tsid, so its leaf is the tagless one in either form."""
    from greptimedb_b200.plan import PromRangeExec
    tags = list(table["tags"])
    metric_engine = metric_engine and bool(tags)
    key = dict(tag_columns=["__tsid"], label_columns=tags) if metric_engine else dict(tag_columns=tags)
    n = PromRangeExec(ctx, fn or "", start, end, interval, range_ms, table["time_index"], table["field"],
                      lookback_delta=lookback if fn is None else None, **key, **kw)
    for b in table_batches(table, metric_engine, splits):
        n.push(b)
    return n


def build(ctx, expr, tables, case, metric_engine):
    """The plan of a golden `expr` (see the fixture's _source) with every leaf in the given form"""
    from greptimedb_b200.plan import AggregatePlan, BinaryPlan, HistogramQuantilePlan, ScalarPlan, SetOpPlan, TopkPlan
    kind = expr[0]
    rec = lambda e: build(ctx, e, tables, case, metric_engine)
    grid = (case["start"], case["end"], case["interval"])
    if kind == "sel":
        return leaf(ctx, tables[expr[1]], metric_engine, *grid, lookback=expr[2])
    if kind == "range":
        return leaf(ctx, tables[expr[2]], metric_engine, *grid, fn=expr[1], range_ms=expr[3])
    if kind == "fn":
        return rec(expr[2]).function(expr[1])
    if kind == "scalar":
        return rec(expr[3]).scalar_op(expr[1], expr[2])
    if kind == "gt":
        return rec(expr[2]).scalar_op(">", expr[1])
    if kind == "bin":
        return BinaryPlan(ctx, expr[1], rec(expr[2]), rec(expr[3]), **expr[4])
    if kind == "or":
        return SetOpPlan(ctx, "or", rec(expr[1]), rec(expr[2]))
    if kind == "agg":
        return AggregatePlan(ctx, expr[1], rec(expr[2]), **expr[3])
    if kind == "topk":
        return TopkPlan(ctx, "topk", expr[1], rec(expr[2]))
    if kind == "hq":
        return HistogramQuantilePlan(ctx, expr[1], rec(expr[2]))
    if kind == "scalar_of":
        return ScalarPlan(ctx, rec(expr[1]))
    raise ValueError(kind)


def value_column(batch, time_index, labels):
    names = [n for n in batch.schema.names if n not in (time_index, "__tsid") and n not in labels]
    assert len(names) == 1, batch.schema.names
    return names[0]


def rows_of(batch, time_index, labels):
    """-> sorted [(labels.., ts ms, value)] of a result batch; a label the batch lacks reads as NULL"""
    import pyarrow as pa
    if batch.num_columns == 0:
        return []
    v = value_column(batch, time_index, labels)
    ts = batch.column(time_index).cast(pa.int64()).to_pylist()
    vals = batch.column(v).to_pylist()
    labs = [batch.column(l).to_pylist() if l in batch.schema.names else [None] * batch.num_rows for l in labels]
    return sorted((tuple(col[i] for col in labs) + (ts[i], vals[i]) for i in range(batch.num_rows)),
                  key=lambda r: tuple(_null_first(x) for x in r[:-2]) + r[-2:])


def expected_of(case, labels):
    return sorted((tuple(lab.get(l) for l in labels) + (ts, float(v)) for lab, ts, v in case["expected"]),
                  key=lambda r: tuple(_null_first(x) for x in r[:-2]) + r[-2:])


# ---- the CPU restatement: a leaf divided on __tsid, and the row-literal node helpers above it ---------------------------
def oracle_leaf(table, metric_engine, start, end, interval, fn=None, range_ms=0, lookback=300_000):
    """The leaf on the CPU over the table's batches: series divided where `__tsid` changes (metric_engine) or where the
    label tuple does, each series labelled by its first row -> (tag names, rows [(labels.., ts, value)])"""
    import numpy as np
    import pyarrow as pa

    from oracle import oracle as orc
    tags = list(table["tags"])
    if not table["series"]:
        return tags, []
    metric_engine = metric_engine and bool(tags)
    batch = pa.Table.from_batches(table_batches(table, metric_engine, splits=3)).combine_chunks().to_batches()[0]
    ts = np.array(batch.column(table["time_index"]).cast(pa.int64()).to_pylist(), np.int64)
    val = np.array(batch.column(table["field"]).to_pylist(), np.float64)
    labels = [batch.column(t).to_pylist() for t in tags]
    key = batch.column("__tsid").to_pylist() if metric_engine else list(zip(*labels)) if tags else [()] * len(ts)
    starts = [i for i in range(len(ts)) if i == 0 or key[i] != key[i - 1]]
    offsets = np.array(starts + [len(ts)], np.uint64)
    series = [tuple(col[i] for col in labels) for i in starts]
    if fn is None:
        out, valid = orc.instant_query(ts, val, offsets, start, end, interval, lookback)
    else:
        out, valid = orc.range_query(orc.make_params(fn, start, end, interval, range_ms), ts, val, None, offsets)
    T = orc.num_steps(start, end, interval)
    rows = [lab + (start + k * interval, float(out[s, k])) for s, lab in enumerate(series) for k in range(T)
            if (int(valid[s, k // 32]) >> (k % 32)) & 1]
    return tags, rows


def oracle_eval(expr, tables, case, metric_engine):
    """A golden `expr` on the CPU -> (tag names, rows [(labels.., ts, value)])"""
    from tests import aggregate_oracle as agg
    from tests import binary_oracle as bor
    from tests import histogram_node_oracle as hno
    from tests import set_oracle as sor
    from tests import topk_oracle as tor
    from tests.instant_fn_oracle import apply
    rec = lambda e: oracle_eval(e, tables, case, metric_engine)
    grid = (case["start"], case["end"], case["interval"])
    as_dicts = lambda tags, rows: [(r[-1], dict(zip(tags, r[:-2])), r[-2]) for r in rows]
    from_dicts = lambda tags, rows: (list(tags), [tuple(lab.get(t) for t in tags) + (ts, v) for v, lab, ts in rows])
    kind = expr[0]
    if kind == "sel":
        return oracle_leaf(tables[expr[1]], metric_engine, *grid, lookback=expr[2])
    if kind == "range":
        return oracle_leaf(tables[expr[2]], metric_engine, *grid, fn=expr[1].replace("prom_", ""), range_ms=expr[3])
    if kind == "fn":
        tags, rows = rec(expr[2])
        return tags, [r[:-1] + (float(apply(expr[1], r[-1])),) for r in rows]
    if kind in ("scalar", "gt"):
        tags, rows = rec(expr[3] if kind == "scalar" else expr[2])
        op, x = (expr[1], expr[2]) if kind == "scalar" else (">", expr[1])
        return tags, bor.scalar_rows(rows, op, x)
    if kind == "bin":
        return bor.binary_rows(rec(expr[2]), rec(expr[3]), expr[1], **expr[4])
    if kind == "or":
        return sor.setop_rows(rec(expr[1]), rec(expr[2]), "or")
    if kind == "agg":
        tags, rows = rec(expr[2])
        out, names = agg.aggregate_rows(as_dicts(tags, rows), tags, expr[1], **expr[3])
        return from_dicts(names, out)
    if kind == "topk":
        tags, rows = rec(expr[2])
        return from_dicts(tags, tor.topk_rows(False, expr[1], as_dicts(tags, rows), tags))
    if kind == "hq":
        tags, rows = rec(expr[2])
        out, names = hno.histogram_node(as_dicts(tags, rows), tags, expr[1])
        return from_dicts(names, out)
    if kind == "scalar_of":   # scalar(): the one series' value at each step, NaN where there is not exactly one
        _, rows = rec(expr[1])
        start, end, step = grid
        at = {}
        for r in rows:
            at.setdefault(r[-2], []).append(r[-1])
        return [], [(t, at[t][0] if len(at.get(t, [])) == 1 else math.nan) for t in range(start, end + 1, step)]
    raise ValueError(kind)
