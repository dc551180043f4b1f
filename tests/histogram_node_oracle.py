"""Row-literal restatement of histogram_quantile(φ, <child>) over any child (create_histogram_plan,
src/query/src/promql/planner.rs:3041-3108; HistogramFold, src/promql/src/extension_plan/histogram_fold.rs).

The child's exported rows are taken as they are: without the `le` tag the result is empty (the reference's
EmptyRelation); otherwise the rows are sorted as HistogramFold requires its input (the other tags, NULL last, then ts,
then CAST(le AS Float64) ascending with NaN and NULL last, :431-467; ties keep row order) and folded by
oracle.histogram_fold_rows, the restatement of fold_buf and the safe mode.  Rows are (value, {tag: label}, ts), as in
the other row-literal oracles."""
import math

import numpy as np

from oracle import oracle as orc
from tests import aggregate_oracle as ago
from tests.binary_helpers import dense_rows, table_arrays


def _nulls_last(v):
    return (1, "") if v is None else (0, v)


def _le_order(label):
    x = orc.parse_f64_rust(label)
    return (1, 0.0) if math.isnan(x) else (0, x)


def histogram_node(rows, tags, phi, le="le"):
    """rows [(value, {tag: label}, ts)] of a child with tag names `tags` -> ([(value, {tag: label}, ts)] in the
    reference's output order, the output tag names)"""
    if le not in tags:
        return [], []
    others = [t for t in tags if t != le]
    srt = sorted(rows, key=lambda r: (tuple(_nulls_last(r[1].get(t)) for t in others), r[2], _le_order(r[1].get(le))))
    lit = [(tuple(lab.get(t) for t in others), ts, lab.get(le), v) for v, lab, ts in srt]
    return [(v, dict(zip(others, key)), ts) for key, ts, v in orc.histogram_fold_rows(lit, phi)], others


def batch_rows(batch, tags, time_index, value):
    """An exported pyarrow batch -> rows [(value, {tag: label}, ts)] in batch order"""
    cols = {n: batch.column(i).to_pylist() for i, n in enumerate(batch.schema.names)}
    ts = batch.column(batch.schema.names.index(time_index)).cast("int64").to_pylist()
    return [(cols[value][i], {t: cols[t][i] for t in tags}, ts[i]) for i in range(batch.num_rows)]


def golden_child_rows(table, case):
    """A golden case's child on the CPU oracle: the instant selector or the range function over `table` (series
    restricted to the case's matchers), then its aggregate, if any -> (rows, tag names)"""
    child = case["child"]
    series = [s for s in table["series"] if all(s[k] == v for k, v in child.get("matchers", {}).items())]
    labels, ts, val, offsets = table_arrays(dict(table, series=series))
    start, end, interval = case["start"], case["end"], case["interval"]
    if child["kind"] == "instant":
        out, valid = orc.instant_query(ts, val, offsets, start, end, interval, child["lookback"])
    else:
        p = orc.make_params(child["function"][len("prom_"):], start, end, interval, child["range"])
        out, valid = orc.range_query(p, ts, val, None, offsets)
    tags = list(table["tags"])
    _, dense = dense_rows(tags, labels, out, valid, start + interval * np.arange(out.shape[1], dtype=np.int64))
    rows = [(r[-1], dict(zip(tags, r[:-2])), r[-2]) for r in dense]
    if "aggregate" in child:
        rows, tags = ago.aggregate_rows(rows, tags, child["aggregate"], by=child.get("by"))
    return rows, tags


def same_value(a, b):
    """Two result values agree: equal, or both NaN"""
    return (math.isnan(a) and math.isnan(b)) or a == b
