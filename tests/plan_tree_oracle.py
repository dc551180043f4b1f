"""PromQL expression trees with two interpretations: `build` makes the plan-node handles of greptimedb_b200.plan, and
`evaluate` composes the row-literal oracles of tests/ bottom-up from the tables' rows (test infrastructure; CPU only).

A tree is a `Node(kind, children, args)`; one constructor per plan node and stage:
  leaf(table, fn=None, range=0)        the instant selector (fn None) or fn(table[range]) of a range function
  vector(s) / time()                   EmptyMetric literal / time()
  binary(op, lhs, rhs, ...)            BinaryPlan (on | ignoring, bool, label_side)
  setop(op, lhs, rhs, ...)             SetOpPlan (on | ignoring)
  aggregate(op, child, ...)            AggregatePlan (the seven accumulators, group, quantile; by | without)
  topk(op, k, child, ...)              TopkPlan (by | without)
  sort(function, child, labels)        SortPlan
  label_join(child, dst, sep, *srcs)   LabelJoinPlan
  label_replace(child, dst, repl, src, regex)  LabelReplacePlan over the patterns in REGEXES
  scalar_op(child, op, s, ...)         the `node op scalar` stage
  function(child, name, *args)         the instant-function stage, unary minus as "negative", the calendar functions
  subquery(fn, child, range)           SubqueryPlan fn(child[range:interval]); the child lives on the inner grid
Tables are dicts {"time_index", "field", "tags", "series": [{tag: label or None, "ts": [..], "val": [..]}]}; one grid
(start, end, interval) serves the whole tree.

What the interpreter carries between nodes is what the device carries: a grid of rows, each a series (one label tuple)
with a cell per step.  A row is (value, {tag: label}, ts, rid, pin, maybe): `rid` is the row's position in the node's
grid as a tuple that sorts like the device's row order (a binary pair is (lhs rid + rhs rid), `or` puts (0,) + lhs before
(1,) + rhs), so the child's row-major order — which fixes a sum's addend order, sort's and topk's ties and `or`'s first
rhs row — is the order of (rid, ts).

Unpinned cells (DESIGN.md §2): the GPU's and x86's default NaN differ in sign and payload, so a NaN an operation
computes is only a NaN: its pin is "nan".  A node that orders or compares such a cell cannot know what the device
decided: a comparison makes the row `maybe` (it may exist or not) and a `bool` value "any"; sort and topk leave the order
of a partition holding one open (topk keeps every member as `maybe`); min / max / quantile give "any"; a NaN copied from a
sample keeps its bits ("bits").  `export` is the node's rows in the reference's output order where it pins one (sort,
topk, aggregate), else in row-major order.
"""
from __future__ import annotations

import math
import re
import struct
from dataclasses import dataclass, field

import numpy as np

from oracle import oracle as orc
from tests import aggregate_oracle as ago
from tests import binary_oracle as bor
from tests import instant_fn_oracle as ifo
from tests import set_oracle as sor
from tests import sort_oracle as soo
from tests import time_fn_oracle as tfo
from tests import topk_oracle as tko
from tests.range_values import nan_with_payload, series_values

LOOKBACK = 300_000
BITS, NAN, ANY = "bits", "nan", "any"
COPYING_RANGE_FNS = ("min_over_time", "max_over_time", "last_over_time")
# the device's names of the exact instant functions -> the oracle's
EXACT_FNS = {"abs": "abs", "ceil": "ceil", "floor": "floor", "sqrt": "sqrt", "prom_round": "round", "degrees": "deg",
             "radians": "rad", "signum": "sgn", "clamp": "clamp", "clamp_min": "clamp_min", "clamp_max": "clamp_max",
             "negative": "negative"}
# the calendar functions (K19): Int32 on the device, so the generator puts an arithmetic stage on top of each
CALENDAR = ("minute", "hour", "month", "year", "day_of_month", "day_of_week", "day_of_year", "days_in_month")
# label_replace patterns the plan's regex engine and Python's `re` read alike
REGEXES = ("(.*)", "h(.*)", "(a|b)(.*)", "", "[0-9]+", "(.)(.)?")


# ---- trees -------------------------------------------------------------------------------------------------------------
@dataclass(eq=False)
class Node:
    kind: str
    children: tuple = ()
    args: dict = field(default_factory=dict)

    def subtrees(self):
        """post-order: every subtree before its parent"""
        for c in self.children:
            yield from c.subtrees()
        yield self

    def size(self):
        return sum(1 for _ in self.subtrees())

    def depth(self):
        return 1 + max((c.depth() for c in self.children), default=0)


def leaf(table, fn=None, range=0):
    return Node("leaf", (), {"table": table, "fn": fn, "range": range})


def vector(s):
    return Node("vector", (), {"s": float(s)})


def time():
    return Node("time")


def binary(op, lhs, rhs, return_bool=False, on=None, ignoring=None, label_side="rhs"):
    return Node("binary", (lhs, rhs), {"op": op, "bool": return_bool, "on": on, "ignoring": ignoring,
                                        "label_side": label_side})


def setop(op, lhs, rhs, on=None, ignoring=None):
    return Node("setop", (lhs, rhs), {"op": op, "on": on, "ignoring": ignoring})


def aggregate(op, child, param=None, by=None, without=None):
    return Node("aggregate", (child,), {"op": op, "param": param, "by": by, "without": without})


def topk(op, k, child, by=None, without=None):
    return Node("topk", (child,), {"op": op, "k": float(k), "by": by, "without": without})


def sort(function, child, labels=()):
    return Node("sort", (child,), {"function": function, "labels": list(labels)})


def label_join(child, dst, sep, *srcs):
    return Node("label_join", (child,), {"dst": dst, "sep": sep, "srcs": list(srcs)})


def label_replace(child, dst, replacement, src, regex):
    return Node("label_replace", (child,), {"dst": dst, "replacement": replacement, "src": src, "regex": regex})


def scalar_op(child, op, s, on_left=False, return_bool=False):
    return Node("scalar_op", (child,), {"op": op, "s": float(s), "on_left": on_left, "bool": return_bool})


def function(child, name, *args):
    return Node("function", (child,), {"name": name, "args": [float(a) for a in args]})


def subquery(fn, child, range):
    return Node("subquery", (child,), {"fn": fn, "range": int(range)})


def child_grid(n: Node, grid):
    """the grid n's children are evaluated on: a subquery's inner grid start - range + interval .. end"""
    if n.kind != "subquery":
        return grid
    start, end, step = grid
    return start - n.args["range"] + step, end, step


def _mod(a):
    return (f" by ({', '.join(a['by'])})" if a.get("by") is not None else
            f" without ({', '.join(a['without'])})" if a.get("without") is not None else "")


def _match(a):
    return (f" on({', '.join(a['on'])})" if a.get("on") is not None else
            f" ignoring({', '.join(a['ignoring'])})" if a.get("ignoring") is not None else "")


def promql(n: Node) -> str:
    """The tree as PromQL text (plan-only details such as label_side in a comment)"""
    a, c = n.args, [promql(x) for x in n.children]
    if n.kind == "leaf":
        return a["table"] if a["fn"] is None else f"{a['fn']}({a['table']}[{a['range'] // 1000}s])"
    if n.kind == "vector":
        return f"vector({a['s']!r})"
    if n.kind == "time":
        return "time()"
    if n.kind == "binary":
        side = "" if a["label_side"] == "rhs" else " /*labels of lhs*/"
        return f"({c[0]} {a['op']}{' bool' if a['bool'] else ''}{_match(a)}{side} {c[1]})"
    if n.kind == "setop":
        return f"({c[0]} {a['op']}{_match(a)} {c[1]})"
    if n.kind == "aggregate":
        p = f"{a['param']!r}, " if a["op"] == "quantile" else ""
        return f"{a['op']}{_mod(a)} ({p}{c[0]})"
    if n.kind == "topk":
        return f"{a['op']}{_mod(a)} ({a['k']!r}, {c[0]})"
    if n.kind == "sort":
        return f"{a['function']}({', '.join([c[0]] + [repr(l) for l in a['labels']])})"
    if n.kind == "label_join":
        return f"label_join({c[0]}, {a['dst']!r}, {a['sep']!r}, {', '.join(repr(s) for s in a['srcs'])})"
    if n.kind == "label_replace":
        return f"label_replace({c[0]}, {a['dst']!r}, {a['replacement']!r}, {a['src']!r}, {a['regex']!r})"
    if n.kind == "scalar_op":
        b = " bool" if a["bool"] else ""
        return f"({a['s']!r} {a['op']}{b} {c[0]})" if a["on_left"] else f"({c[0]} {a['op']}{b} {a['s']!r})"
    if n.kind == "subquery":
        return f"{a['fn']}({c[0]}[{a['range'] // 1000}s:])"
    if n.kind == "function":
        if a["name"] == "negative":
            return f"-{c[0]}"
        return f"{a['name']}({', '.join([c[0]] + [repr(x) for x in a['args']])})"
    raise ValueError(n.kind)


# ---- the device side ----------------------------------------------------------------------------------------------------
def table_series(table):
    """the table's series in the order the leaf is fed (tag tuples by the plan's label order: "", NULL, strings)"""
    tags = table["tags"]
    return sorted(table["series"], key=lambda s: tuple(ago.label_order(s[t]) for t in tags))


def table_batch(table):
    import pyarrow as pa
    series = [s for s in table_series(table) if len(s["ts"])]
    cols = {table["time_index"]: pa.array([t for s in series for t in s["ts"]], pa.timestamp("ms")),
            table["field"]: pa.array(np.array([v for s in series for v in s["val"]], np.float64), pa.float64())}
    for t in table["tags"]:
        cols[t] = pa.array([s[t] for s in series for _ in s["ts"]], pa.string())
    return pa.RecordBatch.from_pydict(cols) if series else None


def build(ctx, n: Node, tables, grid):
    """The plan-node handle of tree n (every leaf a fresh PromRangeExec fed its table)"""
    from greptimedb_b200 import plan as P
    start, end, step = grid
    a = n.args
    kids = [build(ctx, c, tables, child_grid(n, grid)) for c in n.children]
    if n.kind == "leaf":
        t = tables[a["table"]]
        fn = a["fn"]
        ex = P.PromRangeExec(ctx, "prom_" + fn if fn else "", start, end, step, a["range"], t["time_index"], t["field"],
                             t["tags"], lookback_delta=None if fn else LOOKBACK)
        b = table_batch(t)
        if b is not None:
            ex.push(b)
        return ex
    if n.kind == "vector":
        return P.EmptyMetricPlan(ctx, start, end, step, "literal", literal=a["s"])
    if n.kind == "time":
        return P.EmptyMetricPlan(ctx, start, end, step, "time")
    if n.kind == "binary":
        return P.BinaryPlan(ctx, a["op"], kids[0], kids[1], return_bool=a["bool"], on=a["on"], ignoring=a["ignoring"],
                            label_side=a["label_side"])
    if n.kind == "setop":
        return P.SetOpPlan(ctx, a["op"], kids[0], kids[1], on=a["on"], ignoring=a["ignoring"])
    if n.kind == "aggregate":
        return P.AggregatePlan(ctx, a["op"], kids[0], param=a["param"], by=a["by"], without=a["without"])
    if n.kind == "topk":
        return P.TopkPlan(ctx, a["op"], a["k"], kids[0], by=a["by"], without=a["without"])
    if n.kind == "sort":
        return P.SortPlan(ctx, a["function"], kids[0], a["labels"])
    if n.kind == "label_join":
        return P.LabelJoinPlan(ctx, kids[0], a["dst"], a["sep"], *a["srcs"])
    if n.kind == "label_replace":
        return P.LabelReplacePlan(ctx, kids[0], a["dst"], a["replacement"], a["src"], a["regex"])
    if n.kind == "scalar_op":
        return kids[0].scalar_op(a["op"], a["s"], scalar_on_left=a["on_left"], return_bool=a["bool"])
    if n.kind == "function":
        return kids[0].function(a["name"], *a["args"])
    if n.kind == "subquery":
        return P.SubqueryPlan(ctx, "prom_" + a["fn"], kids[0], start, end, step, a["range"])
    raise ValueError(n.kind)


# ---- the row-literal side -----------------------------------------------------------------------------------------------
@dataclass
class Row:
    value: float
    labels: dict
    ts: int
    rid: tuple
    pin: str = BITS
    maybe: bool = False


@dataclass
class Result:
    tags: list
    rows: list          # the grid's cells in row-major order: what a parent node reads
    export: list        # the rows execute() emits, in the reference's order where it pins one
    ordered: bool = False  # whether `export`'s order is pinned


def bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def _row_major(rows):
    return sorted(rows, key=lambda r: (r.rid, r.ts))


def _result(tags, rows, export=None, ordered=False):
    rows = _row_major(rows)
    return Result(list(tags), rows, rows if export is None else export, ordered)


def _computed_pin(value, *inputs):
    """pin of a value an operation computed from cells of the given pins"""
    if ANY in inputs:
        return ANY
    return NAN if math.isnan(value) else BITS


def _cmp_open(op, x, px, y, py):
    """whether the comparison `x op y` of cells pinned px / py could come out either way on the device: a NaN of open
    sign orders below or above every number, but equals none"""
    if ANY in (px, py):
        return True
    if BITS == px == py:
        return False
    if op in ("==", "!="):
        return math.isnan(x) and math.isnan(y)
    return True


def grid_steps(grid):
    start, end, step = grid
    return [start + k * step for k in range(orc.num_steps(start, end, step))]


def _leaf(n, tables, grid):
    a, t = n.args, tables[n.args["table"]]
    start, end, step = grid
    series = [s for s in table_series(t) if len(s["ts"])]
    ts = np.array([x for s in series for x in s["ts"]], np.int64)
    val = np.array([v for s in series for v in s["val"]], np.float64)
    offsets = np.cumsum([0] + [len(s["ts"]) for s in series]).astype(np.uint64)
    steps = grid_steps(grid)
    if not series or not steps:
        return _result(t["tags"], [])
    if a["fn"] is None:
        out, valid = orc.instant_query(ts, val, offsets, start, end, step, LOOKBACK)
    else:
        out, valid = orc.range_query(orc.make_params(a["fn"], start, end, step, a["range"]), ts, val, None, offsets,
                                     rescan=True)
    copies = a["fn"] is None or a["fn"] in COPYING_RANGE_FNS
    rows = []
    for r, s in enumerate(series):
        for k, t_ in enumerate(steps):
            if (int(valid[r, k // 32]) >> (k % 32)) & 1:
                v = float(out[r, k])
                rows.append(Row(v, {g: s[g] for g in t["tags"]}, t_, (r,), BITS if copies else _computed_pin(v)))
    return _result(t["tags"], rows)


def _scalar_op(n, child):
    a = n.args
    is_cmp = bor._op_id(a["op"]) >= bor._EQ
    out = []
    for r in child.rows:
        v = bor.scalar_value(a["op"], a["s"], r.value, a["on_left"], a["bool"])
        if is_cmp and _cmp_open(a["op"], r.value, r.pin, a["s"], BITS):   # it read a cell whose bits are open
            if a["bool"]:
                out.append(Row(0.0 if v is None else v, r.labels, r.ts, r.rid, ANY, r.maybe))
            else:
                out.append(Row(r.value, r.labels, r.ts, r.rid, r.pin, True))
            continue
        if v is None:
            continue
        pin = r.pin if (is_cmp and not a["bool"]) else BITS if is_cmp else _computed_pin(v, r.pin)
        out.append(Row(v, r.labels, r.ts, r.rid, pin, r.maybe))
    return _result(child.tags, out)


def apply_function(name, v, args):
    if name == "negative":
        return -v
    return float(ifo.apply(EXACT_FNS.get(name, name), np.array([v]), *args)[0])


def _function(n, child):
    a = n.args
    out = []
    if a["name"] in CALENDAR:   # f(eval ts) at every valid cell: the cell's value is not read
        return _result(child.tags, [Row(float(tfo.step_value(a["name"], r.ts)), r.labels, r.ts, r.rid, BITS, r.maybe)
                                    for r in child.rows])
    for r in child.rows:
        v = apply_function(a["name"], r.value, a["args"])
        out.append(Row(v, r.labels, r.ts, r.rid, _computed_pin(v, r.pin), r.maybe))
    return _result(child.tags, out)


def _binary(n, lhs, rhs):
    a = n.args
    keys = bor.binary_key_columns(lhs.tags, rhs.tags, a["on"], a["ignoring"])
    is_cmp = bor._op_id(a["op"]) >= bor._EQ
    is_filter = is_cmp and not a["bool"]
    from_lhs = is_filter or a["label_side"] == "lhs"
    table = {}
    for r in rhs.rows:
        table.setdefault((tuple(r.labels.get(k) for k in keys), r.ts), []).append(r)
    out = []
    for l in lhs.rows:
        for r in table.get((tuple(l.labels.get(k) for k in keys), l.ts), []):
            v = bor.binary_value(a["op"], l.value, r.value, a["bool"])
            maybe = l.maybe or r.maybe
            side = l if from_lhs else r
            if is_cmp and _cmp_open(a["op"], l.value, l.pin, r.value, r.pin):
                if is_filter:
                    out.append(Row(l.value, side.labels, l.ts, l.rid + r.rid, l.pin, True))
                else:
                    out.append(Row(0.0 if v is None else v, side.labels, l.ts, l.rid + r.rid, ANY, maybe))
                continue
            if v is None:
                continue
            pin = l.pin if is_filter else BITS if is_cmp else _computed_pin(v, l.pin, r.pin)
            out.append(Row(v, side.labels, l.ts, l.rid + r.rid, pin, maybe))
    return _result(lhs.tags if from_lhs else rhs.tags, out)


def _setop(n, lhs, rhs):
    a, op = n.args, n.args["op"]
    keys, out_tags = sor.setop_key_columns(op, lhs.tags, rhs.tags, a["on"], a["ignoring"])
    key = lambda r: (tuple(r.labels.get(k) for k in keys), r.ts)
    if op != "or":
        # left.distinct(): a cell equal to an earlier one in labels, ts and value bits goes
        seen, distinct = {}, []
        for r in lhs.rows:
            d = (tuple(sorted(r.labels.items(), key=lambda kv: kv[0])), r.ts)
            earlier = seen.setdefault(d, [])
            if any(e.pin == BITS and r.pin == BITS and bits(e.value) == bits(r.value) and not e.maybe for e in earlier):
                continue
            open_ = any(e.pin != BITS or r.pin != BITS or e.maybe for e in earlier
                        if not (e.pin == BITS and r.pin == BITS and bits(e.value) != bits(r.value)))
            earlier.append(r)
            distinct.append((r, open_))
        sure, unsure = set(), set()
        for r in rhs.rows:
            (unsure if r.maybe else sure).add(key(r))
        out = []
        for r, open_ in distinct:
            k = key(r)
            present = k in sure
            if present == (op == "and") or k in unsure and k not in sure:
                out.append(Row(r.value, r.labels, r.ts, r.rid, r.pin, r.maybe or open_ or (k in unsure and not present)))
        return _result(lhs.tags, out)
    widen = lambda r: {t: r.labels.get(t) for t in out_tags}
    out = [Row(r.value, widen(r), r.ts, (0,) + r.rid, r.pin, r.maybe) for r in lhs.rows]
    sure, unsure = set(), set()
    for r in lhs.rows:
        (unsure if r.maybe else sure).add(key(r))
    for r in rhs.rows:
        k = key(r)
        if k in sure:
            continue
        out.append(Row(r.value, widen(r), r.ts, (1,) + r.rid, r.pin, r.maybe or k in unsure))
        (unsure if r.maybe or k in unsure else sure).add(k)
    return _result(out_tags, out)


def _aggregate(n, child):
    a, op = n.args, n.args["op"]
    names = ago.group_names(child.tags, a["by"], a["without"])
    buckets = {}
    for r in child.rows:
        buckets.setdefault((tuple(r.labels.get(g) for g in names), r.ts), []).append(r)
    groups = sorted({g for g, _ in buckets}, key=lambda g: tuple(ago.label_order(x) for x in g))
    gix = {g: i for i, g in enumerate(groups)}
    out = []
    for (g, ts), members in buckets.items():
        sure = [m for m in members if not m.maybe]
        v = ago.accumulate(op, [m.value for m in sure] or [m.value for m in members], a["param"])
        pins = {m.pin for m in members}
        if op == "group":
            pin = BITS
        elif len(sure) != len(members):
            pin = ANY
        elif op == "count":
            pin = BITS
        elif ANY in pins or (NAN in pins and op in ("min", "max", "quantile")):
            pin = ANY
        else:
            pin = NAN if math.isnan(v) else BITS
        out.append(Row(v, dict(zip(names, g)), ts, (gix[g],), pin, not sure))
    rows = _row_major(out)
    return Result(names, rows, rows, True)


def _topk(n, child):
    a = n.args
    bottom = a["op"] == "bottomk"
    modifier, labels = ("by", a["by"]) if a["by"] is not None else ("without", a["without"]) \
        if a["without"] is not None else (None, ())
    gcols = tko.group_columns(child.tags, modifier, labels)
    parts = {}
    for r in child.rows:
        parts.setdefault((tuple(r.labels.get(g) for g in gcols), r.ts), []).append(r)
    kept, exported, ordered = [], [], True
    # export order: group labels, ts, rank; the plan layer orders NULL group labels by its one label order, where the
    # reference puts them last (DESIGN.md §2, "Known divergence: where NULL labels sort")
    for key in sorted(parts, key=lambda p: (tuple(ago.label_order(x) for x in p[0]), p[1])):
        members = parts[key]
        if any(m.pin != BITS or m.maybe for m in members):   # the ranking read an open cell: any member may stay
            ordered = False
            if tko.kept_ranks(a["k"], len(members)):
                chosen = [Row(m.value, m.labels, m.ts, m.rid, m.pin, True) for m in members]
                kept += chosen
                exported += chosen
            continue
        lit = [(m.value, m.labels, m.ts) for m in members]
        ranked = tko.topk_rows(bottom, a["k"], lit, child.tags, modifier, labels)
        by_id = {id(t): m for t, m in zip(lit, members)}
        chosen = [by_id[id(t)] for t in ranked]
        kept += chosen
        exported += chosen
    return Result(child.tags, _row_major(kept), exported, ordered)


def _sort(n, child):
    a = n.args
    lit = [(r.value, r.labels, r.ts) for r in child.rows]
    by_id = {id(t): r for t, r in zip(lit, child.rows)}
    order = [by_id[id(t)] for t in soo.sort_rows(a["function"], lit, a["labels"])]
    by_label = a["function"].startswith("sort_by_label")
    ordered = by_label or all(r.pin == BITS and not r.maybe for r in child.rows)
    return Result(child.tags, child.rows, order, ordered)


def _subquery(n, child, grid):
    """every grid row of the child is one series whose samples are its valid cells, NaN included (filter_nan off)"""
    a = n.args
    start, end, step = grid
    series = {}
    for r in child.rows:
        series.setdefault(r.rid, []).append(r)
    steps = grid_steps(grid)
    if not series or not steps:
        return _result(child.tags, [])
    cells = [c for rows in series.values() for c in rows]
    ts = np.array([c.ts for c in cells], np.int64)
    val = np.array([c.value for c in cells], np.float64)
    offsets = np.cumsum([0] + [len(rows) for rows in series.values()]).astype(np.uint64)
    out, valid = orc.range_query(orc.make_params(a["fn"], start, end, step, a["range"], filter_nan=False), ts, val, None,
                                 offsets, rescan=True)
    rows = []
    for i, (rid, members) in enumerate(series.items()):
        open_ts = [m.ts for m in members if m.pin != BITS or m.maybe]
        for k, t_ in enumerate(steps):
            # a window over an open cell or a row that may not exist: any value, and the window may be empty
            in_window = [x for x in open_ts if t_ - a["range"] < x <= t_]
            window = [m for m in members if t_ - a["range"] < m.ts <= t_]
            maybe = bool(window) and all(m.maybe for m in window)
            if (int(valid[i, k // 32]) >> (k % 32)) & 1:
                v = float(out[i, k])
                pin = ANY if in_window else BITS if a["fn"] in COPYING_RANGE_FNS else _computed_pin(v)
                rows.append(Row(v, members[0].labels, t_, rid, pin, maybe))
    return _result(child.tags, rows)


def _with_label(child, dst, value_of):
    tags = [t for t in child.tags if t != dst] + [dst]
    out = []
    for r in child.rows:
        lab = {t: r.labels.get(t) for t in child.tags if t != dst}
        lab[dst] = value_of(r)
        out.append(Row(r.value, lab, r.ts, r.rid, r.pin, r.maybe))
    return _result(tags, out)


def _label_join(n, child):
    a = n.args
    # concat_ws: a NULL source, or one that is no tag, is skipped; an empty one is joined
    return _with_label(child, a["dst"], lambda r: a["sep"].join(
        v for v in (r.labels.get(s) for s in a["srcs"] if s in child.tags) if v is not None))


def label_replace_value(regex, replacement, value):
    """the expanded replacement where the whole value matches, else None (Rust's `$1` / `${1}` expansion; a group that
    did not take part is "")"""
    m = re.fullmatch(regex, value, re.DOTALL)
    if m is None:
        return None
    def group(g):
        i = int(g.group(1).strip("{}"))
        return (m.group(i) or "") if i <= m.re.groups else ""
    return re.sub(r"\$(\d+|\{\d+\})", group, replacement)


def _label_replace(n, child):
    a = n.args
    src, dst = a["src"], a["dst"]
    if src in child.tags:
        if a["regex"] == "":
            return child
        def value_of(r):
            v = r.labels.get(src)
            if v is None:
                return None
            new = label_replace_value(a["regex"], a["replacement"], v)
            return v if new is None else new
        return _with_label(child, dst, value_of)
    if a["replacement"] == "":
        return child
    return _with_label(child, dst, lambda r: a["replacement"])


def evaluate(n: Node, tables, grid) -> Result:
    """Row-literal result of tree n over the tables' rows on the grid (start, end, interval)"""
    kids = [evaluate(c, tables, child_grid(n, grid)) for c in n.children]
    if n.kind == "subquery":
        return _subquery(n, kids[0], grid)
    if n.kind == "leaf":
        return _leaf(n, tables, grid)
    if n.kind in ("vector", "time"):
        rows = [Row(n.args["s"] if n.kind == "vector" else t / 1000.0, {}, t, (0,)) for t in grid_steps(grid)]
        return _result([], rows)
    return {"binary": _binary, "setop": _setop}[n.kind](n, *kids) if len(kids) == 2 else {
        "scalar_op": _scalar_op, "function": _function, "aggregate": _aggregate, "topk": _topk, "sort": _sort,
        "label_join": _label_join, "label_replace": _label_replace}[n.kind](n, kids[0])


# ---- seeded tables and trees --------------------------------------------------------------------------------------------
STEPS = (1, 31, 32, 33, 64, 65, 200)
TAG_VALUES = ("a0", "a1", "b0", "", None, "h7", "h12")
RANGE_FNS = ("rate", "increase", "delta", "idelta", "sum_over_time", "avg_over_time", "min_over_time",
             "max_over_time", "last_over_time", "count_over_time", "resets", "changes", "stddev_over_time")
SUBQUERY_FNS = ("max_over_time", "min_over_time", "last_over_time", "sum_over_time", "avg_over_time",
                "count_over_time", "changes", "resets", "delta", "stddev_over_time")
ARITH = ("+", "-", "*", "/", "%")
CMP = ("==", "!=", ">", "<", ">=", "<=")
AGG_OPS = ("sum", "avg", "count", "min", "max", "stddev", "stdvar", "group", "quantile")
# the table schemas: two plain ones and one whose tags include `zone`, which holds NULLs and empty strings
SCHEMAS = {"m1": ["host", "job"], "m2": ["host", "job", "zone"], "m3": ["host"]}


def make_grid(rng):
    T = int(rng.choice(STEPS))
    step = int(rng.choice([15_000, 30_000, 60_000]))
    start = 1_700_000_000_000 + int(rng.integers(0, step))     # not aligned to the samples
    return start, start + (T - 1) * step, step


def make_series(rng, grid, labels):
    """one series: a value class of tests/range_values.py on scrapes that may start mid-grid, with the odd duplicate
    timestamp; some series have no sample in reach of the grid at all"""
    start, end, step = grid
    scrape = int(rng.choice([10_000, 15_000, 20_000, 45_000]))
    lo = start - 2 * LOOKBACK if rng.random() < 0.7 else start + int(rng.integers(0, end - start + 1))
    if rng.random() < 0.08:
        lo = end + LOOKBACK + 1   # no sample where the grid looks
    n = max(1, min(600, (end - lo) // scrape + 1))
    ts = lo + scrape * np.arange(n, dtype=np.int64) + rng.integers(0, scrape // 4, n)
    ts = np.sort(ts)
    if n > 3 and rng.random() < 0.3:
        i = int(rng.integers(1, n))
        ts[i] = ts[i - 1]
    # (ordinary classes weigh double: the special ones make NaNs, which only have to be NaNs, in most operations)
    cls = str(rng.choice(["counter", "counter", "counter", "gauge", "gauge", "offset", "offset", "ties", "huge",
                          "inf", "zeros", "subnormal", "const", "nan"]))
    val = series_values(cls, n, rng)
    if rng.random() < 0.1:
        m = rng.random(n) < 0.2
        val[m] = nan_with_payload(rng, int(m.sum()))
    return dict(labels, ts=[int(x) for x in ts], val=[float(x) for x in val])


def make_tables(rng, grid):
    tables = {}
    for name, tags in SCHEMAS.items():
        n = int(rng.integers(0, 9)) if name != "m1" else int(rng.integers(1, 9))
        seen, series = set(), []
        for _ in range(4 * n):
            if len(series) == n:
                break
            lab = tuple(str(rng.choice(TAG_VALUES[:4] if t == "host" else TAG_VALUES[:3])) if t != "zone" else
                        TAG_VALUES[int(rng.integers(0, len(TAG_VALUES)))] for t in tags)
            if lab in seen:
                continue
            seen.add(lab)
            series.append(make_series(rng, grid, dict(zip(tags, lab))))
        tables[name] = {"time_index": "ts", "field": "val", "tags": list(tags), "series": series}
    return tables


class TreeGen:
    """Random trees of depth <= 4 and <= 8 nodes that the plan accepts.  It does not read the contract table of
    tests/test_gpu_plan_contract.py: it draws only Float64 nodes over Utf8-keyed tables, whose contracts accept every
    node kind drawn here, and steers around the two refusals that remain (key columns that do not match, a literal
    EmptyMetric on the lhs of a filter).  A refused tree fails the test."""

    def __init__(self, rng, tables, grid):
        self.rng, self.tables, self.grid = rng, tables, grid
        self.labels = 0

    def pick(self, seq):
        return seq[int(self.rng.integers(0, len(seq)))]

    def leaf_node(self):
        r = self.rng.random()
        if r < 0.08:
            return vector(self.pick([1.0, -0.0, 2.5, 1e308, math.inf]))
        if r < 0.14:
            return time()
        table = self.pick([t for t, v in self.tables.items() if v["series"]] or ["m1"])
        if self.rng.random() < 0.5:
            return leaf(table)
        return leaf(table, self.pick(RANGE_FNS), self.grid[2] * int(self.rng.integers(1, 5)))

    def tags_of(self, n):
        return evaluate(n, self.tables, self.grid).tags

    def draw(self, depth, budget):
        """a tree of at most `depth` levels and `budget` nodes"""
        if depth <= 1 or budget <= 1 or self.rng.random() < 0.05:
            return self.leaf_node()
        kind = self.pick(["scalar_op", "function", "binary", "binary", "setop", "aggregate", "aggregate", "topk",
                          "sort", "label_join", "label_replace", "subquery", "calendar"])
        if kind == "calendar":
            if depth < 3 or budget < 3:
                return self.leaf_node()
            # hour(x) etc. are Int32, which most nodes refuse: an arithmetic stage makes the value Float64 again
            inner = function(self.draw(depth - 2, budget - 2), self.pick(CALENDAR))
            return scalar_op(inner, self.pick(ARITH), self.pick([1.0, 0.5, -2.0, 7.0]))
        if kind in ("binary", "setop"):
            if budget < 3:
                return self.leaf_node()
            split = int(self.rng.integers(1, budget - 1))
            lhs, rhs = self.draw(depth - 1, split), self.draw(depth - 1, budget - 1 - split)
            return self.binary_node(lhs, rhs) if kind == "binary" else self.setop_node(lhs, rhs)
        child = self.draw(depth - 1, budget - 1)
        tags = self.tags_of(child)
        rng = self.rng
        if kind == "scalar_op":
            op = self.pick(ARITH + CMP)
            s = self.pick([0.0, -0.0, 1.0, 2.0, 0.5, -3.0, 100.0, 1e-310])
            return scalar_op(child, op, s, on_left=bool(rng.random() < 0.3), return_bool=op in CMP and rng.random() < 0.4)
        if kind == "subquery":
            return subquery(self.pick(SUBQUERY_FNS), child, self.grid[2] * int(rng.integers(1, 5)))
        if kind == "function":
            name = self.pick(list(EXACT_FNS))
            args = {"prom_round": [self.pick([0.0, 0.5, 10.0])], "clamp": [-5.0, 5.0], "clamp_min": [0.0],
                    "clamp_max": [1.0]}.get(name, [])
            return function(child, name, *args)
        mod = self.modifier(tags)
        if kind == "aggregate":
            op = self.pick(AGG_OPS)
            return aggregate(op, child, param=self.pick([0.0, 0.5, 0.9, 1.0]) if op == "quantile" else None, **mod)
        if kind == "topk":
            return topk(self.pick(["topk", "bottomk"]), self.pick([1, 2, 3, 0.5, 100]), child, **mod)
        if kind == "sort":
            fn = self.pick(soo.FUNCTIONS)
            if fn.startswith("sort_by_label"):
                if not tags:
                    fn = "sort"
                else:
                    return sort(fn, child, list(rng.permutation(tags)[:int(rng.integers(1, len(tags) + 1))]))
            return sort(fn, child)
        self.labels += 1
        dst = f"d{self.labels}"
        if kind == "label_join":
            srcs = [str(t) for t in rng.permutation(tags + ["nope"])[:int(rng.integers(1, len(tags) + 2))]]
            return label_join(child, dst, self.pick(["-", "", ","]), *srcs)
        src = self.pick(tags + ["nope"])
        return label_replace(child, dst, self.pick(["x$1", "$1$2", "${1}y", "lit", ""]), src, self.pick(REGEXES))

    def modifier(self, tags):
        r = self.rng.random()
        pool = tags + ["nope"]
        sub = [str(t) for t in self.rng.permutation(pool)[:int(self.rng.integers(0, len(pool) + 1))]]
        return {"by": sub} if r < 0.4 else {"without": sub} if r < 0.7 else {}

    def matching(self, ltags, rtags):
        r = self.rng.random()
        common = [t for t in ltags if t in rtags]
        sub = [str(t) for t in self.rng.permutation(common)[:int(self.rng.integers(0, len(common) + 1))]]
        return {"on": sub} if r < 0.35 else {"ignoring": sub} if r < 0.55 else {}

    def binary_node(self, lhs, rhs):
        op = self.pick(ARITH + CMP)
        cmp_ = op in CMP
        ret_bool = cmp_ and self.rng.random() < 0.4
        # a filtering comparison with a literal EmptyMetric lhs is not supported, and one with time() on the lhs
        # filters the rhs (the reference's scalar lhs): draw the EmptyMetric on the rhs
        if cmp_ and not ret_bool and _base(lhs).kind in ("vector", "time"):
            lhs, rhs = rhs, lhs
            if _base(lhs).kind in ("vector", "time"):
                ret_bool = True
        ltags, rtags = self.tags_of(lhs), self.tags_of(rhs)
        m = self.matching(ltags, rtags)
        side = "lhs" if (not rtags and ltags) or self.rng.random() < 0.2 else "rhs"
        try:
            bor.binary_key_columns(ltags, rtags, m.get("on"), m.get("ignoring"))
        except KeyError:
            m = {"on": []}
        return binary(op, lhs, rhs, return_bool=ret_bool, label_side=side, **m)

    def setop_node(self, lhs, rhs):
        op = self.pick(["and", "or", "unless"])
        ltags, rtags = self.tags_of(lhs), self.tags_of(rhs)
        m = self.matching(ltags, rtags)
        try:
            sor.setop_key_columns(op, ltags, rtags, m.get("on"), m.get("ignoring"))
        except KeyError:
            m = {"on": []}
        return setop(op, lhs, rhs, **m)


def _base(n):
    """the node a chain of stages and label functions sits on"""
    while n.kind in ("scalar_op", "function", "label_replace", "label_join"):
        n = n.children[0]
    return n


def draw_case(seed):
    """-> (tree, tables, grid) of one seed: the same seed draws the same case"""
    rng = np.random.default_rng(seed)
    grid = make_grid(rng)
    tables = make_tables(rng, grid)
    gen = TreeGen(rng, tables, grid)
    while True:
        # a tree whose result is a quarter or more unpinned cells checks little: draw another
        tree = gen.draw(4, 8)
        rows = evaluate(tree, tables, grid).export
        if 4 * sum(1 for r in rows if r.maybe or r.pin != BITS) < len(rows) or not rows:
            return tree, tables, grid
