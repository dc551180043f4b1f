"""pyarrow <-> GpuPromRangeExec (C++ plan layer, csrc/b2p_plan.cpp) over the Arrow C Data Interface.

`PromRangeExec` takes the constructor arguments of the reference's plan nodes with their own names
(SeriesDivide tag_columns/time_index, SeriesNormalize offset/need_filter_out_nan, RangeManipulate
start/end/interval/range/field column, the prom_* UDF name, optional by-label aggregate) and is fed
pyarrow RecordBatches exactly like the reference's tests feed a MemoryExec.  `scalar_op` puts `node op number` on
top of any node, `function` an instant-vector function (abs, clamp_min, prom_round, ...; the two chain in call order),
`BinaryPlan` combines two nodes (`lhs op rhs`, vector matching on labels), `SetOpPlan` applies `and` / `or` / `unless`
to two nodes, `ScalarPlan` is scalar(node), `TopkPlan` is topk / bottomk(k, node) [by | without (labels)],
`SubqueryPlan` is fn(node[range:step]), `HistogramQuantilePlan` is histogram_quantile(phi, node), `SortPlan` is
sort / sort_desc / sort_by_label / sort_by_label_desc(node), `AbsentPlan` is absent(node), `EmptyMetricPlan` is
time(), vector(s) or a number as a one-row node, `LabelReplacePlan` / `LabelJoinPlan` are label_replace / label_join over
any node; `PromRangeExec.timestamp()` is timestamp(<selector>).  `label_regex_check` / `label_regex_replace` run the
label_replace regex engine on one string, no device needed.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Union

from . import _lib
from .engine import B2PError, Context, make_params, op_id, setop_id, topk_bottom


class _ArrowArray(C.Structure):
    _fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                ("n_children", C.c_int64), ("buffers", C.c_void_p), ("children", C.c_void_p),
                ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


class _ArrowSchema(C.Structure):
    _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
                ("n_children", C.c_int64), ("children", C.c_void_p), ("dictionary", C.c_void_p),
                ("release", C.c_void_p), ("private_data", C.c_void_p)]


def _cstr_array(items: Sequence[str]):
    arr = (C.c_char_p * max(len(items), 1))()
    for i, s in enumerate(items):
        arr[i] = s.encode()
    return arr


class _PlanNode:
    """What every node handle has: scalar operators on top, execute, close."""
    _h = None

    def scalar_op(self, op, scalar: float, scalar_on_left: bool = False, return_bool: bool = False) -> "_PlanNode":
        """`node op scalar` (or `scalar op node`) on top of this node; calls chain in order.  Returns self."""
        rc = self._L.b2p_plan_set_scalar_op(self._h, op_id(op), float(scalar), int(bool(scalar_on_left)),
                                            int(bool(return_bool)))
        if rc != 0:
            raise B2PError(rc, self._L.b2p_plan_last_error().decode())
        return self

    def function(self, name: str, *args: float) -> "_PlanNode":
        """`name(node, args...)` on top of this node, `name` as the reference's projection shows it ("abs", "radians",
        "degrees", "signum", "prom_round", "clamp", "clamp_min", ...); chains with scalar_op in call order.  Returns
        self."""
        arr = (C.c_double * max(len(args), 1))(*[float(a) for a in args])
        rc = self._L.b2p_plan_set_function(self._h, name.encode(), arr, len(args))
        if rc != 0:
            raise B2PError(rc, self._L.b2p_plan_last_error().decode())
        return self

    def _set_sharded(self):
        rc = self._L.b2p_plan_set_sharded(self._h)
        if rc != 0:
            raise B2PError(rc, self._L.b2p_plan_last_error().decode())
        return self

    def execute(self):
        """-> pyarrow.RecordBatch with the rows the reference's plan would emit."""
        import pyarrow as pa
        arr, sch = _ArrowArray(), _ArrowSchema()
        rc = self._L.b2p_plan_execute(self._h, C.addressof(arr), C.addressof(sch))
        if rc != 0:
            raise B2PError(rc, self._L.b2p_plan_last_error().decode())
        return pa.RecordBatch._import_from_c(C.addressof(arr), C.addressof(sch))

    def close(self):
        if getattr(self, "_h", None):
            self._L.b2p_plan_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


class PromRangeExec(_PlanNode):
    """The range / instant leaf.  `field_column` is one field name, or a sequence of them for a table with several
    Float64 field columns: every field is selected at once and execute() emits one value column per field.
    `label_columns` makes it a metric-engine leaf: `tag_columns` is the one UInt64 `__tsid` column the series divide
    on, and the label columns (Utf8) travel beside it, read at each series' first row; `by_columns` and `le_column` then
    name label columns.  Nodes above read the labels; a UInt64 `__tsid` column is exported last where the reference
    keeps it."""

    def __init__(self, ctx: Context, function: str, start: int, end: int, interval: int, range: int, time_index: str,
                 field_column: Union[str, Sequence[str]], tag_columns: Sequence[str], offset: int = 0,
                 need_filter_out_nan: bool = True, param0: float = 0.0, param1: float = 0.0,
                 aggregate: Optional[str] = None, by_columns: Sequence[str] = (), lookback_delta: Optional[int] = None,
                 histogram_quantile: Optional[float] = None, le_column: str = "le",
                 label_columns: Optional[Sequence[str]] = None):
        self._L = _lib.load()
        self._ctx = ctx
        p = make_params(0, start, end, interval, range, offset=offset, filter_nan=need_filter_out_nan, param0=param0,
                        param1=param1)
        fields = [field_column] if isinstance(field_column, str) else list(field_column)
        tags, by, fa = _cstr_array(tag_columns), _cstr_array(by_columns), _cstr_array(fields)
        self._h = self._L.b2p_plan_range_create_fields(ctx._h, function.encode(), C.byref(p), time_index.encode(), fa,
                                                       len(fields), tags, len(tag_columns), (aggregate or "").encode(),
                                                       by, len(by_columns))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())
        if label_columns is not None:       # the metric-engine form: __tsid plus label columns
            rc = self._L.b2p_plan_set_label_columns(self._h, _cstr_array(list(label_columns)), len(label_columns))
            if rc != 0:
                raise B2PError(rc, self._L.b2p_plan_last_error().decode())
        if lookback_delta is not None:      # instant-vector selector (InstantManipulate) instead of a range function
            self._L.b2p_plan_set_instant(self._h, int(lookback_delta))
        if histogram_quantile is not None:  # HistogramFold on top
            rc = self._L.b2p_plan_set_histogram_quantile(self._h, le_column.encode(), float(histogram_quantile))
            if rc != 0:
                raise B2PError(rc, self._L.b2p_plan_last_error().decode())

    def timestamp(self, lookback_delta: int = 300_000) -> "PromRangeExec":
        """timestamp(<selector>): the instant form whose value is each chosen sample's timestamp in seconds (no value
        column read, no stale-NaN test); execute() emits one Float64 column `value`.  Returns self."""
        rc = self._L.b2p_plan_set_timestamp(self._h, int(lookback_delta))
        if rc != 0:
            raise B2PError(rc, self._L.b2p_plan_last_error().decode())
        return self

    def push(self, batch) -> None:
        """Feed one pyarrow.RecordBatch (moved into the plan through the C Data Interface)."""
        arr, sch = _ArrowArray(), _ArrowSchema()
        batch._export_to_c(C.addressof(arr), C.addressof(sch))
        rc = self._L.b2p_plan_push_batch(self._h, C.addressof(arr), C.addressof(sch))
        if rc != 0:
            raise B2PError(rc, self._L.b2p_plan_last_error().decode())

    def num_series(self) -> int:
        return int(self._L.b2p_plan_num_series(self._h))

    def sharded(self) -> "PromRangeExec":
        """Mark the leaf's aggregate or HistogramFold stage sharded (b2p_plan_set_sharded): every rank pushes its own
        shard of series and execute() gives every rank the aggregate or histogram_quantile over the union, through the
        context's communicator (without one, the unsharded node).  A leaf without such a stage raises.  Returns
        self."""
        return self._set_sharded()


class BinaryPlan(_PlanNode):
    """`lhs op rhs` over two nodes (PromRangeExec or BinaryPlan), matched like the reference's inner join on the tag
    columns of the rhs (narrowed by `on` / `ignoring`) and the time index.  `label_side` names the node whose tag
    columns an arithmetic / `bool` result carries ("rhs" unless the rhs has no tags, for two sides over one table).
    The children stay usable (push batches into them before execute()) and are kept alive by this node."""

    def __init__(self, ctx: Context, op, lhs: _PlanNode, rhs: _PlanNode, return_bool: bool = False,
                 on: Optional[Sequence[str]] = None, ignoring: Optional[Sequence[str]] = None,
                 label_side: str = "rhs"):
        if on is not None and ignoring is not None:
            raise ValueError("on and ignoring are exclusive")
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (lhs, rhs)
        matching, labels = (b"on", list(on)) if on is not None else (b"ignoring", list(ignoring)) if ignoring is not None \
            else (None, [])
        arr = _cstr_array(labels)
        self._h = self._L.b2p_plan_binary_create(ctx._h, op_id(op), int(bool(return_bool)), lhs._h, rhs._h, matching,
                                                 arr, len(labels), label_side.encode())
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class SetOpPlan(_PlanNode):
    """`lhs and / or / unless rhs` over two nodes (any node handle).  `and` / `unless` keep the lhs rows and columns and
    match on each side's tags narrowed by `on` / `ignoring` (the two must agree); `or` emits the lhs rows, then the rhs
    rows no lhs row (or earlier rhs row) of the same key covers, with the time index first and then the union of the tags
    and the value column in name order.  The children stay usable and are kept alive by this node."""

    def __init__(self, ctx: Context, op, lhs: _PlanNode, rhs: _PlanNode, on: Optional[Sequence[str]] = None,
                 ignoring: Optional[Sequence[str]] = None):
        if on is not None and ignoring is not None:
            raise ValueError("on and ignoring are exclusive")
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (lhs, rhs)
        matching, labels = (b"on", list(on)) if on is not None else (b"ignoring", list(ignoring)) if ignoring is not None \
            else (None, [])
        arr = _cstr_array(labels)
        self._h = self._L.b2p_plan_setop_create(ctx._h, setop_id(op), lhs._h, rhs._h, matching, arr, len(labels))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class ScalarPlan(_PlanNode):
    """scalar(child): a tagless one-row node over the child's steps.  The child's one series (every row one label
    tuple) as it is, or NaN at every step when the child has no rows or two or more series.  The child stays usable
    and is kept alive by this node."""

    def __init__(self, ctx: Context, child: _PlanNode):
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        self._h = self._L.b2p_plan_scalar_create(ctx._h, child._h)
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class TopkPlan(_PlanNode):
    """topk(k, child) / bottomk(k, child) (op "topk" | "bottomk") per (group labels, step), with `by` or `without`
    labels (neither: one group per step).  Cells rank by value in the f64 total order, then by the child's tags (NULL
    first).  Nodes above see the child's rows with the kept cells; execute() emits {value, tags.., time index} by group
    labels, ts, rank.  The child stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, op, k: float, child: _PlanNode, by: Optional[Sequence[str]] = None,
                 without: Optional[Sequence[str]] = None):
        if by is not None and without is not None:
            raise ValueError("by and without are exclusive")
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        modifier, labels = (b"by", list(by)) if by is not None else (b"without", list(without)) if without is not None \
            else (None, [])
        arr = _cstr_array(labels)
        self._h = self._L.b2p_plan_topk_create(ctx._h, topk_bottom(op), float(k), child._h, modifier, arr, len(labels))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class AggregatePlan(_PlanNode):
    """op(child) per (group labels, step), with `by` or `without` labels (neither: one group per step): op is one of sum
    avg count min max stddev stdvar group quantile (param = phi).  Members fold in the child's row order; execute()
    emits {group labels.., time index, value} with rows in group label order.  The child may be any node; it stays
    usable and is kept alive by this node."""

    def __init__(self, ctx: Context, op: str, child: _PlanNode, param: Optional[float] = None,
                 by: Optional[Sequence[str]] = None, without: Optional[Sequence[str]] = None):
        if by is not None and without is not None:
            raise ValueError("by and without are exclusive")
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        modifier, labels = (b"by", list(by)) if by is not None else (b"without", list(without)) if without is not None \
            else (None, [])
        arr = _cstr_array(labels)
        phi = 0.0 if param is None else float(param)  # (-0.0 stays -0.0: it names the column Float64(-0))
        self._h = self._L.b2p_plan_aggregate_create(ctx._h, op.encode(), phi, child._h, modifier, arr, len(labels))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())

    def sharded(self) -> "AggregatePlan":
        """Mark the node sharded (b2p_plan_set_sharded): every rank runs the plan over its own shard of series and
        execute() gives every rank the aggregate over the union, through the context's communicator (without one, the
        unsharded node).  The child subtree must be row-local.  Returns self."""
        return self._set_sharded()


class CountValuesPlan(_PlanNode):
    """count_values(label, child) per (group labels, step), with `by` or `without` labels (neither: one group per step):
    one row per distinct value (by bits) of the group's cells at the step.  Nodes above see rows labelled with the group
    labels whose value is the count; execute() emits {count(<child value>) Int64, group labels.., time index,
    <label> Float64} by group labels, ts, value (Float64 counts under an element-wise stage).  The child may be any
    node; it stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, label: str, child: _PlanNode, by: Optional[Sequence[str]] = None,
                 without: Optional[Sequence[str]] = None):
        if by is not None and without is not None:
            raise ValueError("by and without are exclusive")
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        modifier, labels = (b"by", list(by)) if by is not None else (b"without", list(without)) if without is not None \
            else (None, [])
        arr = _cstr_array(labels)
        self._h = self._L.b2p_plan_count_values_create(ctx._h, label.encode(), child._h, modifier, arr, len(labels))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())

    def sharded(self) -> "CountValuesPlan":
        """Mark the node sharded (b2p_plan_set_sharded): every rank runs the plan over its own shard of series and
        execute() gives every rank count_values over the union, through the context's communicator (without one, the
        unsharded node).  The child subtree must be row-local.  Returns self."""
        return self._set_sharded()


class SubqueryPlan(_PlanNode):
    """function(child[range:step]): RangeManipulate(start, end, interval, range) directly over any node, then the range
    function `function` ("prom_max_over_time", ...; param0 / param1 as for PromRangeExec).  Build the child on the inner
    grid: start - range + step .. end every step (step = the subquery's step, or interval when it has none).  Each
    child row is one series whose samples are its valid cells, NaN included.  Rows and labels are the child's; execute()
    emits {time index, value, tags..}.  The child stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, function: str, child: _PlanNode, start: int, end: int, interval: int, range: int,
                 param0: float = 0.0, param1: float = 0.0, offset: int = 0):
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        p = make_params(0, start, end, interval, range, offset=offset, filter_nan=False, param0=param0, param1=param1)
        self._h = self._L.b2p_plan_subquery_create(ctx._h, function.encode(), C.byref(p), child._h)
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class HistogramQuantilePlan(_PlanNode):
    """histogram_quantile(phi, child) over any node: the child's rows that agree on every tag but `le` form one
    histogram, its buckets in numeric `le` order (+Inf last).  One row per histogram in label order, labelled with the
    child's tags without `le`; execute() keeps the child's column layout without `le` and its value name.  A child
    without the `le` tag gives an empty batch with no columns.  The child stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, phi: float, child: _PlanNode, le: str = "le"):
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        self._h = self._L.b2p_plan_histogram_quantile_create(ctx._h, le.encode(), float(phi), child._h)
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())

    def sharded(self) -> "HistogramQuantilePlan":
        """Mark the node sharded (b2p_plan_set_sharded): every rank runs the plan over its own shard of series, which
        may split a histogram's buckets across ranks, and execute() gives every rank the node over every rank's child
        rows in rank order, through the context's communicator (without one, the unsharded node).  The child subtree
        must be row-local.  Returns self."""
        return self._set_sharded()


class SortPlan(_PlanNode):
    """sort(child) / sort_desc(child) (function "sort" | "sort_desc": the cells by value in the f64 total order) or
    sort_by_label(child, labels..) / sort_by_label_desc (the rows by the listed labels, byte order, NULL last); equal keys
    keep the child's row-major order.  execute() emits {time index, value, tags..} in that order; nodes above see the
    child's result unchanged.  The child stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, function: str, child: _PlanNode, labels: Sequence[str] = ()):
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        labels = list(labels)
        arr = _cstr_array(labels)
        self._h = self._L.b2p_plan_sort_create(ctx._h, function.encode(), child._h, arr, len(labels))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class AbsentPlan(_PlanNode):
    """absent(child): one row over the grid start, start + interval, .. <= end with the value 1.0 at every step at which
    no child row has a valid cell (NaN counts as present).  `labels` are the (name, value) equality matchers of the
    argument's selector in matcher order: a name given twice keeps its last value, names are ordered byte-wise.
    execute() emits {time_index, value_column, labels..}.  The child is any node, built on the same grid when it has
    rows; it stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, child: _PlanNode, start: int, end: int, interval: int, time_index: str,
                 value_column: str, labels: Sequence[tuple] = ()):
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        labels = list(labels)
        names, values = _cstr_array([n for n, _ in labels]), _cstr_array([v for _, v in labels])
        self._h = self._L.b2p_plan_absent_create(ctx._h, int(start), int(end), int(interval), time_index.encode(),
                                                 value_column.encode(), names, values, len(labels), child._h)
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class EmptyMetricPlan(_PlanNode):
    """EmptyMetric: one tagless row over start, start + interval, .. <= end (none when start > end), every cell valid.
    kind "none" exports only the time index; "time" is time() (value t / 1000, named `<time_index> / Float64(1000)`);
    "literal" is vector(s), pi() or a number (`literal` at every step, named value_column).  The calendar functions
    without an argument are .function("hour") etc. on this node."""

    KINDS = {"none": 0, "time": 1, "literal": 2}

    def __init__(self, ctx: Context, start: int, end: int, interval: int, kind: str = "time", literal: float = 0.0,
                 time_index: str = "time", value_column: str = "value"):
        self._L = _lib.load()
        self._ctx = ctx
        self._h = self._L.b2p_plan_empty_metric_create(ctx._h, int(start), int(end), int(interval), time_index.encode(),
                                                       value_column.encode(), self.KINDS[kind], float(literal))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class LabelReplacePlan(_PlanNode):
    """label_replace(child, dst, replacement, src, regex): dst = the expanded replacement where the whole src value
    matches `regex` (Rust `regex` syntax, the supported subset), the src value where it does not, NULL where it is NULL;
    the literal replacement on every row when src is not a tag; a no-op when src is a tag and regex is "", or src is not
    a tag and replacement is "".  The child's values and rows are kept; nodes above see dst as the last tag, execute()
    emits {time index, values.., dst, tags..}.  The child stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, child: _PlanNode, dst: str, replacement: str, src: str, regex: str):
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        self._h = self._L.b2p_plan_label_replace_create(ctx._h, child._h, dst.encode(), replacement.encode(),
                                                        src.encode(), regex.encode())
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


class LabelJoinPlan(_PlanNode):
    """label_join(child, dst, separator, *srcs): dst = the source labels' values joined by `separator`, skipping a
    source that is "", absent or NULL on the row (concat_ws); a tag named dst is replaced.  Layout as for
    LabelReplacePlan.  The child stays usable and is kept alive by this node."""

    def __init__(self, ctx: Context, child: _PlanNode, dst: str, separator: str, *srcs: str):
        self._L = _lib.load()
        self._ctx = ctx
        self._children = (child,)
        arr = _cstr_array(list(srcs))
        self._h = self._L.b2p_plan_label_join_create(ctx._h, child._h, dst.encode(), separator.encode(), arr, len(srcs))
        if not self._h:
            raise B2PError(-1, self._L.b2p_plan_last_error().decode())


REGEX_OK, REGEX_INVALID, REGEX_UNSUPPORTED = 0, 1, 2


def label_regex_check(regex: str) -> int:
    """REGEX_OK, REGEX_INVALID (Rust's regex crate rejects it) or REGEX_UNSUPPORTED (valid in Rust, refused here)."""
    return int(_lib.load().b2p_label_regex_check(regex.encode()))


def label_regex_replace(regex: str, replacement: str, value: str) -> str:
    """regexp_replace(value, "^(?s:" + regex + ")$", replacement) as label_replace evaluates one label value."""
    L = _lib.load()
    need = C.c_uint64(0)
    cap = 256
    while True:
        buf = C.create_string_buffer(cap)
        rc = L.b2p_label_regex_replace(regex.encode(), replacement.encode(), value.encode(), buf, cap, C.byref(need))
        if rc == 0:
            return buf.raw[:need.value].decode()
        if rc != -5:  # B2P_E_TOO_LARGE: retry with room for the result
            raise B2PError(rc, L.b2p_plan_last_error().decode())
        cap = need.value + 1
