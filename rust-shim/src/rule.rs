//! `GpuPromRewrite` — the `PhysicalOptimizerRule` that swaps the PromQL range-query sub-tree for one `GpuPromRangeExec`.
//!
//! Shape matched (bottom-up, exactly what `TQL ANALYZE (0, 10, '5s') rate(test[10s])` prints —
//! tests/cases/standalone/tql-explain-analyze/analyze.result:154-177 — and `tsid_column.result:124-130` for the
//! aggregate on top):
//!
//! ```text
//!   [SortPreservingMergeExec / SortExec(labels, ts)]                                  (planner.rs:443-449)
//!   [AggregateExec(FinalPartitioned) <- RepartitionExec <- AggregateExec(Partial)]    prom_aggr_expr_to_plan
//!   FilterExec: prom_fn(...)@i IS NOT NULL [AND ..]                                   planner.rs:1063, 2774-2791
//!   ProjectionExec: expr=[ts, prom_fn(ts_range, val, ts, range_ms) as .., tags..]     planner.rs:1012-1101
//!                   (one prom_fn call per field column of a multi-field table, planner.rs:2180)
//!   PromRangeManipulateExec: req range=[..], interval=[..], eval range=[..]           range_manipulate.rs
//!   PromSeriesNormalizeExec: offset=[..], time index=[..], filter NaN: [..]           normalize.rs
//!   PromSeriesDivideExec: tags=[..]                                                   series_divide.rs
//!   <input: CooperativeExec <- SeriesScan / MergeScanExec>
//! ```
//!
//! Binary operators on top of an already rewritten `GpuPromRangeExec` (planner.rs:556-777, 3436-3546):
//!
//! ```text
//!   ProjectionExec: expr=[.., col op Float64(c) | Float64(c) op col, ..]   (arithmetic, or a comparison with `bool`)
//!   FilterExec: col cmp Float64(c)                                        (comparison without `bool`)
//!     <- GpuPromRangeExec                     => the same node with b2p_plan_set_scalar_op appended
//!
//!   ProjectionExec | FilterExec <- HashJoinExec(Inner, on = [(tag, tag).., (ts, ts)])
//!     <- GpuPromRangeExec, GpuPromRangeExec   => `match_binary_join`: the b2p_plan_binary_create arguments
//! ```
//!
//! Instant-vector functions (planner.rs:2368-2413) and scalar() (planner.rs:3141-3183):
//!
//! ```text
//!   ProjectionExec: expr=[.., fn(col [, Float64(c)..]), ..]   (abs .. atanh, radians, degrees, signum, prom_round, clamp*)
//!     <- GpuPromRangeExec                     => the same node with b2p_plan_set_function appended
//!
//!   ScalarCalculateExec(start, end, interval, time index, tag columns, field)
//!     <- GpuPromRangeExec                     => `match_scalar`: the b2p_plan_scalar_create child
//! ```
//!
//! Set operators (planner.rs:3549-3906):
//!
//! ```text
//!   HashJoinExec(LeftSemi | LeftAnti, on = [(tag, tag).., (ts, ts)])      (`and` / `unless`)
//!     <- AggregateExec(group by every column, no aggregates) <- GpuPromRangeExec   (left.distinct())
//!     <- GpuPromRangeExec
//!   UnionDistinctOnExec(compare_keys) <- GpuPromRangeExec, GpuPromRangeExec         (`or`)
//!                                           => `match_set_op`: the b2p_plan_setop_create arguments
//! ```
//!
//! topk / bottomk (planner.rs:454-541, 2963-3016):
//!
//! ```text
//!   ProjectionExec(value, tags.., ts) <- SortExec(group labels, ts, rank)
//!     <- FilterExec(rank <= Float64(k))
//!     <- BoundedWindowAggExec(row_number() PARTITION BY group labels, ts ORDER BY value, tags)
//!     <- GpuPromRangeExec                     => `match_topk`: the b2p_plan_topk_create arguments
//! ```
//!
//! The aggregate node over any rewritten node (prom_aggr_expr_to_plan, planner.rs:334-452, create_aggregate_exprs
//! 2808-2897):
//!
//! ```text
//!   AggregateExec(Final | FinalPartitioned) <- RepartitionExec <- AggregateExec(Partial, group labels + ts)
//!     <- GpuPromRangeExec                     => `match_aggregate_node`: the b2p_plan_aggregate_create arguments
//!         (sum avg count min max stddev_pop var_pop, quantile(Float64(φ), col), max(Float64(1)) = group)
//! ```
//!
//! count_values (planner.rs:402-445):
//!
//! ```text
//!   ProjectionExec(count, group labels.., ts, label) <- SortExec(group labels, ts, value)
//!     <- ProjectionExec(count, group labels.., ts, value AS label, value)
//!     <- AggregateExec(Final | FinalPartitioned) <- RepartitionExec
//!     <- AggregateExec(Partial, group labels + ts + value, count(value))
//!     <- GpuPromRangeExec                     => `match_count_values`: the b2p_plan_count_values_create arguments
//! ```
//!
//! Subqueries fn(<expr>[range:step]) (planner.rs:292-332):
//!
//! ```text
//!   FilterExec(prom_fn IS NOT NULL) <- ProjectionExec(prom_fn(..)) <- PromRangeManipulateExec (no SeriesNormalize)
//!     <- GpuPromRangeExec (one series per batch: no by-label aggregate, no HistogramFold)
//!                                           => `match_subquery`: the b2p_plan_subquery_create arguments
//! ```
//!
//! histogram_quantile over a rewritten node (create_histogram_plan, planner.rs:3041-3108):
//!
//! ```text
//!   HistogramFoldExec(le, field, ts, φ) <- SortExec(tags.., ts, CAST(le AS Float64)) [<- RepartitionExec]
//!     <- GpuPromRangeExec (Utf8 tags including le, without its own HistogramFold)
//!                                           => `match_histogram_quantile`: the b2p_plan_histogram_quantile_create arguments
//! ```
//!
//! sort / sort_desc / sort_by_label / sort_by_label_desc over a rewritten node (planner.rs:1060-1089, 2743-2772):
//!
//! ```text
//!   [SortPreservingMergeExec <-] SortExec(value ASC | DESC NULLS FIRST  |  tags.. ASC | DESC NULLS LAST)
//!     <- FilterExec(value IS NOT NULL) <- ProjectionExec(ts, value, tags..)
//!     <- GpuPromRangeExec                     => `match_sort`: the b2p_plan_sort_create arguments
//! ```
//!
//! absent over a rewritten node (create_absent_plan, planner.rs:3186-3245):
//!
//! ```text
//!   PromAbsentExec(start, end, step, ts, value, fake labels) <- SortExec(ts)
//!     <- AggregateExec(group by ts, first_value(field)) [<- RepartitionExec <- AggregateExec(Partial)]
//!     <- GpuPromRangeExec (on the same grid)   => `match_absent`: the b2p_plan_absent_create arguments
//! ```
//!
//! The time family (planner.rs:905-965, 2222-2300, 3994-4009; empty_metric.rs):
//!
//! ```text
//!   EmptyMetricExec(start, end, interval, expr: none | CAST(CAST(ts AS Int64) AS Float64) / 1000 | Float64(c))
//!     [<- under ProjectionExec(date_part(..))]  => `match_empty_metric`: the b2p_plan_empty_metric_create arguments
//!   InstantManipulateExec <- ProjectionExec(ts, CAST(CAST(ts AS Int64) AS Float64) / 1000 AS value, tags..)
//!     <- SeriesNormalize <- SeriesDivide       => a timestamp leaf (b2p_plan_set_timestamp)
//!   ProjectionExec(date_part(Utf8(part), ts) | days_in_month's date_part(..) | (- col))
//!     <- GpuPromRangeExec                     => the same node with the calendar / `negative` stage appended
//!   ProjectionExec(the child's columns, unchanged) <- GpuPromRangeExec      (timestamp(<any other expression>))
//!                                             => the child itself
//! ```
//!
//! label_replace / label_join (planner.rs:2306-2356, 2504-2700):
//!
//! ```text
//!   ProjectionExec(ts, values.., regexp_replace(tag, "^(?s:re)$", r) | Utf8(r) | concat_ws(sep, tag | NULL, ..) AS dst,
//!     tags..) <- GpuPromRangeExec              => `match_label`: the b2p_plan_label_{replace,join}_create arguments
//! ```
//!
//! Over a table with several field columns the rule takes the shapes the library evaluates per field (the leaf, the
//! aggregate node with one aggregate per field, sort by every field, subqueries, absent, the binary zip) and leaves on
//! the CPU those the library refuses there (the leaf's own aggregate, filtering comparisons over two or more fields,
//! topk / bottomk, count_values, group, scalar, set operators with a multi-field side, histogram_quantile).
//!
//! Every sub-tree the rule rewrites starts at a range selector, whose field columns must be Float64: over an Int64
//! (BIGINT) column the library evaluates only the instant selector and the nodes above it (DESIGN §1 a25), which this
//! rule does not rewrite, so a query over an Int64 column stays on the CPU as a whole.
//!
//! Anything that does not match exactly is left alone — the CPU operators keep running for it.  The rule lives in the
//! `promql` crate (src/promql/src/gpu/rule.rs) so that it can read the nodes' fields; the handful of `pub(crate)`
//! getters it needs are listed in `rust-shim/README.md`.
use std::sync::Arc;

use datafusion::arrow::datatypes::{DataType, SchemaRef};
use datafusion::common::tree_node::{Transformed, TreeNode};
use datafusion::common::{Result as DataFusionResult, ScalarValue};
use datafusion::config::ConfigOptions;
use datafusion::common::JoinType;
use datafusion::logical_expr::Operator;
use datafusion::physical_expr::expressions::{BinaryExpr, CastExpr, Column, IsNotNullExpr, Literal, NegativeExpr};
use datafusion::physical_expr::{PhysicalExpr, ScalarFunctionExpr};
use datafusion::physical_optimizer::PhysicalOptimizerRule;
use datafusion::physical_plan::aggregates::{AggregateExec, AggregateMode};
use datafusion::physical_plan::filter::FilterExec;
use datafusion::physical_plan::joins::HashJoinExec;
use datafusion::physical_plan::projection::ProjectionExec;
use datafusion::physical_plan::repartition::RepartitionExec;
use datafusion::physical_plan::sorts::sort::SortExec;
use datafusion::physical_plan::sorts::sort_preserving_merge::SortPreservingMergeExec;
use datafusion::physical_plan::windows::BoundedWindowAggExec;
use datafusion::physical_plan::ExecutionPlan;

use crate::exec::{GpuPromRangeExec, GpuPromRangeParams, GpuPromStage};
use crate::ffi::{B2pBinOp, B2pEmptyMetricKind, B2pFn, B2pSetOp};
// In-tree these are `crate::extension_plan::{..}`; named here the way the reference names them.
use promql::extension_plan::{
    AbsentExec, EmptyMetricExec, HistogramFoldExec, InstantManipulateExec, RangeManipulateExec, ScalarCalculateExec,
    SeriesDivideExec, SeriesNormalizeExec, UnionDistinctOnExec,
};

/// The projection indices a `FilterExec` keeps rows on: `c IS NOT NULL`, or the conjunction of such tests that closes a
/// multi-field selector (`create_empty_values_filter_expr`, planner.rs:2774-2791), in ascending order; `None` for any
/// other predicate.
fn not_null_columns(pred: &Arc<dyn PhysicalExpr>) -> Option<Vec<usize>> {
    let mut out = Vec::new();
    let mut stack = vec![pred.clone()];
    while let Some(e) = stack.pop() {
        if let Some(b) = e.as_any().downcast_ref::<BinaryExpr>() {
            if *b.op() != Operator::And {
                return None;
            }
            stack.push(b.left().clone());
            stack.push(b.right().clone());
            continue;
        }
        let not_null = e.as_any().downcast_ref::<IsNotNullExpr>()?;
        out.push(not_null.arg().as_any().downcast_ref::<Column>()?.index());
    }
    out.sort_unstable();
    out.dedup();
    Some(out)
}

/// The closing pair of a range selector or a subquery, `FilterExec(<its IS NOT NULL tests>) <- ProjectionExec(plain
/// columns, one prom_fn call per field column)` (planner.rs:1012-1101, 2180, 2774-2791): the filtered columns are exactly
/// the calls, every call is the same function with the same literal arguments, call i reads its value column as
/// `prom_fn(ts_range, <field>, ..)`, and every other projected expression is a plain column.
struct FieldUdfs {
    function: String,
    params: (f64, f64),
    /// the value column each call reads, in projection order (the RangeManipulate's field columns)
    fields: Vec<String>,
    input: Arc<dyn ExecutionPlan>,
}

/// The label columns of a metric-engine scan (planner.rs:1725-1800, 1834): when SeriesDivide runs on `__tsid` alone,
/// the Utf8 columns of its input other than the time index, the fields and `__tsid`, which travel beside the id and
/// which the nodes above read.  Empty for any other divide.
fn metric_engine_labels(tags: &[String], schema: &SchemaRef, time_index: &str, fields: &[String]) -> Vec<String> {
    if tags != [String::from("__tsid")] {
        return vec![];
    }
    schema
        .fields()
        .iter()
        .filter(|f| {
            f.name() != time_index
                && f.name() != "__tsid"
                && !fields.contains(f.name())
                && matches!(f.data_type(), DataType::Utf8)
        })
        .map(|f| f.name().clone())
        .collect()
}

fn match_field_udfs(plan: &Arc<dyn ExecutionPlan>) -> Option<FieldUdfs> {
    let filter = plan.as_any().downcast_ref::<FilterExec>()?;
    let filtered = not_null_columns(filter.predicate())?;
    let projection = filter.input().as_any().downcast_ref::<ProjectionExec>()?;
    let mut function: Option<String> = None;
    let mut params: Option<(f64, f64)> = None;
    let (mut fields, mut calls) = (Vec::new(), Vec::new());
    for (i, e) in projection.expr().iter().enumerate() {
        if e.expr.as_any().downcast_ref::<Column>().is_some() {
            continue;
        }
        let udf = e.expr.as_any().downcast_ref::<ScalarFunctionExpr>()?;
        let name = udf.name();
        B2pFn::from_udf_name(name)?;
        // UDF arguments (planner.rs:2438-2474): (ts_range, value_range [, ts] [, range_length | scalar params ..])
        let p = scalar_params(name, udf.args())?;
        if function.get_or_insert_with(|| name.to_string()).as_str() != name {
            return None;
        }
        let bits = |q: (f64, f64)| (q.0.to_bits(), q.1.to_bits());
        if bits(*params.get_or_insert(p)) != bits(p) {
            return None;
        }
        fields.push(udf.args().get(1)?.as_any().downcast_ref::<Column>()?.name().to_string());
        calls.push(i);
    }
    if calls.is_empty() || calls != filtered {
        return None;
    }
    Some(FieldUdfs { function: function?, params: params?, fields, input: projection.input().clone() })
}

#[derive(Debug)]
pub struct GpuPromRewrite {
    device: i32,
}

impl GpuPromRewrite {
    pub fn new(device: i32) -> Self {
        Self { device }
    }

    /// `FilterExec(prom_fn IS NOT NULL [AND ..]) <- ProjectionExec(prom_fn(..) per field) <- RangeManipulate <- Normalize
    /// <- Divide <- input`, one call per field column of the RangeManipulate, in its order (`match_field_udfs`); the time
    /// index and the tags are plain columns, which the node emits unchanged.
    fn match_range_subtree(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<(GpuPromRangeParams, Arc<dyn ExecutionPlan>)> {
        let udfs = match_field_udfs(plan)?;
        let range_exec = udfs.input.as_any().downcast_ref::<RangeManipulateExec>()?;
        let normalize = range_exec.input().as_any().downcast_ref::<SeriesNormalizeExec>()?;
        let divide = normalize.input().as_any().downcast_ref::<SeriesDivideExec>()?;
        if !range_exec.field_columns().iter().eq(udfs.fields.iter()) {
            return None;
        }
        // the library's range leaf takes Float64 field columns only: a range function over an Int64 (BIGINT) column is
        // refused at push (DESIGN §1 a25), and so is everything built on such a leaf (subquery, histogram_quantile,
        // arithmetic between two Int64 sides, `or`, a filter over an Int64 lhs, a multi-field sort with an Int64 field),
        // so any other field type keeps the whole sub-tree on the CPU
        let schema = divide.input().schema();
        for field in range_exec.field_columns() {
            if schema.field_with_name(field).ok()?.data_type() != &DataType::Float64 {
                return None;
            }
        }
        let (param0, param1) = udfs.params;
        let params = GpuPromRangeParams {
            function: udfs.function,
            start: range_exec.start(),
            end: range_exec.end(),
            interval: range_exec.interval(),
            range: range_exec.range(),
            time_index_column: range_exec.time_index_column().to_string(),
            field_columns: range_exec.field_columns().to_vec(),
            offset: normalize.offset(),
            need_filter_out_nan: normalize.need_filter_out_nan(),
            tag_columns: divide.tag_columns().to_vec(),
            label_columns: metric_engine_labels(divide.tag_columns(), &divide.input().schema(),
                                                range_exec.time_index_column(), range_exec.field_columns()),
            param0,
            param1,
            lookback_delta: 0,
            timestamp: false,
            aggregate: None,
            by_columns: vec![],
            histogram: None,
            stages: vec![],
        };
        Some((params, divide.input().clone()))
    }

    /// `AggregateExec(FinalPartitioned) <- RepartitionExec <- AggregateExec(Partial) <- <range sub-tree>` with ONE
    /// aggregate expression among sum / avg / count / min / max / stddev_pop / var_pop and group-by = label columns +
    /// time index (agg_modifier_to_col, planner.rs:1400-1480).
    fn match_aggregate(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<(GpuPromRangeParams, Arc<dyn ExecutionPlan>)> {
        let fin = plan.as_any().downcast_ref::<AggregateExec>()?;
        if !matches!(fin.mode(), AggregateMode::FinalPartitioned | AggregateMode::Final) {
            return None;
        }
        let repart = fin.input().as_any().downcast_ref::<RepartitionExec>()?;
        let partial = repart.input().as_any().downcast_ref::<AggregateExec>()?;
        if !matches!(partial.mode(), AggregateMode::Partial) || partial.aggr_expr().len() != 1 {
            return None;
        }
        let (mut params, input) = self.match_range_subtree(partial.input())?;
        if params.field_columns.len() != 1 {
            return None; // the library refuses the leaf's aggregate stage over several fields: `match_aggregate_node`
        }
        let agg = match partial.aggr_expr()[0].fun().name() {
            "sum" => "sum",
            "avg" => "avg",
            "count" => "count",
            "min" => "min",
            "max" => "max",
            "stddev_pop" => "stddev",
            "var_pop" => "stdvar",
            // quantile / count_values are not all-reduce-able here (match_aggregate_node, match_count_values; topk:
            // match_topk)
            _ => return None,
        };
        let mut by = Vec::new();
        for (expr, _name) in partial.group_expr().expr() {
            let col = expr.as_any().downcast_ref::<Column>()?;
            if col.name() != params.time_index_column {
                if !params.labels().iter().any(|t| t == col.name()) {
                    return None;
                }
                by.push(col.name().to_string());
            }
        }
        params.aggregate = Some(agg.to_string());
        params.by_columns = by;
        Some((params, input))
    }
}

/// What `b2p_plan_binary_create` takes for `lhs op rhs` over two rewritten nodes.
#[derive(Debug)]
pub struct GpuPromBinarySpec {
    pub op: B2pBinOp,
    pub return_bool: bool,
    pub lhs: GpuPromRangeParams,
    pub rhs: GpuPromRangeParams,
    /// the join's tag keys, passed as `on(..)`
    pub on: Vec<String>,
    /// "lhs" | "rhs": the side whose tag columns the projection emits (planner.rs:696-711)
    pub label_side: &'static str,
}

/// What `b2p_plan_setop_create` takes for `lhs and | or | unless rhs` over two rewritten nodes.
#[derive(Debug)]
pub struct GpuPromSetOpSpec {
    pub op: B2pSetOp,
    pub lhs: GpuPromRangeParams,
    pub rhs: GpuPromRangeParams,
    /// passed as `on(..)`: the join's tag keys (`and` / `unless`), or UnionDistinctOn's compare keys (`or`)
    pub on: Vec<String>,
}

/// What `b2p_plan_scalar_create` takes for `scalar(child)` over a rewritten node.
#[derive(Debug)]
pub struct GpuPromScalarSpec {
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_topk_create` takes for a matched topk / bottomk: the op, the literal k, the group labels (passed as
/// `by`, in the window's partition order, the time index left out) and the child node.
#[derive(Debug, Clone)]
pub struct GpuPromTopkSpec {
    pub bottom: bool,
    pub k: f64,
    pub by: Vec<String>,
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_aggregate_create` takes for an aggregate over a rewritten node: the op name, its literal parameter
/// (quantile's φ, else 0), the group labels (passed as `by`, in the group-by order, the time index left out) and the child.
#[derive(Debug, Clone)]
pub struct GpuPromAggregateSpec {
    pub op: &'static str,
    pub param: f64,
    pub by: Vec<String>,
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_count_values_create` takes for a matched count_values: the label (the value column's alias), the
/// group labels (passed as `by`, in the group-by order, the time index and the value left out) and the child node.
#[derive(Debug, Clone)]
pub struct GpuPromCountValuesSpec {
    pub label: String,
    pub by: Vec<String>,
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_subquery_create` takes for a matched subquery: the range function, RangeManipulate's outer grid and
/// range, the function's literal arguments and the child node (evaluated on the inner grid).
#[derive(Debug, Clone)]
pub struct GpuPromSubquerySpec {
    pub function: String,
    pub start: i64,
    pub end: i64,
    pub interval: i64,
    pub range: i64,
    pub param0: f64,
    pub param1: f64,
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_histogram_quantile_create` takes for a matched HistogramFold: the le column, the literal φ and the
/// child node.
#[derive(Debug, Clone)]
pub struct GpuPromHistogramQuantileSpec {
    pub le_column: String,
    pub phi: f64,
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_sort_create` takes for a matched sort: the function ("sort" | "sort_desc" | "sort_by_label" |
/// "sort_by_label_desc"), the labels of the sort_by_label forms in key order and the child node.
#[derive(Debug, Clone)]
pub struct GpuPromSortSpec {
    pub function: String,
    pub labels: Vec<String>,
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_absent_create` takes for a matched absent: the grid, the output's time index and value column names,
/// the fake labels (the equality matchers of the argument's selector, as `Absent::try_new` kept them: one per name, by
/// name) and the child node.
#[derive(Debug, Clone)]
pub struct GpuPromAbsentSpec {
    pub start: i64,
    pub end: i64,
    pub interval: i64,
    pub time_index: String,
    pub value_column: String,
    pub labels: Vec<(String, String)>,
    pub child: GpuPromRangeParams,
}

/// What `b2p_plan_label_replace_create` / `b2p_plan_label_join_create` take for a matched label projection: label_replace
/// (dst, replacement, src, the raw regex) when `join` is false, label_join (dst, separator in `replacement`, srcs with
/// "" for a NULL source) when it is true, and the child node.
#[derive(Debug, Clone)]
pub struct GpuPromLabelSpec {
    pub join: bool,
    pub dst: String,
    pub replacement: String,
    pub src: String,
    pub regex: String,
    pub srcs: Vec<String>,
    pub child: GpuPromRangeParams,
}

/// Whether the library evaluates a label_replace regex (`b2p_label_regex_check` == 0): a pattern it reports invalid or
/// unsupported keeps the query on the CPU, which gives the reference's error or result itself.
fn label_regex_supported(regex: &str) -> bool {
    let Ok(c) = std::ffi::CString::new(regex) else { return false };
    // SAFETY: a host-only call on a NUL-terminated string that outlives it
    unsafe { crate::ffi::b2p_label_regex_check(c.as_ptr()) == 0 }
}

/// `^(?s:<raw>)$` -> raw: the pattern build_regexp_replace_label_expr wrapped (planner.rs:2579)
fn unwrap_label_regex(wrapped: &str) -> Option<&str> {
    wrapped.strip_prefix("^(?s:")?.strip_suffix(")$")
}

fn utf8_literal(e: &Arc<dyn PhysicalExpr>) -> Option<String> {
    match scalar_literal(e)? {
        ScalarValue::Utf8(Some(v)) => Some(v.clone()),
        _ => None,
    }
}

/// The instant-vector functions the library evaluates, by ScalarFunctionExpr::name(), with the number of literal
/// arguments after the value column (planner.rs:2368-2413; prom_round always gets its to_nearest, 0.0 when omitted).
const INSTANT_FNS: &[(&str, usize)] = &[
    ("abs", 0), ("ceil", 0), ("floor", 0), ("sqrt", 0), ("exp", 0), ("ln", 0), ("log2", 0), ("log10", 0),
    ("sin", 0), ("cos", 0), ("tan", 0), ("asin", 0), ("acos", 0), ("atan", 0), ("sinh", 0), ("cosh", 0),
    ("tanh", 0), ("asinh", 0), ("acosh", 0), ("atanh", 0), ("prom_round", 1), ("degrees", 0), ("radians", 0),
    ("signum", 0), ("clamp", 2), ("clamp_min", 1), ("clamp_max", 1),
];

/// DataFusion operator -> b2p_binop; `pow` / `atan2` arrive as scalar functions (planner.rs:3915-3990).
fn binop_of(expr: &Arc<dyn PhysicalExpr>) -> Option<(B2pBinOp, Arc<dyn PhysicalExpr>, Arc<dyn PhysicalExpr>, bool)> {
    // `bool`: CAST(cmp AS Float64)
    let (expr, cast) = match expr.as_any().downcast_ref::<CastExpr>() {
        Some(c) => (c.expr().clone(), true),
        None => (expr.clone(), false),
    };
    if let Some(b) = expr.as_any().downcast_ref::<BinaryExpr>() {
        let op = match b.op() {
            Operator::Plus => B2pBinOp::Add,
            Operator::Minus => B2pBinOp::Sub,
            Operator::Multiply => B2pBinOp::Mul,
            Operator::Divide => B2pBinOp::Div,
            Operator::Modulo => B2pBinOp::Mod,
            Operator::Eq => B2pBinOp::Eq,
            Operator::NotEq => B2pBinOp::Ne,
            Operator::Gt => B2pBinOp::Gt,
            Operator::Lt => B2pBinOp::Lt,
            Operator::GtEq => B2pBinOp::Ge,
            Operator::LtEq => B2pBinOp::Le,
            _ => return None,
        };
        if cast != op.is_comparison() {
            return None;
        }
        return Some((op, b.left().clone(), b.right().clone(), cast));
    }
    let f = expr.as_any().downcast_ref::<ScalarFunctionExpr>()?;
    let op = match f.name() {
        "power" => B2pBinOp::Pow,
        "atan2" => B2pBinOp::Atan2,
        _ => return None,
    };
    Some((op, f.args().first()?.clone(), f.args().get(1)?.clone(), false))
}

fn float_literal(e: &Arc<dyn PhysicalExpr>) -> Option<f64> {
    match e.as_any().downcast_ref::<Literal>()?.value() {
        ScalarValue::Float64(Some(v)) => Some(*v),
        _ => None,
    }
}

fn scalar_literal(e: &Arc<dyn PhysicalExpr>) -> Option<&ScalarValue> {
    Some(e.as_any().downcast_ref::<Literal>()?.value())
}

fn column_named(e: &Arc<dyn PhysicalExpr>, name: &str) -> bool {
    e.as_any().downcast_ref::<Column>().is_some_and(|c| c.name() == name)
}

/// `CAST(CAST(<ts> AS Int64) AS Float64) / Float64(1000)`: build_special_time_expr (empty_metric.rs:393-402), the
/// value of time() and of timestamp()
fn is_special_time_expr(e: &Arc<dyn PhysicalExpr>, ts: &str) -> bool {
    let Some(b) = e.as_any().downcast_ref::<BinaryExpr>() else { return false };
    if *b.op() != Operator::Divide || float_literal(b.right()) != Some(1000.0) {
        return false;
    }
    let Some(outer) = b.left().as_any().downcast_ref::<CastExpr>() else { return false };
    let Some(inner) = outer.expr().as_any().downcast_ref::<CastExpr>() else { return false };
    outer.cast_type() == &DataType::Float64 && inner.cast_type() == &DataType::Int64 && column_named(inner.expr(), ts)
}

/// The calendar function (the library's stage name) of a `date_part(Utf8(field), ts)` projection, or of days_in_month's
/// `date_part(Utf8("day"), date_trunc(Utf8("month"), ts) + IntervalYearMonth(1) - IntervalDayTime(1 day))`
/// (planner.rs:2222-2300); `None` for any other expression, which stays on the CPU.
fn calendar_fn(e: &Arc<dyn PhysicalExpr>, ts: &str) -> Option<&'static str> {
    let f = e.as_any().downcast_ref::<ScalarFunctionExpr>()?;
    if f.name() != "date_part" {
        return None;
    }
    let [field, arg] = f.args() else { return None };
    let ScalarValue::Utf8(Some(field)) = scalar_literal(field)? else { return None };
    if column_named(arg, ts) {
        return match field.as_str() {
            "minute" => Some("minute"),
            "hour" => Some("hour"),
            "month" => Some("month"),
            "year" => Some("year"),
            "day" => Some("day_of_month"),
            "dow" => Some("day_of_week"),
            "doy" => Some("day_of_year"),
            _ => None,
        };
    }
    if field != "day" {
        return None;
    }
    // `date_trunc(..) + (1 month - 1 day)`: the interval either as the planner wrote it or folded into one literal
    let plus = arg.as_any().downcast_ref::<BinaryExpr>()?;
    if *plus.op() != Operator::Plus {
        return None;
    }
    let one_month_less_a_day = match scalar_literal(plus.right()) {
        Some(ScalarValue::IntervalMonthDayNano(Some(v))) => v.months == 1 && v.days == -1 && v.nanoseconds == 0,
        Some(_) => false,
        None => {
            let minus = plus.right().as_any().downcast_ref::<BinaryExpr>()?;
            *minus.op() == Operator::Minus
                && matches!(scalar_literal(minus.left()), Some(ScalarValue::IntervalYearMonth(Some(1))))
                && matches!(scalar_literal(minus.right()),
                            Some(ScalarValue::IntervalDayTime(Some(d))) if d.days == 1 && d.milliseconds == 0)
        }
    };
    let trunc = plus.left().as_any().downcast_ref::<ScalarFunctionExpr>()?;
    let [unit, col] = trunc.args() else { return None };
    let month = matches!(scalar_literal(unit), Some(ScalarValue::Utf8(Some(u))) if u == "month");
    (one_month_less_a_day && trunc.name() == "date_trunc" && month && column_named(col, ts)).then_some("days_in_month")
}

/// The one projected expression of a `ProjectionExec` that is not a plain column (`None` when there are none or two).
fn single_expression(p: &ProjectionExec) -> Option<Arc<dyn PhysicalExpr>> {
    let mut value = None;
    for e in p.expr() {
        if e.expr.as_any().downcast_ref::<Column>().is_none() {
            if value.is_some() {
                return None;
            }
            value = Some(e.expr.clone());
        }
    }
    value
}

/// What `b2p_plan_empty_metric_create` takes for a matched `EmptyMetricExec`, and the calendar stage of `hour()` etc.
/// without an argument (a `date_part` projection over it).
#[derive(Debug, Clone)]
pub struct GpuPromEmptyMetricSpec {
    pub start: i64,
    pub end: i64,
    pub interval: i64,
    pub time_index: String,
    pub value_column: String,
    pub kind: B2pEmptyMetricKind,
    pub literal: f64,
    pub stages: Vec<GpuPromStage>,
}

impl GpuPromRewrite {
    /// `ProjectionExec(col op lit)` / `FilterExec(col cmp lit)` over a `GpuPromRangeExec` -> the node's parameters with
    /// the scalar operator appended; every other projected expression must be a plain column.
    fn match_scalar_op(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<(GpuPromRangeParams, Arc<dyn ExecutionPlan>)> {
        let (expr, input, filter) = if let Some(f) = plan.as_any().downcast_ref::<FilterExec>() {
            (f.predicate().clone(), f.input().clone(), true)
        } else {
            let p = plan.as_any().downcast_ref::<ProjectionExec>()?;
            let mut value = None;
            for e in p.expr() {
                if e.expr.as_any().downcast_ref::<Column>().is_none() {
                    if value.is_some() {
                        return None;
                    }
                    value = Some(e.expr.clone());
                }
            }
            (value?, p.input().clone(), false)
        };
        let node = input.as_any().downcast_ref::<GpuPromRangeExec>()?;
        let (op, l, r, return_bool) = binop_of(&expr)?;
        if filter != (op.is_comparison() && !return_bool) {
            return None;
        }
        if filter && node.params().field_columns.len() != 1 {
            return None; // refused over several fields (planner.rs:3976-3981)
        }
        let (scalar, on_left) = match (float_literal(&l), float_literal(&r)) {
            (None, Some(v)) if l.as_any().downcast_ref::<Column>().is_some() => (v, false),
            (Some(v), None) if r.as_any().downcast_ref::<Column>().is_some() => (v, true),
            _ => return None,
        };
        let mut params = node.params().clone();
        params.stages.push(GpuPromStage::ScalarOp(op, scalar, on_left, return_bool));
        Some((params, node.input().clone()))
    }

    /// `ProjectionExec(fn(col, lit..))` over a `GpuPromRangeExec` -> the node's parameters with the function appended
    /// as one more stage; every other projected expression must be a plain column.
    fn match_function(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<(GpuPromRangeParams, Arc<dyn ExecutionPlan>)> {
        let p = plan.as_any().downcast_ref::<ProjectionExec>()?;
        let mut value = None;
        for e in p.expr() {
            if e.expr.as_any().downcast_ref::<Column>().is_none() {
                if value.is_some() {
                    return None;
                }
                value = Some(e.expr.clone());
            }
        }
        let value = value?;
        let node = p.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        // a calendar function of the node's eval time, or unary minus (planner.rs:552): stages without arguments
        let stage = calendar_fn(&value, &node.params().time_index_column).or_else(|| {
            let neg = value.as_any().downcast_ref::<NegativeExpr>()?;
            neg.arg().as_any().downcast_ref::<Column>().map(|_| "negative")
        });
        if let Some(name) = stage {
            let mut params = node.params().clone();
            params.stages.push(GpuPromStage::Function(name.to_string(), vec![]));
            return Some((params, node.input().clone()));
        }
        let f = value.as_any().downcast_ref::<ScalarFunctionExpr>()?;
        let name = f.name();
        let &(_, n_args) = INSTANT_FNS.iter().find(|(n, _)| *n == name)?;
        let (col, lits) = f.args().split_first()?;
        col.as_any().downcast_ref::<Column>()?;
        if lits.len() != n_args {
            return None;
        }
        let args = lits.iter().map(float_literal).collect::<Option<Vec<f64>>>()?;
        let mut params = node.params().clone();
        params.stages.push(GpuPromStage::Function(name.to_string(), args));
        Some((params, node.input().clone()))
    }

    /// `InstantManipulateExec <- ProjectionExec(ts, CAST(CAST(ts AS Int64) AS Float64) / 1000 AS value, tags..) <-
    /// SeriesNormalize <- SeriesDivide <- input`: timestamp(<selector>) (planner.rs:905-909, 951-965) -> a timestamp
    /// leaf.  The leaf reads no value; it is given the scan's first Float64 or Int64 column, which every batch carries.
    fn match_timestamp_leaf(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<(GpuPromRangeParams, Arc<dyn ExecutionPlan>)> {
        let instant = plan.as_any().downcast_ref::<InstantManipulateExec>()?;
        let p = instant.input().as_any().downcast_ref::<ProjectionExec>()?;
        let normalize = p.input().as_any().downcast_ref::<SeriesNormalizeExec>()?;
        let divide = normalize.input().as_any().downcast_ref::<SeriesDivideExec>()?;
        let ts = instant.time_index_column();
        if !is_special_time_expr(&single_expression(p)?, ts) {
            return None;
        }
        let tags = divide.tag_columns();
        let schema = divide.input().schema();
        let field = schema.fields().iter().find(|f| {
            f.name() != ts
                && !tags.contains(f.name())
                && matches!(f.data_type(), DataType::Float64 | DataType::Int64)
        })?;
        let params = GpuPromRangeParams {
            function: String::new(),
            start: instant.start(),
            end: instant.end(),
            interval: instant.interval(),
            range: 0,
            time_index_column: ts.to_string(),
            field_columns: vec![field.name().clone()],
            offset: normalize.offset(),
            need_filter_out_nan: normalize.need_filter_out_nan(),
            tag_columns: tags.to_vec(),
            label_columns: metric_engine_labels(tags, &schema, ts, &[field.name().clone()]),
            param0: 0.0,
            param1: 0.0,
            lookback_delta: instant.lookback_delta(),
            timestamp: true,
            aggregate: None,
            by_columns: vec![],
            histogram: None,
            stages: vec![],
        };
        Some((params, divide.input().clone()))
    }

    /// `ProjectionExec` of the child's columns in the child's order over a `GpuPromRangeExec`: what the reference plans
    /// for timestamp(<any other expression>), whose `timestamp_fn` flag reaches only a vector selector
    /// (planner.rs:244-290, 2358-2366) -> the child itself.
    fn match_passthrough(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<(GpuPromRangeParams, Arc<dyn ExecutionPlan>)> {
        let p = plan.as_any().downcast_ref::<ProjectionExec>()?;
        let node = p.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let child = node.schema();
        if p.expr().len() != child.fields().len() {
            return None;
        }
        for (i, e) in p.expr().iter().enumerate() {
            let c = e.expr.as_any().downcast_ref::<Column>()?;
            if c.index() != i || e.alias != *child.field(i).name() {
                return None;
            }
        }
        Some((node.params().clone(), node.input().clone()))
    }

    /// `[ProjectionExec(date_part(..)) <-] EmptyMetricExec` (empty_metric.rs; time(), vector(s), pi(), a literal, and
    /// the calendar functions without an argument) -> the arguments of `b2p_plan_empty_metric_create` and its stage.
    pub fn match_empty_metric(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromEmptyMetricSpec> {
        let (input, stage) = match plan.as_any().downcast_ref::<ProjectionExec>() {
            Some(p) => {
                let ts = p.input().schema().field(0).name().clone();
                (p.input().clone(), Some(calendar_fn(&single_expression(p)?, &ts)?))
            }
            None => (plan.clone(), None),
        };
        let em = input.as_any().downcast_ref::<EmptyMetricExec>()?;
        let schema = em.schema();
        let time_index = schema.field(0).name().clone();
        let (kind, literal) = match em.expr() {
            None => (B2pEmptyMetricKind::None, 0.0),
            Some(e) if is_special_time_expr(e, &time_index) => (B2pEmptyMetricKind::Time, 0.0),
            Some(e) => (B2pEmptyMetricKind::Literal, float_literal(e)?),
        };
        let value_column = if schema.fields().len() > 1 { schema.field(1).name().clone() } else { String::new() };
        Some(GpuPromEmptyMetricSpec {
            start: em.start(),
            end: em.end(),
            interval: em.interval(),
            time_index,
            value_column,
            kind,
            literal,
            stages: stage.map(|n| GpuPromStage::Function(n.to_string(), vec![])).into_iter().collect(),
        })
    }

    /// `ScalarCalculateExec <- GpuPromRangeExec` -> the child of `b2p_plan_scalar_create` (no Rust execution node for the
    /// scalar node yet, as for the binary join).
    pub fn match_scalar(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromScalarSpec> {
        let s = plan.as_any().downcast_ref::<ScalarCalculateExec>()?;
        let child = s.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        if child.params().field_columns.len() != 1 {
            return None; // refused over several fields (planner.rs:3155-3160)
        }
        Some(GpuPromScalarSpec { child: child.params().clone() })
    }

    /// `ProjectionExec <- SortExec <- FilterExec(rank <= k) <- BoundedWindowAggExec(row_number()) <- GpuPromRangeExec`
    /// (prom_topk_bottomk_to_plan, planner.rs:454-541) -> the arguments of `b2p_plan_topk_create`.  The window's partition
    /// keys other than the time index become `by(..)`; the first sort key's direction tells topk (descending) from bottomk.
    pub fn match_topk(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromTopkSpec> {
        let p = plan.as_any().downcast_ref::<ProjectionExec>()?;
        let sort = p.input().as_any().downcast_ref::<SortExec>()?;
        let filter = sort.input().as_any().downcast_ref::<FilterExec>()?;
        let window = filter.input().as_any().downcast_ref::<BoundedWindowAggExec>()?;
        let [w] = window.window_expr() else { return None };
        if w.name() != "row_number()" && !w.name().starts_with("row_number") {
            return None;
        }
        let child = window.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        if child.params().field_columns.len() != 1 {
            return None; // refused over several fields (planner.rs:2969-2974)
        }
        // rank <= Float64(k) (the UInt64 rank is cast to Float64, planner.rs:475)
        let pred = filter.predicate().as_any().downcast_ref::<BinaryExpr>()?;
        if *pred.op() != Operator::LtEq {
            return None;
        }
        let k = float_literal(pred.right())?;
        let order = w.order_by();
        let bottom = !order.first()?.options.descending;
        let ts = &child.params().time_index_column;
        let mut by = Vec::new();
        for e in w.partition_by() {
            let c = e.as_any().downcast_ref::<Column>()?;
            if c.name() != ts.as_str() {
                by.push(c.name().to_string());
            }
        }
        Some(GpuPromTopkSpec { bottom, k, by, child: child.params().clone() })
    }

    /// `AggregateExec(Final) <- RepartitionExec <- AggregateExec(Partial)` over a `GpuPromRangeExec` -> the arguments of
    /// `b2p_plan_aggregate_create`.  `quantile(Float64(φ), col)` needs a literal φ; `max(Float64(1))` is `group`
    /// (planner.rs:2836-2838).  A non-literal φ and group columns that are not tags of the child stay on the CPU;
    /// count_values (which groups by the value column too) is `match_count_values`.  Over a child with F field columns
    /// the reference plans one aggregate of the same op per field (planner.rs:2824-2866): F aggregate expressions, the
    /// i-th over the child's i-th value column; `group()` is refused there (planner.rs:2815-2823) and stays on the CPU.
    pub fn match_aggregate_node(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromAggregateSpec> {
        let fin = plan.as_any().downcast_ref::<AggregateExec>()?;
        if !matches!(fin.mode(), AggregateMode::FinalPartitioned | AggregateMode::Final) {
            return None;
        }
        let repart = fin.input().as_any().downcast_ref::<RepartitionExec>()?;
        let partial = repart.input().as_any().downcast_ref::<AggregateExec>()?;
        let [a, rest @ ..] = partial.aggr_expr() else { return None };
        if !matches!(partial.mode(), AggregateMode::Partial) {
            return None;
        }
        let child = partial.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        if 1 + rest.len() != child.params().field_columns.len() {
            return None;
        }
        let args = a.expressions();
        let first_literal = args.first().and_then(float_literal);
        if !rest.is_empty() {
            // the child's output is {time index, value per field, tags..}: aggregate i reads value column i
            let schema = child.schema();
            for (i, e) in partial.aggr_expr().iter().enumerate() {
                let e_args = e.expressions();
                if e.fun().name() != a.fun().name()
                    || e_args.first().and_then(float_literal).map(f64::to_bits) != first_literal.map(f64::to_bits)
                {
                    return None;
                }
                let col = e_args.last()?.as_any().downcast_ref::<Column>()?;
                if col.name() != schema.field(1 + i).name().as_str() {
                    return None;
                }
            }
        }
        let (op, param) = match a.fun().name() {
            "sum" => ("sum", 0.0),
            "avg" => ("avg", 0.0),
            "count" => ("count", 0.0),
            "min" => ("min", 0.0),
            "max" if first_literal == Some(1.0) => ("group", 0.0),
            "max" => ("max", 0.0),
            "stddev_pop" => ("stddev", 0.0),
            "var_pop" => ("stdvar", 0.0),
            "quantile" => ("quantile", first_literal?),
            _ => return None,
        };
        if op == "group" && !rest.is_empty() {
            return None;
        }
        // every group column other than the time index must be one of the child's tags: count_values (planned as
        // count with the value column among the group columns, planner.rs:420-424, 2833) goes to match_count_values,
        // and any other grouping the node cannot express stays on the CPU
        let params = child.params();
        let mut by = Vec::new();
        for (expr, _name) in partial.group_expr().expr() {
            let c = expr.as_any().downcast_ref::<Column>()?;
            if c.name() != params.time_index_column {
                if !params.labels().iter().any(|t| t == c.name()) {
                    return None;
                }
                by.push(c.name().to_string());
            }
        }
        // keep_tsid (planner.rs:347-416) needs no check here: the child is a range-function or timestamp leaf, whose
        // projection drops __tsid in the reference and in the library alike, so neither keeps it above
        Some(GpuPromAggregateSpec { op, param, by, child: params.clone() })
    }

    /// `ProjectionExec <- SortExec <- ProjectionExec(value AS label) <- AggregateExec(Final) <- RepartitionExec <-
    /// AggregateExec(Partial, groupBy [tags.., ts, value], count(value))` over a `GpuPromRangeExec` (planner.rs:402-445)
    /// -> the arguments of `b2p_plan_count_values_create`.  Exactly one group column is neither the time index nor a
    /// tag of the child: the counted value, which must be count's argument; the inner projection names its alias.
    pub fn match_count_values(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromCountValuesSpec> {
        let top = plan.as_any().downcast_ref::<ProjectionExec>()?;
        let sort = top.input().as_any().downcast_ref::<SortExec>()?;
        let inner = sort.input().as_any().downcast_ref::<ProjectionExec>()?;
        let fin = inner.input().as_any().downcast_ref::<AggregateExec>()?;
        if !matches!(fin.mode(), AggregateMode::FinalPartitioned | AggregateMode::Final) {
            return None;
        }
        let repart = fin.input().as_any().downcast_ref::<RepartitionExec>()?;
        let partial = repart.input().as_any().downcast_ref::<AggregateExec>()?;
        let [a] = partial.aggr_expr() else { return None };
        if !matches!(partial.mode(), AggregateMode::Partial) || a.fun().name() != "count" {
            return None;
        }
        let child = partial.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let params = child.params();
        if params.field_columns.len() != 1 {
            return None; // refused over several fields (planner.rs:2874-2879)
        }
        let mut by = Vec::new();
        let mut value = None;
        for (expr, _name) in partial.group_expr().expr() {
            let c = expr.as_any().downcast_ref::<Column>()?;
            if c.name() == params.time_index_column {
                continue;
            }
            if params.labels().iter().any(|t| t == c.name()) {
                by.push(c.name().to_string());
            } else if value.replace(c.name().to_string()).is_some() {
                return None;
            }
        }
        let value = value?;
        let [arg] = a.expressions().as_slice() else { return None };
        if arg.as_any().downcast_ref::<Column>()?.name() != value {
            return None;
        }
        let label = inner.expr().iter().find_map(|e| {
            let c = e.expr.as_any().downcast_ref::<Column>()?;
            (c.name() == value && e.alias != value).then(|| e.alias.clone())
        })?;
        Some(GpuPromCountValuesSpec { label, by, child: params.clone() })
    }

    /// `FilterExec(prom_fn IS NOT NULL) <- ProjectionExec(prom_fn(..)) <- RangeManipulate <- GpuPromRangeExec`, the
    /// subquery fn(<expr>[range:step]) (prom_subquery_expr_to_plan, planner.rs:292-332: no SeriesNormalize between the
    /// RangeManipulate and the inner plan) -> the arguments of `b2p_plan_subquery_create`.  The reference's
    /// RangeManipulate windows every input batch as one series (range_manipulate.rs:603-630) and the node windows every
    /// child row, so only a child that hands one series per batch is taken: a range or instant node (SeriesDivide's
    /// batches), with or without element-wise stages, or its aggregate without `by` (one series).  An aggregate by labels
    /// or a HistogramFold child stays on the CPU.  Over a multi-field child the function is projected once per field
    /// and the filter is the conjunction of their IS NOT NULL (planner.rs:292-332), as for the leaf (`match_field_udfs`).
    pub fn match_subquery(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromSubquerySpec> {
        let udfs = match_field_udfs(plan)?;
        let range_exec = udfs.input.as_any().downcast_ref::<RangeManipulateExec>()?;
        if range_exec.range() <= 0 || !range_exec.field_columns().iter().eq(udfs.fields.iter()) {
            return None;
        }
        let child = range_exec.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let params = child.params();
        if params.histogram.is_some() || (params.aggregate.is_some() && !params.by_columns.is_empty()) {
            return None;
        }
        if range_exec.field_columns().len() != params.field_columns.len() {
            return None;
        }
        let (param0, param1) = udfs.params;
        Some(GpuPromSubquerySpec {
            function: udfs.function,
            start: range_exec.start(),
            end: range_exec.end(),
            interval: range_exec.interval(),
            range: range_exec.range(),
            param0,
            param1,
            child: params.clone(),
        })
    }

    /// `HistogramFoldExec <- SortExec(tags.., ts, CAST(le AS Float64)) [<- RepartitionExec] <- GpuPromRangeExec`
    /// (create_histogram_plan, planner.rs:3041-3108) -> the arguments of `b2p_plan_histogram_quantile_create`.  The
    /// child must be a `GpuPromRangeExec` (a range or instant leaf, or the leaf with its aggregate stage, with or without
    /// element-wise stages) whose Utf8 tag columns include the le column; the library's node accepts any node, but
    /// this matcher only builds the ones the rule rewrites into a `GpuPromRangeExec`.  Left on the CPU: a leaf that
    /// already carries its own HistogramFold, and a `__tsid`-keyed input.  The reference strips `__tsid` with a
    /// `ProjectionExec` before the fold (strip_tsid_column, planner.rs:3064), so such an input does not match here
    /// even when its leaf carries the labels (a metric-engine leaf): that shape stays on the CPU until this matcher
    /// looks through the strip projection.  A label-less id-keyed node carries no le label at all.
    pub fn match_histogram_quantile(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromHistogramQuantileSpec> {
        let fold = plan.as_any().downcast_ref::<HistogramFoldExec>()?;
        let mut input = fold.input().clone();
        if let Some(s) = input.as_any().downcast_ref::<SortExec>() {
            input = s.input().clone();
        }
        if let Some(r) = input.as_any().downcast_ref::<RepartitionExec>() {
            input = r.input().clone();
        }
        let child = input.as_any().downcast_ref::<GpuPromRangeExec>()?;
        let le_column = fold.input().schema().field(fold.le_column_index()).name().to_string();
        // several fields: the reference folds the first one only (a FIXME, planner.rs:3084-3092); the library refuses
        if child.params().histogram.is_some()
            || child.params().field_columns.len() != 1
            || !child.params().labels().iter().any(|t| *t == le_column)
        {
            return None;
        }
        Some(GpuPromHistogramQuantileSpec { le_column, phi: fold.quantile(), child: child.params().clone() })
    }

    /// `[SortPreservingMergeExec <-] SortExec(keys) <- FilterExec(value IS NOT NULL) <- ProjectionExec(ts, value, tags..)
    /// <- GpuPromRangeExec` (planner.rs:1060-1089, 2743-2772) -> the arguments of `b2p_plan_sort_create`.  The keys must
    /// be the value column alone, NULLS FIRST (ascending: sort, descending: sort_desc), or one or more tag columns of the
    /// child, all in one direction, NULLS LAST (sort_by_label / sort_by_label_desc).  Any other key stays on the CPU: the
    /// time index, a column that is not a tag, mixed directions or null orderings.  The projection must pass the time
    /// index, the value and the tags through as plain columns.  Over a multi-field child the filter is the conjunction
    /// of the value columns' IS NOT NULL and sort / sort_desc key on every value column in order (planner.rs:1066-1071,
    /// 2743-2749), which the library's multi-key sort reproduces.
    pub fn match_sort(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromSortSpec> {
        let plan = match plan.as_any().downcast_ref::<SortPreservingMergeExec>() {
            Some(m) => m.input(),
            None => plan,
        };
        let sort = plan.as_any().downcast_ref::<SortExec>()?;
        let filter = sort.input().as_any().downcast_ref::<FilterExec>()?;
        let value_indices = not_null_columns(filter.predicate())?;
        let projection = filter.input().as_any().downcast_ref::<ProjectionExec>()?;
        let child = projection.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let params = child.params();
        if value_indices.len() != params.field_columns.len() {
            return None;
        }
        let mut names = Vec::new();
        for e in projection.expr() {
            e.expr.as_any().downcast_ref::<Column>()?;
            names.push(e.alias.clone());
        }
        let values = value_indices.iter().map(|&i| names.get(i).cloned()).collect::<Option<Vec<String>>>()?;
        let keys: Vec<(String, bool, bool)> = sort
            .expr()
            .iter()
            .map(|k| {
                let c = k.expr.as_any().downcast_ref::<Column>()?;
                Some((c.name().to_string(), k.options.descending, k.options.nulls_first))
            })
            .collect::<Option<_>>()?;
        let (_, descending, nulls_first) = keys.first()?.clone();
        if keys.iter().any(|(_, d, n)| *d != descending || *n != nulls_first) {
            return None;
        }
        if keys.iter().map(|k| &k.0).eq(values.iter()) {
            if !nulls_first {
                return None;
            }
            let function = if descending { "sort_desc" } else { "sort" };
            return Some(GpuPromSortSpec { function: function.to_string(), labels: vec![], child: params.clone() });
        }
        if nulls_first || params.id_only() {
            return None;
        }
        let mut labels = Vec::new();
        for (name, _, _) in &keys {
            if !params.labels().iter().any(|t| t == name) || !names.iter().any(|n| n == name) {
                return None;
            }
            labels.push(name.clone());
        }
        let function = if descending { "sort_by_label_desc" } else { "sort_by_label" };
        Some(GpuPromSortSpec { function: function.to_string(), labels, child: params.clone() })
    }

    /// `ProjectionExec(plain columns, one generated `<expr> AS dst`) <- GpuPromRangeExec`, the projection
    /// label_replace / label_join plan (planner.rs:1012-1101, 2306-2356, 2518-2700), with `<expr>` one of
    /// `regexp_replace(<tag column>, Utf8("^(?s:<raw>)$"), Utf8(r))`, `Utf8(r)` (a source that is not a tag) or
    /// `concat_ws(Utf8(sep), <tag column> | NULL, ..)` -> the arguments of `b2p_plan_label_replace_create` /
    /// `b2p_plan_label_join_create`.  A regex the library does not support, a source column that is not a tag of the
    /// child (the time index or a value column), a label-less id-keyed child and every other shape stay on the CPU.  No-op
    /// label_replace plans have no generated expression: `match_passthrough` takes them.
    pub fn match_label(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromLabelSpec> {
        let p = plan.as_any().downcast_ref::<ProjectionExec>()?;
        let child = p.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let params = child.params();
        if params.id_only() {
            return None;
        }
        let mut generated = None;
        for e in p.expr() {
            if e.expr.as_any().downcast_ref::<Column>().is_none() {
                if generated.is_some() {
                    return None;
                }
                generated = Some((e.expr.clone(), e.alias.clone()));
            }
        }
        let (expr, dst) = generated?;
        let tag = |e: &Arc<dyn PhysicalExpr>| {
            let c = e.as_any().downcast_ref::<Column>()?;
            params.labels().iter().any(|t| t == c.name()).then(|| c.name().to_string())
        };
        let spec = |join, replacement: String, src: String, regex: String, srcs: Vec<String>| GpuPromLabelSpec {
            join,
            dst: dst.clone(),
            replacement,
            src,
            regex,
            srcs,
            child: params.clone(),
        };
        if let Some(r) = utf8_literal(&expr) {
            return (!r.is_empty()).then(|| spec(false, r, String::new(), String::new(), vec![]));
        }
        let f = expr.as_any().downcast_ref::<ScalarFunctionExpr>()?;
        match f.name() {
            "regexp_replace" => {
                let [src, pattern, replacement] = f.args() else { return None };
                let src = tag(src)?;
                let pattern = utf8_literal(pattern)?;
                let raw = unwrap_label_regex(&pattern)?;
                if !label_regex_supported(raw) {
                    return None;
                }
                Some(spec(false, utf8_literal(replacement)?, src, raw.to_string(), vec![]))
            }
            "concat_ws" => {
                let (sep, args) = f.args().split_first()?;
                let srcs = args
                    .iter()
                    .map(|a| match scalar_literal(a) {
                        Some(ScalarValue::Null) | Some(ScalarValue::Utf8(None)) => Some(String::new()),
                        Some(_) => None,
                        None => tag(a),
                    })
                    .collect::<Option<Vec<String>>>()?;
                if srcs.is_empty() {
                    return None;
                }
                Some(spec(true, utf8_literal(sep)?, String::new(), String::new(), srcs))
            }
            _ => None,
        }
    }

    /// `PromAbsentExec <- SortExec(ts) <- AggregateExec(ts, first_value(field)) [<- RepartitionExec <-
    /// AggregateExec(Partial)] <- GpuPromRangeExec` (create_absent_plan, planner.rs:3186-3245) -> the arguments of
    /// `b2p_plan_absent_create`.  The aggregate must group by the time index alone with one `first_value`, and the child
    /// must be evaluated on the absent node's grid: the node reads the child's validity per step of that grid, where
    /// the reference compares the aggregate's timestamps with its cursor.  Anything else stays on the CPU.
    pub fn match_absent(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromAbsentSpec> {
        let absent = plan.as_any().downcast_ref::<AbsentExec>()?;
        let sort = absent.input().as_any().downcast_ref::<SortExec>()?;
        let agg = sort.input().as_any().downcast_ref::<AggregateExec>()?;
        let mut input = agg.input().clone();
        if matches!(agg.mode(), AggregateMode::Final | AggregateMode::FinalPartitioned) {
            let repart = input.as_any().downcast_ref::<RepartitionExec>()?;
            let partial = repart.input().as_any().downcast_ref::<AggregateExec>()?;
            if !matches!(partial.mode(), AggregateMode::Partial) {
                return None;
            }
            input = partial.input().clone();
        } else if !matches!(agg.mode(), AggregateMode::Single | AggregateMode::SinglePartitioned) {
            return None;
        }
        let [a] = agg.aggr_expr() else { return None };
        if a.fun().name() != "first_value" {
            return None;
        }
        let child = input.as_any().downcast_ref::<GpuPromRangeExec>()?;
        let params = child.params();
        let [(ts, _)] = agg.group_expr().expr() else { return None };
        if ts.as_any().downcast_ref::<Column>()?.name() != params.time_index_column {
            return None;
        }
        if (params.start, params.end, params.interval) != (absent.start(), absent.end(), absent.step()) {
            return None;
        }
        Some(GpuPromAbsentSpec {
            start: absent.start(),
            end: absent.end(),
            interval: absent.step(),
            time_index: absent.time_index_column().to_string(),
            value_column: absent.value_column().to_string(),
            labels: absent.fake_labels().to_vec(),
            child: params.clone(),
        })
    }

    /// `ProjectionExec | FilterExec <- HashJoinExec(Inner, tags.. + ts)` over two `GpuPromRangeExec` -> the arguments of
    /// `b2p_plan_binary_create`.  The join keys become `on(..)`; the projection's tag columns tell the label side.  Over
    /// multi-field sides the projection holds one expression per zipped pair, min(F_l, F_r) of them, all of one operator
    /// (planner.rs:712-777, 3401-3414); a filtering comparison over two or more pairs is refused there and stays here.
    pub fn match_binary_join(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromBinarySpec> {
        let (exprs, join_plan) = if let Some(f) = plan.as_any().downcast_ref::<FilterExec>() {
            (vec![f.predicate().clone()], f.input().clone())
        } else {
            let p = plan.as_any().downcast_ref::<ProjectionExec>()?;
            let values: Vec<_> = p
                .expr()
                .iter()
                .filter(|e| e.expr.as_any().downcast_ref::<Column>().is_none())
                .map(|e| e.expr.clone())
                .collect();
            (values, p.input().clone())
        };
        let join = join_plan.as_any().downcast_ref::<HashJoinExec>()?;
        if *join.join_type() != JoinType::Inner || join.filter().is_some() {
            return None;
        }
        let lhs = join.left().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let rhs = join.right().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let pairs = lhs.params().field_columns.len().min(rhs.params().field_columns.len());
        let (op, _, _, return_bool) = binop_of(exprs.first()?)?;
        for e in &exprs[1..] {
            let (o, _, _, b) = binop_of(e)?;
            if o != op || b != return_bool {
                return None;
            }
        }
        let filter = op.is_comparison() && !return_bool;
        if (filter && pairs != 1) || (!filter && exprs.len() != pairs) {
            return None;
        }
        let mut on = Vec::new();
        let mut has_ts = false;
        for (l, r) in join.on() {
            let (l, r) = (l.as_any().downcast_ref::<Column>()?, r.as_any().downcast_ref::<Column>()?);
            if l.name() != r.name() {
                return None;
            }
            if l.name() == rhs.params().time_index_column {
                has_ts = true;
            } else {
                on.push(l.name().to_string());
            }
        }
        if !has_ts {
            return None;
        }
        // a projection emits the tag columns of one side: the lhs's when every projected tag column is on the lhs of the
        // join's output schema (planner.rs:696-711)
        let label_side = match plan.as_any().downcast_ref::<ProjectionExec>() {
            Some(p) => {
                let n_left = join.left().schema().fields().len();
                let from_left = p.expr().iter().filter_map(|e| e.expr.as_any().downcast_ref::<Column>()).all(|c| c.index() < n_left);
                if from_left { "lhs" } else { "rhs" }
            }
            None => "lhs",
        };
        Some(GpuPromBinarySpec { op, return_bool, lhs: lhs.params().clone(), rhs: rhs.params().clone(), on, label_side })
    }

    /// `HashJoinExec(LeftSemi | LeftAnti, tags.. + ts) <- AggregateExec(distinct) <- GpuPromRangeExec` (and / unless,
    /// planner.rs:3549-3703) or `UnionDistinctOnExec` (or, planner.rs:3707-3906) over two `GpuPromRangeExec` -> the
    /// arguments of `b2p_plan_setop_create`.  The join keys / compare keys become `on(..)`.
    pub fn match_set_op(&self, plan: &Arc<dyn ExecutionPlan>) -> Option<GpuPromSetOpSpec> {
        if let Some(u) = plan.as_any().downcast_ref::<UnionDistinctOnExec>() {
            let lhs = u.left().as_any().downcast_ref::<GpuPromRangeExec>()?;
            let rhs = u.right().as_any().downcast_ref::<GpuPromRangeExec>()?;
            if lhs.params().field_columns.len() != 1 || rhs.params().field_columns.len() != 1 {
                return None; // refused (planner.rs:3718-3730)
            }
            let on = u.compare_keys().clone();
            return Some(GpuPromSetOpSpec { op: B2pSetOp::Or, lhs: lhs.params().clone(), rhs: rhs.params().clone(), on });
        }
        let join = plan.as_any().downcast_ref::<HashJoinExec>()?;
        let op = match join.join_type() {
            JoinType::LeftSemi => B2pSetOp::And,
            JoinType::LeftAnti => B2pSetOp::Unless,
            _ => return None,
        };
        if join.filter().is_some() {
            return None;
        }
        // left.distinct(): an AggregateExec that groups by every column and computes nothing
        let distinct = join.left().as_any().downcast_ref::<AggregateExec>()?;
        if !distinct.aggr_expr().is_empty() {
            return None;
        }
        let lhs = distinct.input().as_any().downcast_ref::<GpuPromRangeExec>()?;
        let rhs = join.right().as_any().downcast_ref::<GpuPromRangeExec>()?;
        if lhs.params().field_columns.len() != 1 {
            return None; // refused (planner.rs:3656-3661)
        }
        let mut on = Vec::new();
        let mut has_ts = false;
        for (l, r) in join.on() {
            let (l, r) = (l.as_any().downcast_ref::<Column>()?, r.as_any().downcast_ref::<Column>()?);
            if l.name() != r.name() {
                return None;
            }
            if l.name() == rhs.params().time_index_column {
                has_ts = true;
            } else {
                on.push(l.name().to_string());
            }
        }
        if !has_ts {
            return None;
        }
        Some(GpuPromSetOpSpec { op, lhs: lhs.params().clone(), rhs: rhs.params().clone(), on })
    }
}

/// The scalar UDF arguments the kernels take as (param0, param1); `None` when an argument is not a literal.
fn scalar_params(function: &str, args: &[Arc<dyn PhysicalExpr>]) -> Option<(f64, f64)> {
    let lit = |e: &Arc<dyn PhysicalExpr>| -> Option<f64> {
        match e.as_any().downcast_ref::<Literal>()?.value() {
            ScalarValue::Float64(Some(v)) => Some(*v),
            ScalarValue::Int64(Some(v)) => Some(*v as f64),
            _ => None,
        }
    };
    Some(match function {
        // prom_quantile_over_time(ts_range, value_range, phi); prom_predict_linear(ts_range, value_range, t)
        "prom_quantile_over_time" | "prom_predict_linear" => (lit(args.get(2)?)?, 0.0),
        // prom_holt_winters(ts_range, value_range, sf, tf)
        "prom_holt_winters" | "prom_double_exponential_smoothing" => (lit(args.get(2)?)?, lit(args.get(3)?)?),
        _ => (0.0, 0.0),
    })
}

impl PhysicalOptimizerRule for GpuPromRewrite {
    fn optimize(&self, plan: Arc<dyn ExecutionPlan>, _config: &ConfigOptions) -> DataFusionResult<Arc<dyn ExecutionPlan>> {
        plan.transform_down(|node| {
            // the widest match first: aggregate over the range sub-tree, then the range sub-tree alone
            let matched = self
                .match_aggregate(&node)
                .or_else(|| self.match_range_subtree(&node))
                .or_else(|| self.match_timestamp_leaf(&node))
                .or_else(|| self.match_scalar_op(&node))
                .or_else(|| self.match_function(&node))
                .or_else(|| self.match_passthrough(&node));
            match matched {
                Some((params, input)) => {
                    // the replaced node's schema is kept verbatim, so parents (Sort, CoalesceBatches, MergeScan ..) see no change
                    let exec = GpuPromRangeExec::try_new(params, self.device, input, node.schema())?;
                    Ok(Transformed::yes(Arc::new(exec) as Arc<dyn ExecutionPlan>))
                }
                None => Ok(Transformed::no(node)),
            }
        })
        .map(|t| t.data)
    }

    fn name(&self) -> &str {
        "GpuPromRewrite"
    }

    /// The node keeps the schema of what it replaces.
    fn schema_check(&self) -> bool {
        true
    }
}
