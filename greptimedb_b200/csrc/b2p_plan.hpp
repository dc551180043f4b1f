// b2p_plan.hpp — C++17 host side above the C ABI: the reference's operator interface for this path,
// over the Arrow C Data Interface (what arrow-rs `FFI_ArrowArray` / pyarrow `_export_to_c` produce).
//
// The reference plans    SeriesDivide(tag_columns, time_index)            series_divide.rs:83-110
//                     -> SeriesNormalize(offset, time_index, need_filter_out_nan, tag_columns)  normalize.rs:66-83
//                     -> RangeManipulate(start, end, interval, range, time_index, field_columns) range_manipulate.rs:86-110
//                     -> Projection(prom_xxx(ts_range, field, ts, range))   src/query/src/promql/planner.rs:1012-1101
//                     -> Filter(field IS NOT NULL)                           planner.rs:1063
//                    [-> Aggregate(by-labels + ts, [sum|avg|count|min|max|stddev|stdvar](field)).sort(...)  planner.rs:334-452]
// PromRangePlan is that whole sub-tree as ONE node: same constructor arguments (names and meaning),
// input = RecordBatches sorted by (tag columns, time index) like SeriesDivideExec requires
// (series_divide.rs:410-440), output = the rows the reference's Filter (or Aggregate+Sort) would emit.
// Errors mirror DataFusionError kinds: Plan (bad arguments / missing column, like field_not_found,
// range_manipulate.rs:127-133), Execution (wrong column type, range_manipulate.rs:700-705), Internal.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/b200promql.h"

namespace b2p {

enum class ErrorKind { Plan, Execution, Internal };
struct PlanError : std::runtime_error {
  ErrorKind kind;
  PlanError(ErrorKind k, const std::string& m) : std::runtime_error(m), kind(k) {}
};

using Millisecond = int64_t;  // extension_plan.rs:42

// An imported Arrow struct array (= RecordBatch); owns the C structs and releases them.
class RecordBatch {
 public:
  RecordBatch(ArrowArray* array, ArrowSchema* schema);  // moves *array / *schema in
  ~RecordBatch();
  RecordBatch(const RecordBatch&) = delete;
  RecordBatch& operator=(const RecordBatch&) = delete;
  int64_t num_rows() const { return array_.length; }
  int find(const std::string& name) const;  // -1 when absent
  const ArrowArray& column(int i) const { return *array_.children[i]; }
  const ArrowSchema& field(int i) const { return *schema_.children[i]; }
  int64_t offset() const { return array_.offset; }

 private:
  ArrowArray array_;
  ArrowSchema schema_;
};

struct PromRangePlanArgs {
  // prom_* UDF name exactly as the planner writes it ("prom_rate", "prom_avg_over_time", ... planner.rs:2183-2221)
  std::string function;
  // RangeManipulate::new
  Millisecond start = 0, end = 0, interval = 0, range = 0;
  std::string time_index;
  // RangeManipulate field_columns: 1 to B2P_MAX_FIELDS Float64 columns, every one selected (planner.rs:2180)
  std::vector<std::string> field_columns;
  // SeriesNormalize::new
  Millisecond offset = 0;
  bool need_filter_out_nan = true;
  // SeriesDivide::new — Utf8 tag columns, or one UInt64 column (__tsid, TagIdentifier::Id)
  std::vector<std::string> tag_columns;
  // a metric-engine leaf (planner.rs:1725-1800): the Utf8 label columns that travel beside the one UInt64 id tag
  // column.  Series still divide on the id; each series takes its labels from its first row (RangeManipulate's
  // take([0; T])).  The metric engine gives one tsid one label set; this node does not check it.
  std::vector<std::string> label_columns;
  // UDF scalar arguments (quantile phi / predict_linear t / smoothing sf, tf)
  double param0 = 0.0, param1 = 0.0;
  // optional prom_aggr_expr_to_plan stage: "", "sum", "avg", "count", "min", "max", "stddev", "stdvar"
  std::string aggregate;
  std::vector<std::string> by_columns;  // must be a subset of tag_columns (label_columns on a metric-engine leaf)
  // function == "" selects the instant-vector form instead: InstantManipulate::new(start, end, lookback_delta,
  // interval, time_index, field_column) (instant_manipulate.rs:189-208); `range` is ignored
  Millisecond lookback_delta = 300000;
  // optional HistogramFold::new(le_column, field, time_index, quantile) on top (histogram_fold.rs:104-130):
  // le_column must be one of tag_columns; every histogram must expose the same bucket bounds
  bool histogram = false;
  std::string le_column;
  double quantile = 0.0;
};

// A label value: a Utf8 string, or NULL (std::nullopt).  NULL equals NULL and differs from every string, as the
// reference's joins compare keys (NullEquality::NullEqualsNull).
using Label = std::optional<std::string>;

// The label tuples of a node's rows: the tag names and, per row, either one UInt64 id (the single tag column is an id
// such as __tsid) or one Label per tag.  Rows of a metric-engine table may also carry their __tsid beside the label
// values (`tsid`): every match, group, order and rewrite reads the values; only the binary node's one-to-one join
// reads the ids, and the export adds them as a UInt64 column `__tsid` after every other column.
struct Labels {
  std::vector<std::string> names;
  bool id_keyed = false;
  bool tsid = false;                       // the rows carry __tsid in `ids` beside `values` (never with id_keyed)
  std::vector<uint64_t> ids;               // [row] when id_keyed or tsid
  std::vector<std::vector<Label>> values;  // [tag][row] when not id_keyed (empty when it is)

  int column(const std::string& name) const;  // -1 when absent
  std::vector<int> columns(const std::vector<std::string>& names) const;
  // row r's value in column c: NULL when c < 0 (a tag the node lacks); an id reads as its decimal string
  Label value(int c, uint32_t r) const;
  // sets `key` to the key of row r over `cols`, read as value() reads them: two keys are equal iff the tuples are
  void key(uint32_t r, const std::vector<int>& cols, std::string& key) const;
  Labels gather(const std::vector<uint32_t>& rows) const;  // the given rows, in that order
  static bool less(const Label& a, const Label& b);         // the order of label values in sorted output
  // drops the __tsid beside the values: the node's projection lists the time index, values and tags only
  void drop_tsid() {
    if (!tsid) return;
    tsid = false;
    ids.clear();
  }
};

// The column order of an exported batch
enum class Columns {
  TimeValueTags,  // {time index, value, tags..}: range and instant nodes, and the filters over them
  TagsTimeValue,  // {tags.., time index, value}: the by-label aggregate, and arithmetic between two vectors
  TimeSorted,     // {time index, then the tags and the value column in name order}: `or`
  ValueTagsTime,  // {value, tags.., time index}: topk / bottomk
  CountTagsTimeLabel,  // {count, tags.., time index, counted value}: count_values
  None,                // no column at all: histogram_quantile over a child without the le tag (an EmptyRelation)
  TimeValueLastTag,    // {time index, value, the last tag, the other tags..}: label_replace / label_join, whose new tag
                       // is the last one for the nodes above and comes first among the tags in its own projection
};

// The type of a value column.  An Int64 cell holds the bits of its int64_t in the 8-byte slot of the grid.  An Int32 cell
// (a calendar function's date_part) and a Count cell (count_values' count, exported as Int64) hold their exact value as a
// double, so those two change only the export: every node reads them as Float64.
enum class ValueType { Float64, Int64, Int32, Count };

// count_values' counted value, a column of each of its rows: its name, its type (Float64, or Int64 cells holding int64_t
// bits) and the cells [rows x T].  Nodes that keep the rows keep it; nodes that build new rows drop it.
struct CountedColumn {
  std::string name;
  ValueType type;
  std::vector<double> values;
};

// What a node computed, before it becomes Arrow: F dense [rows x T] grids (one per field) under one validity, the eval
// timestamps and one label tuple per row.  Exported, row r emits one Arrow row per valid step k (rows in order, steps
// ascending) with F value columns.  One bitmap serves every field because no node that accepts F >= 2 clears a bit for
// one field and not another: element-wise stages, arithmetic and `bool` keep bits, a join's bits are its presence, a
// group has a cell wherever a member has, sort keeps bits, and the one per-value filter (a filtering comparison) is
// refused for F >= 2 (DESIGN §8).
struct NodeResult {
  int64_t T = 0;
  uint32_t Tw = 0;
  uint32_t rows = 0;
  uint32_t F = 1;                // fields; whatever sets F sets types
  std::vector<int64_t> eval_ts;  // [T]
  std::vector<double> val;       // [F x rows x T], field f at f * rows * T; empty when rows == 0 or T == 0
  std::vector<uint32_t> valid;   // [rows x Tw]
  std::string time_index;
  std::vector<std::string> value_names;  // [F]
  std::vector<ValueType> types{ValueType::Float64};  // [F] as the reference types each value column (DESIGN §1 a25)
  Labels labels;
  Columns columns = Columns::TimeValueTags;
  // when not empty, the export emits these cells (row * T + step), in this order, instead of rows then steps; a cell
  // whose bit a later stage cleared is skipped
  std::vector<uint64_t> cell_order;
  std::optional<CountedColumn> counted;  // the rows of a count_values result, and of the nodes that keep them
  // an EmptyMetric row: time() (scalar-typed in PromQL) or a literal (a scalar, or vector(s)); read by the binary node.
  // The aggregate node, topk and count_values pass their child's on, so sum(vector(1)) > x is refused as vector(1) > x
  // is: this layer does not model the matching of either
  bool scalar_like = false, literal_row = false;
  bool is(uint32_t f, ValueType t) const { return f < types.size() && types[f] == t; }
  bool has(ValueType t) const { return std::find(types.begin(), types.end(), t) != types.end(); }
  bool valid_at(uint32_t r, int64_t k) const { return (valid[(size_t)r * Tw + (size_t)(k >> 5)] >> (k & 31)) & 1u; }
  size_t grid() const { return (size_t)rows * (size_t)T; }
  double* field(uint32_t f) { return val.data() + f * grid(); }
  const double* field(uint32_t f) const { return val.data() + f * grid(); }
};

// One element-wise stage on top of a node's result: `node op scalar` / `scalar op node` (b2p_plan_set_scalar_op), or an
// instant-vector function (b2p_plan_set_function).  A node applies its stages in the order they were added.
struct Stage {
  bool is_fn = false;
  int op = 0;                 // enum b2p_binop; enum b2p_ifn when is_fn
  int part = -1;              // enum b2p_step_part of a calendar stage (is_fn; `op` unused)
  double scalar = 0.0;
  bool scalar_on_left = false, return_bool = false;
  std::string fn_name;        // the function as the reference's projection names it ("abs", "prom_round", ...)
  std::vector<double> args;   // its literal arguments after the value column
};

// A plan node: computes its result (step 1), then exports it as one Arrow batch (step 2).
class PlanNode {
 public:
  explicit PlanNode(b2p_ctx* ctx) : ctx_(ctx) {}
  virtual ~PlanNode() = default;
  // the node's result with its element-wise stages applied
  void run(NodeResult& r);
  // runs the node and exports the result batch (caller releases it)
  void execute(ArrowArray* out, ArrowSchema* out_schema);
  void add_scalar_op(int op, double scalar, bool scalar_on_left, bool return_bool);
  void add_function(const std::string& name, const std::vector<double>& args);
  // b2p_plan_set_sharded: false on a node without a sharded form
  virtual bool set_sharded() { return false; }

 protected:
  virtual void compute(NodeResult& r) = 0;
  // A sharded node's check before its work: false without a communicator (the node then runs unsharded); with one, a
  // Plan error for a node below that is sharded or not row-local, else true
  bool sharded_run(const char* node) const;
  // the children a sharded node's check walks (the row-local nodes' and the sharded nodes')
  virtual std::vector<const PlanNode*> children() const { return {}; }
  // what the node computes over rows other ranks hold, nullptr when it is row-local
  virtual const char* cross_row() const { return nullptr; }
  bool sharded_ = false;
  // the argument checks every node makes: a NULL context (unless the node does no device work) is an Internal error,
  // then a NULL child a Plan error, "<node>: NULL context" / "<node>: NULL child"
  void require(const char* node, std::initializer_list<const PlanNode*> children, bool device = true) const;
  b2p_ctx* ctx_;

 private:
  std::vector<Stage> stages_;
};

class PromRangePlan : public PlanNode {
 public:
  PromRangePlan(b2p_ctx* ctx, PromRangePlanArgs args);
  // input stream, in order; batches of one partition (sorted by tags, ts)
  void push(std::unique_ptr<RecordBatch> batch);
  int64_t num_series() const { return num_series_; }  // the reference's `num_series` metric (range_manipulate.rs:610-619)
  // switch the node to the instant-vector form (InstantManipulate) / add a HistogramFold on top; before execute()
  int set_instant(Millisecond lookback_delta) {
    args_.function.clear();
    fn_id_ = -1;
    args_.lookback_delta = lookback_delta;
    return 0;
  }
  void set_histogram(const std::string& le_column, double quantile);
  // the metric-engine form: `names` are Utf8 label columns beside the one UInt64 id tag column (before push())
  void set_label_columns(std::vector<std::string> names);
  // timestamp(<selector>): the instant form whose value is the chosen sample's timestamp in seconds (K4's timestamp
  // mode); the result is one Float64 column named `value` whatever the table's fields
  int set_timestamp(Millisecond lookback_delta) {
    timestamp_ = true;
    return set_instant(lookback_delta);
  }

 protected:
  // runs the sub-plan on the device
  void compute(NodeResult& r) override;

 private:
  PromRangePlanArgs args_;
  int fn_id_;
  int agg_id_;
  bool timestamp_ = false;
  std::vector<int64_t> ts_;
  std::vector<std::vector<double>> val_;  // [field][row]; an Int64 field's rows hold int64_t bits
  std::vector<ValueType> types_;          // [field], set by the first batch
  // F >= 2: each field's Arrow validity bitmap re-based to bit 0 of the first row (empty while the field has no NULL)
  std::vector<std::vector<uint8_t>> present_;
  std::vector<uint64_t> offsets_;  // first row of every series (SeriesDivide's output), end marker added by execute()
  Labels series_;                  // [series] the labels of each series' first row
  int64_t num_series_ = 0;
  // last row's key, to continue a series across batch boundaries (series_divide.rs:636-645)
  std::vector<Label> last_key_;
  uint64_t last_id_ = 0;
  bool have_last_ = false;
  void check_key_columns() const;  // by-columns and the le column name a tag or label column
  bool set_sharded() override { return (agg_id_ >= 0 || args_.histogram) && (sharded_ = true); }
  const char* cross_row() const override {
    return agg_id_ >= 0 ? "an aggregate stage" : args_.histogram ? "histogram_quantile" : nullptr;
  }
};

// Label matching modifier of a binary or set operator
enum class Matching { None, On, Ignoring };

// Label modifier of an aggregation (topk / bottomk, the aggregate node)
enum class Modifier { None, By, Without };

// Vector-vector binary operator over two nodes (b2p_plan_binary_create): the reference's ProjectionExec / FilterExec
// over an inner HashJoinExec on (key columns, time index), planner.rs:556-777, 3436-3546.  The join is a match between
// series on the host (hash of the key tuples, O(rows + pairs)); the per-step work is b2p_binary_op.
class BinaryPlan : public PlanNode {
 public:
  BinaryPlan(b2p_ctx* ctx, int op, bool return_bool, std::shared_ptr<PlanNode> lhs, std::shared_ptr<PlanNode> rhs,
             Matching matching, std::vector<std::string> labels, bool labels_from_lhs);

 protected:
  void compute(NodeResult& r) override;

 private:
  int op_;
  bool return_bool_;
  std::shared_ptr<PlanNode> lhs_, rhs_;
  Matching matching_;
  std::vector<std::string> labels_;
  bool labels_from_lhs_;
  const char* cross_row() const override { return "a binary operator"; }
};

// Set operator `and` / `or` / `unless` over two nodes (b2p_plan_setop_create): the reference's left.distinct()
// LeftSemi / LeftAnti HashJoinExec on (key columns, time index), planner.rs:3549-3703, and UnionDistinctOnExec,
// planner.rs:3707-3906.  Labels are matched on the host into one dense key id per row; the per-cell work is b2p_setop.
class SetOpPlan : public PlanNode {
 public:
  SetOpPlan(b2p_ctx* ctx, int op, std::shared_ptr<PlanNode> lhs, std::shared_ptr<PlanNode> rhs, Matching matching,
            std::vector<std::string> labels);

 protected:
  void compute(NodeResult& r) override;

 private:
  int op_;
  std::shared_ptr<PlanNode> lhs_, rhs_;
  Matching matching_;
  std::vector<std::string> labels_;
  const char* cross_row() const override { return "a set operator"; }
};

// scalar(child), the reference's ScalarCalculateExec (planner.rs:3141-3183, scalar_calculate.rs:532-637): a tagless node
// with one row over the child's steps.  The child's label tuples become dense series keys on the host (a tuple with a
// NULL label: B2P_NO_KEY); the decision and the copy are b2p_scalar_calculate.
class ScalarPlan : public PlanNode {
 public:
  ScalarPlan(b2p_ctx* ctx, std::shared_ptr<PlanNode> child);

 protected:
  void compute(NodeResult& r) override;

 private:
  std::shared_ptr<PlanNode> child_;
  const char* cross_row() const override { return "scalar()"; }
};

// topk(k, child) / bottomk(k, child) [by | without (labels)], the reference's Window(row_number()) -> Filter(rank <= k)
// -> Sort(group labels, ts, rank), planner.rs:454-541, 2963-3016.  The host computes each row's group (over the group
// labels) and a tie ordinal from the label tuples in the window's order (tags descending for topk, ascending for
// bottomk, NULL first; identical tuples in row order); the per-step selection is b2p_topk.  The result is the child's
// rows, labels and values with the kept cells' bits, so nodes above see the child's row order; the export emits
// {value, tags.., time index} by group labels (Labels::less), ts, rank.
class TopkPlan : public PlanNode {
 public:
  TopkPlan(b2p_ctx* ctx, bool bottom, double k, std::shared_ptr<PlanNode> child, Modifier modifier,
           std::vector<std::string> labels);

 protected:
  void compute(NodeResult& r) override;

 private:
  bool bottom_;
  double k_;
  std::shared_ptr<PlanNode> child_;
  Modifier modifier_;
  std::vector<std::string> labels_;
  const char* cross_row() const override { return "topk / bottomk"; }
};

// <op>(child) [by | without (labels)] over any node, GpuPromAggregateExec: the reference's Aggregate(group labels + ts,
// op(value)).sort(group labels, ts) (prom_aggr_expr_to_plan, planner.rs:334-452; create_aggregate_exprs 2808-2897).
// Group labels as for TopkPlan; the fold is b2p_group_aggregate (sum avg count min max stddev stdvar, and group as count
// with the value 1.0) or b2p_group_quantile, members in the child's row order.  Rows: the groups in Labels::less order;
// columns {group labels.., time index, <df name>(<child value name>)}.
class AggregatePlan : public PlanNode {
 public:
  AggregatePlan(b2p_ctx* ctx, const std::string& op, double param, std::shared_ptr<PlanNode> child, Modifier modifier,
                std::vector<std::string> labels);

 protected:
  void compute(NodeResult& r) override;

 private:
  int op_;
  std::string df_name_;  // DataFusion's name of the aggregate function ("var_pop", "quantile", ...)
  double param_;
  std::shared_ptr<PlanNode> child_;
  Modifier modifier_;
  std::vector<std::string> labels_;
  bool set_sharded() override { return sharded_ = true; }
  std::vector<const PlanNode*> children() const override { return {child_.get()}; }
  const char* cross_row() const override { return "an aggregate"; }
};

// count_values(label, child) [by | without (labels)], GpuPromCountValuesExec: the reference's Aggregate(groupBy = [group
// labels.., ts, value], count(value)) -> Projection(count, group labels.., ts, value AS label) -> Sort(group labels, ts,
// value), planner.rs:402-445.  Group labels as for AggregatePlan (group_rows / group_columns); the per-step distinct
// values and counts are b2p_count_values.  Rows: per group in Labels::less order, one for each rank of a distinct value
// that occurs at some step, labelled with the group labels and holding the count (named count(<child value name>)), so
// the nodes above count, sum or compare them; the counted values ride along in `counted` for the export.
class CountValuesPlan : public PlanNode {
 public:
  CountValuesPlan(b2p_ctx* ctx, std::string label, std::shared_ptr<PlanNode> child, Modifier modifier,
                  std::vector<std::string> labels);

 protected:
  void compute(NodeResult& r) override;

 private:
  std::string label_;
  std::shared_ptr<PlanNode> child_;
  Modifier modifier_;
  std::vector<std::string> labels_;
  bool set_sharded() override { return sharded_ = true; }
  std::vector<const PlanNode*> children() const override { return {child_.get()}; }
  const char* cross_row() const override { return "count_values"; }
};

// fn(child[range:step]), GpuPromSubqueryExec: the reference's RangeManipulate(start, end, interval, range) directly over
// the inner plan, then Projection(prom_fn) and Filter(IS NOT NULL) (prom_subquery_expr_to_plan, planner.rs:292-332).
// The child is any node, evaluated on its own grid (the reference's start' = start - range + step, step' = step or the
// outer interval, the outer end), which must be regular; its step is read from its eval timestamps.  Every row is one
// series whose samples are its valid cells (NaN included); the windows are b2p_subquery.  Rows and labels: the child's;
// columns {time index, value, tags..}.  The value is named as the reference's projection names it over the child's value
// column: fn(<ti>_range,<child value>) with ,<ti>,Int64(range) for rate / increase / delta and ,Float64(p) per literal
// argument of predict_linear, quantile_over_time and holt_winters, e.g.
// prom_max_over_time(ts_range,prom_rate(ts_range,val)) over a range leaf.
class SubqueryPlan : public PlanNode {
 public:
  SubqueryPlan(b2p_ctx* ctx, std::string function, const b2p_range_params& p, std::shared_ptr<PlanNode> child);

 protected:
  void compute(NodeResult& r) override;

 private:
  std::string function_;
  b2p_range_params p_;
  std::shared_ptr<PlanNode> child_;
  std::vector<const PlanNode*> children() const override { return {child_.get()}; }
};

// histogram_quantile(φ, child), GpuPromHistogramFoldExec: the reference's HistogramFold(le, field, time index, φ) over
// any input (create_histogram_plan, planner.rs:3041-3108; histogram_fold.rs).  The child's rows that agree on every tag
// but le form one histogram (histogram_index, as the range leaf builds it); the fold over the child's grid is
// b2p_histogram_fold.  Rows: the histograms in Labels::less order; labels: the child's tags without le; the value keeps
// the child's value name, and the export the child's column layout (a topk child's cell_order is dropped).  A child
// without the le tag gives no rows and an export without columns (the reference's EmptyRelation).  Plan errors at
// execute: an id-keyed child (this layer's __tsid form has no le label) and a count_values child (its counted value
// would be a Float64 tag of the fold in the reference, which is not modelled here).  Sharded (b2p_plan_set_sharded, over
// a communicator): the histograms are agreed across ranks and b2p_histogram_fold_allgather folds each on one rank; the
// result is the unsharded node's over every rank's child rows in rank order, the same bytes on every rank.  The Int32 /
// Int64 refusals are then decided on the agreed value types, on every rank alike.
class HistogramQuantilePlan : public PlanNode {
 public:
  HistogramQuantilePlan(b2p_ctx* ctx, std::string le_column, double phi, std::shared_ptr<PlanNode> child);
  bool set_sharded() override { return sharded_ = true; }

 protected:
  void compute(NodeResult& r) override;

 private:
  std::string le_column_;
  double phi_;
  std::shared_ptr<PlanNode> child_;
  std::vector<const PlanNode*> children() const override { return {child_.get()}; }
  const char* cross_row() const override { return "histogram_quantile"; }
};

// sort / sort_desc / sort_by_label / sort_by_label_desc (child [, labels]), GpuPromSortExec: the reference's
// Projection(time index, value, tags..) -> Filter(value IS NOT NULL) -> Sort(keys) over the child (planner.rs:1060-1089,
// 2743-2772).  The result is the child's (rows, row order, values and bits, so nodes above see the child) with its export
// order in cell_order: the valid cells by value in the f64 total order (b2p_sort_cells, K14), or the rows ranked by the
// listed labels on the host (byte order, NULL last in both directions) with each row's cells in step order; ties keep
// row-major order.  Columns {time index, value, tags..}; a child without columns stays so.  Plan errors at execute:
// sort_by_label* over a label the child lacks or an id-keyed child, and any sort over a count_values child.
class SortPlan : public PlanNode {
 public:
  SortPlan(b2p_ctx* ctx, const std::string& function, std::shared_ptr<PlanNode> child, std::vector<std::string> labels);

 protected:
  void compute(NodeResult& r) override;

 private:
  bool desc_ = false, by_label_ = false;
  std::shared_ptr<PlanNode> child_;
  std::vector<std::string> labels_;
  const char* cross_row() const override { return "sort"; }
};

// absent(child), GpuPromAbsentExec: the reference's PromAbsentExec(start, end, interval, time index, value column, fake
// labels) over Aggregate(ts, first_value) -> Sort(ts) of the child (create_absent_plan, planner.rs:3186-3245; absent.rs).
// One row over the grid start + k * interval <= end, valid with the value 1.0 at every step at which no child row has a
// valid cell (b2p_absent, K15; NaN cells count as present).  Its labels are the fake labels: a name given twice keeps
// its last value (the reference's HashMap collect), ordered by name byte-wise.  Columns {time index, value, labels..}.
// The child is any node; only its validity is read, so an id-keyed or count_values child is fine.  Plan error at
// execute: a child with rows whose eval timestamps are not this node's grid.
class AbsentPlan : public PlanNode {
 public:
  AbsentPlan(b2p_ctx* ctx, Millisecond start, Millisecond end, Millisecond interval, std::string time_index,
             std::string value_column, const std::vector<std::pair<std::string, std::string>>& labels,
             std::shared_ptr<PlanNode> child);

 protected:
  void compute(NodeResult& r) override;

 private:
  Millisecond start_, end_, interval_;
  std::string time_index_, value_column_;
  std::vector<std::pair<std::string, std::string>> labels_;  // by name, one per name
  std::shared_ptr<PlanNode> child_;
  const char* cross_row() const override { return "absent()"; }
};

// EmptyMetric(start, end, interval, time_index, field_column, field_expr) (empty_metric.rs): one tagless row over
// start + k * interval <= end (none when start > end) with every cell valid, and a value column by `kind`: none
// (B2P_EMPTY_NONE, only the time index), time() (B2P_EMPTY_TIME, `<time index> / Float64(1000)`, K19) or a number
// (B2P_EMPTY_LITERAL: vector(s), pi(), a literal).  `hour()` and the other calendar functions without an argument are a
// calendar stage on this node.  Plan errors at create: interval <= 0, a NULL name, an unknown kind.
class EmptyMetricPlan : public PlanNode {
 public:
  EmptyMetricPlan(b2p_ctx* ctx, Millisecond start, Millisecond end, Millisecond interval, std::string time_index,
                  std::string value_column, int kind, double literal);

 protected:
  void compute(NodeResult& r) override;

 private:
  Millisecond start_, end_, interval_;
  std::string time_index_, value_column_;
  int kind_;
  double literal_;
  const char* cross_row() const override { return "an EmptyMetric row (time(), vector(), a literal), which every rank holds whole"; }
};

// label_replace(child, dst, replacement, src, regex) / label_join(child, dst, separator, srcs..), GpuPromLabelExec: the
// reference's Projection(time index, values.., <label expr> AS dst, tags..) over any node (planner.rs:1012-1101,
// 2306-2356, 2504-2700).  The child's grid, validity, eval timestamps, types, cell order and counted values are moved,
// not copied; only the label tuples change, each distinct source value of label_replace evaluated once (label_join
// concatenates per row, which costs less than a lookup).  Nodes above see dst appended to the tags (label_join first drops a tag named dst); the export is
// {time index, values.., dst, other tags..} (Columns::TimeValueLastTag) whatever the child's layout, because the
// reference's projection always lists its columns so.  A no-op label_replace exports {time index, values.., tags..} and
// keeps the child's flags; a node that adds a label clears scalar_like / literal_row, so the binary node joins a labelled
// vector(1) on labels.  Rows are never merged.  Plan errors: at create, an invalid dst name, a regex Rust rejects, a
// regex outside b2p_regex.hpp's supported list, label_join without sources; at execute, the reference's same-labelset
// error, an id-keyed (__tsid) child, a count_values child (the reference drops its counted-value column here, which
// this layer does not model), dst or a label_join source named like the time index or a value column.
class LabelPlan : public PlanNode {
 public:
  // label_replace
  LabelPlan(b2p_ctx* ctx, std::shared_ptr<PlanNode> child, std::string dst, std::string replacement, std::string src,
            const std::string& regex);
  // label_join
  LabelPlan(b2p_ctx* ctx, std::shared_ptr<PlanNode> child, std::string dst, std::string separator,
            std::vector<std::string> srcs);
  ~LabelPlan() override;

 protected:
  void compute(NodeResult& r) override;

 private:
  std::shared_ptr<PlanNode> child_;
  bool join_;
  std::string dst_, replacement_, src_;  // replacement_ is label_join's separator
  std::vector<std::string> srcs_;
  std::unique_ptr<class LabelRegex> regex_;
  bool empty_regex_ = false;
  std::vector<const PlanNode*> children() const override { return {child_.get()}; }
};

int function_id_from_name(const std::string& prom_name);  // -1 when unknown
int aggregate_id_from_name(const std::string& name);      // -1 when unknown

}  // namespace b2p
