//! `GpuPromRangeExec` — one physical node for the PromQL range-query sub-plan
//!
//! ```text
//! [AggregateExec(Final) <- RepartitionExec <- AggregateExec(Partial) <-]
//! FilterExec(prom_fn IS NOT NULL [AND ..]) <- ProjectionExec(prom_fn(ts_range, val, ts, range) [per field column])
//!    <- PromRangeManipulateExec <- PromSeriesNormalizeExec <- PromSeriesDivideExec <- (scan)
//! ```
//!
//! Trait surface = `RangeManipulateExec`'s (src/promql/src/extension_plan/range_manipulate.rs:427-579); input
//! requirements = `SeriesDivideExec`'s (series_divide.rs:396-440: hash-partitioned on the series key, sorted by
//! (series key, time index)).  The stream moves every input `RecordBatch` into the C++ plan layer through the Arrow C
//! Data Interface (`b2p_plan_push_batch`, zero copy: the plan reads the Arrow values buffers in place) and emits the
//! rows the replaced sub-tree would have emitted (`b2p_plan_execute`).  One `b2p_ctx` — one CUDA stream — per
//! partition: DataFusion polls partitions concurrently (range_manipulate.rs:546-579).
use std::any::Any;
use std::ffi::CString;
use std::pin::Pin;
use std::sync::Arc;
use std::task::{Context, Poll};

use arrow::array::{Array, RecordBatch, StructArray};
use arrow::datatypes::SchemaRef;
use arrow::ffi::{from_ffi, to_ffi, FFI_ArrowArray, FFI_ArrowSchema};
use arrow_schema::SortOptions;
use datafusion::common::{DataFusionError, Result as DataFusionResult, Statistics};
use datafusion::execution::{RecordBatchStream, SendableRecordBatchStream, TaskContext};
use datafusion::physical_expr::expressions::Column as ColumnExpr;
use datafusion::physical_expr::{EquivalenceProperties, LexRequirement, OrderingRequirements, PhysicalSortRequirement};
use datafusion::physical_plan::metrics::{BaselineMetrics, Count, ExecutionPlanMetricsSet, MetricBuilder, MetricValue, MetricsSet};
use datafusion::physical_plan::{DisplayAs, DisplayFormatType, Distribution, ExecutionPlan, PlanProperties};
use futures::{ready, Stream, StreamExt};

use crate::ffi;

pub type Millisecond = i64; // src/promql/src/extension_plan.rs:42

/// Constructor arguments of the replaced nodes, under their own names.
#[derive(Clone, Debug)]
pub struct GpuPromRangeParams {
    /// `prom_*` ScalarUDF of the Projection (planner.rs:2183-2221); empty = instant-vector selector (InstantManipulate).
    pub function: String,
    // RangeManipulate::new (range_manipulate.rs:86-110)
    pub start: Millisecond,
    pub end: Millisecond,
    pub interval: Millisecond,
    pub range: Millisecond,
    pub time_index_column: String,
    /// RangeManipulate's field columns (1..=64 Float64 columns), every one selected; the node emits one value column per
    /// field in this order (b2p_plan_range_create_fields).
    pub field_columns: Vec<String>,
    // SeriesNormalize::new (normalize.rs:66-83)
    pub offset: Millisecond,
    pub need_filter_out_nan: bool,
    // SeriesDivide::new (series_divide.rs:83-110): Utf8 tag columns, or the single `__tsid: UInt64` column
    pub tag_columns: Vec<String>,
    /// A metric-engine scan (planner.rs:1725-1800): the Utf8 label columns that travel beside the `__tsid` tag column
    /// (b2p_plan_set_label_columns); empty otherwise.
    pub label_columns: Vec<String>,
    // UDF scalars: quantile phi / predict_linear t / smoothing factors
    pub param0: f64,
    pub param1: f64,
    /// InstantManipulate::new lookback (instant_manipulate.rs:189-208) when `function` is empty.
    pub lookback_delta: Millisecond,
    /// timestamp(<selector>): the instant form whose value is the chosen sample's timestamp in seconds
    /// (b2p_plan_set_timestamp, planner.rs:905-909, 951-965); `function` is empty.
    pub timestamp: bool,
    /// prom_aggr_expr_to_plan (planner.rs:334-452): "sum" | "avg" | "count" | "min" | "max" | "stddev" | "stdvar".
    pub aggregate: Option<String>,
    pub by_columns: Vec<String>,
    /// HistogramFold::new(le_column, .., quantile) on top (histogram_fold.rs:104-130).
    pub histogram: Option<(String, f64)>,
    /// Element-wise stages on top, in order: `node op scalar` projections / filters and instant-vector functions.
    pub stages: Vec<GpuPromStage>,
}

impl GpuPromRangeParams {
    /// The label columns the nodes above group, match, order and rewrite on: a metric-engine leaf's label columns,
    /// otherwise its tag columns.
    pub fn labels(&self) -> &[String] {
        if self.label_columns.is_empty() { &self.tag_columns } else { &self.label_columns }
    }

    /// The label-less `__tsid` form: the one tag column is the id and no label travels beside it.
    pub fn id_only(&self) -> bool {
        self.label_columns.is_empty() && self.tag_columns == [String::from("__tsid")]
    }
}

/// One element-wise stage of a `GpuPromRangeExec` (b2p_plan_set_scalar_op / b2p_plan_set_function).
#[derive(Clone, Debug)]
pub enum GpuPromStage {
    /// `node op scalar` (or `scalar op node`): (op, scalar, scalar_on_left, return_bool)
    ScalarOp(ffi::B2pBinOp, f64, bool, bool),
    /// `name(node, args..)`, `name` as the projection's ScalarFunctionExpr::name() ("abs", "prom_round", "clamp", ..)
    Function(String, Vec<f64>),
}

#[derive(Debug)]
pub struct GpuPromRangeExec {
    params: GpuPromRangeParams,
    device: i32,
    input: Arc<dyn ExecutionPlan>,
    output_schema: SchemaRef,
    properties: Arc<PlanProperties>,
    metric: ExecutionPlanMetricsSet,
}

const METRIC_NUM_SERIES: &str = "num_series"; // the reference's metric name (range_manipulate.rs:610-619)

impl GpuPromRangeExec {
    /// `output_schema` is the schema of the node this one replaces (the Filter's, or the final Aggregate's / the
    /// HistogramFold's): the rule copies it from the matched sub-tree, so parents see no difference.
    pub fn try_new(params: GpuPromRangeParams, device: i32, input: Arc<dyn ExecutionPlan>, output_schema: SchemaRef) -> DataFusionResult<Self> {
        if params.interval <= 0 {
            return Err(DataFusionError::Plan("GpuPromRangeExec: interval must be positive".into()));
        }
        if !params.function.is_empty() && ffi::B2pFn::from_udf_name(&params.function).is_none() {
            return Err(DataFusionError::Plan(format!("GpuPromRangeExec: unknown range function {}", params.function)));
        }
        let in_props = input.properties();
        let properties = Arc::new(PlanProperties::new(
            EquivalenceProperties::new(output_schema.clone()),
            in_props.partitioning.clone(),
            in_props.emission_type,
            in_props.boundedness,
        ));
        Ok(Self { params, device, input, output_schema, properties, metric: ExecutionPlanMetricsSet::new() })
    }

    pub fn params(&self) -> &GpuPromRangeParams {
        &self.params
    }

    /// the scan the node reads (what a rule stacking more onto the node rebuilds it over)
    pub fn input(&self) -> &Arc<dyn ExecutionPlan> {
        &self.input
    }
}

impl ExecutionPlan for GpuPromRangeExec {
    fn as_any(&self) -> &dyn Any {
        self
    }

    fn name(&self) -> &str {
        "GpuPromRangeExec"
    }

    fn schema(&self) -> SchemaRef {
        self.output_schema.clone()
    }

    fn properties(&self) -> &Arc<PlanProperties> {
        &self.properties
    }

    // SeriesDivideExec::required_input_distribution (series_divide.rs:396-408)
    fn required_input_distribution(&self) -> Vec<Distribution> {
        if self.params.tag_columns.is_empty() {
            return vec![Distribution::SinglePartition];
        }
        let schema = self.input.schema();
        vec![Distribution::HashPartitioned(
            self.params
                .tag_columns
                .iter()
                .map(|tag| Arc::new(ColumnExpr::new_with_schema(tag, &schema).unwrap()) as _)
                .collect(),
        )]
    }

    // SeriesDivideExec::required_input_ordering (series_divide.rs:410-440): (tags asc nulls first, time index asc)
    fn required_input_ordering(&self) -> Vec<Option<OrderingRequirements>> {
        let schema = self.input.schema();
        let opts = Some(SortOptions { descending: false, nulls_first: true });
        let mut exprs: Vec<PhysicalSortRequirement> = self
            .params
            .tag_columns
            .iter()
            .map(|tag| PhysicalSortRequirement { expr: Arc::new(ColumnExpr::new_with_schema(tag, &schema).unwrap()), options: opts })
            .collect();
        exprs.push(PhysicalSortRequirement {
            expr: Arc::new(ColumnExpr::new_with_schema(&self.params.time_index_column, &schema).unwrap()),
            options: opts,
        });
        vec![Some(OrderingRequirements::Hard(vec![LexRequirement::new(exprs).unwrap()]))]
    }

    fn maintains_input_order(&self) -> Vec<bool> {
        // rows come out series-major in input order; with an aggregate they are re-sorted by (labels, ts) like the
        // reference's `.sort(group_exprs)` (planner.rs:443-449)
        vec![self.params.aggregate.is_none() && self.params.histogram.is_none()]
    }

    fn children(&self) -> Vec<&Arc<dyn ExecutionPlan>> {
        vec![&self.input]
    }

    fn with_new_children(self: Arc<Self>, children: Vec<Arc<dyn ExecutionPlan>>) -> DataFusionResult<Arc<dyn ExecutionPlan>> {
        assert!(!children.is_empty());
        Ok(Arc::new(Self::try_new(self.params.clone(), self.device, children[0].clone(), self.output_schema.clone())?))
    }

    fn execute(&self, partition: usize, context: Arc<TaskContext>) -> DataFusionResult<SendableRecordBatchStream> {
        let baseline_metric = BaselineMetrics::new(&self.metric, partition);
        let num_series = Count::new();
        MetricBuilder::new(&self.metric)
            .with_partition(partition)
            .build(MetricValue::Count { name: METRIC_NUM_SERIES.into(), count: num_series.clone() });
        let input = self.input.execute(partition, context)?;
        // missing columns panic in the reference (range_manipulate.rs:504-516); the plan layer reports them as
        // DataFusionError::Plan("No field named ..") on the first batch instead
        let plan = PlanHandle::create(self.device, &self.params)?;
        Ok(Box::pin(GpuPromRangeStream {
            input,
            plan: Some(plan),
            output_schema: self.output_schema.clone(),
            metric: baseline_metric,
            num_series,
            done: false,
        }))
    }

    fn metrics(&self) -> Option<MetricsSet> {
        Some(self.metric.clone_inner())
    }

    fn partition_statistics(&self, _partition: Option<usize>) -> DataFusionResult<Statistics> {
        Ok(Statistics::new_unknown(&self.schema()))
    }
}

impl DisplayAs for GpuPromRangeExec {
    fn fmt_as(&self, t: DisplayFormatType, f: &mut std::fmt::Formatter) -> std::fmt::Result {
        match t {
            DisplayFormatType::Default | DisplayFormatType::Verbose | DisplayFormatType::TreeRender => write!(
                f,
                "GpuPromRangeExec: fn=[{}], req range=[{}..{}], interval=[{}], eval range=[{}], offset=[{}], time index=[{}], fields={:?}, tags={:?}{}{}",
                if self.params.function.is_empty() { "instant" } else { &self.params.function },
                self.params.start,
                self.params.end,
                self.params.interval,
                self.params.range,
                self.params.offset,
                self.params.time_index_column,
                self.params.field_columns,
                self.params.tag_columns,
                self.params.aggregate.as_ref().map(|a| format!(", aggr=[{a} by {:?}]", self.params.by_columns)).unwrap_or_default(),
                self.params.histogram.as_ref().map(|(le, q)| format!(", histogram_quantile=[{q}, le={le}]")).unwrap_or_default(),
            ),
        }
    }
}

/// Owns the `b2p_ctx` of one partition and the plan object living on it.
struct PlanHandle {
    ctx: *mut ffi::b2p_ctx,
    plan: *mut ffi::b2p_plan,
}
// SAFETY: the context and the plan are only ever touched by the stream that owns the handle; the library keeps no
// thread affinity (its error string is thread-local and read right after a failing call on the same thread).
unsafe impl Send for PlanHandle {}

impl PlanHandle {
    fn create(device: i32, p: &GpuPromRangeParams) -> DataFusionResult<Self> {
        // SAFETY: plain FFI calls with pointers that outlive them.
        unsafe {
            let ctx = ffi::b2p_create(device);
            if ctx.is_null() {
                return Err(DataFusionError::Execution(ffi::last_error()));
            }
            let c = |s: &str| CString::new(s).expect("column names contain no NUL");
            let function = c(&p.function);
            let time_index = c(&p.time_index_column);
            let fields: Vec<CString> = p.field_columns.iter().map(|s| c(s)).collect();
            let field_ptrs: Vec<*const std::os::raw::c_char> = fields.iter().map(|s| s.as_ptr()).collect();
            let tags: Vec<CString> = p.tag_columns.iter().map(|s| c(s)).collect();
            let tag_ptrs: Vec<*const std::os::raw::c_char> = tags.iter().map(|s| s.as_ptr()).collect();
            let by: Vec<CString> = p.by_columns.iter().map(|s| c(s)).collect();
            let by_ptrs: Vec<*const std::os::raw::c_char> = by.iter().map(|s| s.as_ptr()).collect();
            let aggregate = c(p.aggregate.as_deref().unwrap_or(""));
            let params = ffi::B2pRangeParams {
                fn_id: 0, // taken from `function`
                filter_nan: p.need_filter_out_nan as i32,
                start: p.start,
                end: p.end,
                interval: p.interval,
                range: p.range,
                offset: p.offset,
                param0: p.param0,
                param1: p.param1,
            };
            let plan = ffi::b2p_plan_range_create_fields(
                ctx, function.as_ptr(), &params, time_index.as_ptr(), field_ptrs.as_ptr(), field_ptrs.len() as i32,
                tag_ptrs.as_ptr(), tag_ptrs.len() as i32, aggregate.as_ptr(), by_ptrs.as_ptr(), by_ptrs.len() as i32,
            );
            if plan.is_null() {
                let e = ffi::plan_last_error();
                ffi::b2p_destroy(ctx);
                return Err(DataFusionError::Plan(e));
            }
            let h = Self { ctx, plan };
            if !p.label_columns.is_empty() {
                let labels: Vec<CString> = p.label_columns.iter().map(|s| c(s)).collect();
                let label_ptrs: Vec<*const std::os::raw::c_char> = labels.iter().map(|s| s.as_ptr()).collect();
                if ffi::b2p_plan_set_label_columns(plan, label_ptrs.as_ptr(), label_ptrs.len() as i32) != ffi::B2P_OK {
                    return Err(DataFusionError::Plan(ffi::plan_last_error()));
                }
            }
            let instant = if p.timestamp {
                ffi::b2p_plan_set_timestamp(plan, p.lookback_delta)
            } else if p.function.is_empty() {
                ffi::b2p_plan_set_instant(plan, p.lookback_delta)
            } else {
                ffi::B2P_OK
            };
            if instant != ffi::B2P_OK {
                return Err(DataFusionError::Plan(ffi::plan_last_error()));
            }
            if let Some((le, q)) = &p.histogram {
                let le = c(le);
                if ffi::b2p_plan_set_histogram_quantile(plan, le.as_ptr(), *q) != ffi::B2P_OK {
                    return Err(DataFusionError::Plan(ffi::plan_last_error()));
                }
            }
            for stage in &p.stages {
                let rc = match stage {
                    GpuPromStage::ScalarOp(op, scalar, on_left, return_bool) => {
                        ffi::b2p_plan_set_scalar_op(plan, *op as i32, *scalar, *on_left as i32, *return_bool as i32)
                    }
                    GpuPromStage::Function(name, args) => {
                        let name = c(name);
                        ffi::b2p_plan_set_function(plan, name.as_ptr(), args.as_ptr(), args.len() as i32)
                    }
                };
                if rc != ffi::B2P_OK {
                    return Err(DataFusionError::Plan(ffi::plan_last_error()));
                }
            }
            Ok(h)
        }
    }

    /// Moves one input batch into the plan (Arrow C Data Interface; the plan reads the buffers in place).
    fn push(&mut self, batch: RecordBatch) -> DataFusionResult<()> {
        let data = StructArray::from(batch).into_data();
        let (mut array, mut schema) = to_ffi(&data).map_err(|e| DataFusionError::ArrowError(Box::new(e), None))?;
        // SAFETY: on success the library has taken over both release callbacks and zeroed ours (C Data Interface move);
        // on failure they are still ours and drop normally.
        let rc = unsafe { ffi::b2p_plan_push_batch(self.plan, &mut array as *mut FFI_ArrowArray, &mut schema as *mut FFI_ArrowSchema) };
        map_rc(rc, ffi::plan_last_error)
    }

    fn execute(&mut self, schema: &SchemaRef) -> DataFusionResult<(RecordBatch, i64)> {
        let mut array = FFI_ArrowArray::empty();
        let mut out_schema = FFI_ArrowSchema::empty();
        // SAFETY: both structs are valid, empty, and exclusively ours; the library fills them with owned data.
        let rc = unsafe { ffi::b2p_plan_execute(self.plan, &mut array, &mut out_schema) };
        map_rc(rc, ffi::plan_last_error)?;
        // SAFETY: the structs were just produced by a conforming exporter.
        let data = unsafe { from_ffi(array, &out_schema) }.map_err(|e| DataFusionError::ArrowError(Box::new(e), None))?;
        let batch = RecordBatch::from(StructArray::from(data));
        // column names are the reference's (checked by tests/test_gpu_plan.py); types already match the replaced node's
        let batch = batch.with_schema(schema.clone()).map_err(|e| DataFusionError::ArrowError(Box::new(e), None))?;
        // SAFETY: plain getter.
        let n = unsafe { ffi::b2p_plan_num_series(self.plan) };
        Ok((batch, n))
    }
}

impl Drop for PlanHandle {
    fn drop(&mut self) {
        // SAFETY: created by us, destroyed exactly once.
        unsafe {
            ffi::b2p_plan_destroy(self.plan);
            ffi::b2p_destroy(self.ctx);
        }
    }
}

/// Error mapping of INTEGRATION.md: INVALID / TOO_LARGE -> Plan, UNSORTED -> Internal (the reference would silently
/// mis-split series on unsorted input, series_divide.rs:622-670), NOMEM -> ResourcesExhausted, else Execution
/// (the variants the reference's own stream returns, range_manipulate.rs:625, 650-652, 701-705).
fn map_rc(rc: std::os::raw::c_int, msg: impl Fn() -> String) -> DataFusionResult<()> {
    match rc {
        ffi::B2P_OK => Ok(()),
        ffi::B2P_E_INVALID | ffi::B2P_E_TOO_LARGE => Err(DataFusionError::Plan(msg())),
        ffi::B2P_E_UNSORTED => Err(DataFusionError::Internal(msg())),
        ffi::B2P_E_NOMEM => Err(DataFusionError::ResourcesExhausted(msg())),
        _ => Err(DataFusionError::Execution(msg())),
    }
}

pub struct GpuPromRangeStream {
    input: SendableRecordBatchStream,
    plan: Option<PlanHandle>,
    output_schema: SchemaRef,
    metric: BaselineMetrics,
    num_series: Count,
    done: bool,
}

impl RecordBatchStream for GpuPromRangeStream {
    fn schema(&self) -> SchemaRef {
        self.output_schema.clone()
    }
}

impl Stream for GpuPromRangeStream {
    type Item = DataFusionResult<RecordBatch>;

    /// Collect-then-execute: the partition's batches are moved into the plan as they arrive (their H2D copies are
    /// chunked and double-buffered inside `b2p_range_eval`), the kernels run when the input is exhausted, and the
    /// result is one batch.  An empty input batch is skipped (the reference's `InstantManipulateStream` parks
    /// without a waker there, instant_manipulate.rs:447-450 — not replicated).
    fn poll_next(mut self: Pin<&mut Self>, cx: &mut Context<'_>) -> Poll<Option<Self::Item>> {
        if self.done {
            return Poll::Ready(None);
        }
        let poll = loop {
            match ready!(self.input.poll_next_unpin(cx)) {
                Some(Ok(batch)) => {
                    if batch.num_rows() == 0 {
                        continue;
                    }
                    let timer = std::time::Instant::now();
                    let r = self.plan.as_mut().expect("plan alive until done").push(batch);
                    self.metric.elapsed_compute().add_elapsed(timer);
                    if let Err(e) = r {
                        self.done = true;
                        break Poll::Ready(Some(Err(e)));
                    }
                }
                Some(Err(e)) => {
                    self.done = true;
                    break Poll::Ready(Some(Err(e)));
                }
                None => {
                    self.done = true;
                    let timer = std::time::Instant::now();
                    let schema = self.output_schema.clone();
                    let r = self.plan.as_mut().expect("plan alive until done").execute(&schema);
                    self.metric.elapsed_compute().add_elapsed(timer);
                    self.plan = None; // frees the device buffers of this partition
                    break match r {
                        Ok((batch, n)) => {
                            self.num_series.add(n.max(0) as usize);
                            if batch.num_rows() == 0 { Poll::Ready(None) } else { Poll::Ready(Some(Ok(batch))) }
                        }
                        Err(e) => Poll::Ready(Some(Err(e))),
                    };
                }
            }
        };
        self.metric.record_poll(poll)
    }
}
