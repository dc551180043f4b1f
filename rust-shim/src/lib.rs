//! GPU execution of GreptimeDB's PromQL range-query sub-plan on an H100 (`libb200promql.so`).
//!
//! * [`ffi`]   — `#[repr(C)]` / `extern "C"` mirror of every declaration in `include/b200promql.h`
//!               (layouts are checked from the C side by `tests/layout.c`).
//! * [`exec`]  — `GpuPromRangeExec`: one DataFusion `ExecutionPlan` that replaces
//!               `SeriesDivide -> SeriesNormalize -> RangeManipulate -> Projection(prom_*) -> Filter [-> Aggregate]`
//!               (trait surface of `RangeManipulateExec`, src/promql/src/extension_plan/range_manipulate.rs:427-579).
//! * [`rule`]  — `GpuPromRewrite`: the `PhysicalOptimizerRule` that finds that sub-tree (shape pinned by
//!               tests/cases/standalone/tql-explain-analyze/analyze.result:154-177) and swaps the node in; registered
//!               next to the other physical rules in `QueryEngineState::new`
//!               (src/query/src/query_engine/state.rs:179-211).
//!
//! Nothing else of the reference changes: the PromQL parser, planner, `SeriesScan` and every other operator stay as they are.
pub mod exec;
pub mod ffi;
pub mod rule;

pub use exec::{GpuPromRangeExec, GpuPromRangeParams};
pub use rule::GpuPromRewrite;

/// Hook for `QueryEngineState::new` (state.rs:179-211): after `EnforceSorting` (index 7), before `WindowedSortPhysicalRule`.
///
/// ```ignore
/// physical_optimizer.rules.insert(8, greptime_promql_b200::physical_rule(device_for_this_datanode));
/// ```
pub fn physical_rule(device: i32) -> std::sync::Arc<dyn datafusion::physical_optimizer::PhysicalOptimizerRule + Send + Sync> {
    std::sync::Arc::new(GpuPromRewrite::new(device))
}
