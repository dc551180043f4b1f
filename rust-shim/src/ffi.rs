//! `extern "C"` mirror of `include/b200promql.h` — one item per declaration, same order as the header.
//!
//! Layout contract: `B2pRangeParams` is `struct b2p_range_params` (64 bytes, fields in header order; checked from
//! the C side by `rust-shim/tests/layout.c` and from Python by `tests/test_abi.py::test_params_struct_layout_matches_oracle`).
//! Every other type crossing the boundary is an opaque pointer, a fixed-width integer, `f64`, or the Arrow C Data
//! Interface structs (`arrow::ffi::FFI_ArrowArray` / `FFI_ArrowSchema`, which are `#[repr(C)]` copies of `struct
//! ArrowArray` / `struct ArrowSchema`).
#![allow(non_camel_case_types, clippy::too_many_arguments)]

use std::os::raw::{c_char, c_int, c_void};

use arrow::ffi::{FFI_ArrowArray, FFI_ArrowSchema};

pub const B2P_OK: c_int = 0;
pub const B2P_E_INVALID: c_int = -1;
pub const B2P_E_CUDA: c_int = -2;
pub const B2P_E_UNSORTED: c_int = -3;
pub const B2P_E_NOMEM: c_int = -4;
pub const B2P_E_TOO_LARGE: c_int = -5;
pub const B2P_COMM_ID_BYTES: usize = 128;

/// `enum b2p_fn` — the reference's UDF names in comments (src/query/src/promql/planner.rs:2183-2221).
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum B2pFn {
    Rate = 0,             // prom_rate      ExtrapolatedRate<true, true>
    Increase = 1,         // prom_increase  ExtrapolatedRate<true, false>
    Delta = 2,            // prom_delta     ExtrapolatedRate<false, false>
    Irate = 3,            // prom_irate
    Idelta = 4,           // prom_idelta
    Resets = 5,           // prom_resets
    Changes = 6,          // prom_changes
    CountOverTime = 7,    // prom_count_over_time
    SumOverTime = 8,      // prom_sum_over_time
    AvgOverTime = 9,      // prom_avg_over_time
    MinOverTime = 10,     // prom_min_over_time
    MaxOverTime = 11,     // prom_max_over_time
    LastOverTime = 12,    // prom_last_over_time
    PresentOverTime = 13, // prom_present_over_time
    AbsentOverTime = 14,  // prom_absent_over_time
    StdvarOverTime = 15,  // prom_stdvar_over_time
    StddevOverTime = 16,  // prom_stddev_over_time
    Deriv = 17,           // prom_deriv
    PredictLinear = 18,   // prom_predict_linear      param0 = t (seconds)
    QuantileOverTime = 19, // prom_quantile_over_time  param0 = phi
    HoltWinters = 20,     // prom_double_exponential_smoothing  param0 = sf, param1 = tf
}

impl B2pFn {
    /// The `prom_*` ScalarUDF name the planner writes into the Projection -> the kernel id.
    pub fn from_udf_name(name: &str) -> Option<Self> {
        Some(match name {
            "prom_rate" => Self::Rate,
            "prom_increase" => Self::Increase,
            "prom_delta" => Self::Delta,
            "prom_irate" => Self::Irate,
            "prom_idelta" => Self::Idelta,
            "prom_resets" => Self::Resets,
            "prom_changes" => Self::Changes,
            "prom_count_over_time" => Self::CountOverTime,
            "prom_sum_over_time" => Self::SumOverTime,
            "prom_avg_over_time" => Self::AvgOverTime,
            "prom_min_over_time" => Self::MinOverTime,
            "prom_max_over_time" => Self::MaxOverTime,
            "prom_last_over_time" => Self::LastOverTime,
            "prom_present_over_time" => Self::PresentOverTime,
            "prom_absent_over_time" => Self::AbsentOverTime,
            "prom_stdvar_over_time" => Self::StdvarOverTime,
            "prom_stddev_over_time" => Self::StddevOverTime,
            "prom_deriv" => Self::Deriv,
            "prom_predict_linear" => Self::PredictLinear,
            "prom_quantile_over_time" => Self::QuantileOverTime,
            "prom_holt_winters" | "prom_double_exponential_smoothing" => Self::HoltWinters,
            _ => return None,
        })
    }
}

/// `enum b2p_agg` — aggregators of `create_aggregate_exprs` (planner.rs:2808-2897).
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum B2pAgg {
    Sum = 0,
    Avg = 1,
    Count = 2,
    Min = 3,
    Max = 4,
    Stddev = 5,
    Stdvar = 6,
}

/// `enum b2p_binop` — PromQL binary operators (planner.rs:3915-3990); the comparisons order f64 by IEEE totalOrder.
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum B2pBinOp {
    Add = 0,
    Sub = 1,
    Mul = 2,
    Div = 3,
    Mod = 4,
    Pow = 5,
    Atan2 = 6,
    Eq = 7,
    Ne = 8,
    Gt = 9,
    Lt = 10,
    Ge = 11,
    Le = 12,
}

/// `enum b2p_setop` — PromQL set operators (planner.rs:3549-3906).
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum B2pSetOp {
    And = 0,
    Or = 1,
    Unless = 2,
}

/// `enum b2p_ifn` — PromQL instant-vector math functions (planner.rs:2368-2413).
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum B2pIfn {
    Abs = 0,
    Ceil = 1,
    Floor = 2,
    Sqrt = 3,
    Exp = 4,
    Ln = 5,
    Log2 = 6,
    Log10 = 7,
    Sin = 8,
    Cos = 9,
    Tan = 10,
    Asin = 11,
    Acos = 12,
    Atan = 13,
    Sinh = 14,
    Cosh = 15,
    Tanh = 16,
    Asinh = 17,
    Acosh = 18,
    Atanh = 19,
    Round = 20,
    Deg = 21,
    Rad = 22,
    Sgn = 23,
    Clamp = 24,
    ClampMin = 25,
    ClampMax = 26,
    // 27 is B2P_IFN__COUNT, no function
    /// unary minus: the sign bit flipped
    Neg = 28,
}

/// `enum b2p_step_part`: what `b2p_step_fn` computes from an eval timestamp (time() in seconds, the calendar parts).
#[repr(i32)]
#[derive(Debug, Clone, Copy, PartialEq, Eq)]
pub enum B2pStepPart {
    Time = 0,
    Minute = 1,
    Hour = 2,
    DayOfMonth = 3,
    DayOfWeek = 4,
    DayOfYear = 5,
    Month = 6,
    Year = 7,
    DaysInMonth = 8,
}

/// `enum b2p_empty_metric_kind`: the value column of `b2p_plan_empty_metric_create`.
#[repr(i32)]
#[derive(Debug, Clone, Copy, PartialEq, Eq)]
pub enum B2pEmptyMetricKind {
    /// only the time index (EmptyMetric without a field expression)
    None = 0,
    /// time(): the eval timestamp in seconds
    Time = 1,
    /// vector(s), pi() or a number literal
    Literal = 2,
}

/// `B2P_NO_KEY`: the key of a row that no row of the other side matches (scalar(): a row with a NULL label).
pub const B2P_NO_KEY: u32 = 0xFFFF_FFFF;

impl B2pBinOp {
    /// true for `== != > < >= <=` (a filter without `bool`)
    pub fn is_comparison(self) -> bool {
        self as i32 >= B2pBinOp::Eq as i32
    }
}

/// `struct b2p_range_params`: RangeManipulate::new(start, end, interval, range, ..) (range_manipulate.rs:86-110),
/// SeriesNormalize::new(offset, .., need_filter_out_nan, ..) (normalize.rs:66-83) and the UDF scalars.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct B2pRangeParams {
    pub fn_id: i32,
    pub filter_nan: i32,
    pub start: i64,
    pub end: i64,
    pub interval: i64,
    pub range: i64,
    pub offset: i64,
    pub param0: f64,
    pub param1: f64,
}
const _: () = assert!(std::mem::size_of::<B2pRangeParams>() == 64);
const _: () = assert!(std::mem::align_of::<B2pRangeParams>() == 8);

#[repr(C)]
pub struct b2p_ctx {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct b2p_group_index {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct b2p_plan {
    _opaque: [u8; 0],
}

#[link(name = "b200promql")]
extern "C" {
    // ---- context ------------------------------------------------------------------------------------------
    pub fn b2p_create(device: c_int) -> *mut b2p_ctx;
    pub fn b2p_destroy(ctx: *mut b2p_ctx);
    pub fn b2p_last_error() -> *const c_char;
    pub fn b2p_version() -> *const c_char;
    pub fn b2p_set_stream(ctx: *mut b2p_ctx, cuda_stream: *mut c_void) -> c_int;
    pub fn b2p_use_own_stream(ctx: *mut b2p_ctx) -> c_int;
    pub fn b2p_sync(ctx: *mut b2p_ctx) -> c_int;
    pub fn b2p_num_steps(start: i64, end: i64, interval: i64) -> i64;
    pub fn b2p_last_slow_series(ctx: *mut b2p_ctx) -> i64;
    pub fn b2p_last_h2d_bytes(ctx: *mut b2p_ctx) -> i64;
    pub fn b2p_last_warp_tier_series(ctx: *mut b2p_ctx) -> i64;
    pub fn b2p_last_kernel_ms(ctx: *mut b2p_ctx, stage: c_int) -> f64;
    pub fn b2p_launch_count(ctx: *mut b2p_ctx) -> i64;

    // ---- device-pointer API (asynchronous on the context's stream) -----------------------------------------
    pub fn b2p_series_offsets_dev(ctx: *mut b2p_ctx, sid: *const u32, n_rows: u64, n_series: u32, offsets: *mut u64) -> c_int;
    pub fn b2p_range_eval_dev(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, val: *const f64, offsets: *const u64,
        n_rows: u64, n_series: u32, out: *mut f64, valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_range_udf_dev(
        ctx: *mut b2p_ctx, fn_id: i32, ts: *const i64, val: *const f64, n_rows: u64, packed_ranges: *const i64,
        eval_ts: *const i64, n_win: u64, range_length: i64, param0: f64, param1: f64, out: *mut f64, valid: *mut u8,
    ) -> c_int;
    pub fn b2p_instant_select_dev(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        val: *const f64, offsets: *const u64, n_rows: u64, n_series: u32, out: *mut f64, valid_words: *mut u32,
    ) -> c_int;
    /// Selectors over a table with several Float64 field columns (1 ..= 64): `vals` / `outs` are host arrays of
    /// n_fields device pointers, one validity bitmap for all fields.  The range form drops a row from every field when
    /// any field is NaN (filter_nan) and keeps a cell only where every field's result is valid; the instant form picks
    /// the row once, with the stale-NaN test on field 0.  `field_valid` (nullable) holds each field's Arrow validity
    /// bitmap: calls the device cannot reproduce over NULL slots are refused (see the header).
    pub fn b2p_range_eval_fields_dev(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, vals: *const *const f64,
        field_valid: *const *const u8, n_fields: i32,
        offsets: *const u64, n_rows: u64, n_series: u32, outs: *const *mut f64, valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_instant_select_fields_dev(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        vals: *const *const f64, field_valid: *const *const u8, n_fields: i32, offsets: *const u64, n_rows: u64,
        n_series: u32,
        outs: *const *mut f64, valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_group_aggregate_dev(
        ctx: *mut b2p_ctx, agg: i32, vals: *const f64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_group_index_create_dev(
        ctx: *mut b2p_ctx, gid: *const u32, n_series: u32, n_groups: u32, out_index: *mut *mut b2p_group_index,
    ) -> c_int;
    pub fn b2p_group_index_destroy(ctx: *mut b2p_ctx, index: *mut b2p_group_index);
    pub fn b2p_group_aggregate_indexed_dev(
        ctx: *mut b2p_ctx, agg: i32, vals: *const f64, valid_words: *const u32, index: *const b2p_group_index, t: u64,
        out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_range_group_sum_indexed_dev(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, val: *const f64, offsets: *const u64, n_rows: u64,
        n_series: u32, index: *const b2p_group_index, g_lo: u32, g_hi: u32, out_sum: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_range_group_sum_fused(ctx: *mut b2p_ctx, p: *const B2pRangeParams, index: *const b2p_group_index) -> c_int;
    pub fn b2p_range_group_sum_dev(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, val: *const f64, offsets: *const u64, n_rows: u64,
        n_series: u32, gid: *const u32, n_groups: u32, out_sum: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_group_aggregate_partial_dev(
        ctx: *mut b2p_ctx, agg: i32, vals: *const f64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32, out_mean: *mut f64,
    ) -> c_int;
    pub fn b2p_group_finalize_dev(ctx: *mut b2p_ctx, agg: i32, val: *mut f64, cnt: *const u32, n: u64) -> c_int;

    // ---- multi-GPU: the library's own NCCL communicator ---------------------------------------------------------
    pub fn b2p_comm_unique_id(out_id: *mut c_void, bytes: usize) -> c_int;
    pub fn b2p_comm_init(ctx: *mut b2p_ctx, id: *const c_void, bytes: usize, n_ranks: c_int, rank: c_int) -> c_int;
    pub fn b2p_comm_destroy(ctx: *mut b2p_ctx) -> c_int;
    pub fn b2p_allreduce_partials_dev(ctx: *mut b2p_ctx, agg: i32, val: *mut f64, cnt: *mut u32, mean: *mut f64, n: u64) -> c_int;
    pub fn b2p_allreduce_columns_dev(ctx: *mut b2p_ctx, sum: *mut f64, cnt: *mut u64, n_cols: u32) -> c_int;
    /// Int64 partials of sum / min / max (K3's Int64 fold) and their cross-rank merge.
    pub fn b2p_group_aggregate_partial_i64_dev(
        ctx: *mut b2p_ctx, agg: i32, vals: *const i64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_allreduce_partials_i64_dev(ctx: *mut b2p_ctx, agg: i32, val: *mut f64, cnt: *mut u32, n: u64) -> c_int;
    /// Ranks of the context's communicator (0 without one); this rank in `rank`.
    pub fn b2p_comm_ranks(ctx: *mut b2p_ctx, rank: *mut i32) -> i32;
    /// Host-pointer sharded by-label aggregate: partials, all-reduce, finalise (collective).
    pub fn b2p_group_aggregate_allreduce(
        ctx: *mut b2p_ctx, agg: i32, vals: *const f64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_group_aggregate_allreduce_i64(
        ctx: *mut b2p_ctx, agg: i32, vals: *const i64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    /// The group-label agreement's exchange: every rank's block size, then every rank's block (host buffers).
    pub fn b2p_group_keys_sizes(ctx: *mut b2p_ctx, bytes: u64, sizes: *mut u64) -> c_int;
    pub fn b2p_group_keys_allgather(ctx: *mut b2p_ctx, block: *const c_void, sizes: *const u64, out: *mut c_void) -> c_int;
    pub fn b2p_last_group_keys_bytes(ctx: *mut b2p_ctx) -> i64;
    pub fn b2p_range_group_sum_allreduce_dev(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, val: *const f64, offsets: *const u64, n_rows: u64,
        n_series: u32, index: *const b2p_group_index, n_tiles: i32, out_sum: *mut f64, out_cnt: *mut u32,
    ) -> c_int;

    // ---- HistogramFold / wide scan --------------------------------------------------------------------------------
    pub fn b2p_histogram_quantile_dev(
        ctx: *mut b2p_ctx, phi: f64, le: *const f64, n_buckets: u32, rates: *const f64, valid_words: *const u32,
        n_hist: u32, t: u64, out: *mut f64, out_valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_histogram_fold_dev(
        ctx: *mut b2p_ctx, phi: f64, hist_off: *const u32, bucket_series: *const u32, bucket_le: *const f64,
        n_hist: u32, rates: *const f64, valid_words: *const u32, t: u64, out: *mut f64, out_valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_histogram_fold_allgather(
        ctx: *mut b2p_ctx, phi: f64, rates: *const f64, valid_words: *const u32, n_rows: u32, t: u64,
        row_hist: *const u32, row_le: *const f64, n_hist: u32, out: *mut f64, out_valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_range_histogram_fold_allgather(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, val: *const f64, sid: *const u32,
        offsets_host: *const u64, n_samples: u64, n_series: u32, phi: f64, row_hist: *const u32, row_le: *const f64,
        n_hist: u32, out: *mut f64, out_valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_histogram_shard_owners(counts: *const u32, n_ranks: i32, n_hist: u32, owner: *mut u32) -> c_int;
    pub fn b2p_histogram_shard_index(
        hist: *const u32, le: *const f64, rank: *const u32, row: *const u32, n: u32, n_hist: u32, hist_off: *mut u32,
        bucket_series: *mut u32, bucket_le: *mut f64,
    ) -> c_int;
    pub fn b2p_row_move_dev(
        ctx: *mut b2p_ctx, input: *const f64, in_valid: *const u32, src: *const u32, dst: *const u32, n: u32, t: u64,
        out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_column_reduce_dev(
        ctx: *mut b2p_ctx, cols: *const *const f64, n_cols: u32, n_rows: u64, out_sum: *mut f64, out_cnt: *mut u64,
    ) -> c_int;

    // ---- binary operators ---------------------------------------------------------------------------------------------
    pub fn b2p_binary_op_dev(
        ctx: *mut b2p_ctx, op: i32, return_bool: i32, lhs: *const f64, lhs_valid: *const u32, lhs_row: *const u32,
        n_lhs_rows: u32, rhs: *const f64, rhs_valid: *const u32, rhs_row: *const u32, n_rhs_rows: u32, n_pairs: u64,
        t: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_scalar_op_dev(
        ctx: *mut b2p_ctx, op: i32, return_bool: i32, scalar_on_left: i32, scalar: f64, vals: *const f64,
        valid: *const u32, n_rows: u64, t: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_count_valid_words_dev(ctx: *mut b2p_ctx, cnt: *const u32, n_rows: u64, t: u64, valid_words: *mut u32) -> c_int;
    pub fn b2p_setop_dev(
        ctx: *mut b2p_ctx, op: i32, lhs: *const f64, lhs_valid: *const u32, lhs_key: *const u32, n_lhs_rows: u32,
        rhs: *const f64, rhs_valid: *const u32, rhs_key: *const u32, n_rhs_rows: u32, n_keys: u32, t: u64,
        out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_instant_fn_dev(
        ctx: *mut b2p_ctx, fn_: i32, arg0: f64, arg1: f64, vals: *const f64, valid: *const u32, n_rows: u64, t: u64,
        out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_scalar_calculate_dev(
        ctx: *mut b2p_ctx, vals: *const f64, valid: *const u32, row_key: *const u32, n_rows: u32, t: u64,
        out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    /// topk (bottom = 0) / bottomk per (group, step); writes validity words only (`out_valid` may be `valid`).
    pub fn b2p_topk_dev(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, vals: *const f64, valid: *const u32, index: *const b2p_group_index,
        tie: *const u32, t: u64, out_valid: *mut u32,
    ) -> c_int;
    /// topk / bottomk over rows sharded across the communicator's ranks: this rank's kept cells; `tie` distinct across
    /// every rank.  Without a communicator (one rank) the words of `b2p_topk_dev`.
    pub fn b2p_topk_allgather_dev(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, vals: *const f64, valid: *const u32, index: *const b2p_group_index,
        tie: *const u32, t: u64, out_valid: *mut u32,
    ) -> c_int;
    /// Bytes of this rank's candidate blocks in the last sharded topk.
    pub fn b2p_last_exchange_bytes(ctx: *mut b2p_ctx) -> i64;
    /// The steps of the sharded topk; `group_sizes` is a host array of the global member counts [n_groups].
    pub fn b2p_topk_shard_plan(
        ctx: *mut b2p_ctx, k: f64, group_sizes: *const u32, n_groups: u32, t: u64, n_ranks: i32, n_batches: *mut u32,
        n_rounds: *mut u32, slots: *mut u32, block_bytes: *mut u64, state_bytes: *mut u64,
    ) -> c_int;
    pub fn b2p_topk_shard_candidates_dev(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, vals: *const f64, valid: *const u32, index: *const b2p_group_index,
        tie: *const u32, t: u64, group_sizes: *const u32, n_ranks: i32, batch: u32, round: u32, state: *mut c_void,
        block: *mut c_void,
    ) -> c_int;
    pub fn b2p_topk_shard_merge_dev(
        ctx: *mut b2p_ctx, k: f64, group_sizes: *const u32, n_groups: u32, t: u64, n_ranks: i32, batch: u32,
        round: u32, blocks: *const c_void, state: *mut c_void,
    ) -> c_int;
    pub fn b2p_topk_shard_mark_dev(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, vals: *const f64, valid: *const u32, index: *const b2p_group_index,
        tie: *const u32, t: u64, group_sizes: *const u32, n_ranks: i32, batch: u32, state: *const c_void,
        out_valid: *mut u32,
    ) -> c_int;
    /// quantile(phi) per (group, step) into out_val / out_cnt [n_groups x T]; cnt 0 = no row.
    pub fn b2p_group_quantile_dev(
        ctx: *mut b2p_ctx, phi: f64, vals: *const f64, valid: *const u32, index: *const b2p_group_index, t: u64,
        out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    /// Host-pointer form of `b2p_quantile_allreduce_dev` (gid over the global group ids).
    pub fn b2p_quantile_allreduce(
        ctx: *mut b2p_ctx, phi: f64, vals: *const f64, valid: *const u32, gid: *const u32, n_rows: u32, n_groups: u32,
        t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    /// Host-pointer sharded count_values: merged rows from `out_goff`, at most `cap_rows` of them (collective).
    pub fn b2p_count_values_allgather(
        ctx: *mut b2p_ctx, vals: *const f64, valid: *const u32, gid: *const u32, n_rows: u32, n_groups: u32, t: u64,
        cap_rows: u64, out_goff: *mut u32, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_count_values_allgather_i64(
        ctx: *mut b2p_ctx, vals: *const i64, valid: *const u32, gid: *const u32, n_rows: u32, n_groups: u32, t: u64,
        cap_rows: u64, out_goff: *mut u32, out_val: *mut i64, out_cnt: *mut u32,
    ) -> c_int;
    /// quantile(phi) by label over rows sharded across the communicator's ranks: every rank receives the full
    /// [n_groups x T] result.  Without a communicator (one rank) the output of `b2p_group_quantile_dev`.
    pub fn b2p_quantile_allreduce_dev(
        ctx: *mut b2p_ctx, phi: f64, vals: *const f64, valid: *const u32, index: *const b2p_group_index, t: u64,
        out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    /// The steps of the sharded quantile: batches, then per batch and pass a rank's block and the advance over the
    /// merged blocks (`live`: cells left, read back).
    pub fn b2p_quantile_shard_plan(
        ctx: *mut b2p_ctx, n_groups: u32, t: u64, n_batches: *mut u32, block_bytes: *mut u64, state_bytes: *mut u64,
    ) -> c_int;
    pub fn b2p_quantile_shard_pass_dev(
        ctx: *mut b2p_ctx, phi: f64, vals: *const f64, valid: *const u32, index: *const b2p_group_index, t: u64,
        batch: u32, pass: u32, block: *mut c_void,
    ) -> c_int;
    pub fn b2p_quantile_shard_advance_dev(
        ctx: *mut b2p_ctx, phi: f64, n_groups: u32, t: u64, batch: u32, pass: u32, blocks: *const c_void,
        n_blocks: u32, out_val: *mut f64, out_cnt: *mut u32, live: *mut u64,
    ) -> c_int;
    /// count_values per (group, step) into out_val / out_cnt [n_series x T], rows in the index's member order: a group's
    /// j-th row holds its j-th smallest distinct value (by bits, f64 total order) and its multiplicity; cnt 0 = none.
    pub fn b2p_count_values_dev(
        ctx: *mut b2p_ctx, vals: *const f64, valid: *const u32, index: *const b2p_group_index, t: u64,
        out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    /// count_values by label over rows sharded across the communicator's ranks, from each rank's
    /// `b2p_count_values_dev` output.  `heights` (host) is every rank's row of h_r(g) [n_ranks x n_groups] (one row
    /// without a communicator); group g gets the sum over ranks of its heights as output rows.
    pub fn b2p_count_values_shard_heights_dev(
        ctx: *mut b2p_ctx, local_cnt: *const u32, index: *const b2p_group_index, t: u64, heights: *mut u32,
    ) -> c_int;
    pub fn b2p_count_values_allgather_dev(
        ctx: *mut b2p_ctx, local_val: *const f64, local_cnt: *const u32, index: *const b2p_group_index, t: u64,
        heights: *const u32, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_count_values_allgather_i64_dev(
        ctx: *mut b2p_ctx, local_val: *const i64, local_cnt: *const u32, index: *const b2p_group_index, t: u64,
        heights: *const u32, out_val: *mut i64, out_cnt: *mut u32,
    ) -> c_int;
    /// The steps of the sharded count_values: batches, then per batch every rank's block and the merge over the
    /// gathered blocks ([keys of rank 0 .. R-1][counts of rank 0 .. R-1]).
    pub fn b2p_count_values_shard_plan(
        ctx: *mut b2p_ctx, heights: *const u32, n_ranks: i32, n_groups: u32, t: u64, n_batches: *mut u32,
        block_bytes: *mut u64,
    ) -> c_int;
    pub fn b2p_count_values_shard_pack_dev(
        ctx: *mut b2p_ctx, local_val: *const f64, local_cnt: *const u32, index: *const b2p_group_index, t: u64,
        heights: *const u32, n_ranks: i32, rank: i32, batch: u32, block: *mut c_void,
    ) -> c_int;
    pub fn b2p_count_values_shard_pack_i64_dev(
        ctx: *mut b2p_ctx, local_val: *const i64, local_cnt: *const u32, index: *const b2p_group_index, t: u64,
        heights: *const u32, n_ranks: i32, rank: i32, batch: u32, block: *mut c_void,
    ) -> c_int;
    pub fn b2p_count_values_shard_merge_dev(
        ctx: *mut b2p_ctx, heights: *const u32, n_ranks: i32, n_groups: u32, t: u64, batch: u32, blocks: *const c_void,
        out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_count_values_shard_merge_i64_dev(
        ctx: *mut b2p_ctx, heights: *const u32, n_ranks: i32, n_groups: u32, t: u64, batch: u32, blocks: *const c_void,
        out_val: *mut i64, out_cnt: *mut u32,
    ) -> c_int;
    /// fn(<child>[range:step]) over a child's grid [n_rows x T_inner] on the inner steps inner_start + k * inner_interval:
    /// every valid cell of a row is one sample of its series (NaN included); p is the outer grid, range and function
    /// (offset and filter_nan 0).  out [n_rows x T] / out_valid [n_rows x Tw] as b2p_range_eval_dev.
    pub fn b2p_subquery_dev(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, inner_start: i64, inner_interval: i64, vals: *const f64,
        valid: *const u32, n_rows: u32, t_inner: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    /// sort / sort_desc (K14): the valid cells of a device grid [n_rows x T] as cell indices row * T + k in value order
    /// (f64 total order, ties in row-major order); `out_n` is a device u64.  Synchronises the context's stream once.
    pub fn b2p_sort_cells_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const f64, valid: *const u32, n_rows: u32, t: u64, out_cells: *mut u64,
        out_n: *mut u64,
    ) -> c_int;
    /// sort / sort_desc over several fields: `vals` is a host array of n_fields device grids sharing `valid`; the cells
    /// in lexicographic order over the fields (field 0 first), equal tuples in row-major order.
    pub fn b2p_sort_cells_fields_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const *const f64, n_fields: i32, valid: *const u32, n_rows: u32, t: u64,
        out_cells: *mut u64, out_n: *mut u64,
    ) -> c_int;
    /// sort / sort_desc over rows sharded across the communicator's ranks: every rank's count of valid cells (host
    /// `counts` [n_ranks], one entry without a communicator), then every rank's sorted run, exchanged and merged into
    /// the global cells row_id[r] * t + k and their values on every rank.  `row_id` (device) is strictly increasing.
    pub fn b2p_sort_shard_counts_dev(
        ctx: *mut b2p_ctx, valid: *const u32, n_rows: u32, t: u64, counts: *mut u64,
    ) -> c_int;
    pub fn b2p_sort_cells_allgather_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const f64, valid: *const u32, row_id: *const u32, n_rows: u32, t: u64,
        counts: *const u64, out_cells: *mut u64, out_vals: *mut f64,
    ) -> c_int;
    pub fn b2p_sort_cells_allgather_fields_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const *const f64, n_fields: i32, valid: *const u32, row_id: *const u32,
        n_rows: u32, t: u64, counts: *const u64, out_cells: *mut u64, out_vals: *const *mut f64,
    ) -> c_int;
    pub fn b2p_sort_cells_allgather_i64_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const i64, valid: *const u32, row_id: *const u32, n_rows: u32, t: u64,
        counts: *const u64, out_cells: *mut u64, out_vals: *mut i64,
    ) -> c_int;
    /// The steps of the sharded sort: every rank's block ([keys of field 0 .. F-1][global cells], `count` entries),
    /// and the merge over the blocks laid back to back in rank order.
    pub fn b2p_sort_shard_pack_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const *const f64, n_fields: i32, valid: *const u32, row_id: *const u32,
        n_rows: u32, t: u64, count: u64, block: *mut c_void,
    ) -> c_int;
    pub fn b2p_sort_shard_pack_i64_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const i64, valid: *const u32, row_id: *const u32, n_rows: u32, t: u64,
        count: u64, block: *mut c_void,
    ) -> c_int;
    pub fn b2p_sort_shard_merge_dev(
        ctx: *mut b2p_ctx, desc: i32, n_fields: i32, counts: *const u64, n_ranks: i32, blocks: *const c_void,
        out_cells: *mut u64, out_vals: *const *mut f64,
    ) -> c_int;
    pub fn b2p_sort_shard_merge_i64_dev(
        ctx: *mut b2p_ctx, desc: i32, counts: *const u64, n_ranks: i32, blocks: *const c_void, out_cells: *mut u64,
        out_vals: *mut i64,
    ) -> c_int;
    /// Int64 (BIGINT) value columns: the cells hold i64 bits in the same 8-byte slots.  The instant selector with field 0
    /// Int64 (no stale-NaN test); the by-label aggregate (sum wrapping, min / max signed, written as i64 bits; avg,
    /// stddev, stdvar over (f64)i64); topk / count_values / sort ranking by signed value; the Float64 coercion.
    pub fn b2p_instant_select_fields_i64_dev(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        vals: *const *const f64, field_valid: *const *const u8, n_fields: i32, offsets: *const u64, n_rows: u64,
        n_series: u32, outs: *const *mut f64, valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_group_aggregate_i64_dev(
        ctx: *mut b2p_ctx, agg: i32, vals: *const i64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_topk_i64_dev(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, vals: *const i64, valid: *const u32, index: *const b2p_group_index,
        tie: *const u32, t: u64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_count_values_i64_dev(
        ctx: *mut b2p_ctx, vals: *const i64, valid: *const u32, index: *const b2p_group_index, t: u64,
        out_val: *mut i64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_sort_cells_i64_dev(
        ctx: *mut b2p_ctx, desc: i32, vals: *const i64, valid: *const u32, n_rows: u32, t: u64, out_cells: *mut u64,
        out_n: *mut u64,
    ) -> c_int;
    pub fn b2p_i64_to_f64_dev(ctx: *mut b2p_ctx, vals: *const i64, n: u64, out: *mut f64) -> c_int;
    /// absent (K15): out_valid [Tw] = the steps at which no row of the device grid's validity [n_rows x Tw] has a bit
    /// (bits past T cleared), out [T] = 1.0 there and 0.0 elsewhere.  Only validity words are read; no host round trip.
    pub fn b2p_absent_dev(
        ctx: *mut b2p_ctx, valid: *const u32, n_rows: u32, t: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;

    // ---- host-side helper (no device work): SeriesDivide + cadence scan of one sorted batch ---------------------------
    /// The merge of the group-label agreement over R blocks (host only).
    pub fn b2p_group_keys_merge(
        blocks: *const *const c_void, sizes: *const u64, n_ranks: i32, rank: i32, out_table: *mut c_void,
        out_table_bytes: *mut u64, n_groups: *mut u32, local_to_global: *mut u32,
    ) -> c_int;
    pub fn b2p_host_scan_series(
        ts: *const i64, sid: *const u32, offsets_in: *const u64, n_rows: u64, n_series: u32, sid_base: u32,
        offsets_out: *mut u64, t0: *mut i64, cadence: *mut i64, all_regular: *mut i32,
    ) -> c_int;

    // ---- host-pointer API (synchronous) ------------------------------------------------------------------------------
    pub fn b2p_range_eval(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, val: *const f64, sid: *const u32,
        offsets_host: *const u64, n_rows: u64, n_series: u32, out: *mut f64, valid_words: *mut u32, out_ts: *mut i64,
    ) -> c_int;
    pub fn b2p_range_udf(
        ctx: *mut b2p_ctx, fn_id: i32, ts: *const i64, val: *const f64, n_rows: u64, packed_ranges: *const i64,
        eval_ts: *const i64, n_win: u64, range_length: i64, param0: f64, param1: f64, out: *mut f64, valid: *mut u8,
    ) -> c_int;
    pub fn b2p_instant_select(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        val: *const f64, sid: *const u32, offsets_host: *const u64, n_rows: u64, n_series: u32, out: *mut f64,
        valid_words: *mut u32,
    ) -> c_int;
    /// Host-pointer forms of the two multi-field selectors (synchronous, one staged copy).
    pub fn b2p_range_eval_fields(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, vals: *const *const f64,
        field_valid: *const *const u8, n_fields: i32,
        sid: *const u32, offsets_host: *const u64, n_rows: u64, n_series: u32, outs: *const *mut f64,
        valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_instant_select_fields(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        vals: *const *const f64, field_valid: *const *const u8, n_fields: i32, sid: *const u32,
        offsets_host: *const u64, n_rows: u64,
        n_series: u32, outs: *const *mut f64, valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_group_aggregate(
        ctx: *mut b2p_ctx, agg: i32, vals: *const f64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_histogram_quantile(
        ctx: *mut b2p_ctx, phi: f64, le: *const f64, n_buckets: u32, rates: *const f64, valid_words: *const u32,
        n_hist: u32, t: u64, out: *mut f64, out_valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_range_histogram_fold(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, ts: *const i64, val: *const f64, sid: *const u32,
        offsets_host: *const u64, n_rows: u64, n_series: u32, phi: f64, hist_off: *const u32,
        bucket_series: *const u32, bucket_le: *const f64, n_hist: u32, out: *mut f64, out_valid_words: *mut u32,
    ) -> c_int;
    /// HistogramFold over any host grid [n_rows x T]; a malformed index is B2P_E_INVALID before anything is launched.
    pub fn b2p_histogram_fold(
        ctx: *mut b2p_ctx, phi: f64, hist_off: *const u32, bucket_series: *const u32, bucket_le: *const f64,
        n_hist: u32, rates: *const f64, valid_words: *const u32, n_rows: u32, t: u64, out: *mut f64,
        out_valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_binary_op(
        ctx: *mut b2p_ctx, op: i32, return_bool: i32, lhs: *const f64, lhs_valid: *const u32, lhs_row: *const u32,
        n_lhs_rows: u32, rhs: *const f64, rhs_valid: *const u32, rhs_row: *const u32, n_rhs_rows: u32, n_pairs: u64,
        t: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_scalar_op(
        ctx: *mut b2p_ctx, op: i32, return_bool: i32, scalar_on_left: i32, scalar: f64, vals: *const f64,
        valid: *const u32, n_rows: u64, t: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_setop(
        ctx: *mut b2p_ctx, op: i32, lhs: *const f64, lhs_valid: *const u32, lhs_key: *const u32, n_lhs_rows: u32,
        rhs: *const f64, rhs_valid: *const u32, rhs_key: *const u32, n_rhs_rows: u32, n_keys: u32, t: u64,
        out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_instant_fn(
        ctx: *mut b2p_ctx, fn_: i32, arg0: f64, arg1: f64, vals: *const f64, valid: *const u32, n_rows: u64, t: u64,
        out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_scalar_calculate(
        ctx: *mut b2p_ctx, vals: *const f64, valid: *const u32, row_key: *const u32, n_rows: u32, t: u64,
        out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_topk(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, vals: *const f64, valid: *const u32, gid: *const u32, n_rows: u32,
        n_groups: u32, tie: *const u32, t: u64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_group_quantile(
        ctx: *mut b2p_ctx, phi: f64, vals: *const f64, valid: *const u32, gid: *const u32, n_rows: u32, n_groups: u32,
        t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_count_values(
        ctx: *mut b2p_ctx, vals: *const f64, valid: *const u32, gid: *const u32, n_rows: u32, n_groups: u32, t: u64,
        out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_subquery(
        ctx: *mut b2p_ctx, p: *const B2pRangeParams, inner_start: i64, inner_interval: i64, vals: *const f64,
        valid: *const u32, n_rows: u32, t_inner: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;
    /// Host-pointer form of b2p_sort_cells_dev (synchronous); `out_cells` has room for n_rows * T entries.
    pub fn b2p_sort_cells(
        ctx: *mut b2p_ctx, desc: i32, vals: *const f64, valid: *const u32, n_rows: u32, t: u64, out_cells: *mut u64,
        out_n: *mut u64,
    ) -> c_int;
    /// Host-pointer form of b2p_sort_cells_fields_dev (synchronous).
    pub fn b2p_sort_cells_fields(
        ctx: *mut b2p_ctx, desc: i32, vals: *const *const f64, n_fields: i32, valid: *const u32, n_rows: u32, t: u64,
        out_cells: *mut u64, out_n: *mut u64,
    ) -> c_int;
    /// Host-pointer forms of the Int64 calls (synchronous).
    pub fn b2p_instant_select_fields_i64(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        vals: *const *const f64, field_valid: *const *const u8, n_fields: i32, sid: *const u32,
        offsets_host: *const u64, n_rows: u64, n_series: u32, outs: *const *mut f64, valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_group_aggregate_i64(
        ctx: *mut b2p_ctx, agg: i32, vals: *const i64, valid_words: *const u32, gid: *const u32, n_series: u32,
        n_groups: u32, t: u64, out_val: *mut f64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_topk_i64(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, vals: *const i64, valid: *const u32, gid: *const u32, n_rows: u32,
        n_groups: u32, tie: *const u32, t: u64, out_valid: *mut u32,
    ) -> c_int;
    pub fn b2p_count_values_i64(
        ctx: *mut b2p_ctx, vals: *const i64, valid: *const u32, gid: *const u32, n_rows: u32, n_groups: u32, t: u64,
        out_val: *mut i64, out_cnt: *mut u32,
    ) -> c_int;
    pub fn b2p_sort_cells_i64(
        ctx: *mut b2p_ctx, desc: i32, vals: *const i64, valid: *const u32, n_rows: u32, t: u64, out_cells: *mut u64,
        out_n: *mut u64,
    ) -> c_int;
    pub fn b2p_i64_to_f64(ctx: *mut b2p_ctx, vals: *const i64, n: u64, out: *mut f64) -> c_int;
    /// Host-pointer form of b2p_absent_dev (synchronous).
    pub fn b2p_absent(
        ctx: *mut b2p_ctx, valid: *const u32, n_rows: u32, t: u64, out: *mut f64, out_valid: *mut u32,
    ) -> c_int;

    // ---- functions of the eval step and timestamp() ---------------------------------------------------------------------
    /// K19: `part` (enum b2p_step_part: time, minute, hour, day_of_month, day_of_week, day_of_year, month, year,
    /// days_in_month) of eval_ts[k] at every valid cell of a [n_rows x t] grid; validity is read, never written.
    pub fn b2p_step_fn_dev(
        ctx: *mut b2p_ctx, part: i32, eval_ts: *const i64, valid: *const u32, n_rows: u64, t: u64, out: *mut f64,
    ) -> c_int;
    pub fn b2p_step_fn(
        ctx: *mut b2p_ctx, part: i32, eval_ts: *const i64, valid: *const u32, n_rows: u64, t: u64, out: *mut f64,
    ) -> c_int;
    /// timestamp(<selector>): the instant selector with the chosen sample's (ts + offset) / 1000 as the value; no value
    /// column, no stale-NaN test.
    pub fn b2p_instant_timestamp_dev(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        offsets: *const u64, n_rows: u64, n_series: u32, out: *mut f64, valid_words: *mut u32,
    ) -> c_int;
    pub fn b2p_instant_timestamp(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, lookback: i64, offset: i64, ts: *const i64,
        sid: *const u32, offsets_host: *const u64, n_rows: u64, n_series: u32, out: *mut f64, valid_words: *mut u32,
    ) -> c_int;

    // ---- plan-level API over the Arrow C Data Interface -----------------------------------------------------------------
    pub fn b2p_plan_range_create(
        ctx: *mut b2p_ctx, function: *const c_char, p: *const B2pRangeParams, time_index: *const c_char,
        field_column: *const c_char, tag_columns: *const *const c_char, n_tags: i32, aggregate: *const c_char,
        by_columns: *const *const c_char, n_by: i32,
    ) -> *mut b2p_plan;
    /// The range / instant leaf over 1..=64 Float64 field columns, every one selected; one value column per field.
    pub fn b2p_plan_range_create_fields(
        ctx: *mut b2p_ctx, function: *const c_char, p: *const B2pRangeParams, time_index: *const c_char,
        field_columns: *const *const c_char, n_fields: i32, tag_columns: *const *const c_char, n_tags: i32,
        aggregate: *const c_char, by_columns: *const *const c_char, n_by: i32,
    ) -> *mut b2p_plan;
    pub fn b2p_plan_set_instant(plan: *mut b2p_plan, lookback_delta: i64) -> c_int;
    pub fn b2p_plan_set_histogram_quantile(plan: *mut b2p_plan, le_column: *const c_char, quantile: f64) -> c_int;
    /// The metric-engine leaf: Utf8 label columns beside the one UInt64 `__tsid` tag column (before the first push).
    pub fn b2p_plan_set_label_columns(plan: *mut b2p_plan, names: *const *const c_char, n: i32) -> c_int;
    /// Marks an aggregate node, or a leaf with an aggregate stage, sharded over the context's communicator.
    pub fn b2p_plan_set_sharded(plan: *mut b2p_plan) -> c_int;
    pub fn b2p_plan_set_scalar_op(plan: *mut b2p_plan, op: i32, scalar: f64, scalar_on_left: i32, return_bool: i32) -> c_int;
    /// The node shares ownership of both children; their handles stay valid and must still be destroyed.
    pub fn b2p_plan_binary_create(
        ctx: *mut b2p_ctx, op: i32, return_bool: i32, lhs: *mut b2p_plan, rhs: *mut b2p_plan, matching: *const c_char,
        labels: *const *const c_char, n_labels: i32, label_side: *const c_char,
    ) -> *mut b2p_plan;
    /// Ownership as for b2p_plan_binary_create.
    pub fn b2p_plan_setop_create(
        ctx: *mut b2p_ctx, op: i32, lhs: *mut b2p_plan, rhs: *mut b2p_plan, matching: *const c_char,
        labels: *const *const c_char, n_labels: i32,
    ) -> *mut b2p_plan;
    /// `name` as the reference's projection shows it (ScalarFunctionExpr::name): "abs", "radians", "prom_round", ...
    pub fn b2p_plan_set_function(plan: *mut b2p_plan, name: *const c_char, args: *const f64, n_args: i32) -> c_int;
    /// Ownership as for b2p_plan_binary_create.
    pub fn b2p_plan_scalar_create(ctx: *mut b2p_ctx, child: *mut b2p_plan) -> *mut b2p_plan;
    /// EmptyMetric: one tagless row over start..=end by interval; `kind` 0 = only the time index, 1 = time(),
    /// 2 = `literal` (vector(s), pi(), a number).
    pub fn b2p_plan_empty_metric_create(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, time_index: *const c_char, value_column: *const c_char,
        kind: i32, literal: f64,
    ) -> *mut b2p_plan;
    /// timestamp(<selector>) on a range node: the instant form whose value is the sample's timestamp in seconds.
    pub fn b2p_plan_set_timestamp(plan: *mut b2p_plan, lookback_delta: i64) -> c_int;
    /// label_replace(child, dst, replacement, src, regex); ownership of `child` as for b2p_plan_binary_create.
    pub fn b2p_plan_label_replace_create(
        ctx: *mut b2p_ctx, child: *mut b2p_plan, dst: *const c_char, replacement: *const c_char, src: *const c_char,
        regex: *const c_char,
    ) -> *mut b2p_plan;
    /// label_join(child, dst, separator, srcs..); ownership of `child` as for b2p_plan_binary_create.
    pub fn b2p_plan_label_join_create(
        ctx: *mut b2p_ctx, child: *mut b2p_plan, dst: *const c_char, separator: *const c_char,
        srcs: *const *const c_char, n_srcs: i32,
    ) -> *mut b2p_plan;
    /// Host only: 0 = a label_replace regex the library evaluates, 1 = Rust's regex crate rejects it, 2 = valid in Rust
    /// but outside the library's supported list (the query stays on the CPU).
    pub fn b2p_label_regex_check(regex: *const c_char) -> c_int;
    /// Host only: regexp_replace(input, "^(?s:" + regex + ")$", replacement) into `out` (NUL-terminated, `cap` bytes);
    /// `out_len` gets the result's length.
    pub fn b2p_label_regex_replace(
        regex: *const c_char, replacement: *const c_char, input: *const c_char, out: *mut c_char, cap: u64,
        out_len: *mut u64,
    ) -> c_int;
    /// `modifier`: NULL, "by" or "without"; ownership of `child` as for b2p_plan_binary_create.
    pub fn b2p_plan_topk_create(
        ctx: *mut b2p_ctx, bottom: i32, k: f64, child: *mut b2p_plan, modifier: *const c_char,
        labels: *const *const c_char, n_labels: i32,
    ) -> *mut b2p_plan;
    /// `op`: sum avg count min max stddev stdvar group quantile (`param` = phi); `modifier`: NULL, "by" or "without";
    /// ownership of `child` as for b2p_plan_binary_create.
    pub fn b2p_plan_aggregate_create(
        ctx: *mut b2p_ctx, op: *const c_char, param: f64, child: *mut b2p_plan, modifier: *const c_char,
        labels: *const *const c_char, n_labels: i32,
    ) -> *mut b2p_plan;
    /// count_values(`label`, child); `modifier`: NULL, "by" or "without"; ownership of `child` as for
    /// b2p_plan_binary_create.
    pub fn b2p_plan_count_values_create(
        ctx: *mut b2p_ctx, label: *const c_char, child: *mut b2p_plan, modifier: *const c_char,
        labels: *const *const c_char, n_labels: i32,
    ) -> *mut b2p_plan;
    /// `function`(child[range:step]): RangeManipulate(p.start, p.end, p.interval, p.range) directly over the child (built
    /// on the inner grid); offset and filter_nan must be 0.  Ownership of `child` as for b2p_plan_binary_create.
    pub fn b2p_plan_subquery_create(
        ctx: *mut b2p_ctx, function: *const c_char, p: *const B2pRangeParams, child: *mut b2p_plan,
    ) -> *mut b2p_plan;
    /// histogram_quantile(`phi`, child) over any node; `le_column` NULL means "le".  Ownership of `child` as for
    /// b2p_plan_binary_create.
    pub fn b2p_plan_histogram_quantile_create(
        ctx: *mut b2p_ctx, le_column: *const c_char, phi: f64, child: *mut b2p_plan,
    ) -> *mut b2p_plan;
    /// `function` ("sort" | "sort_desc" | "sort_by_label" | "sort_by_label_desc") over any node; `labels` for the
    /// sort_by_label forms only.  Ownership of `child` as for b2p_plan_binary_create.
    pub fn b2p_plan_sort_create(
        ctx: *mut b2p_ctx, function: *const c_char, child: *mut b2p_plan, labels: *const *const c_char, n_labels: i32,
    ) -> *mut b2p_plan;
    /// absent(child) over the grid (start, end, interval); `label_names` / `label_values` are the equality matchers of the
    /// argument's selector in matcher order.  Ownership of `child` as for b2p_plan_binary_create.
    pub fn b2p_plan_absent_create(
        ctx: *mut b2p_ctx, start: i64, end: i64, interval: i64, time_index: *const c_char, value_column: *const c_char,
        label_names: *const *const c_char, label_values: *const *const c_char, n_labels: i32, child: *mut b2p_plan,
    ) -> *mut b2p_plan;
    /// MOVES the batch: on success the release callbacks now belong to the plan.
    pub fn b2p_plan_push_batch(plan: *mut b2p_plan, batch: *mut FFI_ArrowArray, schema: *mut FFI_ArrowSchema) -> c_int;
    pub fn b2p_plan_execute(plan: *mut b2p_plan, out: *mut FFI_ArrowArray, out_schema: *mut FFI_ArrowSchema) -> c_int;
    pub fn b2p_plan_num_series(plan: *mut b2p_plan) -> i64;
    pub fn b2p_plan_destroy(plan: *mut b2p_plan);
    pub fn b2p_plan_last_error() -> *const c_char;

    // ---- bench / test utility ------------------------------------------------------------------------------------------
    pub fn b2p_synth_fill_dev(
        ctx: *mut b2p_ctx, series_begin: u64, n_series: u64, n_samples: u32, t0: i64, scrape_ms: i64, jitter_ms: u32,
        with_resets: i32, seed: u64, ts: *mut i64, val: *mut f64, sid: *mut u32,
    ) -> c_int;
}

/// The library's thread-local error message as an owned string.
pub fn last_error() -> String {
    // SAFETY: b2p_last_error returns a NUL-terminated string owned by the library, valid until the next call on this thread.
    unsafe { std::ffi::CStr::from_ptr(b2p_last_error()).to_string_lossy().into_owned() }
}
pub fn plan_last_error() -> String {
    // SAFETY: as above.
    unsafe { std::ffi::CStr::from_ptr(b2p_plan_last_error()).to_string_lossy().into_owned() }
}
