/*
 * b200promql.h — C ABI of libb200promql.so: an H100 (sm_90a) evaluator for GreptimeDB's
 * PromQL range-query hot path.  Plain pointers and sizes only (no torch / Arrow C++ types), so
 * the reference's Rust host can bind it with `extern "C"` / cxx (see INTEGRATION.md).
 *
 * What each entry point replaces in the reference (paths relative to the greptimedb tree):
 *
 *   b2p_series_offsets_dev     SeriesDivideStream::poll_next + find_first_diff_row
 *                              src/promql/src/extension_plan/series_divide.rs:540-620, 622-670
 *   b2p_range_eval[_dev]       SeriesNormalizeStream::normalize            normalize.rs:388-431
 *                            + RangeManipulateStream::calculate_range/manipulate
 *                                                                          range_manipulate.rs:636-772
 *                            + Projection(prom_* ScalarUDF):  ExtrapolatedRate::calc
 *                              functions/extrapolate_rate.rs:133-288, IDelta::calc idelta.rs:113-153,
 *                              #[range_fn] loop common/macro/src/range_fn.rs:189-229 over
 *                              aggr_over_time.rs:35-179, resets.rs:33-48, changes.rs:33-48,
 *                              deriv.rs:32-40, predict_linear.rs:163-199, quantile.rs:201-225,
 *                              double_exponential_smoothing.rs:226-258
 *                            + Filter(value IS NOT NULL)  src/query/src/promql/planner.rs:1063
 *                              (expressed as the validity bitmap)
 *   b2p_range_udf[_dev]        one prom_* ScalarUDF call over a RangeArray (packed i64 keys
 *                              offset | len<<32, src/promql/src/range_array.rs:247-254) — the narrow
 *                              boundary: Fn(&[ColumnarValue]) -> ColumnarValue, extrapolate_rate.rs:90-96
 *   b2p_instant_select[_dev]   InstantManipulateStream::manipulate         instant_manipulate.rs:473-585
 *   b2p_range_eval_fields[_dev], b2p_instant_select_fields[_dev]
 *                              the same two over a table with several field columns: RangeManipulate field_columns
 *                              range_manipulate.rs:70-153, the UDF per field planner.rs:2180, the all-fields
 *                              IS NOT NULL filter planner.rs:2774-2791
 *   b2p_group_aggregate[_dev]  DataFusion AggregateExec(Partial+Final) planned by
 *                              prom_aggr_expr_to_plan src/query/src/promql/planner.rs:334-452
 *                              (sum/avg/count/min/max/stddev/stdvar by labels + eval ts)
 *   b2p_histogram_quantile[_dev] HistogramFoldStream::fold_buf + evaluate_row
 *                              histogram_fold.rs:754-820, 1046-1118
 *   b2p_histogram_fold[_dev]   the same fold over an explicit (histogram -> buckets in le order) index and any grid:
 *                              safe mode histogram_fold.rs:834-981 + evaluate_row :1046-1118
 *   b2p_column_reduce_dev      avg_over_time over a wide table (config 5): per-column sum,count
 *   b2p_binary_op[_dev]        vector-vector arithmetic / comparison: ProjectionExec / FilterExec over the inner
 *                              HashJoinExec on (tag columns, time index), planner.rs:556-777, 3436-3546; the join is a
 *                              host-side series match that yields (lhs row, rhs row) pairs
 *   b2p_scalar_op[_dev]        vector-scalar arithmetic / comparison (ProjectionExec / FilterExec, planner.rs:556-777)
 *   b2p_instant_fn[_dev]       instant-vector math functions: the Projection of planner.rs:2368-2413 (DataFusion math
 *                              builtins, prom_round round.rs:52-105, clamp / clamp_min / clamp_max clamp.rs:75-325)
 *   b2p_scalar_calculate[_dev] scalar(): ScalarCalculateStream, scalar_calculate.rs:532-637
 *   b2p_absent[_dev]           absent(): AbsentStream over Aggregate(ts, first_value) -> Sort(ts), absent.rs,
 *                              planner.rs:3186-3245
 *   b2p_setop[_dev]            set operators: `and` / `unless` = left.distinct() LeftSemi / LeftAnti HashJoinExec on
 *                              (key columns, time index), planner.rs:3549-3703; `or` = UnionDistinctOnExec,
 *                              planner.rs:3707-3906, union_distinct_on.rs:338-577; the key match is done by the caller
 *   b2p_topk[_dev]             topk / bottomk: Window(row_number() OVER (PARTITION BY group labels, ts ORDER BY value,
 *                              tags)) -> Filter(row_number <= k), planner.rs:454-541, 2963-3016; the caller groups the
 *                              rows and ranks the label tuples
 *   b2p_group_quantile[_dev]   quantile by label: Aggregate(quantile(φ, value)), QuantileAccumulator::evaluate,
 *                              quantile_aggr.rs:110-116, quantile.rs:201-225
 *   b2p_count_values[_dev]     count_values by label: Aggregate(groupBy = [labels.., ts, value], count(value)) ->
 *                              Sort(labels, ts, value), planner.rs:402-445
 *   b2p_subquery[_dev]         fn(<expr>[range:step]): RangeManipulate directly over the inner plan + Projection(prom_fn)
 *                              + Filter, planner.rs:292-332
 *   b2p_sort_cells[_dev]       sort / sort_desc: Filter(value IS NOT NULL) -> Sort(value ASC | DESC, NULLS FIRST),
 *                              planner.rs:1060-1089, 2743-2772
 *   b2p_sort_cells_fields[_dev] the same over several fields: Sort(f0, f1, .. ASC | DESC, NULLS FIRST),
 *                              planner.rs:1066-1071, 2743-2749
 *   b2p_*_i64[_dev]            the instant selector, the by-label aggregate, topk / bottomk, count_values and sort over
 *                              an Int64 (BIGINT) value column; b2p_i64_to_f64[_dev] the Float64 coercion of one
 *
 * Data layout (HBM, struct-of-arrays, all row-sorted by (series id, timestamp) exactly like
 * the reference's required_input_ordering, series_divide.rs:410-440):
 *   ts[n_rows]   int64  ms since epoch (Millisecond = i64, extension_plan.rs:42)
 *   val[n_rows]  f64
 *   sid[n_rows]  uint32 dense series id 0..n_series-1, non-decreasing (host-side renumbering of
 *                __tsid: UInt64 / tag tuples, SURVEY.md appendix C-9)
 *   offsets[n_series+1] uint64 row offset of each series (product of b2p_series_offsets_dev)
 * Result layout: dense grid.  T = b2p_num_steps(start,end,interval) global eval steps
 *   t_k = start + k*interval; out[s*T + k] f64, valid bit k of series s in
 *   valid_words[s*Tw + (k>>5)] bit (k&31), Tw = (T+31)/32.  valid=0 <=> the reference emits no
 *   row for (series, t_k) (trimmed step, empty window, null result, NaN-stale); out is 0.0 there.
 *
 * Conventions: every function returns 0 (B2P_OK) or a negative B2P_E_*; b2p_last_error() gives a
 * thread-local message.  *_dev functions take DEVICE pointers, enqueue on the context's stream and
 * return without synchronising; call b2p_sync() before reading results — it also completes the
 * rare slow-path fix-ups.  Host-pointer functions copy H2D, run, copy D2H and synchronise.
 * A b2p_ctx is bound to one device and one stream; use one context per calling thread/partition
 * (DataFusion calls execute(partition) concurrently — range_manipulate.rs:546-579).
 * All column pointers must be 16-byte aligned.
 */
#ifndef B200PROMQL_H
#define B200PROMQL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B2P_API __attribute__((visibility("default")))
#else
#define B2P_API
#endif

#define B2P_OK 0
#define B2P_E_INVALID (-1)  /* bad argument */
#define B2P_E_CUDA (-2)     /* CUDA runtime error */
#define B2P_E_UNSORTED (-3) /* sid column not non-decreasing / id >= n_series */
#define B2P_E_NOMEM (-4)
#define B2P_E_TOO_LARGE (-5) /* n_series * T exceeds what the dense grid supports */

/* Range functions (UDF names in the reference: prom_rate, prom_increase, ...). */
enum b2p_fn {
  B2P_FN_RATE = 0,             /* ExtrapolatedRate<true,true>   */
  B2P_FN_INCREASE = 1,         /* ExtrapolatedRate<true,false>  */
  B2P_FN_DELTA = 2,            /* ExtrapolatedRate<false,false> */
  B2P_FN_IRATE = 3,            /* IDelta<true>  */
  B2P_FN_IDELTA = 4,           /* IDelta<false> */
  B2P_FN_RESETS = 5,
  B2P_FN_CHANGES = 6,
  B2P_FN_COUNT_OVER_TIME = 7,
  B2P_FN_SUM_OVER_TIME = 8,
  B2P_FN_AVG_OVER_TIME = 9,
  B2P_FN_MIN_OVER_TIME = 10,
  B2P_FN_MAX_OVER_TIME = 11,
  B2P_FN_LAST_OVER_TIME = 12,
  B2P_FN_PRESENT_OVER_TIME = 13,
  B2P_FN_ABSENT_OVER_TIME = 14,
  B2P_FN_STDVAR_OVER_TIME = 15,
  B2P_FN_STDDEV_OVER_TIME = 16,
  B2P_FN_DERIV = 17,
  B2P_FN_PREDICT_LINEAR = 18,    /* param0 = t (seconds, i64 in the reference) */
  B2P_FN_QUANTILE_OVER_TIME = 19,/* param0 = phi */
  B2P_FN_HOLT_WINTERS = 20,      /* param0 = sf, param1 = tf */
  B2P_FN__COUNT = 21
};

/* Aggregators of the by-label aggregate (create_aggregate_exprs, planner.rs:2808-2897). */
enum b2p_agg { B2P_AGG_SUM = 0, B2P_AGG_AVG = 1, B2P_AGG_COUNT = 2, B2P_AGG_MIN = 3, B2P_AGG_MAX = 4,
               B2P_AGG_STDDEV = 5, B2P_AGG_STDVAR = 6 };

/* PromQL binary operators (planner.rs:3915-3990): arithmetic on Float64 operands, then the comparisons, which order
 * floats by IEEE 754 totalOrder like arrow-rs' cmp kernels (NaN == NaN, -0.0 < +0.0, +NaN above +inf). */
enum b2p_binop { B2P_OP_ADD = 0, B2P_OP_SUB = 1, B2P_OP_MUL = 2, B2P_OP_DIV = 3, B2P_OP_MOD = 4, B2P_OP_POW = 5,
                 B2P_OP_ATAN2 = 6, B2P_OP_EQ = 7, B2P_OP_NE = 8, B2P_OP_GT = 9, B2P_OP_LT = 10, B2P_OP_GE = 11,
                 B2P_OP_LE = 12 };

/* PromQL instant-vector math functions (planner.rs:2368-2413): element-wise over a node's value column, validity
 * unchanged.  ROUND takes arg0 = to_nearest (0: to an integer); CLAMP takes arg0 = lo, arg1 = hi; CLAMP_MIN takes arg0 = lo
 * (hi = f64::MAX); CLAMP_MAX takes arg0 = hi (lo = -f64::MAX).  The other functions take no argument. */
enum b2p_ifn { B2P_IFN_ABS = 0, B2P_IFN_CEIL = 1, B2P_IFN_FLOOR = 2, B2P_IFN_SQRT = 3, B2P_IFN_EXP = 4, B2P_IFN_LN = 5,
               B2P_IFN_LOG2 = 6, B2P_IFN_LOG10 = 7, B2P_IFN_SIN = 8, B2P_IFN_COS = 9, B2P_IFN_TAN = 10, B2P_IFN_ASIN = 11,
               B2P_IFN_ACOS = 12, B2P_IFN_ATAN = 13, B2P_IFN_SINH = 14, B2P_IFN_COSH = 15, B2P_IFN_TANH = 16,
               B2P_IFN_ASINH = 17, B2P_IFN_ACOSH = 18, B2P_IFN_ATANH = 19, B2P_IFN_ROUND = 20, B2P_IFN_DEG = 21,
               B2P_IFN_RAD = 22, B2P_IFN_SGN = 23, B2P_IFN_CLAMP = 24, B2P_IFN_CLAMP_MIN = 25, B2P_IFN_CLAMP_MAX = 26,
               B2P_IFN__COUNT = 27 /* the math functions above; 27 itself is no function */,
               B2P_IFN_NEG = 28 /* unary minus: the sign bit flipped (-0.0, a NaN's sign), as Rust's f64 Neg */ };

/* Functions of the eval step alone (b2p_step_fn): time() in seconds, and the calendar parts of the UTC millisecond
 * timestamp as DataFusion's date_part gives them (planner.rs:2222-2300, 3994-4009): DAY_OF_WEEK counts from Sunday = 0,
 * DAY_OF_YEAR from 1, DAYS_IN_MONTH is the last day of the step's month. */
enum b2p_step_part { B2P_STEP_TIME = 0, B2P_STEP_MINUTE = 1, B2P_STEP_HOUR = 2, B2P_STEP_DAY_OF_MONTH = 3,
                     B2P_STEP_DAY_OF_WEEK = 4, B2P_STEP_DAY_OF_YEAR = 5, B2P_STEP_MONTH = 6, B2P_STEP_YEAR = 7,
                     B2P_STEP_DAYS_IN_MONTH = 8, B2P_STEP__COUNT = 9 };

/* PromQL set operators; they work per (match key, step) cell and copy cells, never compute values. */
enum b2p_setop { B2P_SET_AND = 0, B2P_SET_OR = 1, B2P_SET_UNLESS = 2 };
#define B2P_NO_KEY 0xFFFFFFFFu /* a row whose labels no row of the other side has */

/* Parameters of the fused sub-plan.  Field-for-field the arguments of
 * RangeManipulate::new(start,end,interval,range,..) (range_manipulate.rs:86-110),
 * SeriesNormalize::new(offset,..,need_filter_out_nan,..) (normalize.rs:66-83) and the UDF scalars. */
typedef struct b2p_range_params {
  int32_t fn_id;      /* enum b2p_fn */
  int32_t filter_nan; /* need_filter_out_nan: 1 for every range selector (planner.rs:1383) */
  int64_t start;      /* ms */
  int64_t end;        /* ms, inclusive */
  int64_t interval;   /* ms, > 0 */
  int64_t range;      /* ms; also prom_rate's range_length argument (planner.rs:2438-2474) */
  int64_t offset;     /* ms, added to every timestamp */
  double param0;
  double param1;
} b2p_range_params;

typedef struct b2p_ctx b2p_ctx;

/* ---- context ------------------------------------------------------------------------- */
B2P_API b2p_ctx* b2p_create(int device);            /* NULL on failure (see b2p_last_error) */
B2P_API void b2p_destroy(b2p_ctx* ctx);
B2P_API const char* b2p_last_error(void);
B2P_API const char* b2p_version(void);
/* Enqueue on an existing cudaStream_t (e.g. the caller's current stream); NULL is the legacy default
 * stream.  b2p_use_own_stream() goes back to the context's private non-blocking stream. */
B2P_API int b2p_set_stream(b2p_ctx* ctx, void* cuda_stream);
B2P_API int b2p_use_own_stream(b2p_ctx* ctx);
/* Wait for the stream, finish slow-path fix-ups, surface deferred errors (B2P_E_UNSORTED, ...). */
B2P_API int b2p_sync(b2p_ctx* ctx);
B2P_API int64_t b2p_num_steps(int64_t start, int64_t end, int64_t interval);
/* Series the last range/instant call routed to the exact slow path, summed over the chunks of a chunked b2p_range_eval
 * and over the tiles of a tiled call (diagnostic; after b2p_sync). */
B2P_API int64_t b2p_last_slow_series(b2p_ctx* ctx);
/* bytes the last b2p_range_eval (host-pointer call) copied host -> device: fewer than 20 B/row when chunks of equally
 * spaced series went over as (offsets, first timestamp, cadence) descriptors instead of their timestamp / id columns */
B2P_API int64_t b2p_last_h2d_bytes(b2p_ctx* ctx);
/* Series the first tier (or the opt-in thread tier) handed to the warp-per-series kernel in the last range call,
 * summed over the chunks of a chunked b2p_range_eval and over the tiles of a tiled call (diagnostic; after b2p_sync). */
B2P_API int64_t b2p_last_warp_tier_series(b2p_ctx* ctx);
/* CUDA-event time (ms) of the kernels of the last *_dev / host call, by stage index:
 * 0 = series_offsets, 1 = range/instant fast kernel, 2 = slow-path kernel, 3 = aggregate /
 * histogram / reduce / binary-operator kernel.  Valid after b2p_sync(). */
B2P_API double b2p_last_kernel_ms(b2p_ctx* ctx, int stage);
/* Kernels launched by this context since creation (the bench's gpu_launches claim). */
B2P_API int64_t b2p_launch_count(b2p_ctx* ctx);

/* ---- device-pointer API (asynchronous) --------------------------------------------------- */
/* SeriesDivide: offsets[s] = the first row whose id is >= s, offsets[n_series] = n_rows.  sid must be 16-byte aligned
 * (B2P_E_INVALID before any launch).  Ids that decrease somewhere, or an id >= n_series, are B2P_E_UNSORTED from the
 * next b2p_sync; the offsets such a column leaves are all 0 (every series empty), so a call queued on them before the
 * verdict, such as b2p_range_eval_dev, reads no row. */
B2P_API int b2p_series_offsets_dev(b2p_ctx* ctx, const uint32_t* sid, uint64_t n_rows, uint32_t n_series,
                           uint64_t* offsets /* [n_series+1] */);
B2P_API int b2p_range_eval_dev(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts, const double* val,
                       const uint64_t* offsets, uint64_t n_rows, uint32_t n_series,
                       double* out /* [n_series*T] */, uint32_t* valid_words /* [n_series*Tw] */);
B2P_API int b2p_range_udf_dev(b2p_ctx* ctx, int32_t fn_id, const int64_t* ts, const double* val, uint64_t n_rows,
                      const int64_t* packed_ranges /* [n_win] offset | len<<32 */,
                      const int64_t* eval_ts /* [n_win] or NULL */, uint64_t n_win, int64_t range_length,
                      double param0, double param1, double* out /* [n_win] */, uint8_t* valid /* [n_win] */);
B2P_API int b2p_instant_select_dev(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                           int64_t offset, const int64_t* ts, const double* val, const uint64_t* offsets,
                           uint64_t n_rows, uint32_t n_series, double* out, uint32_t* valid_words);
/* timestamp(<selector>): the instant selector of b2p_instant_select_dev with the value column replaced by the sample's
 * timestamp, as the reference projects ts / 1000 before InstantManipulate (planner.rs:905-909, 951-965): the chosen
 * row's ts + offset as (double)t / 1000.0.  No value column is read, so there is no stale-NaN test: a selected
 * stale-NaN sample is kept, whatever the table's value type. */
B2P_API int b2p_instant_timestamp_dev(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                      int64_t offset, const int64_t* ts, const uint64_t* offsets, uint64_t n_rows,
                                      uint32_t n_series, double* out, uint32_t* valid_words);
/* Multi-field tables (Influx line protocol / OTLP ingest: cpu(usage_user, usage_system, ..)): one timestamp column and
 * n_fields Float64 value columns over the same rows, 1 <= n_fields <= B2P_MAX_FIELDS.  `vals` and `outs` are HOST
 * arrays of n_fields DEVICE pointers: vals[f] is field f's column [n_rows], outs[f] its grid [n_series*T].  There is
 * one validity bitmap for all fields.
 *
 * b2p_range_eval_fields_dev: the reference's RangeManipulate with field_columns (range_manipulate.rs:70-153), the prom_*
 * UDF projected once per field (planner.rs:2180) and Filter(every field IS NOT NULL) (planner.rs:2774-2791).
 *   - With p->filter_nan, a row in which ANY field is NaN is dropped for every field, as SeriesNormalize's filter over
 *     all Float64 columns does (normalize.rs:415-428).  The union is taken on context copies of the value columns
 *     (8 B per field and row of scratch); the caller's columns are never written.
 *   - The windows come from the timestamps alone; each field runs the range tiers of b2p_range_eval_dev over the same
 *     offsets, and a (series, step) cell is valid only where every field's result is.  A cell whose bit is 0 holds
 *     0.0 or the value its own field computed there.
 *   - The call synchronises once (the slow path's fix-ups must land before the conjunction), then enqueues the
 *     conjunction; call b2p_sync() before reading the results, as for every *_dev call.
 *   - n_fields == 1 is exactly b2p_range_eval_dev.
 * b2p_instant_select_fields_dev: InstantManipulate over every field (instant_manipulate.rs:473-585).  The step's row is
 * chosen once: the lookback search and the stale-NaN test read field 0 only (planner.rs:922), and every field is
 * taken from that row, NaN or not.  n_fields == 1 is exactly b2p_instant_select_dev.
 *
 * NULL slots.  `field_valid` (may be NULL, as may any entry: no NULL slot) is a host array of n_fields DEVICE pointers
 * to each field's Arrow validity bitmap (bit r of byte r/8, 1 = a value), (n_rows + 7) / 8 bytes.  vals[f] holds the
 * field's value buffer as it is, NULL slots included.  The reference reads NULL slots in two ways:
 *   - rate, increase, delta, irate, idelta, resets, changes, last_over_time, quantile_over_time and holt_winters read
 *     the value buffer (`values()`), count / present / absent_over_time only the window's length, and the NaN filter
 *     the buffer value (`value(i)`): the range call reproduces them from vals alone and ignores the bitmaps;
 *   - sum / avg / min / max_over_time (arrow's null-skipping aggregates), stdvar / stddev_over_time (a NULL slot
 *     panics) and deriv / predict_linear (`is_null` skipped, functions.rs:126-144): a range call of these functions
 *     whose bitmaps hold a NULL slot in rows [0, n_rows) is refused with B2P_E_INVALID naming the field.
 * The instant selector exports a NULL slot of the chosen row as a NULL in that field of an emitted row, which one
 * validity bitmap cannot carry: an instant call whose bitmaps hold a NULL slot is refused the same way.  Checking the
 * bitmaps synchronises once; with field_valid NULL nothing is read. */
#define B2P_MAX_FIELDS 64
B2P_API int b2p_range_eval_fields_dev(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts,
                                      const double* const* vals, const uint8_t* const* field_valid,
                                      int32_t n_fields, const uint64_t* offsets,
                                      uint64_t n_rows, uint32_t n_series, double* const* outs, uint32_t* valid_words);
B2P_API int b2p_instant_select_fields_dev(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                          int64_t offset, const int64_t* ts, const double* const* vals,
                                          const uint8_t* const* field_valid, int32_t n_fields,
                                          const uint64_t* offsets, uint64_t n_rows,
                                          uint32_t n_series, double* const* outs, uint32_t* valid_words);
/* gid[s] in [0,n_groups) (or >= n_groups to drop the series).  members_* is scratch-free: the
 * library builds the group->series CSR itself.  out_val/out_cnt are [n_groups*T]; cnt==0 <=> the
 * group has no row at that step.  Partial results of several shards/GPUs combine by adding
 * out_val (SUM/COUNT) and out_cnt — see b2p_group_finalize_dev. */
B2P_API int b2p_group_aggregate_dev(b2p_ctx* ctx, int32_t agg, const double* vals, const uint32_t* valid_words,
                            const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                            double* out_val, uint32_t* out_cnt);
/* group -> member-series index of one gid[] assignment (the by-labels of a query do not change between
 * its batches): built once (radix sort + read-back of the largest group size; synchronises), reused by
 * b2p_group_aggregate_indexed_dev / b2p_range_group_sum_indexed_dev.  Replaces the hash table of string
 * keys DataFusion's AggregateExec builds per input row (planner.rs:334-452, SURVEY.md 8 a10). */
typedef struct b2p_group_index b2p_group_index;
B2P_API int b2p_group_index_create_dev(b2p_ctx* ctx, const uint32_t* gid /* device, [n_series] */, uint32_t n_series,
                               uint32_t n_groups, b2p_group_index** out_index);
B2P_API void b2p_group_index_destroy(b2p_ctx* ctx, b2p_group_index* index);
B2P_API int b2p_group_aggregate_indexed_dev(b2p_ctx* ctx, int32_t agg, const double* vals, const uint32_t* valid_words,
                                    const b2p_group_index* index, uint64_t T, double* out_val, uint32_t* out_cnt);
/* sum by (..)(fn(..)): range function + by-label partial SUM / COUNT of groups [g_lo, g_hi), ADDED into
 * out_sum / out_cnt [n_groups*T] (zero them first; shards, chunks and group ranges chain by accumulation).
 * rate / increase / delta with the first tier's query shape (32-bit time domain, range >= interval, start >= 0)
 * and reasonably balanced groups run FUSED: series are walked group by group, a group's rows of out_sum / out_cnt
 * belong to one warp and are updated in member order — no [n_series*T] intermediate, no atomics on the common
 * path, asynchronous (b2p_range_group_sum_fused() tells).  At most one fused call is outstanding per context: the
 * next range call synchronises first.  Everything else takes two passes through context scratch of
 * n_series*T*8 + n_series*Tw*4 bytes, synchronises in between, and needs the whole group range [0, n_groups). */
B2P_API int b2p_range_group_sum_indexed_dev(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts, const double* val,
                                    const uint64_t* offsets, uint64_t n_rows, uint32_t n_series,
                                    const b2p_group_index* index, uint32_t g_lo, uint32_t g_hi, double* out_sum,
                                    uint32_t* out_cnt);
B2P_API int b2p_range_group_sum_fused(b2p_ctx* ctx, const b2p_range_params* p, const b2p_group_index* index); /* 1/0 */
/* Same with a one-off index built from gid (device, [n_series]); synchronous. */
B2P_API int b2p_range_group_sum_dev(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts, const double* val,
                            const uint64_t* offsets, uint64_t n_rows, uint32_t n_series, const uint32_t* gid,
                            uint32_t n_groups, double* out_sum, uint32_t* out_cnt);
/* Partial state of one rank / shard for a later cross-rank merge: SUM / AVG -> (sum, cnt); COUNT -> cnt;
 * MIN / MAX -> (extreme, cnt); STDDEV / STDVAR -> (cnt, mean in out_mean, M2 in out_val). */
B2P_API int b2p_group_aggregate_partial_dev(b2p_ctx* ctx, int32_t agg, const double* vals, const uint32_t* valid_words,
                                    const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                    double* out_val, uint32_t* out_cnt, double* out_mean /* stddev / stdvar, else NULL */);
/* After the cross-GPU merge: AVG = sum/cnt in place; COUNT = (double)cnt; STDVAR = M2/cnt; STDDEV = sqrt(M2/cnt). */
B2P_API int b2p_group_finalize_dev(b2p_ctx* ctx, int32_t agg, double* val, const uint32_t* cnt, uint64_t n);

/* ---- multi-GPU (one process / context per GPU): NCCL communicator owned by the context ----------------
 * Series are hash-sharded over the ranks (SURVEY.md 8e; the reference hash-partitions on the series key,
 * series_divide.rs:396-408) and the by-label partials merge with one all-reduce, the analogue of the reference's
 * __sum_state (datanode) / __sum_merge (frontend) split, src/query/src/dist_plan/commutativity.rs:85-113, 158-191.
 * libnccl.so.2 is bound with dlopen at the first call (no link dependency; B2P_NCCL_LIB overrides the name).
 * Rank 0 calls b2p_comm_unique_id and ships the B2P_COMM_ID_BYTES to the other ranks by any means (the reference
 * would use its own RPC); every rank then calls b2p_comm_init (collective). */
#define B2P_COMM_ID_BYTES 128
B2P_API int b2p_comm_unique_id(void* out_id, size_t bytes);
B2P_API int b2p_comm_init(b2p_ctx* ctx, const void* id, size_t bytes, int n_ranks, int rank);
B2P_API int b2p_comm_destroy(b2p_ctx* ctx);
/* In-place merge of every rank's partials [n] on the context's stream (asynchronous): SUM / AVG / COUNT add val and
 * cnt; MIN / MAX reduce val with min / max in the f64::total_cmp order of the single-pass aggregate (+NaN greatest,
 * -NaN least, -0.0 < +0.0; groups absent on a rank are neutral) and add cnt; STDDEV / STDVAR merge
 * the (cnt, mean, M2 = val) states.  A context without communicator and n_ranks == 1 returns at once. */
B2P_API int b2p_allreduce_partials_dev(b2p_ctx* ctx, int32_t agg, double* val, uint32_t* cnt, double* mean, uint64_t n);
/* Wide avg_over_time (config 5): per-column (sum, count) of every rank added in place. */
B2P_API int b2p_allreduce_columns_dev(b2p_ctx* ctx, double* sum, uint64_t* cnt, uint32_t n_cols);
/* Int64 partials of SUM / MIN / MAX (any other aggregator is B2P_E_INVALID): exactly b2p_group_aggregate_i64_dev's output
 * (K3's Int64 fold: wrapping sum, signed min / max; int64_t bits in out_val, 0 where cnt is 0), which is already the
 * state another rank's partial merges with. */
B2P_API int b2p_group_aggregate_partial_i64_dev(b2p_ctx* ctx, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                                                const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                                double* out_val, uint32_t* out_cnt);
/* In-place merge of every rank's Int64 partials [n] (asynchronous): SUM adds the bits as uint64 (ncclSum; modular
 * addition is the wrapping sum whatever the rank order), MIN / MAX reduce them as int64 (ncclMin / ncclMax) after a
 * group absent on a rank took INT64_MAX / INT64_MIN, and a group absent everywhere reads 0; cnt is added.  Without a
 * communicator and n_ranks == 1 it returns at once. */
B2P_API int b2p_allreduce_partials_i64_dev(b2p_ctx* ctx, int32_t agg, double* val, uint32_t* cnt, uint64_t n);
/* The number of ranks of the context's communicator (0 without one) and, in *rank (may be NULL), this rank (0 without
 * one).  No device work. */
B2P_API int32_t b2p_comm_ranks(b2p_ctx* ctx, int32_t* rank);
/* Host-pointer forms of the sharded by-label aggregate, what a sharded plan node runs: this rank's rows (vals / valid /
 * gid as for b2p_group_aggregate, gid over the n_groups GLOBAL group ids, any rank may have no row) become its partials
 * (b2p_group_aggregate_partial_dev / _i64_dev), every rank's are merged (b2p_allreduce_partials_dev / _i64_dev) and
 * finalised (b2p_group_finalize_dev); out_val / out_cnt [n_groups x T] come back as b2p_group_aggregate writes them over
 * the union of the ranks' rows.  Float64: every aggregator; Int64: sum, min and max.  Collective: every rank calls with
 * the same agg, n_groups and T.  Synchronous. */
B2P_API int b2p_group_aggregate_allreduce(b2p_ctx* ctx, int32_t agg, const double* vals, const uint32_t* valid_words,
                                          const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                          double* out_val, uint32_t* out_cnt);
B2P_API int b2p_group_aggregate_allreduce_i64(b2p_ctx* ctx, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                                              const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                              double* out_val, uint32_t* out_cnt);
/* The group-label agreement's exchange of exact bytes (the plan layer's sharded nodes; the blocks are
 * b2p_group_keys_merge's).  b2p_group_keys_sizes: this rank's block size `bytes`; one ncclAllGather of the 8-byte sizes
 * fills the HOST array sizes [n_ranks] (row r: rank r), the same on every rank; without a communicator sizes[0] = bytes.
 * b2p_group_keys_allgather: every rank's block, back to back in rank order, into the HOST buffer out (sum of sizes
 * bytes): this rank's block goes to its place in one device buffer, then one ncclBroadcast per rank with bytes, in one
 * NCCL group (no block is padded).  b2p_last_group_keys_bytes() then gives this rank's block bytes (the all-gather of
 * the sizes adds 8 B per rank).  Both synchronise the stream. */
B2P_API int b2p_group_keys_sizes(b2p_ctx* ctx, uint64_t bytes, uint64_t* sizes);
B2P_API int b2p_group_keys_allgather(b2p_ctx* ctx, const void* block, const uint64_t* sizes, void* out);
B2P_API int64_t b2p_last_group_keys_bytes(b2p_ctx* ctx);
/* sum by (..)(fn(..)) over ALL ranks: this rank's fused partials, computed in n_tiles group ranges; each range's rows
 * of out_sum / out_cnt are all-reduced on a high-priority communication stream as soon as they are complete, while
 * the next range computes (kernel time of the last tile's all-reduce: b2p_last_kernel_ms(ctx, 4)).  On return
 * (stream order) out_sum / out_cnt hold the merged partials on every rank. */
B2P_API int b2p_range_group_sum_allreduce_dev(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts,
                                      const double* val, const uint64_t* offsets, uint64_t n_rows, uint32_t n_series,
                                      const b2p_group_index* index, int32_t n_tiles, double* out_sum, uint32_t* out_cnt);
/* rates is the dense matrix of n_hist*n_buckets series (bucket b of histogram h = series
 * h*n_buckets+b, le ascending, last = +Inf).  out [n_hist*T], out_valid_words [n_hist*Tw]. */
B2P_API int b2p_histogram_quantile_dev(b2p_ctx* ctx, double phi, const double* le, uint32_t n_buckets,
                               const double* rates, const uint32_t* valid_words, uint32_t n_hist, uint64_t T,
                               double* out, uint32_t* out_valid_words);
/* HistogramFold over an explicit index (device pointers): histogram h owns buckets hist_off[h] .. hist_off[h+1] of
 * bucket_series / bucket_le, in ascending le order (NaN bounds last); layouts may differ between histograms.  Per
 * (histogram, step) the buckets that have a sample at that step are folded like the reference's safe mode
 * (histogram_fold.rs:834-846, 930-981): none -> no row; fewer than two or no +Inf bound last -> NaN; else
 * evaluate_row (:1046-1118).  b2p_histogram_quantile_dev is the uniform-layout front end of the same kernel. */
B2P_API int b2p_histogram_fold_dev(b2p_ctx* ctx, double phi, const uint32_t* hist_off, const uint32_t* bucket_series,
                           const double* bucket_le, uint32_t n_hist, const double* rates, const uint32_t* valid_words,
                           uint64_t T, double* out, uint32_t* out_valid_words);
/* cols: n_cols column pointers (device array of device pointers), each n_rows f64; NaN rows are
 * skipped (SeriesNormalize filter).  out_sum[n_cols], out_cnt[n_cols] accumulate. */
B2P_API int b2p_column_reduce_dev(b2p_ctx* ctx, const double* const* cols, uint32_t n_cols, uint64_t n_rows,
                          double* out_sum, uint64_t* out_cnt);

/* Binary operator over two dense grids matched into pairs: for pair p and step k, lhs[lhs_row[p]*T + k] op
 * rhs[rhs_row[p]*T + k] -> out[p*T + k], out_valid [n_pairs*Tw].  A cell is valid iff both operands are; a comparison
 * without `bool` (return_bool == 0) also drops the cells where it is false and keeps the lhs value; with `bool` the
 * value is 1.0 / 0.0.  Invalid cells hold 0.0.  Pairs may come in any order and repeat rows (group_left / right).
 * B2P_E_INVALID: unknown op, return_bool on an arithmetic op; a row index >= n_lhs_rows / n_rhs_rows is found on the
 * device (that pair's cells are written invalid) and reported by b2p_sync. */
B2P_API int b2p_binary_op_dev(b2p_ctx* ctx, int32_t op /* enum b2p_binop */, int32_t return_bool, const double* lhs,
                              const uint32_t* lhs_valid, const uint32_t* lhs_row /* [n_pairs] */, uint32_t n_lhs_rows,
                              const double* rhs, const uint32_t* rhs_valid, const uint32_t* rhs_row /* [n_pairs] */,
                              uint32_t n_rhs_rows, uint64_t n_pairs, uint64_t T, double* out, uint32_t* out_valid);
/* One grid against a number: `scalar op vals` (scalar_on_left) or `vals op scalar`; a filtering comparison keeps the
 * vector's value.  out / out_valid may be vals / valid (in place). */
B2P_API int b2p_scalar_op_dev(b2p_ctx* ctx, int32_t op, int32_t return_bool, int32_t scalar_on_left, double scalar,
                              const double* vals, const uint32_t* valid, uint64_t n_rows, uint64_t T, double* out,
                              uint32_t* out_valid);
/* cnt [n_rows*T] of a by-label aggregate (0 <=> no row) -> valid_words [n_rows*Tw], so that a finalized aggregate
 * feeds b2p_binary_op_dev without a host round trip. */
B2P_API int b2p_count_valid_words_dev(b2p_ctx* ctx, const uint32_t* cnt, uint64_t n_rows, uint64_t T,
                                      uint32_t* valid_words);

/* Set operator over two dense grids whose rows carry dense match-key ids (the caller matches the labels, as for
 * b2p_binary_op; lhs_key / rhs_key [rows] in [0, n_keys) or B2P_NO_KEY).  Per step k:
 *   and:    lhs row r keeps its cell iff some rhs row with the same key has a cell at k; B2P_NO_KEY rows keep nothing
 *   unless: lhs row r keeps its cell iff no rhs row with the same key has one; B2P_NO_KEY rows keep every cell
 *   or:     every lhs cell; an rhs cell iff no lhs row and no EARLIER rhs row (row order) with the same key has one;
 *           B2P_NO_KEY rhs rows keep every cell
 * and / unless: out [n_lhs_rows x T], out_valid [n_lhs_rows x Tw]; out / out_valid may be lhs / lhs_valid (in place);
 * rhs (the values) is not read and may be NULL.  or: out [(n_lhs_rows + n_rhs_rows) x T] = the lhs rows, then the rhs
 * rows; out_valid likewise; out must not overlap the inputs.  A kept cell is a bit copy of the input (NaN payloads,
 * -0.0); every other cell is 0.0.  The library groups the rows by key itself.  B2P_E_INVALID: unknown op; a key
 * >= n_keys other than B2P_NO_KEY is found on the device (that row is written invalid) and reported by b2p_sync. */
B2P_API int b2p_setop_dev(b2p_ctx* ctx, int32_t op /* enum b2p_setop */, const double* lhs, const uint32_t* lhs_valid,
                          const uint32_t* lhs_key, uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid,
                          const uint32_t* rhs_key, uint32_t n_rhs_rows, uint32_t n_keys, uint64_t T, double* out,
                          uint32_t* out_valid);

/* Instant-vector function `fn` (enum b2p_ifn) over a dense grid: out[r*T + k] = fn(vals[r*T + k]) where the validity
 * bit is set, 0.0 elsewhere; out_valid = valid (copied when out_valid != valid).  out / out_valid may be vals / valid
 * (in place).  abs ceil floor sqrt round deg rad sgn clamp* are bit-identical to the reference's Rust; the
 * transcendental functions are CUDA's, within the ulp bound DESIGN.md section 2 states.  B2P_E_INVALID: unknown fn;
 * a clamp bound pair with lo > hi (clamp_min(v, +inf) and clamp_max(v, -inf) included). */
B2P_API int b2p_instant_fn_dev(b2p_ctx* ctx, int32_t fn /* enum b2p_ifn */, double arg0, double arg1, const double* vals,
                               const uint32_t* valid, uint64_t n_rows, uint64_t T, double* out, uint32_t* out_valid);
/* K19: a function of the eval step (enum b2p_step_part) at every valid cell of a dense grid: out[r*T + k] =
 * f(eval_ts[k]) where bit k of row r is set, 0.0 elsewhere; valid is read, never written.  TIME is (double)ts / 1000.0
 * (one IEEE division, as build_special_time_expr, empty_metric.rs:393-402); the calendar parts are integers in Float64
 * cells, proleptic Gregorian in UTC, negative epochs included.  A step whose year is outside [-262143, 262143] (chrono's
 * date range) is written 0.0 and found on the device: B2P_E_INVALID from b2p_sync.  eval_ts [T] is a device array.
 * B2P_E_INVALID: an unknown part, a NULL argument. */
B2P_API int b2p_step_fn_dev(b2p_ctx* ctx, int32_t part /* enum b2p_step_part */, const int64_t* eval_ts,
                            const uint32_t* valid, uint64_t n_rows, uint64_t T, double* out);
/* scalar(v), the reference's ScalarCalculate (scalar_calculate.rs:532-637), over the whole grid: row_key[r] is a dense
 * series id (< n_rows) or B2P_NO_KEY for a row whose labels include a NULL.  When every row with a cell carries one key
 * (a B2P_NO_KEY row: only while it has exactly one cell), out [T] / out_valid [Tw] are that series' cells, bit copies;
 * otherwise (no cells, or two or more series) out is NaN at every step with every bit valid.  Two rows of one key with
 * a cell at the same step, or a key >= n_rows other than B2P_NO_KEY, are found on the device (B2P_E_INVALID from
 * b2p_sync).  No host round trip between the two passes. */
B2P_API int b2p_scalar_calculate_dev(b2p_ctx* ctx, const double* vals, const uint32_t* valid, const uint32_t* row_key,
                                     uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid);
/* absent(v) (K15), the reference's AbsentStream (absent.rs) over the grid of its child: the steps at which no row has a
 * valid cell.  out_valid [Tw] word w = ~(OR over rows of valid[r * Tw + w]) with the bits past T cleared, and out [T]
 * = 1.0 where that bit is set, 0.0 elsewhere.  A valid cell counts whatever its value (NaN included); the values are
 * never read, only the validity words (bits past T in a row's last word are ignored).  No rows: every step is set.
 * Asynchronous: no host round trip; scratch is 4 B per output word from the context.  valid may be NULL only when
 * n_rows == 0, out / out_valid only when T == 0.  B2P_E_INVALID: a NULL argument; B2P_E_TOO_LARGE: T > 32 * (2^32 - 1). */
B2P_API int b2p_absent_dev(b2p_ctx* ctx, const uint32_t* valid, uint32_t n_rows, uint64_t T, double* out,
                           uint32_t* out_valid);

/* topk(k, v) / bottomk(k, v) per (group, step) over a dense grid whose rows are grouped by `index` (a row whose group id
 * is >= n_groups belongs to no group and keeps nothing).  A cell's rank key is (value in the f64 total order, tie[row]),
 * compared descending for topk (bottom == 0) and ascending for bottomk; tie [rows] must be distinct per row (the caller
 * derives it from the label tuples in the direction of the op, b2p_plan.cpp), so the order is strict and the result
 * deterministic.  The ranks kept follow the reference's Filter(row_number <= k) on Float64: floor(k) for finite k >= 1,
 * none for k < 1, -inf and -NaN, all for +inf and +NaN.  Per (group, step) exactly the min(kept ranks, valid cells) best
 * cells keep their bit.  Only out_valid [rows x Tw] is written (bits at or past T are 0); it may be valid (in place).
 * vals is never written: topk is a filter, and every consumer reads a cell only where its bit is set.  Scratch comes
 * from the context and is bounded (b2p_aggregation.cu, topk_run).  B2P_E_INVALID: a NULL argument. */
B2P_API int b2p_topk_dev(b2p_ctx* ctx, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                         const b2p_group_index* index, const uint32_t* tie, uint64_t T, uint32_t* out_valid);

/* topk / bottomk over rows sharded across ranks (Float64 only).  Every rank passes its own rows as for b2p_topk_dev: its
 * index over the same n_groups global group ids, and tie values distinct across ALL ranks (the row's global ordinal in
 * the op's direction, derived from the label tuples by the caller); each series lies whole on one rank.  On return (stream
 * order) out_valid holds this rank's kept cells, and the union over the ranks is bit for bit what b2p_topk_dev writes
 * over the concatenation of every rank's rows with the same gid and tie.
 *
 * kk is the rank count of b2p_topk_dev's k.  From the global member count of each group: kk = 0 keeps nothing, kk >= the
 * largest group keeps every valid cell, and otherwise a group of at most kk members keeps every valid cell and the
 * others (G_x groups, "exchanged") are exchanged.  Per (exchanged group, step) and round, each rank sends its best
 * slots = min(kk, 32) keys (f64 total-order key and tie, 12 B) below the previous round's bound plus a 4-byte count; a
 * merge over the ranks' blocks finds the kk-th best key, and each rank keeps its own cells at or above it: the global
 * top kk of a group are among the union of each rank's own top kk.  kk <= 32 takes one round and marks the kept cells
 * from the rank's own candidates; kk > 32 takes ceil(kk / 32) rounds and then reads the values once more.
 * The (exchanged group, 32-step tile) units are cut into batches whose blocks and state fit the context's cap
 * (128 MB; B2P_TOPK_EXCHANGE_BYTES at b2p_create, which must be the same on every rank).
 *
 * b2p_topk_allgather_dev: the whole call over the context's communicator: one all-reduce of the n_groups x 4 B member
 * counts and one read-back of them (synchronises once), then per batch and round three ncclAllGather calls in one group.
 * Without a communicator and n_ranks == 1 (no b2p_comm_init) it gives b2p_topk_dev's words.  b2p_last_exchange_bytes()
 * then gives the bytes of this rank's candidate blocks:
 *     rounds x G_x x 32 ceil(T / 32) x (12 slots + 4),
 * 0 when no group has more than kk members globally (the all-reduce of the counts is not included).
 *
 * The steps it is built from, so that one GPU can run R ranks (one context each) through the same kernels.  group_sizes
 * is a HOST array of the n_groups global member counts; every step derives the same exchange from (k, group_sizes, T,
 * n_ranks).  b2p_topk_shard_plan gives n_batches, n_rounds (0 without exchanged groups), slots, and the largest block
 * and state of a batch in bytes (0 without exchanged groups).  Then, for every batch b and round r < n_rounds:
 *   b2p_topk_shard_candidates_dev on every rank writes its block (block_bytes of b2p_topk_shard_plan suffice; the
 *     batch's own size is nx x nt x 32 x (12 slots + 4) for its nx groups and nt tiles): three sections, keys hi
 *     [u x slots x 32] u64, ties [u x slots x 32] u32, counts [u x 32] u32 for u = nx x nt units; reads state after
 *     round 0;
 *   the blocks are gathered section by section: [hi of rank 0 .. R-1][ties of rank 0 .. R-1][counts of rank 0 .. R-1];
 *   b2p_topk_shard_merge_dev over the gathered blocks writes the batch's state (state_bytes, device);
 * and b2p_topk_shard_mark_dev(b) on every rank writes its words of batch b from that state; batch 0 also writes every
 * word the exchange does not decide.  A rank's mark must follow its own last candidates step of the batch on the same
 * context (its candidate lists stay in context scratch), before the next batch's. */
B2P_API int b2p_topk_allgather_dev(b2p_ctx* ctx, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                                   const b2p_group_index* index, const uint32_t* tie, uint64_t T, uint32_t* out_valid);
B2P_API int64_t b2p_last_exchange_bytes(b2p_ctx* ctx);
B2P_API int b2p_topk_shard_plan(b2p_ctx* ctx, double k, const uint32_t* group_sizes, uint32_t n_groups, uint64_t T,
                                int32_t n_ranks, uint32_t* n_batches, uint32_t* n_rounds, uint32_t* slots,
                                uint64_t* block_bytes, uint64_t* state_bytes);
B2P_API int b2p_topk_shard_candidates_dev(b2p_ctx* ctx, int32_t bottom, double k, const double* vals,
                                          const uint32_t* valid, const b2p_group_index* index, const uint32_t* tie,
                                          uint64_t T, const uint32_t* group_sizes, int32_t n_ranks, uint32_t batch,
                                          uint32_t round, void* state, void* block);
B2P_API int b2p_topk_shard_merge_dev(b2p_ctx* ctx, double k, const uint32_t* group_sizes, uint32_t n_groups,
                                     uint64_t T, int32_t n_ranks, uint32_t batch, uint32_t round, const void* blocks,
                                     void* state);
B2P_API int b2p_topk_shard_mark_dev(b2p_ctx* ctx, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                                    const b2p_group_index* index, const uint32_t* tie, uint64_t T,
                                    const uint32_t* group_sizes, int32_t n_ranks, uint32_t batch, const void* state,
                                    uint32_t* out_valid);

/* quantile(phi, v) by label (K11, QuantileAccumulator::evaluate, src/promql/src/functions/quantile_aggr.rs:110-116 over
 * quantile_with_scratch, quantile.rs:201-225): per (group, step) the n valid cells of the index's member rows; phi NaN
 * gives NaN, phi < 0 -inf, phi > 1 +inf; otherwise, sorted by f64::total_cmp, rank = phi (n - 1), lo = floor(rank),
 * hi = min(n - 1, lo + 1), w = rank - floor(rank) and the result s[lo] (1 - w) + s[hi] w, evaluated as written (so
 * quantile(0, {1, +inf}) is NaN).  Output out_val / out_cnt [n_groups x T] as b2p_group_aggregate_dev: out_cnt = n, and
 * n = 0 (value 0.0) is "no row".  Rows of the index's gid >= n_groups take part in nothing.  Deterministic; scratch
 * comes from the context and is bounded (b2p_aggregation.cu, quantile_run).  B2P_E_INVALID: a NULL argument. */
B2P_API int b2p_group_quantile_dev(b2p_ctx* ctx, double phi, const double* vals, const uint32_t* valid,
                                   const b2p_group_index* index, uint64_t T, double* out_val, uint32_t* out_cnt);

/* quantile(phi, v) by label over rows sharded across ranks (Float64 only).  Every rank passes its own rows as for
 * b2p_group_quantile_dev, with an index over the same n_groups global group ids; each series lies whole on one rank.  On
 * return (stream order) EVERY rank's out_val / out_cnt [n_groups x T] holds the full result, bit for bit what
 * b2p_group_quantile_dev writes over the concatenation of every rank's rows.
 *
 * The select is K11's radix select on the 64-bit total-order key with 4-bit digits (16 bins).  Per pass each rank
 * histograms the next digit of its keys under the current prefix into a block, the blocks are added (integer counts,
 * so in any order), and every rank advances the same state from the merged counts: the rows never move.  The extreme
 * pass merges the largest key under p_lo (MAX) and the smallest under p_hi (MIN).  A (group, step) is done after at most
 * 17 passes (16 digits and the extreme pass); phi outside [0, 1] or NaN after one (the count).  Per (group, 32-step tile)
 * unit and pass the block is 2 560 B: counts [16 x 32] u32, then r_lo [32] u64, then r_hi [32] u64, each section
 * unit-major over the batch.  The units are cut into batches whose block and state (1 792 B per unit) fit the context's
 * exchange cap (128 MB; B2P_TOPK_EXCHANGE_BYTES at b2p_create, which also bounds the sharded topk's exchange and must be
 * the same on every rank).
 *
 * b2p_quantile_allreduce_dev: the whole call over the context's communicator: per batch and pass, the rank's block, one
 * ncclGroupStart/End of three in-place ncclAllReduce calls (counts u32 SUM, r_lo u64 MAX, r_hi u64 MIN) and the
 * advance, which reads back the count of unfinished cells (so each pass synchronises once).  A batch stops after the
 * pass that leaves none; that count comes from the merged state alone, so every rank makes the same collective calls.
 * Without a communicator and n_ranks == 1 (no b2p_comm_init) it gives b2p_group_quantile_dev's output.
 * b2p_last_exchange_bytes() then gives the bytes of this rank's blocks: sum over batches of passes run x units x 2 560.
 *
 * The steps it is built from, so that one GPU can run R ranks (one context each) through the same kernels.
 * b2p_quantile_shard_plan gives n_batches (0 when n_groups or T is 0) and the largest block and state of a batch in
 * bytes.  Then for every batch b and pass p = 0, 1, .. < 17:
 *   b2p_quantile_shard_pass_dev on every rank zeroes its block (the batch's block is units x 2 560 B, at most
 *     block_bytes) and adds this rank's counts or extremes of the pass into it; pass 0 first clears the batch's
 *     selection state, which the context keeps;
 *   b2p_quantile_shard_advance_dev on every rank merges the n_blocks blocks laid one after another (each the batch's
 *     block size; one all-reduced block, or every rank's block in any order), advances its context's state, writes the
 *     cells it finishes into out_val / out_cnt and returns in *live (host) the count of cells still unfinished; it
 *     synchronises the stream.  The batch is done after the pass whose live is 0.
 * A rank's pass must follow its own previous advance on the same context.  B2P_E_INVALID: a NULL argument, a batch or
 * pass out of range, n_blocks 0, an advance before its batch's pass 0 on the context, no communicator with n_ranks > 1. */
B2P_API int b2p_quantile_allreduce_dev(b2p_ctx* ctx, double phi, const double* vals, const uint32_t* valid,
                                       const b2p_group_index* index, uint64_t T, double* out_val, uint32_t* out_cnt);
/* Host-pointer form of b2p_quantile_allreduce_dev (vals / valid / gid as for b2p_group_quantile, gid over the n_groups
 * global group ids): what a sharded quantile plan node runs.  Synchronous. */
B2P_API int b2p_quantile_allreduce(b2p_ctx* ctx, double phi, const double* vals, const uint32_t* valid,
                                   const uint32_t* gid, uint32_t n_rows, uint32_t n_groups, uint64_t T, double* out_val,
                                   uint32_t* out_cnt);
/* Host-pointer form of the sharded count_values (vals / valid / gid as for b2p_count_values, gid over the n_groups global
 * group ids): what a sharded count_values plan node runs.  b2p_count_values_dev (_i64_dev) over this rank's rows, the
 * heights table of b2p_count_values_shard_heights_dev, then b2p_count_values_allgather_dev (_i64_dev).  out_goff
 * [n_groups + 1] (host) receives the merged rows' offsets, the same on every rank; out_val / out_cnt receive
 * [out_goff[n_groups] x T] rows, which must fit cap_rows (B2P_E_TOO_LARGE otherwise; every rank decides alike when every
 * rank passes the same cap, e.g. the rows of all ranks).  Collective; synchronous. */
B2P_API int b2p_count_values_allgather(b2p_ctx* ctx, const double* vals, const uint32_t* valid, const uint32_t* gid,
                                       uint32_t n_rows, uint32_t n_groups, uint64_t T, uint64_t cap_rows,
                                       uint32_t* out_goff, double* out_val, uint32_t* out_cnt);
B2P_API int b2p_count_values_allgather_i64(b2p_ctx* ctx, const int64_t* vals, const uint32_t* valid, const uint32_t* gid,
                                           uint32_t n_rows, uint32_t n_groups, uint64_t T, uint64_t cap_rows,
                                           uint32_t* out_goff, int64_t* out_val, uint32_t* out_cnt);
B2P_API int b2p_quantile_shard_plan(b2p_ctx* ctx, uint32_t n_groups, uint64_t T, uint32_t* n_batches,
                                    uint64_t* block_bytes, uint64_t* state_bytes);
B2P_API int b2p_quantile_shard_pass_dev(b2p_ctx* ctx, double phi, const double* vals, const uint32_t* valid,
                                        const b2p_group_index* index, uint64_t T, uint32_t batch, uint32_t pass,
                                        void* block);
B2P_API int b2p_quantile_shard_advance_dev(b2p_ctx* ctx, double phi, uint32_t n_groups, uint64_t T, uint32_t batch,
                                           uint32_t pass, const void* blocks, uint32_t n_blocks, double* out_val,
                                           uint32_t* out_cnt, uint64_t* live);

/* count_values(label, v) by label (K12; the reference's Aggregate(groupBy = [group labels.., ts, value], count(value)),
 * planner.rs:402-445): per (group, step) the distinct values of the valid cells of the index's member rows, a value
 * being its bits (-0.0 and +0.0 are two values, and so are NaNs with different bits), in the f64 total order.  Output
 * out_val (f64) / out_cnt (u32) [n_series x T] with rows in the index's member order (a group's rows ordered by row
 * index, the groups by id; rows of gid >= n_groups last): at step k, the group's j-th row holds its j-th smallest
 * distinct value and how many of its cells have it; out_cnt 0 (value 0.0) past the last, and on every row of
 * gid >= n_groups.  Exact and deterministic; scratch comes from the context and is bounded (b2p_aggregation.cu,
 * count_values_run).  B2P_E_INVALID: a NULL argument; B2P_E_TOO_LARGE: a group of more than 67 M members. */
B2P_API int b2p_count_values_dev(b2p_ctx* ctx, const double* vals, const uint32_t* valid, const b2p_group_index* index,
                                 uint64_t T, double* out_val, uint32_t* out_cnt);

/* count_values(label, v) by label over rows sharded across ranks.  Every rank first runs b2p_count_values_dev (or
 * b2p_count_values_i64_dev) over its own rows, with an index over the same n_groups global group ids; each series lies
 * whole on one rank.  That output, local_val / local_cnt [n_rows x T] in the index's member order, is the input here:
 * per (group, step) it is already the rank's distinct values ascending with their multiplicities, and the global
 * answer is the union of the ranks' lists with the counts of equal values added (integer sums: the same bits on every
 * rank whatever the order of the blocks).  No row moves.
 *
 * b2p_count_values_shard_heights_dev: h_r(g), the number of leading rows of group g that have a count at some step
 * (the most distinct values g has at one step on this rank), into the HOST array heights.  With a communicator one
 * ncclAllGather of the n_groups x 4 B vector fills heights [n_ranks x n_groups] (row r: rank r), the same table on every
 * rank; without one (n_ranks == 1) it writes [n_groups].  Reads the table back, so it synchronises the stream.  Group g
 * then has U_g = sum over ranks of h_r(g) output rows (at most its global member count) from out_goff[g] =
 * sum over g' < g of U_g'; the caller sizes out_val / out_cnt [out_goff[n_groups] x T] from the table.
 *
 * b2p_count_values_allgather_dev / _i64_dev: the whole call over the context's communicator.  On return (stream order)
 * every rank's row out_goff[g] + j is bit for bit row goff[g] + j of b2p_count_values_dev (_i64_dev) over the
 * concatenation of every rank's rows with the same gid, j < U_g; count 0 and value 0 past the step's distinct values.
 * Per batch of whole groups over a window of steps each rank packs the first h_r(g) rows of each of its groups as
 * (key u64, count u32) entries, (group, step)-segment-major, padded to the batch's largest rank block (known to every
 * rank from heights), two ncclAllGather calls in one group (keys, counts) gather the blocks, and the merge sorts each
 * (group, step) segment's sum over ranks of h_r(g) entries by key (CUB's segmented sort of pairs) and writes each run
 * of equal keys with the sum of its counts.  A cell past a rank's distinct values is packed as the largest key with
 * count 0; a run whose counts add up to 0 is no value, so the largest positive NaN (or INT64_MAX), whose key is the
 * same, is counted wherever it sorts.  Batches fit the context's exchange cap with their merge scratch (128 MB;
 * B2P_TOPK_EXCHANGE_BYTES at b2p_create, which also bounds the sharded topk's and quantile's exchanges and must be the
 * same on every rank); a group too large for the cap alone is a batch of its own over 32 steps.
 * b2p_last_exchange_bytes() then gives the bytes of this rank's blocks: sum over batches of W_b x (the largest over
 * ranks of the batch's summed h_r(g)) x 12.  Without a communicator and n_ranks == 1 (no b2p_comm_init) the output is
 * the first U_g rows of each group of b2p_count_values_dev.
 *
 * The steps it is built from, so that one GPU can run R ranks (one context each) through the same kernels; heights is
 * the HOST table [n_ranks x n_groups], and every step derives the same batches from (heights, n_ranks, n_groups, T, the
 * cap); no state is kept in the context between calls.  b2p_count_values_shard_plan gives n_batches (0 when no group
 * has a value) and the largest rank block in bytes.  Then for every batch b:
 *   b2p_count_values_shard_pack_dev (_i64_dev) on every rank writes its block, [keys: P u64][counts: P u32] for the
 *     batch's P entries per rank (P x 12 B, at most block_bytes); entries past the rank's own are not written;
 *   the blocks are gathered section by section: [keys of rank 0 .. R-1][counts of rank 0 .. R-1];
 *   b2p_count_values_shard_merge_dev (_i64_dev) over the gathered blocks writes the batch's rows of out_val / out_cnt.
 * B2P_E_INVALID: a NULL argument, a batch out of range, n_ranks > 1 without a communicator in the composed call, a row
 * of heights for this rank (the composed call's, or pack's `rank`) above its own member count of a group;
 * B2P_E_TOO_LARGE: a group or batch too large for CUB's int sizes. */
B2P_API int b2p_count_values_shard_heights_dev(b2p_ctx* ctx, const uint32_t* local_cnt, const b2p_group_index* index,
                                               uint64_t T, uint32_t* heights);
B2P_API int b2p_count_values_allgather_dev(b2p_ctx* ctx, const double* local_val, const uint32_t* local_cnt,
                                           const b2p_group_index* index, uint64_t T, const uint32_t* heights,
                                           double* out_val, uint32_t* out_cnt);
B2P_API int b2p_count_values_allgather_i64_dev(b2p_ctx* ctx, const int64_t* local_val, const uint32_t* local_cnt,
                                               const b2p_group_index* index, uint64_t T, const uint32_t* heights,
                                               int64_t* out_val, uint32_t* out_cnt);
B2P_API int b2p_count_values_shard_plan(b2p_ctx* ctx, const uint32_t* heights, int32_t n_ranks, uint32_t n_groups,
                                        uint64_t T, uint32_t* n_batches, uint64_t* block_bytes);
B2P_API int b2p_count_values_shard_pack_dev(b2p_ctx* ctx, const double* local_val, const uint32_t* local_cnt,
                                            const b2p_group_index* index, uint64_t T, const uint32_t* heights,
                                            int32_t n_ranks, int32_t rank, uint32_t batch, void* block);
B2P_API int b2p_count_values_shard_pack_i64_dev(b2p_ctx* ctx, const int64_t* local_val, const uint32_t* local_cnt,
                                                const b2p_group_index* index, uint64_t T, const uint32_t* heights,
                                                int32_t n_ranks, int32_t rank, uint32_t batch, void* block);
B2P_API int b2p_count_values_shard_merge_dev(b2p_ctx* ctx, const uint32_t* heights, int32_t n_ranks,
                                             uint32_t n_groups, uint64_t T, uint32_t batch, const void* blocks,
                                             double* out_val, uint32_t* out_cnt);
B2P_API int b2p_count_values_shard_merge_i64_dev(b2p_ctx* ctx, const uint32_t* heights, int32_t n_ranks,
                                                 uint32_t n_groups, uint64_t T, uint32_t batch, const void* blocks,
                                                 int64_t* out_val, uint32_t* out_cnt);

/* Subquery fn(<expr>[range:step]) (K13; RangeManipulate(start, end, interval, range) directly over the inner plan,
 * prom_subquery_expr_to_plan, planner.rs:292-332): vals / valid [n_rows x T_inner] are a child's grid on the inner steps
 * inner_start + k * inner_interval (the reference plans them from start - range + inner_interval to end).  Every valid
 * cell of a row is one sample of that row's series, its value a bit copy (no SeriesNormalize: NaN is a sample); p gives
 * the outer grid (start, end, interval), the range, fn_id and param0 / param1 as for b2p_range_eval_dev, whose tiers
 * evaluate the windows over those samples.  Output out [n_rows x T] / out_valid [n_rows x Tw] on the outer grid, row for
 * row, exactly as b2p_range_eval_dev over the same samples.  Each row is one series: the reference's RangeManipulate
 * windows each input batch as one series (range_manipulate.rs:603-630), which is the row's series whenever the child
 * hands it one series per batch.  Scratch comes from the context (16 B per grid cell of a batch of rows, b2p_range.cu,
 * subquery_run); a grid of more than one batch waits for each batch's range call before the next.
 * B2P_E_INVALID: an unknown fn_id, a non-positive interval or inner_interval, a zero range, a non-zero offset or
 * filter_nan, a NULL argument. */
B2P_API int b2p_subquery_dev(b2p_ctx* ctx, const b2p_range_params* p, int64_t inner_start, int64_t inner_interval,
                             const double* vals, const uint32_t* valid, uint32_t n_rows, uint64_t T_inner, double* out,
                             uint32_t* out_valid);

/* sort / sort_desc (K14; the reference's Sort(value ASC | DESC, NULLS FIRST) over the child's rows, planner.rs:1060-1089):
 * the valid cells of vals / valid [n_rows x T] (bits past T in a row's last word are ignored) as cell indices
 * row * T + k into out_cells, ordered by value in the f64 total order (-NaN < -inf < .. < -0.0 < +0.0 < .. < +inf <
 * +NaN), ascending, or descending when desc != 0.  Equal values keep row-major order (row, then step) in both
 * directions: a stable radix sort over the key total_key(v) ^ 2^63, bitwise inverted for desc.  out_cells has room for
 * n_rows * T entries; the first *out_n (a device u64) are written.  The call reads the number of valid cells back
 * once, so it synchronises the context's stream.  Scratch comes from the context (24 B per valid cell and 8 B per row,
 * b2p_sort.cu, sort_run).  B2P_E_INVALID: a NULL argument; B2P_E_NOMEM: the scratch could not be allocated;
 * B2P_E_TOO_LARGE: n_rows >= 2^31 - 1. */
B2P_API int b2p_sort_cells_dev(b2p_ctx* ctx, int32_t desc, const double* vals, const uint32_t* valid, uint32_t n_rows,
                               uint64_t T, uint64_t* out_cells, uint64_t* out_n);
/* sort / sort_desc over a node with several fields (the reference sorts by every field in order, each ASC | DESC NULLS
 * FIRST, planner.rs:1066-1071, 2743-2749): as b2p_sort_cells_dev, ordered lexicographically by the fields' values in
 * the f64 total order, field 0 first, every field in the same direction.  `vals` is a HOST array of n_fields DEVICE
 * grids [n_rows x T] sharing the bitmap `valid`; 1 <= n_fields <= B2P_MAX_FIELDS.  Equal tuples keep row-major order.
 * It is a least-significant-key-first radix sort: the scatter keys on field n_fields - 1, then each earlier field reloads
 * the pairs' keys (sort_rekey_kernel) before another stable sort, so the call makes n_fields radix sorts and
 * n_fields - 1 rekey launches; the scratch stays 24 B per valid cell.  n_fields == 1 is exactly b2p_sort_cells_dev. */
B2P_API int b2p_sort_cells_fields_dev(b2p_ctx* ctx, int32_t desc, const double* const* vals, int32_t n_fields,
                                      const uint32_t* valid, uint32_t n_rows, uint64_t T, uint64_t* out_cells,
                                      uint64_t* out_n);

/* sort / sort_desc over rows sharded across ranks (the reference's MergeSort over a MergeScan of per-datanode sorts,
 * dist_plan/merge_sort.rs, planner.rs:55-98): every rank sorts its own cells with K14, the sorted runs are exchanged,
 * and a merge writes the global order on every rank.  Every rank passes its own vals / valid [n_rows x T] and
 * row_id [n_rows] (device u32), the row's global ordinal in the child's row order: strictly increasing along a rank's
 * rows (distributed.shard_rows keeps the global order; the call checks it) and distinct across ranks (not checked).
 * Local cell (r, k) is global cell row_id[r] * T + k, so T <= 2^32.
 *
 * b2p_sort_shard_counts_dev: this rank's number of valid cells (K13's count).  With a communicator one ncclAllGather of
 * 8 B per rank fills the HOST table counts [n_ranks] (entry r: rank r), the same on every rank; without one it fills
 * counts[0].  Reads the table back, so it synchronises the stream.  N = the sum of counts sizes the outputs.
 *
 * b2p_sort_cells_allgather_dev (_fields_dev, _i64_dev): the whole call over the context's communicator.  On return
 * (stream order) every rank's out_cells [N] holds the global cells and out_vals [N] their values, bit for bit what
 * b2p_sort_cells_dev (_fields_dev, _i64_dev) writes over the global grid whose row i is the row with row_id i: the f64
 * total order (Int64: signed order), ascending or descending, equal values in (row, step) order.  The values are
 * decoded from the exchanged keys (a bijection), so NaN payloads and signed zeros come back bit for bit.  _fields_dev:
 * vals and out_vals are HOST arrays of n_fields device pointers, the keys compared lexicographically as
 * b2p_sort_cells_fields_dev does.  Each rank packs its run as one block, [field 0 keys: n u64] .. [field F-1 keys: n
 * u64][global cells: n u64] (keys flipped for desc), into its place in the gathered buffer, and one ncclBroadcast per
 * rank with cells, rooted there and of that rank's size, in one group, lays every block back to back on every rank;
 * when N == 0 no rank makes a collective call.  b2p_last_exchange_bytes() then gives the bytes this rank sent,
 * n_local x 8 x (n_fields + 1).  The exchange is the answer itself, so it is not cut into batches under
 * B2P_TOPK_EXCHANGE_BYTES.  Scratch per rank: the gathered blocks (N x 8 (F + 1) B), K14's over the local cells (24 B
 * per local valid cell, 8 B per row), and the merge's run buffers (N x 8 (F + 1) B, twice from five ranks with cells
 * on).  The merge is ceil(log2 R) rounds of pairwise merge-path merges (one copy round for one rank), each reading and
 * writing N x 8 (F + 1) B.  Without a communicator and n_ranks == 1 (no b2p_comm_init) it is b2p_sort_cells_dev's
 * order with the values beside it.
 *
 * The steps it is built from, so that one GPU can run R ranks (one context each) through the same kernels; the context
 * keeps no state between them.  counts is the HOST table of every rank's count:
 *   b2p_sort_shard_pack_dev (_i64_dev) writes this rank's block, count = its own entry of the table (8 (F + 1) count B);
 *   the blocks are laid back to back in rank order, block r of counts[r] entries;
 *   b2p_sort_shard_merge_dev (_i64_dev) over them writes out_cells / out_vals on every rank.
 * B2P_E_INVALID: a NULL argument, n_ranks > 1 without a communicator in the composed call, a rank's count that is not
 * its entry of counts, a row_id that is not strictly increasing; B2P_E_TOO_LARGE: T > 2^32 or n_rows >= 2^31 - 1;
 * B2P_E_NOMEM: the scratch could not be allocated. */
B2P_API int b2p_sort_shard_counts_dev(b2p_ctx* ctx, const uint32_t* valid, uint32_t n_rows, uint64_t T,
                                      uint64_t* counts);
B2P_API int b2p_sort_cells_allgather_dev(b2p_ctx* ctx, int32_t desc, const double* vals, const uint32_t* valid,
                                         const uint32_t* row_id, uint32_t n_rows, uint64_t T, const uint64_t* counts,
                                         uint64_t* out_cells, double* out_vals);
B2P_API int b2p_sort_cells_allgather_fields_dev(b2p_ctx* ctx, int32_t desc, const double* const* vals,
                                                int32_t n_fields, const uint32_t* valid, const uint32_t* row_id,
                                                uint32_t n_rows, uint64_t T, const uint64_t* counts,
                                                uint64_t* out_cells, double* const* out_vals);
B2P_API int b2p_sort_cells_allgather_i64_dev(b2p_ctx* ctx, int32_t desc, const int64_t* vals, const uint32_t* valid,
                                             const uint32_t* row_id, uint32_t n_rows, uint64_t T,
                                             const uint64_t* counts, uint64_t* out_cells, int64_t* out_vals);
B2P_API int b2p_sort_shard_pack_dev(b2p_ctx* ctx, int32_t desc, const double* const* vals, int32_t n_fields,
                                    const uint32_t* valid, const uint32_t* row_id, uint32_t n_rows, uint64_t T,
                                    uint64_t count, void* block);
B2P_API int b2p_sort_shard_pack_i64_dev(b2p_ctx* ctx, int32_t desc, const int64_t* vals, const uint32_t* valid,
                                        const uint32_t* row_id, uint32_t n_rows, uint64_t T, uint64_t count,
                                        void* block);
B2P_API int b2p_sort_shard_merge_dev(b2p_ctx* ctx, int32_t desc, int32_t n_fields, const uint64_t* counts,
                                     int32_t n_ranks, const void* blocks, uint64_t* out_cells,
                                     double* const* out_vals);
B2P_API int b2p_sort_shard_merge_i64_dev(b2p_ctx* ctx, int32_t desc, const uint64_t* counts, int32_t n_ranks,
                                         const void* blocks, uint64_t* out_cells, int64_t* out_vals);

/* ---- Int64 (BIGINT) value columns ------------------------------------------------------------------------------
 * An Int64 cell holds the bits of an int64_t in the same 8-byte slot a Float64 cell uses, so every layout above is
 * unchanged and only the calls that read a value as a number have an Int64 form.  The reference reads such a column
 * through the Arrow Int64 type: no stale-NaN test and no NaN filter (instant_manipulate.rs:490-527, normalize.rs:419),
 * integer order and integer equality.  An i64 whose bits are a NaN double is an ordinary integer to every call here. */
/* As b2p_instant_select_fields_dev with field 0 Int64: no staleness test, so every fresh row is selected (the other
 * fields' cells, of either type, are copied bit for bit).  n_fields == 1 is the one-field Int64 selector. */
B2P_API int b2p_instant_select_fields_i64_dev(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval,
                                              int64_t lookback, int64_t offset, const int64_t* ts,
                                              const double* const* vals, const uint8_t* const* field_valid,
                                              int32_t n_fields, const uint64_t* offsets, uint64_t n_rows,
                                              uint32_t n_series, double* const* outs, uint32_t* valid_words);
/* As b2p_group_aggregate_dev over Int64 cells: sum is the two's-complement wrapping sum (DataFusion's Int64 Sum
 * accumulator; wrapping add is associative, so the bits do not depend on the member order), min / max compare signed;
 * these three write the int64_t bits into out_val.  avg, stddev and stdvar read each value as (double)i64 and write
 * Float64 as b2p_group_aggregate_dev does; count writes the Float64 count. */
B2P_API int b2p_group_aggregate_i64_dev(b2p_ctx* ctx, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                                        const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                        double* out_val, uint32_t* out_cnt);
/* As b2p_topk_dev / b2p_count_values_dev / b2p_sort_cells_dev over Int64 cells: cells rank by signed value (key
 * bits ^ 2^63); count_values' distinct values are the int64_t values, written to out_val as int64_t. */
B2P_API int b2p_topk_i64_dev(b2p_ctx* ctx, int32_t bottom, double k, const int64_t* vals, const uint32_t* valid,
                             const b2p_group_index* index, const uint32_t* tie, uint64_t T, uint32_t* out_valid);
B2P_API int b2p_count_values_i64_dev(b2p_ctx* ctx, const int64_t* vals, const uint32_t* valid,
                                     const b2p_group_index* index, uint64_t T, int64_t* out_val, uint32_t* out_cnt);
B2P_API int b2p_sort_cells_i64_dev(b2p_ctx* ctx, int32_t desc, const int64_t* vals, const uint32_t* valid,
                                   uint32_t n_rows, uint64_t T, uint64_t* out_cells, uint64_t* out_n);
/* out[i] = (double)vals[i] (round to nearest even, as an Arrow Int64 -> Float64 cast) for i < n; out may be vals.  The
 * coercion DataFusion applies where a Float64 operator (arithmetic with a Float64 side, a math function, scalar(),
 * quantile) reads an Int64 column. */
B2P_API int b2p_i64_to_f64_dev(b2p_ctx* ctx, const int64_t* vals, uint64_t n, double* out);

/* ---- host-side helper (no device work) -------------------------------------------------------- */
/* The merge of the group-label agreement (b2p_plan_set_sharded), host only, so that one process can play R ranks.  A
 * block is one rank's groups in Labels order (the plan layer's sorted group order: per label "" first, then NULL, then
 * the other strings in byte order), all little-endian: u32 n_groups, u32 n_labels, u32 flags (bit 0: every group carries
 * a u64 __tsid), u32 n_fields, u64 n_rows (the rank's rows: 0 exactly when n_groups is 0), one u8 per field (its value
 * type: 0 Float64, 1 Int64, 2 Int32, 3 a count), then per group [u64 __tsid] and per label a u32 tag (0xFFFFFFFF:
 * NULL, else the byte length) followed by the bytes.  The merge is an R-way merge of the blocks in rank order into the global table (the same block layout,
 * written to out_table, whose capacity must be the sum of sizes; *out_table_bytes its length; its n_rows the sum, its
 * field types those of the blocks with rows), dropping duplicate tuples (a duplicate keeps the lowest rank's __tsid), so every rank derives the identical table from the identical
 * blocks whatever its own rank; *n_groups is the global count and local_to_global [rank's n_groups] maps block `rank`'s
 * groups to their global ids (the table's order).  B2P_E_INVALID: a NULL argument, a block that is truncated, longer
 * than its groups, not strictly in Labels order, unlike block 0 in n_labels, flags or n_fields, or with rows whose field
 * types differ from another block's with rows. */
B2P_API int b2p_group_keys_merge(const void* const* blocks, const uint64_t* sizes, int32_t n_ranks, int32_t rank,
                                 void* out_table, uint64_t* out_table_bytes, uint32_t* n_groups,
                                 uint32_t* local_to_global);
/* SeriesDivide (series_divide.rs:540-670) plus a cadence scan of one sorted batch on the HOST: series boundaries from
 * the id column `sid` (ids sid_base .. sid_base + n_series - 1, non-decreasing), or copied from `offsets_in`
 * (n_series + 1) when sid is NULL, into offsets_out (n_series + 1); and per series t0 = its first timestamp and
 * cadence = ts[1] - ts[0] (0 for series of fewer than two rows).  *all_regular = 1 iff ts[i] == t0 + i * cadence holds
 * for every row of every series — then the timestamp column is fully described by (offsets, t0, cadence), which is what
 * b2p_range_eval sends over PCIe instead of it (8 B/row less; the device rebuilds the column).  Any of t0 / cadence /
 * all_regular may be NULL.  B2P_E_UNSORTED when the ids are not non-decreasing or out of range. */
B2P_API int b2p_host_scan_series(const int64_t* ts, const uint32_t* sid, const uint64_t* offsets_in, uint64_t n_rows,
                         uint32_t n_series, uint32_t sid_base, uint64_t* offsets_out, int64_t* t0, int64_t* cadence,
                         int32_t* all_regular);

/* ---- host-pointer API (synchronous; H2D + kernels + D2H inside) ----------------------------- */
/* sid may be NULL when offsets_host (n_series+1) is given instead. out_ts (may be NULL) receives
 * the T eval timestamps. Pinned host buffers are copied directly; pageable ones are staged.
 * Every host entry below that takes offsets_host refuses, with B2P_E_INVALID and before anything is copied, offsets that
 * decrease or whose last entry exceeds n_rows (the rule of b2p_host_scan_series); rows before offsets_host[0] or past
 * offsets_host[n_series] belong to no series.  An id column that is not non-decreasing or holds an id >= n_series is
 * B2P_E_UNSORTED. */
B2P_API int b2p_range_eval(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts, const double* val,
                   const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series,
                   double* out, uint32_t* valid_words, int64_t* out_ts);
B2P_API int b2p_range_udf(b2p_ctx* ctx, int32_t fn_id, const int64_t* ts, const double* val, uint64_t n_rows,
                  const int64_t* packed_ranges, const int64_t* eval_ts, uint64_t n_win, int64_t range_length,
                  double param0, double param1, double* out, uint8_t* valid);
B2P_API int b2p_instant_select(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                       int64_t offset, const int64_t* ts, const double* val, const uint32_t* sid,
                       const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series, double* out,
                       uint32_t* valid_words);
/* Host-pointer form of b2p_instant_timestamp_dev (synchronous), staged as b2p_instant_select stages. */
B2P_API int b2p_instant_timestamp(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                  int64_t offset, const int64_t* ts, const uint32_t* sid, const uint64_t* offsets_host,
                                  uint64_t n_rows, uint32_t n_series, double* out, uint32_t* valid_words);
/* Host-pointer forms of b2p_range_eval_fields_dev / b2p_instant_select_fields_dev (synchronous): vals[f], field_valid[f]
 * and outs[f] are host columns; sid may be NULL when offsets_host (n_series+1) is given instead.  One staged copy per call (no chunked
 * pipeline): every column must fit on the device at once. */
B2P_API int b2p_range_eval_fields(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts, const double* const* vals,
                                  const uint8_t* const* field_valid, int32_t n_fields, const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows,
                                  uint32_t n_series, double* const* outs, uint32_t* valid_words);
B2P_API int b2p_instant_select_fields(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                      int64_t offset, const int64_t* ts, const double* const* vals,
                                      const uint8_t* const* field_valid, int32_t n_fields, const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows,
                                      uint32_t n_series, double* const* outs, uint32_t* valid_words);
B2P_API int b2p_group_aggregate(b2p_ctx* ctx, int32_t agg, const double* vals, const uint32_t* valid_words,
                        const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val,
                        uint32_t* out_cnt);
B2P_API int b2p_histogram_quantile(b2p_ctx* ctx, double phi, const double* le, uint32_t n_buckets, const double* rates,
                           const uint32_t* valid_words, uint32_t n_hist, uint64_t T, double* out,
                           uint32_t* out_valid_words);
/* histogram_quantile(phi, fn(bucket series)) in one call: samples in (host), rows [n_hist*T] out (host); the dense
 * per-series matrix stays on the device between the range function and the fold.  Index arrays are host pointers. */
B2P_API int b2p_range_histogram_fold(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts, const double* val,
                             const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series,
                             double phi, const uint32_t* hist_off, const uint32_t* bucket_series, const double* bucket_le,
                             uint32_t n_hist, double* out, uint32_t* out_valid_words);
/* Host-pointer form of b2p_histogram_fold_dev (synchronous): rates / valid_words are any [n_rows x T] grid and its
 * bitmap; the index (hist_off [n_hist + 1], bucket_series / bucket_le [hist_off[n_hist]]) as for the device form.  The
 * index is checked on the host before anything is launched: hist_off[0] != 0, a decreasing hist_off or a bucket_series
 * entry >= n_rows is B2P_E_INVALID.  out [n_hist x T], out_valid_words [n_hist x Tw]. */
B2P_API int b2p_histogram_fold(b2p_ctx* ctx, double phi, const uint32_t* hist_off, const uint32_t* bucket_series,
                               const double* bucket_le, uint32_t n_hist, const double* rates, const uint32_t* valid_words,
                               uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid_words);
/* histogram_quantile over bucket rows sharded across ranks (collective and synchronous; every rank calls it with the
 * same n_hist, T and phi).  rates / valid_words are this rank's [n_rows x T] grid and bitmap, row_hist [n_rows] each
 * row's global histogram id (< n_hist) and row_le [n_rows] its parsed bound (NaN: NULL or unparsable).  out
 * [n_hist x T] / out_valid_words [n_hist x Tw] receive the same bytes on every rank: b2p_histogram_fold over every
 * rank's rows concatenated in rank order, each histogram's buckets in the order of b2p_histogram_shard_index (bound
 * ascending, NaN last, ties in (rank, row) order).
 *   1. one all-gather of each rank's bucket count per histogram, [n_ranks x n_hist] u32;
 *   2. owners (b2p_histogram_shard_owners): the rank holding most of a histogram's buckets, the lowest on a tie;
 *   3. batches of contiguous histograms in which every rank's sent and received rows, (8 T + 4 Tw + 24) B each, fit the
 *      context's exchange cap (B2P_TOPK_EXCHANGE_BYTES, equal on every rank; a histogram too large alone is a batch of
 *      its own).  Per batch each rank packs its rows of histograms it does not own (b2p_row_move_dev), grouped by
 *      owner in (histogram, row) order, each with a 24-byte header (bound, histogram, rank, row), and sends them with
 *      ncclSend / ncclRecv in one group; the owner folds its histograms (K5) over [its rows | the received rows]
 *      with the index b2p_histogram_shard_index builds from the headers;
 *   4. every owner's result rows go to every rank (one ncclBroadcast per owner) and are placed in histogram order.
 * The counts table decides everything after it, so every rank derives the same batches, sends and receives: no size
 * is exchanged.  Where every histogram is whole on one rank no bucket row moves.  b2p_last_exchange_bytes() gives the
 * bytes this rank sent: its packed rows with their headers and its result block.  Without a communicator the output
 * is b2p_histogram_fold's over its own rows.  B2P_E_INVALID: a NULL argument; a row_hist entry >= n_hist on any rank
 * (the counts table carries each rank's verdict, so every rank returns it).  B2P_E_TOO_LARGE: more than 2^32 - 1
 * bucket rows over all ranks, also on every rank.  A failure local to one rank — a NULL argument or a bad grid before
 * the first collective, a device allocation or copy failing during the call — returns on that rank only, while the
 * other ranks wait in their next collective; as with the other sharded calls, the caller must then tear down the
 * communicator on every rank.
 *
 * b2p_range_histogram_fold_allgather is the same call over this rank's bucket SERIES: the range function (p, samples
 * as b2p_range_histogram_fold takes them) writes the [n_series x T] rates straight into the fold's grid on the device,
 * row_hist / row_le give each series' histogram and bound.  Whether or not a histogram is split, the dense matrix never
 * leaves the device; where none is split no bucket row is sent and each rank runs K5 over its own series, as
 * b2p_range_histogram_fold would, and only the results are gathered.
 *
 * The steps it is built from, so one GPU can play R ranks through the same code:
 *   b2p_histogram_shard_owners (host only): owner [n_hist] from the counts table [n_ranks x n_hist];
 *   b2p_histogram_shard_index (host only): the fold index over n buckets, each given by its histogram (< n_hist),
 *     bound, source rank and source row: histogram, then bound ascending with NaN last (-0.0 ties +0.0), then
 *     (rank, row).  hist_off [n_hist + 1], bucket_series [n] (the buckets' positions in the input) and bucket_le [n]
 *     are what b2p_histogram_fold[_dev] take.  B2P_E_INVALID: a NULL argument, a hist entry >= n_hist;
 *   b2p_row_move_dev: out row dst[i] = in row src[i] for i < n, T f64 values and Tw u32 words per row, device pointers
 *     (16-byte copies where T is even and both grids are 16-byte aligned). */
B2P_API int b2p_histogram_fold_allgather(b2p_ctx* ctx, double phi, const double* rates, const uint32_t* valid_words,
                                         uint32_t n_rows, uint64_t T, const uint32_t* row_hist, const double* row_le,
                                         uint32_t n_hist, double* out, uint32_t* out_valid_words);
B2P_API int b2p_range_histogram_fold_allgather(b2p_ctx* ctx, const b2p_range_params* p, const int64_t* ts,
                                               const double* val, const uint32_t* sid, const uint64_t* offsets_host,
                                               uint64_t n_samples, uint32_t n_series, double phi,
                                               const uint32_t* row_hist, const double* row_le, uint32_t n_hist,
                                               double* out, uint32_t* out_valid_words);
B2P_API int b2p_histogram_shard_owners(const uint32_t* counts, int32_t n_ranks, uint32_t n_hist, uint32_t* owner);
B2P_API int b2p_histogram_shard_index(const uint32_t* hist, const double* le, const uint32_t* rank, const uint32_t* row,
                                      uint32_t n, uint32_t n_hist, uint32_t* hist_off, uint32_t* bucket_series,
                                      double* bucket_le);
B2P_API int b2p_row_move_dev(b2p_ctx* ctx, const double* in, const uint32_t* in_valid, const uint32_t* src,
                             const uint32_t* dst, uint32_t n, uint64_t T, double* out, uint32_t* out_valid);
/* Host-pointer forms of b2p_binary_op_dev / b2p_scalar_op_dev (synchronous; row-index errors are returned directly). */
B2P_API int b2p_binary_op(b2p_ctx* ctx, int32_t op, int32_t return_bool, const double* lhs, const uint32_t* lhs_valid,
                          const uint32_t* lhs_row, uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid,
                          const uint32_t* rhs_row, uint32_t n_rhs_rows, uint64_t n_pairs, uint64_t T, double* out,
                          uint32_t* out_valid);
B2P_API int b2p_scalar_op(b2p_ctx* ctx, int32_t op, int32_t return_bool, int32_t scalar_on_left, double scalar,
                          const double* vals, const uint32_t* valid, uint64_t n_rows, uint64_t T, double* out,
                          uint32_t* out_valid);
/* Host-pointer form of b2p_setop_dev (synchronous; key errors are returned directly). */
B2P_API int b2p_setop(b2p_ctx* ctx, int32_t op, const double* lhs, const uint32_t* lhs_valid, const uint32_t* lhs_key,
                      uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid, const uint32_t* rhs_key,
                      uint32_t n_rhs_rows, uint32_t n_keys, uint64_t T, double* out, uint32_t* out_valid);

/* Host-pointer form of b2p_topk_dev (synchronous): the rows' group ids gid [n_rows] (>= n_groups: no group) instead of
 * an index, which the call builds itself; errors are returned directly. */
B2P_API int b2p_topk(b2p_ctx* ctx, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                     const uint32_t* gid, uint32_t n_rows, uint32_t n_groups, const uint32_t* tie, uint64_t T,
                     uint32_t* out_valid);

/* Host-pointer form of b2p_group_quantile_dev (synchronous): the rows' group ids gid [n_rows] (>= n_groups: no group)
 * instead of an index, which the call builds itself. */
B2P_API int b2p_group_quantile(b2p_ctx* ctx, double phi, const double* vals, const uint32_t* valid, const uint32_t* gid,
                               uint32_t n_rows, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt);

/* Host-pointer form of b2p_count_values_dev (synchronous): the rows' group ids gid [n_rows] (>= n_groups: no group)
 * instead of an index, which the call builds itself.  out_val / out_cnt [n_rows x T] in the order of a stable sort of the
 * rows by gid. */
B2P_API int b2p_count_values(b2p_ctx* ctx, const double* vals, const uint32_t* valid, const uint32_t* gid,
                             uint32_t n_rows, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt);

/* Host-pointer form of b2p_subquery_dev (synchronous): the grid and its bitmap go to the device, the sample rows are
 * made there. */
B2P_API int b2p_subquery(b2p_ctx* ctx, const b2p_range_params* p, int64_t inner_start, int64_t inner_interval,
                         const double* vals, const uint32_t* valid, uint32_t n_rows, uint64_t T_inner, double* out,
                         uint32_t* out_valid);

/* Host-pointer form of b2p_sort_cells_dev (synchronous): the grid and its bitmap go to the device; out_cells (room for
 * n_rows * T entries, the first *out_n written) and out_n are host pointers. */
B2P_API int b2p_sort_cells(b2p_ctx* ctx, int32_t desc, const double* vals, const uint32_t* valid, uint32_t n_rows,
                           uint64_t T, uint64_t* out_cells, uint64_t* out_n);
/* Host-pointer form of b2p_sort_cells_fields_dev (synchronous): vals[f] are host grids. */
B2P_API int b2p_sort_cells_fields(b2p_ctx* ctx, int32_t desc, const double* const* vals, int32_t n_fields,
                                  const uint32_t* valid, uint32_t n_rows, uint64_t T, uint64_t* out_cells,
                                  uint64_t* out_n);

/* Host-pointer forms of the Int64 calls above (synchronous), staged as their Float64 twins stage. */
B2P_API int b2p_instant_select_fields_i64(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                          int64_t offset, const int64_t* ts, const double* const* vals,
                                          const uint8_t* const* field_valid, int32_t n_fields, const uint32_t* sid,
                                          const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series,
                                          double* const* outs, uint32_t* valid_words);
B2P_API int b2p_group_aggregate_i64(b2p_ctx* ctx, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                                    const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                    double* out_val, uint32_t* out_cnt);
B2P_API int b2p_topk_i64(b2p_ctx* ctx, int32_t bottom, double k, const int64_t* vals, const uint32_t* valid,
                         const uint32_t* gid, uint32_t n_rows, uint32_t n_groups, const uint32_t* tie, uint64_t T,
                         uint32_t* out_valid);
B2P_API int b2p_count_values_i64(b2p_ctx* ctx, const int64_t* vals, const uint32_t* valid, const uint32_t* gid,
                                 uint32_t n_rows, uint32_t n_groups, uint64_t T, int64_t* out_val, uint32_t* out_cnt);
B2P_API int b2p_sort_cells_i64(b2p_ctx* ctx, int32_t desc, const int64_t* vals, const uint32_t* valid, uint32_t n_rows,
                               uint64_t T, uint64_t* out_cells, uint64_t* out_n);
B2P_API int b2p_i64_to_f64(b2p_ctx* ctx, const int64_t* vals, uint64_t n, double* out);

/* Host-pointer forms of b2p_instant_fn_dev / b2p_scalar_calculate_dev (synchronous; device-found errors returned). */
B2P_API int b2p_instant_fn(b2p_ctx* ctx, int32_t fn, double arg0, double arg1, const double* vals, const uint32_t* valid,
                           uint64_t n_rows, uint64_t T, double* out, uint32_t* out_valid);
B2P_API int b2p_scalar_calculate(b2p_ctx* ctx, const double* vals, const uint32_t* valid, const uint32_t* row_key,
                                 uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid);
/* Host-pointer form of b2p_step_fn_dev (synchronous; a step out of range is returned directly). */
B2P_API int b2p_step_fn(b2p_ctx* ctx, int32_t part, const int64_t* eval_ts, const uint32_t* valid, uint64_t n_rows,
                        uint64_t T, double* out);
/* Host-pointer form of b2p_absent_dev (synchronous): valid [n_rows x Tw], out [T] and out_valid [Tw] are host
 * pointers. */
B2P_API int b2p_absent(b2p_ctx* ctx, const uint32_t* valid, uint32_t n_rows, uint64_t T, double* out,
                       uint32_t* out_valid);

/* ---- plan-level API over the Arrow C Data Interface ------------------------------------------------
 * GpuPromRangeExec: the whole sub-tree SeriesDivide -> SeriesNormalize -> RangeManipulate ->
 * Projection(prom_fn) -> Filter(IS NOT NULL) [-> Aggregate(by-labels, ts).sort()] as one node, fed
 * with the RecordBatches the scan produces (arrow-rs `arrow::ffi::to_ffi`, pyarrow `_export_to_c`).
 * Constructor arguments carry the reference's names and meaning (see greptimedb_b200/csrc/b2p_plan.hpp:
 * SeriesDivide::new series_divide.rs:83-110, SeriesNormalize::new normalize.rs:66-83,
 * RangeManipulate::new range_manipulate.rs:86-110, UDF names planner.rs:2183-2221).
 * Input batches must be sorted by (tag columns, time index) — SeriesDivideExec's own requirement.
 * `function` is the UDF name ("prom_rate", ...); p->fn_id is ignored.  tag columns: Utf8, or a single
 * UInt64 id column (with label columns beside it: b2p_plan_set_label_columns).  aggregate: NULL/"" or
 * "sum|avg|count|min|max|stddev|stdvar" with by_columns ⊆ tags, checked at create (⊆ label columns on a
 * metric-engine leaf: a leaf keyed on `__tsid` alone checks a by-column that is not `__tsid` at
 * b2p_plan_set_label_columns and at push instead).
 * b2p_plan_push_batch MOVES the batch (its release callbacks are taken over). b2p_plan_execute
 * fills caller-provided ArrowArray/ArrowSchema structs; the caller releases them. */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif
typedef struct b2p_plan b2p_plan;
B2P_API b2p_plan* b2p_plan_range_create(b2p_ctx* ctx, const char* function, const b2p_range_params* p,
                                        const char* time_index, const char* field_column,
                                        const char* const* tag_columns, int32_t n_tags, const char* aggregate,
                                        const char* const* by_columns, int32_t n_by);
/* The same node over a table with several Float64 field columns (Influx line protocol / OTLP ingest), 1 <= n_fields <=
 * B2P_MAX_FIELDS: every field is selected at once, as b2p_range_eval_fields / b2p_instant_select_fields evaluate them
 * (a NaN in any field drops the row from every field with p->filter_nan; a cell is kept where every field's result
 * is).  b2p_plan_range_create is this call with one field.  The export has columns {time index, one value per field in
 * the given order, tags..}, each value named as the one-field node names its field.  The node's result carries
 * n_fields values per cell under one validity, and the nodes above keep them (DESIGN §8): element-wise stages,
 * arithmetic and `bool` apply per field; a binary node zips the fields pairwise (min of the two counts); an aggregate
 * folds each field; sort orders by every field in turn; subquery applies its function per field; absent reads only
 * validity.  Refused with the reference's Plan errors when a node sees two or more fields: a filtering comparison
 * ("Unsupported expr type: filter on multi-value input"), topk / bottomk, count_values, group, scalar, and / or /
 * unless, and histogram_quantile.  With two or more fields, NULL slots of a field are handed to the device as its Arrow
 * validity bitmap (the calls the reference evaluates differently over a NULL slot are refused at execute, naming the
 * field); with one field a NULL slot is read as NaN, as b2p_plan_range_create always has.  At create: a duplicate field,
 * n_fields out of range, and `aggregate` with two or more fields are Plan errors; at push: a missing field ("No field
 * named ..") is a Plan error and a non-Float64 one an Execution error. */
B2P_API b2p_plan* b2p_plan_range_create_fields(b2p_ctx* ctx, const char* function, const b2p_range_params* p,
                                               const char* time_index, const char* const* field_columns,
                                               int32_t n_fields, const char* const* tag_columns, int32_t n_tags,
                                               const char* aggregate, const char* const* by_columns, int32_t n_by);
/* Turn the node into the instant-vector form: InstantManipulate(start, end, lookback_delta, interval, ...)
 * (instant_manipulate.rs:189-208) instead of RangeManipulate + prom_fn; `function` / range are then ignored. */
B2P_API int b2p_plan_set_instant(b2p_plan* plan, int64_t lookback_delta);
/* The metric-engine form of a leaf (planner.rs:1300-1350, 1725-1800): Prometheus remote write tables divide their
 * series on the one UInt64 tag column `__tsid` (a hash of the label set), and `names` are the n >= 1 Utf8 label
 * columns that travel beside it.  Batches are sorted by (__tsid, time index); series divide on the id alone, and each
 * series takes its label values (NULL allowed) from its first row.  The metric engine gives one id one label set;
 * this node does not check it.  The nodes above group, match, order and rewrite on the label values, as over a leaf
 * keyed on those columns; the by-columns of the aggregate stage and the le column of HistogramFold name label columns.
 * __tsid rides along as a UInt64 column `__tsid`, exported after every other column, where the reference keeps it:
 * the instant selector, unary minus, scalar arithmetic, `bool` and filtering stages, both binary forms (the label side's; two sides
 * that carry it with no on / ignoring join on it one-to-one), `and` / `unless` (the lhs's), `or` (when both sides have
 * it), topk / bottomk, and an aggregate other than count_values that groups on every label column (the group's first
 * member's id, keep_tsid planner.rs:347-416).  Every other node drops it.  Call before the first push and before
 * b2p_plan_set_histogram_quantile: at the call, a leaf whose tag columns are not exactly `__tsid`, no label column,
 * one named like the time index, a field or the tag column, and one given twice are Plan errors; at push, a `__tsid`
 * column that is not UInt64 and a missing label column are Plan errors and a non-Utf8 label column an Execution
 * error. */
B2P_API int b2p_plan_set_label_columns(b2p_plan* plan, const char* const* names, int32_t n);
/* Add HistogramFold(le_column, field, time_index, quantile) (histogram_fold.rs:104-130) on top of the per-series
 * result: series that agree on every tag except `le` form one histogram.  Refused for a node of two or more fields. */
B2P_API int b2p_plan_set_histogram_quantile(b2p_plan* plan, const char* le_column, double quantile);
/* `node op scalar` (or `scalar op node` with scalar_on_left) on top of any node, binary nodes included; calls chain in
 * order (rate(x[1m]) * 60 > 1 is two calls).  Arithmetic and `bool` keep every row (the value column is renamed like
 * the reference's projection); a comparison without `bool` is a filter and keeps the node's value. */
B2P_API int b2p_plan_set_scalar_op(b2p_plan* plan, int32_t op, double scalar, int32_t scalar_on_left, int32_t return_bool);
/* Vector-vector binary node over two nodes (range, instant, aggregate, histogram or binary).  Series are matched on the
 * host like the reference's inner join on (key columns, time index): key = the rhs node's tag columns, intersected with
 * `labels` for matching "on", without them for "ignoring" (matching NULL: all of them); no key when either side has no
 * tags (every row pairs with every row); two id-keyed (__tsid) nodes without a modifier match on the id.  Every lhs
 * series pairs with every rhs series of the same key.  Output rows: {tag columns of label_side ("lhs" | "rhs"), time
 * index, value} for arithmetic / `bool`, the lhs node's rows for a filtering comparison; pairs in lhs then rhs row
 * order, steps ascending.  The node shares ownership of both children: their handles stay usable for push_batch and
 * must still be destroyed.  NULL on error (b2p_plan_last_error); the children are untouched then. */
B2P_API b2p_plan* b2p_plan_binary_create(b2p_ctx* ctx, int32_t op, int32_t return_bool, b2p_plan* lhs, b2p_plan* rhs,
                                         const char* matching /* NULL | "on" | "ignoring" */,
                                         const char* const* labels, int32_t n_labels,
                                         const char* label_side /* "lhs" | "rhs" */);
/* Set operator node over two nodes (range, instant, aggregate, histogram, binary or set).  Labels are matched on the
 * host; both sides must be evaluated on the same steps and carry Utf8 tags (an id-keyed __tsid side is refused: the
 * reference matches set operators on label values).
 *   and / unless: key = each side's tags, kept by "on" (listed) or "ignoring" (not listed); the two key sets must be
 *     equal.  Output: the lhs node's rows and columns, cells filtered; an lhs cell equal in labels, step and value bits
 *     to one of an earlier lhs row is dropped first (the reference's left.distinct()).
 *   or: key = the "on" labels (one that neither side has is an error), or the union of both sides' tags without the
 *     "ignoring" ones, or that union.  Output: the lhs rows, then the rhs rows; columns {lhs time index, then the sorted
 *     union of both sides' tags and the lhs value name}; a tag a side lacks is NULL on its rows.
 * Ownership as for b2p_plan_binary_create.  NULL on error (b2p_plan_last_error). */
B2P_API b2p_plan* b2p_plan_setop_create(b2p_ctx* ctx, int32_t op /* enum b2p_setop */, b2p_plan* lhs, b2p_plan* rhs,
                                        const char* matching /* NULL | "on" | "ignoring" */,
                                        const char* const* labels, int32_t n_labels);
/* Instant-vector function on top of any node, named as the reference's projection shows it: abs ceil floor sqrt exp ln
 * log2 log10 sin cos tan asin acos atan sinh cosh tanh asinh acosh atanh, degrees, radians, signum, negative (unary
 * minus, named (- <value>); refused at execute over an Int64 or Int32 column) (no argument),
 * prom_round (0 or 1: to_nearest, default 0), clamp (lo, hi), clamp_min (lo), clamp_max (hi).  Functions and
 * b2p_plan_set_scalar_op calls form one chain, applied in call order; the value column is renamed like the projection
 * (abs(val), clamp(val,Float64(0),Float64(12))).  B2P_E_INVALID: unknown name or wrong argument count.  A clamp with
 * lo > hi fails at execute, when the node has rows, with the reference's Execution error "min '12' > max '0'".
 * The calendar functions minute hour month year day_of_month day_of_week day_of_year days_in_month (no argument) are
 * K19 over the node's eval timestamps: one value column whatever the node's field count, named
 * date_part(Utf8("<part>"),<time index>) (days_in_month after its whole expression) and typed Int32; labels and
 * validity are kept.  Int32 is accepted by the stages above (read as Float64), by a binary operator against a Float64
 * side (Float64) or as the lhs of a filtering comparison (kept), by and / unless (the lhs kept), by `or` with an Int32
 * side, and by sort*, topk / bottomk and absent; every other node refuses it with a Plan error at execute. */
B2P_API int b2p_plan_set_function(b2p_plan* plan, const char* name, const double* args, int32_t n_args);
/* scalar(child), GpuPromScalarExec: a tagless node with one row over the child's steps, columns {time index,
 * scalar(<value name>)}; usable under scalar operators and functions and as a child of the binary and set nodes (a
 * tagless side pairs with every row).  Ownership as for b2p_plan_binary_create.  NULL on error. */
B2P_API b2p_plan* b2p_plan_scalar_create(b2p_ctx* ctx, b2p_plan* child);
/* topk(k, child) / bottomk(k, child) (bottom != 0) with an optional `by` / `without` modifier, GpuPromTopkExec: groups are
 * (group labels, step), the group labels being the listed ones the child has in the listed order (by), the child's
 * tags that are not listed in name order (without), or none.  Within a group the cells rank by value in the f64 total
 * order, then by every tag in column order (descending for topk, ascending for bottomk, NULL first); identical label
 * tuples rank in row order.  k follows b2p_topk_dev.  Nodes above see the child's rows, labels and values with the
 * kept cells; the export has columns {value, tags.., time index} and rows by group labels, ts, rank.  The child may be
 * any node; an id-keyed (__tsid) child is refused.  Ownership as for b2p_plan_binary_create.  NULL on error. */
B2P_API b2p_plan* b2p_plan_topk_create(b2p_ctx* ctx, int32_t bottom, double k, b2p_plan* child,
                                       const char* modifier /* NULL | "by" | "without" */, const char* const* labels,
                                       int32_t n_labels);
/* <op>(child) with an optional `by` / `without` modifier, GpuPromAggregateExec (prom_aggr_expr_to_plan,
 * planner.rs:334-452): groups are (group labels, step), the group labels as for b2p_plan_topk_create; a group has a row
 * at a step iff one of its members has a cell there, members folding in the child's row order.  op: sum avg count min
 * max stddev stdvar (as b2p_group_aggregate), group (1.0 wherever count does), quantile (param = phi, as
 * b2p_group_quantile_dev).  count_values, topk, bottomk and any other name are refused.  An id-keyed (__tsid) child is
 * only accepted without a modifier (one group per step).  The result has columns {group labels.., time index, value}
 * with rows in group label order; the value is named <df name>(<child's value name>), e.g. var_pop(val),
 * quantile(Float64(0.5),val), max(Float64(1)) for group.  The child may be any node.  Ownership as for
 * b2p_plan_binary_create.  NULL on error (b2p_plan_last_error). */
B2P_API b2p_plan* b2p_plan_aggregate_create(b2p_ctx* ctx, const char* op, double param, b2p_plan* child,
                                            const char* modifier /* NULL | "by" | "without" */,
                                            const char* const* labels, int32_t n_labels);
/* count_values(label, child) with an optional `by` / `without` modifier, GpuPromCountValuesExec (planner.rs:402-445):
 * groups as for b2p_plan_aggregate_create; per (group, step) one row for each distinct value of the child's cells (as
 * b2p_count_values_dev).  Nodes above see one row per (group, rank of the value), with the group labels as its labels
 * and the count as its value, named count(<child's value name>): count(count_values(..)), sum by (..)(count_values(..))
 * and count_values(..) > 1 compose.  The export has columns {count(<child value>) Int64, group labels.., time index,
 * <label> Float64 (the value)} with rows by group labels, ts, value in the f64 total order; with an element-wise stage
 * on top the first column is Float64.  A label equal to a group label, the time index or the count column, and an
 * id-keyed (__tsid) child with a modifier, are Plan errors at execute.  Ownership as for b2p_plan_binary_create.  NULL
 * on error (b2p_plan_last_error). */
B2P_API b2p_plan* b2p_plan_count_values_create(b2p_ctx* ctx, const char* label, b2p_plan* child,
                                               const char* modifier /* NULL | "by" | "without" */,
                                               const char* const* labels, int32_t n_labels);
/* Marks an aggregate node (every op), a count_values node, or a range / instant leaf with an aggregate stage, as
 * SHARDED (before execute): every rank runs the same plan over its own shard of series (each series whole on one rank),
 * and after execute every rank holds the result over the union of the shards, its export identical bit for bit on every
 * rank; nodes above run on that replicated result unchanged.  The node uses the context's communicator (b2p_comm_init);
 * without one it is exactly the unsharded node.  With one, at execute: the ranks agree one group table (each rank's
 * group label tuples, NULL distinct from "", plus the group's __tsid where the aggregate keeps it, its row count and its
 * field types, serialised as b2p_group_keys_merge reads them, exchanged by b2p_group_keys_sizes /
 * b2p_group_keys_allgather and merged on every rank; a rank without rows takes the field types of the ranks with rows,
 * and ranks with rows whose types differ are a Plan error on every rank), then fold over the global group ids:
 * b2p_group_aggregate_allreduce (_i64 for an Int64 sum / min / max; group is count's cells with the value 1.0; an Int64
 * avg / stddev / stdvar / group reads the Float64 coercion), b2p_quantile_allreduce or b2p_count_values_allgather
 * (_i64; at most the rows of all ranks).  Plan errors at execute: a child subtree with a node that is not row-local
 * (binary and set operators, topk, sort, absent, scalar(), count_values, aggregates, histogram_quantile, and an
 * EmptyMetric row, which every rank holds whole; leaves over the rank's series, element-wise stages, label_replace /
 * label_join and subqueries are row-local) or another sharded node below.  Any other node: a Plan error at the call. */
B2P_API int b2p_plan_set_sharded(b2p_plan* plan);
/* function(child[range:step]), GpuPromSubqueryExec (planner.rs:292-332): RangeManipulate(p->start, p->end, p->interval,
 * p->range) directly over the child, then the range function `function` ("prom_max_over_time", ...; p->fn_id is
 * ignored; param0 / param1 as for b2p_plan_range_create) and Filter(IS NOT NULL).  The child is any node; the caller
 * builds it on the inner grid (start - range + step .. end, step = the subquery's step or the outer interval), and
 * its eval timestamps must be a regular grid.  Each child row is one series whose samples are its valid cells, NaN
 * included (b2p_subquery).  Output: the child's rows and labels with columns {time index, value, tags..}, the value
 * named fn(<ti>_range,<child value>) (rate / increase / delta append ,<ti>,Int64(range); predict_linear,
 * quantile_over_time and holt_winters append their literals as Float64(..)), e.g. prom_rate(ts_range,val,ts,Int64(20000)).
 * Plan errors: an unknown function, a non-positive interval, a zero range, a non-zero offset or filter_nan (at create;
 * NULL is returned), a child whose grid is not regular (at execute).  Ownership as for b2p_plan_binary_create. */
B2P_API b2p_plan* b2p_plan_subquery_create(b2p_ctx* ctx, const char* function, const b2p_range_params* p,
                                           b2p_plan* child);
/* histogram_quantile(phi, child), GpuPromHistogramFoldExec (create_histogram_plan, planner.rs:3041-3108; HistogramFold,
 * histogram_fold.rs): the child is any node.  Its rows that agree on every tag except le_column (NULL: "le") form one
 * histogram; its buckets are ordered by le parsed as Rust's str::parse::<f64> (NULL or unparsable: NaN, last), ties in
 * row order, and folded per step as b2p_histogram_fold_dev (the buckets with a cell at that step).  Rows: one per
 * histogram in label order; labels: the child's tags without le; the value keeps the child's value name.  The export
 * keeps the child's column layout without le (a topk child's rank order is dropped).  A child without the le tag gives
 * an empty result (no rows, and an export without columns, as the reference's EmptyRelation); nodes above see no rows
 * over the child's steps.  Plan errors at execute: an id-keyed (__tsid) child, which carries no le; a count_values
 * child, whose counted value would be one more Float64 tag of the fold in the reference, which this layer does not
 * model.  Ownership as for b2p_plan_binary_create.  NULL on error (b2p_plan_last_error). */
B2P_API b2p_plan* b2p_plan_histogram_quantile_create(b2p_ctx* ctx, const char* le_column, double phi, b2p_plan* child);
/* sort(child) / sort_desc(child) / sort_by_label(child, labels..) / sort_by_label_desc(child, labels..),
 * GpuPromSortExec: the reference's Projection(time index, value, tags..) -> Filter(value IS NOT NULL) -> Sort(keys) over
 * the child (planner.rs:1060-1089, 2743-2772).  `function` is "sort" (value ASC), "sort_desc" (value DESC), both NULLS
 * FIRST in the f64 total order (b2p_sort_cells), "sort_by_label" or "sort_by_label_desc" (the listed labels in order,
 * byte-wise, "" before every other string and NULL after every string in both directions, ranked on the host).
 * Equal keys keep the child's row-major order (row, then step).  The export has columns {time index, value, tags..}
 * (tags in the child's order, the value keeps the child's value name) in that order; a child that exports no columns
 * gives the same empty result.  Nodes above see the child's result unchanged (rows, row order, values, bits);
 * element-wise stages on this node apply after the order is fixed, and a cell whose bit a stage clears is not
 * exported.  Plan errors at create (NULL is returned): an unknown function, sort_by_label* without a label, sort /
 * sort_desc with labels.  Plan errors at execute: sort_by_label* naming a label the child lacks or over an id-keyed
 * (__tsid) child, and any sort over a count_values child.  Ownership as for b2p_plan_binary_create. */
B2P_API b2p_plan* b2p_plan_sort_create(b2p_ctx* ctx, const char* function, b2p_plan* child, const char* const* labels,
                                       int32_t n_labels);
/* absent(child), GpuPromAbsentExec: the reference's PromAbsentExec(start, end, interval, time index, value column, fake
 * labels) over Aggregate(ts, first_value(value)) -> Sort(ts) of the child (create_absent_plan, planner.rs:3186-3245;
 * absent.rs).  One row over the grid start + k * interval <= end (none when start > end) with the value 1.0 at every
 * step at which no row of the child has a valid cell (a NaN cell counts as present; b2p_absent).  The labels are the
 * (label_names[i], label_values[i]) pairs, the equality matchers of the argument's selector in matcher order: a name
 * given twice keeps its last value, names are ordered byte-wise, an empty value is kept; the child's own labels play
 * no part.  The export has columns {time_index, value_column, labels..}, Utf8 labels.  The child is any node: one without
 * rows (or without columns) is absent at every step; an id-keyed or a count_values child is fine, because only its
 * validity is read.  Nodes above see one row with these labels; element-wise stages on this node apply to it.  Plan
 * errors at create (NULL is returned): a NULL ctx, child, name or label, interval <= 0, n_labels < 0, a label named like
 * time_index or value_column.  Plan error at execute: a child with rows whose eval timestamps are not this node's
 * grid.  Ownership as for b2p_plan_binary_create. */
B2P_API b2p_plan* b2p_plan_absent_create(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval,
                                         const char* time_index, const char* value_column,
                                         const char* const* label_names, const char* const* label_values,
                                         int32_t n_labels, b2p_plan* child);
/* EmptyMetric(start, end, interval, time_index, value_column, field_expr) (empty_metric.rs), GpuEmptyMetricExec: one
 * tagless row over start + k * interval <= end (no row when start > end) with every cell valid.  kind B2P_EMPTY_NONE
 * exports only the time index (no_field_expr); B2P_EMPTY_TIME is time(), the value (double)t / 1000.0 (K19) named
 * `<time_index> / Float64(1000)`; B2P_EMPTY_LITERAL is vector(s), pi() or a number literal, `literal` at every step,
 * named value_column.  The binary node pairs it with every row of the other side, as it pairs scalar(); the calendar
 * functions without an argument (hour(), ..) are b2p_plan_set_function on this node.  Plan errors at create (NULL is
 * returned): interval <= 0, a NULL name, an unknown kind. */
enum b2p_empty_metric_kind { B2P_EMPTY_NONE = 0, B2P_EMPTY_TIME = 1, B2P_EMPTY_LITERAL = 2 };
B2P_API b2p_plan* b2p_plan_empty_metric_create(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval,
                                               const char* time_index, const char* value_column,
                                               int32_t kind /* enum b2p_empty_metric_kind */, double literal);
/* timestamp(<selector>): turn a range node into the instant form (as b2p_plan_set_instant) whose value is the chosen
 * sample's timestamp in seconds, b2p_instant_timestamp: no value column is read and there is no stale-NaN test, for
 * Float64, Int64 and multi-field tables alike; the result is one Float64 column named `value`.  timestamp() of any
 * other expression keeps its child's values in the reference (its flag reaches only a vector selector, through
 * parentheses, planner.rs:244-290, 2358-2366): that needs no node. */
B2P_API int b2p_plan_set_timestamp(b2p_plan* plan, int64_t lookback_delta);
/* label_replace(child, dst, replacement, src, regex), GpuPromLabelExec: the reference's Projection(time index, values..,
 * regexp_replace(src, "^(?s:" + regex + ")$", replacement) AS dst, tags..) over the child (planner.rs:2330-2352,
 * 2518-2616).  No per-cell work: the child's grid, validity and row order are moved into the result and only the label
 * tuples change, each distinct source value evaluated once (b2p_regex.hpp states the engine).  In the reference's order:
 *   - dst failing ^[a-zA-Z_][a-zA-Z0-9_]*$ or starting with "__": "Invalid destination label name in label_replace(): <dst>";
 *   - regex rejected by Rust's regex crate: "Invalid regular expression in label_replace(): <regex>";
 *   - src a tag of the child and regex "": the child unchanged (a no-op);
 *   - src not a tag ("" included): a no-op when replacement is "", else dst = replacement on every row;
 *   - dst already a tag of the child (on either branch that adds it, dst == src included): "vector cannot contain metrics
 *     with the same labelset";
 *   - else dst = the expanded replacement where the whole src value matches, the src value itself where it does not,
 *     NULL where it is NULL.
 * Rows are never merged: two series that end up with one label tuple stay two rows.  Nodes above see dst appended to the
 * child's tags; the export is {time index, values.., dst, the child's tags..} ({time index, values.., tags..} for a
 * no-op).  A tagless literal or time() child that gains a label is joined on labels by the binary node from then on.
 * Plan errors, at create: the two texts above, a regex that is valid in Rust but outside the supported list
 * (b2p_label_regex_check), then a NULL child (so the first two need no node); at execute: an id-keyed (__tsid) child, a count_values child, dst named like the time index
 * or a value column.  Ownership as for b2p_plan_binary_create.  NULL on error (b2p_plan_last_error). */
B2P_API b2p_plan* b2p_plan_label_replace_create(b2p_ctx* ctx, b2p_plan* child, const char* dst, const char* replacement,
                                                const char* src, const char* regex);
/* label_join(child, dst, separator, srcs..), GpuPromLabelExec: the reference's Projection(time index, values..,
 * concat_ws(separator, src..) AS dst, tags..) (planner.rs:2306-2327, 2619-2700).  A source "" or one the child does not
 * have is NULL, and concat_ws skips NULLs (all NULL gives ""; a NULL tag value is skipped too).  dst is not validated;
 * when it is a tag of the child, that tag is dropped and dst takes its place at the end of the tags.  Layout, moves and
 * rows as for b2p_plan_label_replace_create.  Plan errors, at create: n_srcs == 0 ("Invalid function argument for
 * label_join"); at execute: an id-keyed (__tsid) or count_values child, a source or dst named like the time index or a
 * value column (the reference would read cell values as labels).  Ownership as for b2p_plan_binary_create. */
B2P_API b2p_plan* b2p_plan_label_join_create(b2p_ctx* ctx, b2p_plan* child, const char* dst, const char* separator,
                                             const char* const* srcs, int32_t n_srcs);
/* Host only, no context: what the plan layer makes of a label_replace regex.  0: supported; 1: invalid (Rust's regex
 * crate rejects it); 2: valid in Rust but outside the list in b2p_regex.hpp (the query stays on the CPU).
 * b2p_plan_last_error says why for 1 and 2.  B2P_E_INVALID for a NULL regex. */
B2P_API int b2p_label_regex_check(const char* regex);
/* Host only, no context: regexp_replace(input, "^(?s:" + regex + ")$", replacement) as label_replace evaluates one
 * value.  Writes the result and a terminating NUL to out when it fits in cap bytes; *out_len (when not NULL) gets the
 * result's length either way.  B2P_OK, B2P_E_TOO_LARGE when it does not fit, B2P_E_INVALID for a NULL argument or a
 * regex whose verdict is not 0 (b2p_plan_last_error says why). */
B2P_API int b2p_label_regex_replace(const char* regex, const char* replacement, const char* input, char* out,
                                    uint64_t cap, uint64_t* out_len);
B2P_API int b2p_plan_push_batch(b2p_plan* plan, struct ArrowArray* batch, struct ArrowSchema* schema);
B2P_API int b2p_plan_execute(b2p_plan* plan, struct ArrowArray* out, struct ArrowSchema* out_schema);
B2P_API int64_t b2p_plan_num_series(b2p_plan* plan);
B2P_API void b2p_plan_destroy(b2p_plan* plan);
B2P_API const char* b2p_plan_last_error(void);

/* ---- bench/test utility: synthetic workload generated on the device (BASELINE.md §4) ------- */
B2P_API int b2p_synth_fill_dev(b2p_ctx* ctx, uint64_t series_begin, uint64_t n_series, uint32_t n_samples, int64_t t0,
                       int64_t scrape_ms, uint32_t jitter_ms, int32_t with_resets, uint64_t seed, int64_t* ts,
                       double* val, uint32_t* sid);

#ifdef __cplusplus
}
#endif
#endif
