/*
 * promql_oracle.h — CPU ORACLE for the PromQL range-query hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product path
 * (greptimedb_b200/, libb200promql.so) never links, imports or calls anything here.
 *
 * It is a plain-C restatement of the reference's (GreptimeTeam/greptimedb, Rust)
 * algorithm for the path  SeriesDivide -> SeriesNormalize -> RangeManipulate ->
 * prom_* range UDF -> Filter(IS NOT NULL) -> Aggregate / HistogramFold / InstantManipulate.
 * Every function cites the reference file:line it follows (paths relative to the
 * GreptimeDB source tree).  The reference itself (Rust nightly + ~1000 crates) is not
 * built by this project, so parity is pinned on the reference's OWN unit-test
 * golden vectors (tests/golden/ *.json, ported from the #[test] bodies cited there).
 *
 * Third-party arithmetic that is NOT in the GreptimeDB tree and is restated from its
 * published algorithm (unit-level parity UNPINNED beyond the reference's 1e-4 tests):
 *   - arrow-rs 57.3.0 compute::sum / min / max   (Cargo.lock:318-321) -> orc_arrow_sum/min/max
 *   - datafusion 52.1 (GreptimeTeam fork rev 02b82535) sum/avg/count/min/max accumulators
 *     (Cargo.toml:340) -> orc_group_aggregate (plain sequential f64 +=, nulls skipped)
 */
#ifndef PROMQL_ORACLE_H
#define PROMQL_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Function ids — shared numbering with include/b200promql.h (B2P_FN_*). */
enum {
  ORC_FN_RATE = 0,
  ORC_FN_INCREASE = 1,
  ORC_FN_DELTA = 2,
  ORC_FN_IRATE = 3,
  ORC_FN_IDELTA = 4,
  ORC_FN_RESETS = 5,
  ORC_FN_CHANGES = 6,
  ORC_FN_COUNT_OVER_TIME = 7,
  ORC_FN_SUM_OVER_TIME = 8,
  ORC_FN_AVG_OVER_TIME = 9,
  ORC_FN_MIN_OVER_TIME = 10,
  ORC_FN_MAX_OVER_TIME = 11,
  ORC_FN_LAST_OVER_TIME = 12,
  ORC_FN_PRESENT_OVER_TIME = 13,
  ORC_FN_ABSENT_OVER_TIME = 14,
  ORC_FN_STDVAR_OVER_TIME = 15,
  ORC_FN_STDDEV_OVER_TIME = 16,
  ORC_FN_DERIV = 17,
  ORC_FN_PREDICT_LINEAR = 18,
  ORC_FN_QUANTILE_OVER_TIME = 19,
  ORC_FN_HOLT_WINTERS = 20,
  ORC_FN__COUNT = 21
};

/* Query parameters of the sub-plan (RangeManipulate + SeriesNormalize + UDF scalars). */
typedef struct {
  int32_t fn_id;
  int32_t filter_nan; /* SeriesNormalize.need_filter_out_nan (normalize.rs:417) */
  int64_t start;      /* RangeManipulate.start   (ms) */
  int64_t end;        /* RangeManipulate.end     (ms, inclusive) */
  int64_t interval;   /* RangeManipulate.interval(ms) */
  int64_t range;      /* RangeManipulate.range   (ms); also prom_rate's range_length */
  int64_t offset;     /* SeriesNormalize.offset  (ms, added to every ts) */
  double param0;      /* quantile phi | predict_linear t (seconds) | holt_winters sf */
  double param1;      /* holt_winters tf */
} orc_params;

/* ---- operators -------------------------------------------------------------------- */

/* RangeManipulateStream::calculate_range — range_manipulate.rs:693-772 (literal cursor walk).
 * off/len need capacity orc_num_steps(start,end,interval).  Returns #windows; *out_start /
 * *out_end receive the trimmed (start', end').  */
int64_t orc_calculate_range(const int64_t* ts, size_t n, int64_t start, int64_t end, int64_t interval,
                            int64_t range, uint32_t* off, uint32_t* len, int64_t* out_start,
                            int64_t* out_end);
/* The textbook definition (maximal run with t-range < ts <= t), used to cross-check. */
int64_t orc_calculate_range_definitional(const int64_t* ts, size_t n, int64_t start, int64_t end,
                                         int64_t interval, int64_t range, uint32_t* off, uint32_t* len,
                                         int64_t* out_start, int64_t* out_end);
int64_t orc_num_steps(int64_t start, int64_t end, int64_t interval);

/* SeriesNormalizeStream::normalize — normalize.rs:388-431. Returns kept rows. */
size_t orc_normalize(const int64_t* ts, const double* val, size_t n, int64_t offset, int filter_nan,
                     int64_t* out_ts, double* out_val);

/* SeriesDivideStream::find_first_diff_row — series_divide.rs:622-670 for TagIdentifier::Id.
 * Writes run starts into offsets (capacity n+1); returns number of series (runs). */
size_t orc_series_divide(const uint32_t* sid, size_t n, uint64_t* offsets);

/* InstantManipulateStream::manipulate — instant_manipulate.rs:473-585.
 * val may be NULL (no field column). take_idx/out_ts capacity = orc_num_steps. Returns #rows. */
int64_t orc_instant_manipulate(const int64_t* ts, const double* val, size_t n, int64_t start, int64_t end,
                               int64_t interval, int64_t lookback, uint64_t* take_idx, int64_t* out_ts);

/* HistogramFoldStream::evaluate_row — histogram_fold.rs:1046-1118.
 * *err = 1 when the reference returns Err (callers map it to NaN, histogram_fold.rs:806). */
double orc_histogram_evaluate_row(double quantile, const double* bucket, const double* counter, size_t n,
                                  int* err);

/* ---- range UDFs over explicit windows (RangeArray semantics, range_array.rs:247-254) ---- */

/* Evaluate fn_id over nwin windows (off[i], len[i]) of one series' (ts,val) columns.
 * eval_ts / range_length are used by rate/increase/delta; param0/param1 by quantile/predict/holt.
 * out[i] = value (0.0 where null, like an Arrow builder), valid[i] = 0/1.
 * ExtrapolatedRate::calc extrapolate_rate.rs:133-288 (sliding reset correction :216-238),
 * IDelta::calc idelta.rs:113-153, #[range_fn] loop range_fn.rs:189-229 + aggr_over_time.rs:35-179,
 * resets.rs:33-48, changes.rs:33-48, deriv.rs:32-40, predict_linear.rs:163-199,
 * quantile.rs:201-225, double_exponential_smoothing.rs:226-258. */
void orc_range_udf(int fn_id, const int64_t* ts, const double* val, const uint32_t* off,
                   const uint32_t* len, const int64_t* eval_ts, size_t nwin, int64_t range_length,
                   double param0, double param1, double* out, uint8_t* valid);
/* Same but rate/increase always rescan the window (no sliding correction) — quantifies the ulps. */
void orc_range_udf_rescan(int fn_id, const int64_t* ts, const double* val, const uint32_t* off,
                          const uint32_t* len, const int64_t* eval_ts, size_t nwin, int64_t range_length,
                          double param0, double param1, double* out, uint8_t* valid);

/* primitives exposed for unit tests */
double orc_arrow_sum(const double* v, size_t n);            /* arrow-rs aggregate.rs lanes=8 */
double orc_arrow_min(const double* v, size_t n);            /* total_cmp order */
double orc_arrow_max(const double* v, size_t n);
void orc_compensated_sum_inc(double inc, double* sum, double* comp); /* functions.rs:87-95 */
/* linear_regression_slices functions.rs:118-185; returns 1 if Some */
int orc_linear_regression(const int64_t* ts, const double* val, size_t n, int64_t intercept_time,
                          double* slope, double* intercept);
double orc_quantile(const double* v, size_t n, double q);   /* quantile.rs:201-225 */
double orc_holt_winters(const double* v, size_t n, double sf, double tf);

/* ---- whole sub-plan over many series -------------------------------------------------- */

/* Dense result layout used by the GPU library too: out[s * T + k] for the GLOBAL grid
 * t_k = start + k*interval, k in [0,T), T = orc_num_steps; valid bit (s*Tw + k/32, k%32) with
 * Tw = ceil(T/32) 32-bit words per series.  A (series, step) the reference would not emit
 * (trimmed step, empty window, null result) has valid = 0 and out = 0.0.
 *
 * orc_range_query_faithful: structure-faithful restatement — per series it materialises a batch
 * copy (concat_batches, series_divide.rs:567), normalize's filter copy (normalize.rs:417-430),
 * the ranges Vec + two packed-key arrays + T-long tag take (range_manipulate.rs:636-681), the UDF
 * loop, and the IS NOT NULL filter copy (planner.rs:1063).
 * orc_range_query_flat: algorithm only, flat arrays, no per-series allocation.
 * Both are sequential over [s_begin, s_end). rows of series s = [offsets[s], offsets[s+1]).
 * rescan != 0 evaluates the windows with orc_range_udf_rescan (rate / increase recompute the counter
 * correction of every window) instead of the reference's sliding orc_range_udf. */
void orc_range_query_faithful(const orc_params* p, const int64_t* ts, const double* val,
                              const uint32_t* sid, const uint64_t* offsets, size_t s_begin, size_t s_end,
                              double* out, uint32_t* valid_words, int rescan);
void orc_range_query_flat(const orc_params* p, const int64_t* ts, const double* val,
                          const uint64_t* offsets, size_t s_begin, size_t s_end, double* out,
                          uint32_t* valid_words, int rescan);
/* pthread fan-out over series (hash-partition analogue of target_partitions, state.rs:125-128).
 * Bit 0 of `faithful` selects orc_range_query_faithful, bit ORC_RESCAN the rescan UDF.  Returns 0 on
 * success. */
#define ORC_RESCAN 2
int orc_range_query_mt(const orc_params* p, const int64_t* ts, const double* val, const uint32_t* sid,
                       const uint64_t* offsets, size_t n_series, double* out, uint32_t* valid_words,
                       int n_threads, int faithful);

/* InstantManipulate over many series, dense layout as above (value of the taken row). */
void orc_instant_query(const int64_t* ts, const double* val, const uint64_t* offsets, size_t n_series,
                       int64_t start, int64_t end, int64_t interval, int64_t lookback, int64_t offset,
                       double* out, uint32_t* valid_words);

/* By-label aggregate (planner.rs:334-452; DataFusion accumulators): sequential, series order.
 * op: 0 sum, 1 avg, 2 count, 3 min, 4 max, 5 stddev_pop, 6 var_pop.  out_val[g*T+k], out_cnt[g*T+k]
 * (cnt==0 -> group absent at that step). */
void orc_group_aggregate(int op, const double* vals, const uint32_t* valid_words, const uint32_t* gid,
                         size_t n_series, size_t n_groups, size_t T, double* out_val, uint32_t* out_cnt);

/* histogram_quantile over dense rate matrix: series h*B+b is bucket b of histogram h
 * (le ascending, last +Inf).  A (h,k) row exists iff all B buckets are valid at k (the
 * reference folds only complete groups in optimistic mode, histogram_fold.rs:772-813). */
void orc_histogram_quantile(double phi, const double* le, size_t B, const double* rates,
                            const uint32_t* valid_words, size_t n_hist, size_t T, double* out,
                            uint32_t* out_valid_words);

/* Synthetic workload generator (BASELINE.md §4; value shapes from benches/bench_range_fn.rs:60-82).
 * Identical integer/f64 arithmetic to the CUDA generator in greptimedb_b200/csrc. */
void orc_synth_fill(uint64_t series_begin, uint64_t n_series, uint32_t n_samples, int64_t t0,
                    int64_t scrape_ms, uint32_t jitter_ms, int with_resets, uint64_t seed, int64_t* ts,
                    double* val, uint32_t* sid);

#ifdef __cplusplus
}
#endif
#endif
