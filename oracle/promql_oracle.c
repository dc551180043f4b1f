/*
 * promql_oracle.c — CPU ORACLE (test infrastructure only; see promql_oracle.h).
 *
 * Plain-C restatement of GreptimeDB's PromQL range-query hot path.  Each function names the
 * reference file:line it follows (relative to the GreptimeDB source tree).  Nothing here is derived from
 * the CUDA code; the CUDA code is checked AGAINST this.
 */
#include "promql_oracle.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------
 * helpers
 * ---------------------------------------------------------------------------------------- */

static int64_t rem_euclid_i64(int64_t a, int64_t b) { /* Rust i64::rem_euclid, b > 0 */
  int64_t r = a % b;
  return r < 0 ? r + b : r;
}

int64_t orc_num_steps(int64_t start, int64_t end, int64_t interval) {
  if (interval <= 0 || end < start) return 0;
  return (end - start) / interval + 1;
}

/* f64::total_cmp (Rust std): flip all bits but the sign for negatives, compare as i64. */
static int64_t total_key(double x) {
  int64_t b;
  memcpy(&b, &x, 8);
  b ^= (int64_t)(((uint64_t)(b >> 63)) >> 1);
  return b;
}

/* ------------------------------------------------------------------------------------------
 * RangeManipulateStream::calculate_range        src/promql/src/extension_plan/range_manipulate.rs:693-772
 * Literal restatement of the cursor walk, including its usize arithmetic.  NB (quirk, see
 * DESIGN.md "C-13"): `cursor = range_start_index + start_delta` can overshoot `len`, in which
 * case BOTH while-loops are skipped and the window is reported empty even if samples are inside
 * (t-range, t].  The definitional variant below does not have that behaviour.
 * ---------------------------------------------------------------------------------------- */
int64_t orc_calculate_range(const int64_t* ts, size_t n, int64_t start, int64_t end, int64_t interval,
                            int64_t range, uint32_t* off, uint32_t* len, int64_t* out_start,
                            int64_t* out_end) {
  if (n == 0) { /* :709-711 */
    *out_start = start;
    *out_end = end;
    return 0;
  }
  int64_t first_ts = ts[0];
  int64_t remainder = rem_euclid_i64(first_ts - start, interval); /* :716 */
  int64_t first_ts_aligned = remainder == 0 ? first_ts : first_ts + (interval - remainder);
  int64_t last_ts = ts[n - 1];
  int64_t last_ts_aligned = ((last_ts + range) / interval) * interval; /* :723 aligned to 0 */
  int64_t s = start > first_ts_aligned ? start : first_ts_aligned;
  int64_t e = end < last_ts_aligned ? end : last_ts_aligned;
  *out_start = s;
  *out_end = e;
  if (s > e) return 0; /* :726-728 */

  int64_t nwin = 0;
  size_t range_start_index = 0, last_range_start = 0, start_delta = 0;
  for (int64_t curr_ts = s; curr_ts <= e; curr_ts += interval) { /* :735 */
    int64_t start_ts = curr_ts - range;
    size_t range_start = n;
    size_t range_end = 0;
    size_t cursor = range_start_index + start_delta;
    /* search back to keep the result correct :743-746 */
    while (cursor < n && ts[cursor] > start_ts && cursor > 0) cursor -= 1;
    while (cursor < n) { /* :748-762 */
      int64_t t = ts[cursor];
      if (range_start > cursor && t > start_ts) {
        range_start = cursor;
        range_start_index = range_start;
      }
      if (t <= curr_ts) {
        range_end = range_end > cursor ? range_end : cursor;
      } else {
        range_start_index = range_start_index > 0 ? range_start_index - 1 : 0; /* saturating_sub */
        break;
      }
      cursor += 1;
    }
    if (range_start > range_end) { /* :763-766 */
      off[nwin] = 0;
      len[nwin] = 0;
      start_delta = 0;
    } else {
      off[nwin] = (uint32_t)range_start;
      len[nwin] = (uint32_t)(range_end + 1 - range_start);
      start_delta = range_start - last_range_start;
      last_range_start = range_start;
    }
    nwin++;
  }
  return nwin;
}

int64_t orc_calculate_range_definitional(const int64_t* ts, size_t n, int64_t start, int64_t end,
                                         int64_t interval, int64_t range, uint32_t* off, uint32_t* len,
                                         int64_t* out_start, int64_t* out_end) {
  if (n == 0) {
    *out_start = start;
    *out_end = end;
    return 0;
  }
  int64_t remainder = rem_euclid_i64(ts[0] - start, interval);
  int64_t first_ts_aligned = remainder == 0 ? ts[0] : ts[0] + (interval - remainder);
  int64_t last_ts_aligned = ((ts[n - 1] + range) / interval) * interval;
  int64_t s = start > first_ts_aligned ? start : first_ts_aligned;
  int64_t e = end < last_ts_aligned ? end : last_ts_aligned;
  *out_start = s;
  *out_end = e;
  if (s > e) return 0;
  int64_t nwin = 0;
  size_t lo = 0, hi = 0; /* lo = first idx with ts > t-range ; hi = first idx with ts > t */
  for (int64_t t = s; t <= e; t += interval) {
    while (lo < n && ts[lo] <= t - range) lo++;
    while (hi < n && ts[hi] <= t) hi++;
    if (hi > lo) {
      off[nwin] = (uint32_t)lo;
      len[nwin] = (uint32_t)(hi - lo);
    } else {
      off[nwin] = 0;
      len[nwin] = 0;
    }
    nwin++;
  }
  return nwin;
}

/* ------------------------------------------------------------------------------------------
 * SeriesNormalizeStream::normalize               src/promql/src/extension_plan/normalize.rs:388-431
 * ---------------------------------------------------------------------------------------- */
size_t orc_normalize(const int64_t* ts, const double* val, size_t n, int64_t offset, int filter_nan,
                     int64_t* out_ts, double* out_val) {
  size_t m = 0;
  for (size_t i = 0; i < n; i++) {
    if (filter_nan && isnan(val[i])) continue; /* :417-426 */
    out_ts[m] = ts[i] + offset;                /* :400-406 */
    out_val[m] = val[i];
    m++;
  }
  return m;
}

/* ------------------------------------------------------------------------------------------
 * SeriesDivideStream::find_first_diff_row         src/promql/src/extension_plan/series_divide.rs:622-670
 * For TagIdentifier::Id (:50-80) equal_at is a u64 compare; a series is a maximal run of equal
 * adjacent ids.
 * ---------------------------------------------------------------------------------------- */
size_t orc_series_divide(const uint32_t* sid, size_t n, uint64_t* offsets) {
  size_t ns = 0;
  if (n == 0) {
    offsets[0] = 0;
    return 0;
  }
  offsets[ns++] = 0;
  size_t same_until = 0;
  while (same_until < n - 1) {
    if (sid[same_until] != sid[same_until + 1]) offsets[ns++] = same_until + 1; /* cut :658-667 */
    same_until++;
  }
  offsets[ns] = n;
  return ns;
}

/* ------------------------------------------------------------------------------------------
 * InstantManipulateStream::manipulate            src/promql/src/extension_plan/instant_manipulate.rs:473-585
 * ---------------------------------------------------------------------------------------- */
int64_t orc_instant_manipulate(const int64_t* ts, const double* val, size_t n, int64_t start, int64_t end,
                               int64_t interval, int64_t lookback, uint64_t* take_idx, int64_t* out_ts) {
  if (n == 0) return 0; /* :485-487 */
  int64_t first_ts = ts[0];
  int64_t last_ts = ts[n - 1];
  int64_t last_useful = lookback > 0 ? last_ts + lookback - 1 : last_ts; /* :501-505 */
  int64_t max_start = first_ts > start ? first_ts : start;
  int64_t min_end = last_useful < end ? last_useful : end;
  int64_t aligned_start = start + (max_start - start) / interval * interval; /* :510 */
  int64_t aligned_end = end - (end - min_end) / interval * interval;         /* :511 */
  int64_t m = 0;
  size_t cursor = 0;
  for (int64_t expected = aligned_start; expected <= aligned_end; expected += interval) {
    int matched = 0;
    while (cursor < n) { /* :523-541 */
      int64_t curr = ts[cursor];
      if (curr == expected) {
        if (val != NULL && isnan(val[cursor])) {
          /* ignore the NaN value */
        } else {
          take_idx[m] = cursor;
          out_ts[m] = expected;
          m++;
        }
        matched = 1;
        break; /* continue 'next */
      } else if (curr > expected) {
        break;
      }
      cursor += 1;
    }
    if (matched) continue;
    if (cursor == n) { /* :542-548 */
      cursor -= 1;
      if (ts[cursor] + lookback <= expected) break;
    }
    int64_t curr_ts = ts[cursor]; /* :551 */
    if (curr_ts + lookback <= expected) continue;
    if (curr_ts > expected) { /* :555-572 */
      if (cursor >= 1) {
        size_t prev = cursor - 1;
        int64_t prev_ts = ts[prev];
        if (prev_ts + lookback > expected) {
          if (val != NULL && isnan(val[prev])) continue;
          take_idx[m] = prev;
          out_ts[m] = expected;
          m++;
        }
      }
    } else if (val != NULL && isnan(val[cursor])) {
      /* stale */
    } else {
      take_idx[m] = cursor;
      out_ts[m] = expected;
      m++;
    }
  }
  return m;
}

/* ------------------------------------------------------------------------------------------
 * HistogramFoldStream::evaluate_row              src/promql/src/extension_plan/histogram_fold.rs:1046-1118
 * ---------------------------------------------------------------------------------------- */
double orc_histogram_evaluate_row(double quantile, const double* bucket, const double* counter_in,
                                  size_t n, int* err) {
  *err = 0;
  if (n <= 1) return NAN;
  if (isfinite(bucket[n - 1])) { /* :1051-1055 Err("last bucket should be +Inf") */
    *err = 1;
    return NAN;
  }
  if (quantile < 0.0) return -INFINITY;
  if (quantile > 1.0) return INFINITY;
  if (isnan(quantile)) return NAN;
  for (size_t i = 0; i + 1 < n; i++)
    if (!(bucket[i] <= bucket[i + 1])) return NAN; /* :1071-1073 */
  int needs_fix = 0;
  for (size_t i = 0; i < n; i++)
    if (!isfinite(counter_in[i])) needs_fix = 1;
  for (size_t i = 0; i + 1 < n; i++)
    if (!(counter_in[i] <= counter_in[i + 1])) needs_fix = 1;
  double* fixed = NULL;
  const double* counter = counter_in;
  if (needs_fix) { /* :1079-1091 */
    fixed = (double*)malloc(n * sizeof(double));
    double prev = 0.0;
    for (size_t i = 0; i < n; i++) {
      double v = isfinite(counter_in[i]) ? counter_in[i] : prev;
      if (i > 0 && v < prev) v = prev;
      fixed[i] = v;
      prev = v;
    }
    counter = fixed;
  }
  double total = counter[n - 1];
  double expected_pos = total * quantile;
  size_t fit = 0;
  while (fit < n && counter[fit] < expected_pos) fit++; /* :1097-1099 */
  double result;
  if (fit >= n - 1) {
    result = bucket[n - 2];
  } else {
    double upper_bound = bucket[fit];
    double upper_count = counter[fit];
    double lower_bound = bucket[0] < 0.0 ? bucket[0] : 0.0; /* bucket[0].min(0.0) */
    if (isnan(bucket[0])) lower_bound = 0.0;                /* f64::min ignores NaN */
    double lower_count = 0.0;
    if (fit > 0) {
      lower_bound = bucket[fit - 1];
      lower_count = counter[fit - 1];
    }
    if (fabs(upper_count - lower_count) < 1e-10) {
      result = NAN;
    } else {
      result = lower_bound + (upper_bound - lower_bound) / (upper_count - lower_count) * (expected_pos - lower_count);
    }
  }
  free(fixed);
  return result;
}

/* ------------------------------------------------------------------------------------------
 * arrow-rs 57.3.0 arrow-arith/src/aggregate.rs (third party; restated from the published
 * algorithm — parity unpinned beyond the reference's 1e-4 tests, aggr_over_time.rs:219-309):
 * non-null float sum = LANES independent accumulators over chunks_exact(LANES), remainder
 * added lane-wise, then a halving tree merge.  x86-64 default target features (the reference
 * sets no target-cpu, .cargo/config.toml) -> 8 lanes for f64.
 * min/max fold with ArrowNativeTypeOp::is_lt / is_gt == total_cmp order.
 * ---------------------------------------------------------------------------------------- */
double orc_arrow_sum(const double* v, size_t n) {
  enum { LANES = 8 };
  double acc[LANES];
  for (int i = 0; i < LANES; i++) acc[i] = 0.0;
  size_t full = n / LANES * LANES;
  for (size_t c = 0; c < full; c += LANES)
    for (int i = 0; i < LANES; i++) acc[i] += v[c + i];
  for (size_t i = full; i < n; i++) acc[i - full] += v[i];
  for (int w = LANES; w >= 2; w /= 2)
    for (int i = 0; i < w / 2; i++) acc[i] += acc[i + w / 2];
  return acc[0];
}
double orc_arrow_min(const double* v, size_t n) {
  double m = v[0];
  for (size_t i = 1; i < n; i++)
    if (total_key(v[i]) < total_key(m)) m = v[i];
  return m;
}
double orc_arrow_max(const double* v, size_t n) {
  double m = v[0];
  for (size_t i = 1; i < n; i++)
    if (total_key(v[i]) > total_key(m)) m = v[i];
  return m;
}

/* compensated_sum_inc                             src/promql/src/functions.rs:87-95 */
void orc_compensated_sum_inc(double inc, double* sum, double* comp) {
  double new_sum = *sum + inc;
  if (fabs(*sum) >= fabs(inc)) {
    *comp += (*sum - new_sum) + inc;
  } else {
    *comp += (inc - new_sum) + *sum;
  }
  *sum = new_sum;
}

/* linear_regression_slices                        src/promql/src/functions.rs:118-185 */
int orc_linear_regression(const int64_t* ts, const double* val, size_t n, int64_t intercept_time,
                          double* slope, double* intercept) {
  double count = 0.0, sum_x = 0.0, sum_y = 0.0, sum_xy = 0.0, sum_x2 = 0.0;
  double comp_x = 0.0, comp_y = 0.0, comp_xy = 0.0, comp_x2 = 0.0;
  int const_y = 1, have_init = 0;
  double init_y = 0.0;
  for (size_t i = 0; i < n; i++) {
    double value = val[i];
    double time = (double)ts[i];
    if (!have_init) {
      init_y = value;
      have_init = 1;
    }
    if (const_y && count > 0.0 && value != init_y) const_y = 0;
    count += 1.0;
    double x = (time - (double)intercept_time) / 1e3;
    orc_compensated_sum_inc(x, &sum_x, &comp_x);
    orc_compensated_sum_inc(value, &sum_y, &comp_y);
    orc_compensated_sum_inc(x * value, &sum_xy, &comp_xy);
    orc_compensated_sum_inc(x * x, &sum_x2, &comp_x2);
  }
  if (count < 2.0) return 0;
  if (const_y) {
    if (!isfinite(init_y)) return 0;
    *slope = 0.0;
    *intercept = init_y;
    return 1;
  }
  sum_x += comp_x;
  sum_y += comp_y;
  sum_xy += comp_xy;
  sum_x2 += comp_x2;
  double cov_xy = sum_xy - sum_x * sum_y / count;
  double var_x = sum_x2 - sum_x * sum_x / count;
  *slope = cov_xy / var_x;
  *intercept = sum_y / count - *slope * sum_x / count;
  return 1;
}

static int cmp_total(const void* a, const void* b) {
  int64_t x = total_key(*(const double*)a), y = total_key(*(const double*)b);
  return x < y ? -1 : (x > y ? 1 : 0);
}

/* quantile_with_scratch                           src/promql/src/functions/quantile.rs:201-225 */
double orc_quantile(const double* v, size_t n, double q) {
  if (isnan(q) || n == 0) return NAN;
  if (q < 0.0) return -INFINITY;
  if (q > 1.0) return INFINITY;
  double* s = (double*)malloc(n * sizeof(double));
  memcpy(s, v, n * sizeof(double));
  qsort(s, n, sizeof(double), cmp_total);
  double rank = q * (double)(n - 1);
  size_t lower = (size_t)floor(rank);
  size_t upper = lower + 1 < n - 1 ? lower + 1 : n - 1;
  double weight = rank - floor(rank);
  double r = s[lower] * (1.0 - weight) + s[upper] * weight;
  free(s);
  return r;
}

/* double_exponential_smoothing_impl               src/promql/src/functions/double_exponential_smoothing.rs:216-258 */
double orc_holt_winters(const double* v, size_t n, double sf, double tf) {
  if (isnan(sf) || isnan(tf) || n == 0) return NAN;
  if (sf < 0.0 || tf < 0.0) return -INFINITY;
  if (sf > 1.0 || tf > 1.0) return INFINITY;
  if (n <= 2) return NAN;
  double s0 = 0.0, s1 = v[0], b = v[1] - v[0];
  for (size_t i = 1; i < n; i++) {
    double x = sf * v[i];
    /* calc_trend_value(i-1, tf, s0, s1, b) :216-223 */
    if (i - 1 != 0) {
      double xx = tf * (s1 - s0);
      double yy = (1.0 - tf) * b;
      b = xx + yy;
    }
    double y = (1.0 - sf) * (s1 + b);
    s0 = s1;
    s1 = x + y;
  }
  return s1;
}

/* ------------------------------------------------------------------------------------------
 * Range UDFs over explicit windows.
 * ---------------------------------------------------------------------------------------- */

/* One #[range_fn] body on values[o..o+l] / times[o..o+l]; returns 1 = Some. */
static int range_fn_body(int fn_id, const int64_t* t, const double* v, size_t l, double* r) {
  switch (fn_id) {
    case ORC_FN_AVG_OVER_TIME: /* aggr_over_time.rs:35-37 */
      if (l == 0) return 0;
      *r = orc_arrow_sum(v, l) / (double)l;
      return 1;
    case ORC_FN_MIN_OVER_TIME: /* :46-48 */
      if (l == 0) return 0;
      *r = orc_arrow_min(v, l);
      return 1;
    case ORC_FN_MAX_OVER_TIME: /* :56-58 */
      if (l == 0) return 0;
      *r = orc_arrow_max(v, l);
      return 1;
    case ORC_FN_SUM_OVER_TIME: /* :66-68 */
      if (l == 0) return 0;
      *r = orc_arrow_sum(v, l);
      return 1;
    case ORC_FN_COUNT_OVER_TIME: /* :76-82 */
      if (l == 0) return 0;
      *r = (double)l;
      return 1;
    case ORC_FN_LAST_OVER_TIME: /* :90-92 */
      if (l == 0) return 0;
      *r = v[l - 1];
      return 1;
    case ORC_FN_ABSENT_OVER_TIME: /* :102-104 */
      if (l == 0) {
        *r = 1.0;
        return 1;
      }
      return 0;
    case ORC_FN_PRESENT_OVER_TIME: /* :112-114 */
      if (l == 0) return 0;
      *r = 1.0;
      return 1;
    case ORC_FN_STDVAR_OVER_TIME: { /* :123-144 */
      if (l == 0) return 0;
      long count = 0;
      double mean = 0.0, result = 0.0;
      for (size_t i = 0; i < l; i++) {
        double value = v[i];
        long new_count = count + 1;
        double delta1 = value - mean;
        double new_mean = delta1 / (double)new_count + mean;
        double delta2 = value - new_mean;
        double new_result = result + delta1 * delta2;
        count += 1;
        mean = new_mean;
        result = new_result;
      }
      *r = result / (double)count;
      return 1;
    }
    case ORC_FN_STDDEV_OVER_TIME: { /* :153-179 */
      if (l == 0) return 0;
      double count = 0.0, mean = 0.0, comp_mean = 0.0, dev = 0.0, comp_dev = 0.0;
      for (size_t i = 0; i < l; i++) {
        count += 1.0;
        double cur = v[i];
        double delta = cur - (mean + comp_mean);
        orc_compensated_sum_inc(delta / count, &mean, &comp_mean);
        orc_compensated_sum_inc(delta * (cur - (mean + comp_mean)), &dev, &comp_dev);
      }
      *r = sqrt((dev + comp_dev) / count);
      return 1;
    }
    case ORC_FN_RESETS: { /* resets.rs:33-48 */
      if (l == 0) return 0;
      long num = 0;
      for (size_t i = 1; i < l; i++)
        if (v[i] < v[i - 1]) num++;
      *r = (double)num;
      return 1;
    }
    case ORC_FN_CHANGES: { /* changes.rs:33-48 */
      if (l == 0) return 0;
      long num = 0;
      for (size_t i = 1; i < l; i++)
        if (v[i] != v[i - 1] && !(isnan(v[i]) && isnan(v[i - 1]))) num++;
      *r = (double)num;
      return 1;
    }
    case ORC_FN_DERIV: { /* deriv.rs:32-40 */
      if (l < 2) return 0;
      double slope, icpt;
      if (!orc_linear_regression(t, v, l, t[0], &slope, &icpt)) return 0;
      *r = slope;
      return 1;
    }
    default:
      return 0;
  }
}

static void range_udf_impl(int fn_id, const int64_t* ts, const double* val, const uint32_t* off,
                           const uint32_t* len, const int64_t* eval_ts, size_t nwin, int64_t range_length,
                           double param0, double param1, double* out, uint8_t* valid, int sliding) {
  if (fn_id == ORC_FN_RATE || fn_id == ORC_FN_INCREASE || fn_id == ORC_FN_DELTA) {
    /* ExtrapolatedRate<IS_COUNTER,IS_RATE>::calc    extrapolate_rate.rs:133-288 */
    const int is_counter = fn_id != ORC_FN_DELTA;
    const int is_rate = fn_id == ORC_FN_RATE;
    double range_length_secs = (double)range_length / 1000.0;
    double counter_correction = 0.0;
    size_t prev_offset = SIZE_MAX, prev_length = 0;
    for (size_t index = 0; index < nwin; index++) {
      size_t offset = off[index], length = len[index];
      if (length < 2) { /* :206-210 */
        out[index] = 0.0;
        valid[index] = 0;
        prev_offset = SIZE_MAX;
        continue;
      }
      size_t end = offset + length;
      double first_value = val[offset];
      double last_value = val[end - 1];
      double result_value;
      if (is_counter) {
        if (sliding && prev_offset != SIZE_MAX && offset == prev_offset + 1 && length == prev_length) {
          /* :219-225 */
          if (val[prev_offset + 1] < val[prev_offset]) counter_correction -= val[prev_offset];
          if (val[end - 1] < val[end - 2]) counter_correction += val[end - 2];
        } else { /* :226-233 */
          counter_correction = 0.0;
          for (size_t i = offset; i + 1 < end; i++)
            if (val[i + 1] < val[i]) counter_correction += val[i];
        }
        result_value = last_value - first_value + counter_correction;
      } else {
        result_value = last_value - first_value;
      }
      prev_offset = offset;
      prev_length = length;

      int64_t first_ts = ts[offset];
      int64_t last_ts = ts[end - 1];
      int64_t range_end = eval_ts[index];
      int64_t range_start = range_end - range_length;
      double sampled_interval_ms = (double)(last_ts - first_ts);
      double average_interval_ms = sampled_interval_ms / (double)(length - 1);
      double duration_to_start_ms = (double)(first_ts - range_start);
      double duration_to_end_ms = (double)(range_end - last_ts);
      if (is_counter && result_value > 0.0 && first_value >= 0.0) { /* :254-261 */
        double duration_to_zero = sampled_interval_ms * (first_value / result_value);
        if (duration_to_zero < duration_to_start_ms) duration_to_start_ms = duration_to_zero;
      }
      double extrapolation_threshold = average_interval_ms * 1.1;
      double extrapolated_interval_ms = sampled_interval_ms;
      if (duration_to_start_ms < extrapolation_threshold)
        extrapolated_interval_ms += duration_to_start_ms;
      else
        extrapolated_interval_ms += average_interval_ms / 2.0;
      if (duration_to_end_ms < extrapolation_threshold)
        extrapolated_interval_ms += duration_to_end_ms;
      else
        extrapolated_interval_ms += average_interval_ms / 2.0;
      double factor = extrapolated_interval_ms / sampled_interval_ms;
      if (is_rate) factor /= range_length_secs;
      out[index] = result_value * factor;
      valid[index] = 1;
    }
    return;
  }
  if (fn_id == ORC_FN_IRATE || fn_id == ORC_FN_IDELTA) {
    /* IDelta<IS_RATE>::calc                          idelta.rs:113-153 */
    const int is_rate = fn_id == ORC_FN_IRATE;
    for (size_t index = 0; index < nwin; index++) {
      size_t o = off[index], l = len[index];
      if (l < 2) {
        out[index] = 0.0;
        valid[index] = 0;
        continue;
      }
      size_t last = o + l - 1, prev = last - 1;
      double sampled_interval = (double)(ts[last] - ts[prev]) / 1000.0;
      double last_value = val[last], prev_value = val[prev];
      if (!is_rate) {
        out[index] = last_value - prev_value;
      } else {
        double rv = last_value < prev_value ? last_value : last_value - prev_value;
        out[index] = rv / sampled_interval;
      }
      valid[index] = 1;
    }
    return;
  }
  for (size_t index = 0; index < nwin; index++) {
    size_t o = off[index], l = len[index];
    double r = 0.0;
    int some;
    if (fn_id == ORC_FN_PREDICT_LINEAR) { /* predict_linear.rs:163-199 */
      some = 0;
      if (l >= 2) {
        double slope, icpt;
        if (orc_linear_regression(ts + o, val + o, l, ts[o + l - 1], &slope, &icpt)) {
          /* `t as f64` where t is the i64 second offset argument */
          r = slope * (double)(int64_t)param0 + icpt;
          some = 1;
        }
      }
    } else if (fn_id == ORC_FN_QUANTILE_OVER_TIME) { /* quantile.rs:150-190: always Some */
      r = orc_quantile(val + o, l, param0);
      some = 1;
    } else if (fn_id == ORC_FN_HOLT_WINTERS) {
      r = orc_holt_winters(val + o, l, param0, param1);
      some = 1;
    } else {
      some = range_fn_body(fn_id, ts + o, val + o, l, &r);
    }
    out[index] = some ? r : 0.0;
    valid[index] = (uint8_t)some;
  }
}

void orc_range_udf(int fn_id, const int64_t* ts, const double* val, const uint32_t* off,
                   const uint32_t* len, const int64_t* eval_ts, size_t nwin, int64_t range_length,
                   double param0, double param1, double* out, uint8_t* valid) {
  range_udf_impl(fn_id, ts, val, off, len, eval_ts, nwin, range_length, param0, param1, out, valid, 1);
}
void orc_range_udf_rescan(int fn_id, const int64_t* ts, const double* val, const uint32_t* off,
                          const uint32_t* len, const int64_t* eval_ts, size_t nwin, int64_t range_length,
                          double param0, double param1, double* out, uint8_t* valid) {
  range_udf_impl(fn_id, ts, val, off, len, eval_ts, nwin, range_length, param0, param1, out, valid, 0);
}

/* ------------------------------------------------------------------------------------------
 * Whole sub-plan drivers.
 * ---------------------------------------------------------------------------------------- */

static void scatter_series_result(const orc_params* p, size_t s, int64_t T, int64_t Tw, int64_t start2,
                                  int64_t nwin, const double* r, const uint8_t* v, double* out,
                                  uint32_t* valid_words) {
  /* window j of the series is eval time start2 + j*interval == global step k0 + j */
  int64_t k0 = (start2 - p->start) / p->interval;
  for (int64_t j = 0; j < nwin; j++) {
    int64_t k = k0 + j;
    if (k < 0 || k >= T) continue;
    if (v[j]) {
      out[s * (size_t)T + (size_t)k] = r[j];
      valid_words[s * (size_t)Tw + (size_t)(k >> 5)] |= 1u << (k & 31);
    }
  }
}

typedef void (*range_udf_fn)(int, const int64_t*, const double*, const uint32_t*, const uint32_t*, const int64_t*,
                             size_t, int64_t, double, double, double*, uint8_t*);

void orc_range_query_flat(const orc_params* p, const int64_t* ts, const double* val,
                          const uint64_t* offsets, size_t s_begin, size_t s_end, double* out,
                          uint32_t* valid_words, int rescan) {
  const range_udf_fn udf = rescan ? orc_range_udf_rescan : orc_range_udf;
  int64_t T = orc_num_steps(p->start, p->end, p->interval);
  int64_t Tw = (T + 31) / 32;
  size_t cap = 0;
  for (size_t s = s_begin; s < s_end; s++) {
    size_t n = (size_t)(offsets[s + 1] - offsets[s]);
    if (n > cap) cap = n;
  }
  int64_t* nts = (int64_t*)malloc((cap + 1) * sizeof(int64_t));
  double* nval = (double*)malloc((cap + 1) * sizeof(double));
  uint32_t* off = (uint32_t*)malloc((size_t)(T + 1) * sizeof(uint32_t));
  uint32_t* len = (uint32_t*)malloc((size_t)(T + 1) * sizeof(uint32_t));
  int64_t* ets = (int64_t*)malloc((size_t)(T + 1) * sizeof(int64_t));
  double* r = (double*)malloc((size_t)(T + 1) * sizeof(double));
  uint8_t* v = (uint8_t*)malloc((size_t)(T + 1));
  for (size_t s = s_begin; s < s_end; s++) {
    memset(out + s * (size_t)T, 0, (size_t)T * sizeof(double));
    memset(valid_words + s * (size_t)Tw, 0, (size_t)Tw * sizeof(uint32_t));
    size_t o = (size_t)offsets[s], n = (size_t)(offsets[s + 1] - offsets[s]);
    size_t m = orc_normalize(ts + o, val + o, n, p->offset, p->filter_nan, nts, nval);
    int64_t s2, e2;
    int64_t nwin = orc_calculate_range(nts, m, p->start, p->end, p->interval, p->range, off, len, &s2, &e2);
    int all_empty = 1;
    for (int64_t j = 0; j < nwin; j++)
      if (len[j] != 0) all_empty = 0;
    if (nwin == 0 || all_empty) continue; /* range_manipulate.rs:641-643 */
    for (int64_t j = 0; j < nwin; j++) ets[j] = s2 + j * p->interval;
    udf(p->fn_id, nts, nval, off, len, ets, (size_t)nwin, p->range, p->param0, p->param1, r, v);
    scatter_series_result(p, s, T, Tw, s2, nwin, r, v, out, valid_words);
  }
  free(nts); free(nval); free(off); free(len); free(ets); free(r); free(v);
}

void orc_range_query_faithful(const orc_params* p, const int64_t* ts, const double* val,
                              const uint32_t* sid, const uint64_t* offsets, size_t s_begin, size_t s_end,
                              double* out, uint32_t* valid_words, int rescan) {
  const range_udf_fn udf = rescan ? orc_range_udf_rescan : orc_range_udf;
  int64_t T = orc_num_steps(p->start, p->end, p->interval);
  int64_t Tw = (T + 31) / 32;
  for (size_t s = s_begin; s < s_end; s++) {
    memset(out + s * (size_t)T, 0, (size_t)T * sizeof(double));
    memset(valid_words + s * (size_t)Tw, 0, (size_t)Tw * sizeof(uint32_t));
    size_t o = (size_t)offsets[s], n = (size_t)(offsets[s + 1] - offsets[s]);
    if (n == 0) continue;
    /* SeriesDivide: row-wise id compares (series_divide.rs:658-667) then concat_batches (:567) */
    size_t same_until = 0;
    while (same_until + 1 < n && sid[o + same_until] == sid[o + same_until + 1]) same_until++;
    (void)same_until;
    int64_t* b_ts = (int64_t*)malloc(n * 8);
    double* b_val = (double*)malloc(n * 8);
    uint32_t* b_sid = (uint32_t*)malloc(n * 4);
    memcpy(b_ts, ts + o, n * 8);
    memcpy(b_val, val + o, n * 8);
    memcpy(b_sid, sid + o, n * 4);
    /* SeriesNormalize: biased ts array (normalize.rs:400-406), Vec<bool> filter + filter_record_batch (:417-430) */
    int64_t* n_ts = (int64_t*)malloc(n * 8);
    double* n_val = (double*)malloc(n * 8);
    uint32_t* n_sid = (uint32_t*)malloc(n * 4);
    uint8_t* keep = (uint8_t*)malloc(n);
    size_t m = 0;
    for (size_t i = 0; i < n; i++) keep[i] = !(p->filter_nan && isnan(b_val[i]));
    for (size_t i = 0; i < n; i++)
      if (keep[i]) {
        n_ts[m] = b_ts[i] + p->offset;
        n_val[m] = b_val[i];
        n_sid[m] = b_sid[i];
        m++;
      }
    /* RangeManipulate::manipulate (range_manipulate.rs:636-681) */
    uint32_t* off = (uint32_t*)malloc((size_t)(T + 1) * 4);
    uint32_t* len = (uint32_t*)malloc((size_t)(T + 1) * 4);
    int64_t s2, e2;
    int64_t nwin = orc_calculate_range(n_ts, m, p->start, p->end, p->interval, p->range, off, len, &s2, &e2);
    int all_empty = 1;
    for (int64_t j = 0; j < nwin; j++)
      if (len[j] != 0) all_empty = 0;
    if (nwin > 0 && !all_empty) {
      /* two RangeArray dictionaries: packed i64 keys offset | len<<32 (range_array.rs:247-254) */
      int64_t* keys_val = (int64_t*)malloc((size_t)nwin * 8);
      int64_t* keys_ts = (int64_t*)malloc((size_t)nwin * 8);
      for (int64_t j = 0; j < nwin; j++) {
        keys_val[j] = (int64_t)((uint64_t)off[j] | ((uint64_t)len[j] << 32));
        keys_ts[j] = keys_val[j];
      }
      /* take(tag, [0; T]) (range_manipulate.rs:666-669) + aligned ts array (:671-676) */
      uint32_t* t_sid = (uint32_t*)malloc((size_t)nwin * 4);
      int64_t* ets = (int64_t*)malloc((size_t)nwin * 8);
      for (int64_t j = 0; j < nwin; j++) {
        t_sid[j] = n_sid[0];
        ets[j] = s2 + j * p->interval;
      }
      /* UDF: validates both key arrays match (extrapolate_rate.rs:166-177), unpacks, loops */
      uint32_t* u_off = (uint32_t*)malloc((size_t)nwin * 4);
      uint32_t* u_len = (uint32_t*)malloc((size_t)nwin * 4);
      int same = 1;
      for (int64_t j = 0; j < nwin; j++) {
        if (keys_val[j] != keys_ts[j]) same = 0;
        u_off[j] = (uint32_t)((uint64_t)keys_ts[j] & 0xffffffffu);
        u_len[j] = (uint32_t)((uint64_t)keys_ts[j] >> 32);
      }
      double* r = (double*)malloc((size_t)nwin * 8);
      uint8_t* v = (uint8_t*)malloc((size_t)nwin);
      if (same)
        udf(p->fn_id, n_ts, n_val, u_off, u_len, ets, (size_t)nwin, p->range, p->param0, p->param1, r, v);
      /* Filter value IS NOT NULL (planner.rs:1063): copies the surviving rows of every column */
      double* f_val = (double*)malloc((size_t)nwin * 8);
      int64_t* f_ts = (int64_t*)malloc((size_t)nwin * 8);
      uint32_t* f_sid = (uint32_t*)malloc((size_t)nwin * 4);
      size_t rows = 0;
      for (int64_t j = 0; j < nwin; j++)
        if (same && v[j]) {
          f_val[rows] = r[j];
          f_ts[rows] = ets[j];
          f_sid[rows] = t_sid[j];
          rows++;
        }
      for (size_t q = 0; q < rows; q++) {
        int64_t k = (f_ts[q] - p->start) / p->interval;
        if (k < 0 || k >= T) continue;
        out[s * (size_t)T + (size_t)k] = f_val[q];
        valid_words[s * (size_t)Tw + (size_t)(k >> 5)] |= 1u << (k & 31);
      }
      free(keys_val); free(keys_ts); free(t_sid); free(ets); free(u_off); free(u_len);
      free(r); free(v); free(f_val); free(f_ts); free(f_sid);
    }
    free(off); free(len); free(keep);
    free(b_ts); free(b_val); free(b_sid); free(n_ts); free(n_val); free(n_sid);
  }
}

typedef struct {
  const orc_params* p;
  const int64_t* ts;
  const double* val;
  const uint32_t* sid;
  const uint64_t* offsets;
  size_t s_begin, s_end;
  double* out;
  uint32_t* valid_words;
  int faithful;
} mt_job;

static void* mt_worker(void* arg) {
  mt_job* j = (mt_job*)arg;
  const int rescan = (j->faithful & ORC_RESCAN) != 0;
  if (j->faithful & 1)
    orc_range_query_faithful(j->p, j->ts, j->val, j->sid, j->offsets, j->s_begin, j->s_end, j->out, j->valid_words,
                             rescan);
  else
    orc_range_query_flat(j->p, j->ts, j->val, j->offsets, j->s_begin, j->s_end, j->out, j->valid_words, rescan);
  return NULL;
}

int orc_range_query_mt(const orc_params* p, const int64_t* ts, const double* val, const uint32_t* sid,
                       const uint64_t* offsets, size_t n_series, double* out, uint32_t* valid_words,
                       int n_threads, int faithful) {
  if (n_threads < 1) n_threads = 1;
  if ((size_t)n_threads > n_series && n_series > 0) n_threads = (int)n_series;
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)n_threads);
  mt_job* jobs = (mt_job*)malloc(sizeof(mt_job) * (size_t)n_threads);
  size_t per = (n_series + (size_t)n_threads - 1) / (size_t)n_threads;
  int started = 0;
  for (int i = 0; i < n_threads; i++) {
    size_t b = (size_t)i * per, e = b + per;
    if (b > n_series) b = n_series;
    if (e > n_series) e = n_series;
    mt_job jb = {p, ts, val, sid, offsets, b, e, out, valid_words, faithful};
    jobs[i] = jb;
    if (pthread_create(&th[i], NULL, mt_worker, &jobs[i]) != 0) break;
    started++;
  }
  for (int i = 0; i < started; i++) pthread_join(th[i], NULL);
  int ok = started == n_threads;
  free(th);
  free(jobs);
  return ok ? 0 : -1;
}

void orc_instant_query(const int64_t* ts, const double* val, const uint64_t* offsets, size_t n_series,
                       int64_t start, int64_t end, int64_t interval, int64_t lookback, int64_t offset,
                       double* out, uint32_t* valid_words) {
  int64_t T = orc_num_steps(start, end, interval);
  int64_t Tw = (T + 31) / 32;
  uint64_t* take = (uint64_t*)malloc((size_t)(T + 1) * 8);
  int64_t* ots = (int64_t*)malloc((size_t)(T + 1) * 8);
  size_t cap = 0;
  for (size_t s = 0; s < n_series; s++) {
    size_t n = (size_t)(offsets[s + 1] - offsets[s]);
    if (n > cap) cap = n;
  }
  int64_t* bts = (int64_t*)malloc((cap + 1) * 8);
  for (size_t s = 0; s < n_series; s++) {
    memset(out + s * (size_t)T, 0, (size_t)T * 8);
    memset(valid_words + s * (size_t)Tw, 0, (size_t)Tw * 4);
    size_t o = (size_t)offsets[s], n = (size_t)(offsets[s + 1] - offsets[s]);
    /* SeriesNormalize with need_filter_out_nan=false is only planned when offset != 0
     * (planner.rs:886-928); it just biases ts. */
    for (size_t i = 0; i < n; i++) bts[i] = ts[o + i] + offset;
    int64_t m = orc_instant_manipulate(bts, val + o, n, start, end, interval, lookback, take, ots);
    for (int64_t q = 0; q < m; q++) {
      int64_t k = (ots[q] - start) / interval;
      if (k < 0 || k >= T) continue;
      out[s * (size_t)T + (size_t)k] = val[o + take[q]];
      valid_words[s * (size_t)Tw + (size_t)(k >> 5)] |= 1u << (k & 31);
    }
  }
  free(take); free(ots); free(bts);
}

/* By-label aggregate.  Keys = by-labels + eval ts (planner.rs:1413-1436), accumulators are
 * DataFusion's: sum/avg = plain f64 +=, count = non-null rows, min/max = f64 compare,
 * stddev_pop/var_pop = Welford (datafusion functions-aggregate variance.rs, unpinned). */
void orc_group_aggregate(int op, const double* vals, const uint32_t* valid_words, const uint32_t* gid,
                         size_t n_series, size_t n_groups, size_t T, double* out_val, uint32_t* out_cnt) {
  size_t Tw = (T + 31) / 32;
  double* m2 = NULL;
  double* mean = NULL;
  if (op == 5 || op == 6) {
    m2 = (double*)calloc(n_groups * T, 8);
    mean = (double*)calloc(n_groups * T, 8);
  }
  memset(out_val, 0, n_groups * T * 8);
  memset(out_cnt, 0, n_groups * T * 4);
  for (size_t s = 0; s < n_series; s++) {
    size_t g = gid[s];
    if (g >= n_groups) continue;
    for (size_t k = 0; k < T; k++) {
      if (!((valid_words[s * Tw + (k >> 5)] >> (k & 31)) & 1u)) continue;
      double x = vals[s * T + k];
      size_t idx = g * T + k;
      uint32_t c = out_cnt[idx];
      switch (op) {
        case 0:
        case 1: out_val[idx] += x; break;
        case 2: break;
        /* min / max: the total order of f64::total_cmp (arrow-rs aggregate min / max and DataFusion's MinMax
         * accumulators compare floats that way): a positive NaN is the greatest value, so max() of a group with a
         * NaN member is NaN while min() ignores it (-NaN sorts lowest).  Third-party semantics, restated. */
        case 3: if (c == 0 || total_key(x) < total_key(out_val[idx])) out_val[idx] = x; break;
        case 4: if (c == 0 || total_key(x) > total_key(out_val[idx])) out_val[idx] = x; break;
        default: {
          double new_count = (double)c + 1.0;
          double delta1 = x - mean[idx];
          double new_mean = delta1 / new_count + mean[idx];
          double delta2 = x - new_mean;
          m2[idx] += delta1 * delta2;
          mean[idx] = new_mean;
        }
      }
      out_cnt[idx] = c + 1;
    }
  }
  for (size_t i = 0; i < n_groups * T; i++) {
    uint32_t c = out_cnt[i];
    if (c == 0) {
      out_val[i] = 0.0;
      continue;
    }
    if (op == 1) out_val[i] = out_val[i] / (double)c;
    if (op == 2) out_val[i] = (double)c;
    if (op == 6) out_val[i] = m2[i] / (double)c;
    if (op == 5) out_val[i] = sqrt(m2[i] / (double)c);
  }
  free(m2);
  free(mean);
}

void orc_histogram_quantile(double phi, const double* le, size_t B, const double* rates,
                            const uint32_t* valid_words, size_t n_hist, size_t T, double* out,
                            uint32_t* out_valid_words) {
  size_t Tw = (T + 31) / 32;
  double* counters = (double*)malloc(B * 8);
  memset(out, 0, n_hist * T * 8);
  memset(out_valid_words, 0, n_hist * Tw * 4);
  for (size_t h = 0; h < n_hist; h++) {
    for (size_t k = 0; k < T; k++) {
      int complete = 1;
      for (size_t b = 0; b < B; b++) {
        size_t s = h * B + b;
        if (!((valid_words[s * Tw + (k >> 5)] >> (k & 31)) & 1u)) {
          complete = 0;
          break;
        }
        counters[b] = rates[s * T + k];
      }
      if (!complete) continue;
      int err;
      double r = orc_histogram_evaluate_row(phi, le, counters, B, &err);
      if (err) r = NAN; /* unwrap_or(NaN) histogram_fold.rs:806 */
      out[h * T + k] = r;
      out_valid_words[h * Tw + (k >> 5)] |= 1u << (k & 31);
    }
  }
  free(counters);
}

/* ------------------------------------------------------------------------------------------
 * Synthetic workload (BASELINE.md §4).  Value shapes follow benches/bench_range_fn.rs:60-82
 * (monotonic counter, resetting counter), written in closed form so a GPU thread can produce
 * sample (s,i) independently; every term is a multiple of 0.25 well below 2^53, so the closed
 * form equals the sequential recurrence bit for bit.
 * ---------------------------------------------------------------------------------------- */
static uint64_t mix64(uint64_t x) { /* splitmix64 finaliser */
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

static double synth_value(uint64_t s, uint32_t i, int with_resets) {
  double scale = (double)(1 + s % 13);
  if (!with_resets) {
    /* v[i] = sum_{j<=i} (1 + (j%7)*0.25) */
    uint32_t q = (i + 1) / 7, r = (i + 1) % 7; /* q full cycles then r terms j%7 = 0..r-1 */
    double v = (double)q * 12.25 + (double)r + 0.25 * (double)(r * (r - 1) / 2);
    if (r == 0) v = (double)q * 12.25;
    return v * scale;
  }
  /* reset to 1.0 when i>0 && (i+s)%37==0, else += 1 + (i%5)*0.5 ; v[-1] = 0 */
  uint32_t ph = (uint32_t)((i + s) % 37);
  uint32_t p; /* index of the last reset <= i, or UINT32_MAX if none */
  int has = 0;
  if (i >= ph && (i - ph) > 0) {
    p = i - ph;
    has = 1;
  } else {
    p = 0;
  }
  double v = has ? 1.0 : 0.0;
  uint32_t j0 = has ? p + 1 : 0;
  for (uint32_t j = j0; j <= i; j++) v += 1.0 + (double)(j % 5) * 0.5;
  return v * scale;
}

void orc_synth_fill(uint64_t series_begin, uint64_t n_series, uint32_t n_samples, int64_t t0,
                    int64_t scrape_ms, uint32_t jitter_ms, int with_resets, uint64_t seed, int64_t* ts,
                    double* val, uint32_t* sid) {
  for (uint64_t ls = 0; ls < n_series; ls++) {
    uint64_t s = series_begin + ls;
    for (uint32_t i = 0; i < n_samples; i++) {
      size_t row = (size_t)ls * n_samples + i;
      uint64_t h = mix64(seed ^ mix64(s * 0x100000001B3ull + i));
      int64_t jit = jitter_ms ? (int64_t)(h % jitter_ms) : 0;
      ts[row] = t0 + (int64_t)i * scrape_ms + jit;
      val[row] = synth_value(s, i, with_resets);
      if (sid) sid[row] = (uint32_t)ls;
    }
  }
}
