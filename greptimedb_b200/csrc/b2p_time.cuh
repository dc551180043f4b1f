// b2p_time.cuh — PromQL functions of the eval step alone over dense [rows x T] grids:
//   K19 step_fn_kernel<PART>   f(eval_ts[k]) at every valid cell (r, k): time() and the calendar functions
//
// The reference computes these as projections over the time index column (planner.rs:2222-2300):
//   * time(): `CAST(CAST(ts AS Int64) AS Float64) / 1000.0` (build_special_time_expr, empty_metric.rs:393-402): one
//     round-to-nearest conversion and one IEEE division, never a multiplication by 0.001 (which differs in the last bit);
//   * minute hour month year day_of_month day_of_week day_of_year: DataFusion's date_part('minute' | 'hour' | 'month' |
//     'year' | 'day' | 'dow' | 'doy', ts) on a UTC millisecond timestamp (planner.rs:3994-4009), dow with Sunday = 0 and
//     doy from 1;
//   * days_in_month: date_part('day', date_trunc('month', ts) + 1 month - 1 day), the last day of ts's month.
// The calendar is proleptic Gregorian over integer days, with floor division so that negative epochs work (the
// civil-from-days algorithm of H. Hinnant, "chrono-Compatible Low-Level Date Algorithms").  A step whose year is outside
// [-kMaxYear, kMaxYear] (chrono's NaiveDate range; the exact bound of arrow-rs' timestamp conversion is not in the
// reference tree, DESIGN.md section 8) is not computed: its cells are written 0.0 and bit 6 of the status word is set
// (-> B2P_E_INVALID).
//
// Work unit: a CTA covers W steps and floor(256 / W) rows at a time, W = 256 when T >= 256, T rounded up to a multiple
// of 32 when 32 <= T < 256, and T itself when T < 32: then one warp spans several rows and still writes consecutive
// cells (the rows of a grid are contiguous), so an instant query (T = 1) keeps every lane busy.  Each thread computes f
// of its one step once, in registers, and then streams it down the rows; the kernel's HBM traffic per cell is the
// 8-byte write plus its share of a validity word.  Validity is not changed.
#pragma once
#include <cstdint>

#include "b2p_status.cuh"
#include "b2p_window.cuh"

namespace b2p {

// must equal enum b2p_step_part of the header
enum StepPart {
  kPartTime = 0, kPartMinute, kPartHour, kPartDayOfMonth, kPartDayOfWeek, kPartDayOfYear, kPartMonth, kPartYear,
  kPartDaysInMonth, kPartCount
};
constexpr int64_t kMaxYear = 262143;
constexpr int kStepThreads = 256;

struct StepFnArgs {
  const int64_t* eval_ts;  // [T]
  const uint32_t* valid;   // [n_rows x Tw]
  uint64_t n_rows;
  uint64_t T;
  uint32_t Tw;
  uint32_t W;              // steps per CTA (step_fn_width)
  double* out;             // [n_rows x T]
  Status* status;
};

__host__ __device__ __forceinline__ int64_t floor_div64(int64_t a, int64_t b) {
  const int64_t q = a / b;
  return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q;
}

// days since 1970-01-01 of the proleptic Gregorian date (y, m, d)
__host__ __device__ __forceinline__ int64_t days_from_civil(int64_t y, int64_t m, int64_t d) {
  y -= m <= 2;
  const int64_t era = floor_div64(y, 400);
  const int64_t yoe = y - era * 400;
  const int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + doe - 719468;
}

// the date part PART of the UTC millisecond timestamp ts; false when its year is outside [-kMaxYear, kMaxYear]
template <int PART>
__host__ __device__ __forceinline__ bool step_part(int64_t ts, double* v) {
  if (PART == kPartTime) {
    *v = (double)ts / 1000.0;
    return true;
  }
  const int64_t days = floor_div64(ts, 86400000);
  const int64_t ms = ts % 86400000 + (ts % 86400000 < 0 ? 86400000 : 0);  // (days * 86400000 may not fit in 64 bits)
  // civil from days
  const int64_t z = days + 719468;
  const int64_t era = floor_div64(z, 146097);
  const int64_t doe = z - era * 146097;
  const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const int64_t doy_mar = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const int64_t mp = (5 * doy_mar + 2) / 153;
  const int64_t d = doy_mar - (153 * mp + 2) / 5 + 1;
  const int64_t m = mp < 10 ? mp + 3 : mp - 9;
  const int64_t y = yoe + era * 400 + (m <= 2);
  if (y < -kMaxYear || y > kMaxYear) return false;
  const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
  if (PART == kPartHour) *v = (double)(ms / 3600000);
  if (PART == kPartMinute) *v = (double)(ms / 60000 % 60);
  if (PART == kPartDayOfWeek) *v = (double)(days + 4 - floor_div64(days + 4, 7) * 7);  // 1970-01-01 is a Thursday
  if (PART == kPartDayOfMonth) *v = (double)d;
  if (PART == kPartMonth) *v = (double)m;
  if (PART == kPartYear) *v = (double)y;
  if (PART == kPartDayOfYear) *v = (double)(days - days_from_civil(y, 1, 1) + 1);
  if (PART == kPartDaysInMonth) *v = (double)(m == 2 ? (leap ? 29 : 28) : (m == 4 || m == 6 || m == 9 || m == 11) ? 30 : 31);
  return true;
}

// steps per CTA of K19 for a grid of T steps
inline uint32_t step_fn_width(uint64_t T) {
  if (T >= (uint64_t)kStepThreads) return kStepThreads;
  return T < 32 ? (uint32_t)(T ? T : 1) : (uint32_t)((T + 31) / 32 * 32);
}

template <int PART>
__global__ void __launch_bounds__(kStepThreads) step_fn_kernel(const StepFnArgs a) {
  const uint32_t W = a.W;
  const uint32_t sub = threadIdx.x / W;               // row within the CTA's pass
  const uint64_t k = (uint64_t)blockIdx.x * W + threadIdx.x % W;
  const uint32_t rows_per_pass = kStepThreads / W;
  if (sub >= rows_per_pass) return;                   // (the threads past the last whole row of a pass)
  double v = 0.0;
  bool ok = true;
  if (k < a.T) ok = step_part<PART>(a.eval_ts[k], &v);
  if (!ok) {
    v = 0.0;
    if (blockIdx.y == 0 && sub == 0) atomicOr(&a.status->k0_errors, kStepRangeError);
  }
  if (k >= a.T) return;
  const uint32_t w = (uint32_t)(k >> 5), bit = (uint32_t)(k & 31);
  for (uint64_t r = (uint64_t)blockIdx.y * rows_per_pass + sub; r < a.n_rows; r += (uint64_t)gridDim.y * rows_per_pass) {
    const uint32_t word = a.valid[r * a.Tw + w];
    a.out[r * a.T + k] = ((word >> bit) & 1u) ? v : 0.0;
  }
}

}  // namespace b2p
