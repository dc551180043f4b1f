// b2p_fields.cuh — PromQL selectors over a table with several Float64 field columns (one timestamp column, F value
// columns, the same rows):
//   K16 nan_union_kernel        SeriesNormalize's NaN filter across fields (normalize.rs:415-428): a row is dropped when
//                               ANY Float64 column is NaN, so every field of such a row becomes NaN.  In place, over the
//                               context's copies of the columns; afterwards each range tier drops, per field, exactly
//                               the rows the reference drops for all of them.
//   K17 instant_fields_kernel   InstantManipulate over F fields (instant_manipulate.rs:473-585): one lookback search
//                               per (series, step), the stale-NaN test on field 0 only (the planner hands it the first
//                               field, planner.rs:922), then F gathers from the chosen row.
//   K18 valid_and_kernel        the closing Filter: the conjunction of `IS NOT NULL` over every field
//                               (planner.rs:2774-2791), word by word over F validity bitmaps, bits past T cleared.
//
// HBM traffic: K16 reads 8F B per row and writes 8 B per field it turns into NaN; K17 reads K4's timestamps once and
// writes 8F B per (series, step) plus one validity bit; K18 reads 4F B and writes 4 B per validity word.
#pragma once
#include <cstdint>

#include "b2p_cells.cuh"
#include "b2p_kernels.cuh"

namespace b2p {

constexpr int kMaxFields = B2P_MAX_FIELDS;

// ---- K16 --------------------------------------------------------------------------------------------------------
// F columns of n_rows values, field f at vals + f * stride.  Thread per row: the F loads of a warp are coalesced.
__global__ void __launch_bounds__(256) nan_union_kernel(double* __restrict__ vals, uint64_t stride, int F,
                                                        uint64_t n_rows) {
  const double nan = __longlong_as_double(0x7FF8000000000000ll);  // f64::NAN
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t nan_fields = 0;  // bit f: field f is NaN in this row (F <= 64)
    for (int f = 0; f < F; ++f)
      if (isnan(vals[(uint64_t)f * stride + r])) nan_fields |= 1ull << f;
    if (!nan_fields) continue;
    for (int f = 0; f < F; ++f)
      if (!((nan_fields >> f) & 1ull)) vals[(uint64_t)f * stride + r] = nan;
  }
}

// NULL slots of one field (its Arrow validity bitmap: bit r of byte r / 8, 1 = a value): sets *flag when rows
// [0, n_rows) hold one.  A multi-field call reads it only to refuse the families it cannot reproduce over NULL slots.
__global__ void __launch_bounds__(256) null_slots_kernel(const uint8_t* __restrict__ bitmap, uint64_t n_rows,
                                                         uint32_t* flag) {
  const uint64_t n_bytes = (n_rows + 7) / 8;
  bool any = false;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_bytes; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t left = n_rows - i * 8;
    const uint32_t mask = left >= 8 ? 0xFFu : (1u << left) - 1u;
    any |= (~(uint32_t)bitmap[i] & mask) != 0;
  }
  if (__syncthreads_or(any) && threadIdx.x == 0) atomicOr(flag, 1u);
}

// ---- K17 --------------------------------------------------------------------------------------------------------
struct FieldsInstantArgs {
  InstantArgs g;                   // grid, lookback, offsets, timestamps and the validity bitmap; g.val is field 0
  int F;
  const double* vals[kMaxFields];  // field columns [n_rows]
  double* outs[kMaxFields];        // [n_series x T] per field
};

// K4 (instant_kernel) with F gathers: warp per series, lane per eval step.  STALE_TEST = false when field 0 is Int64
// (b2p_instant_select_fields_i64): the reference looks for stale NaNs through a Float64 downcast only
// (instant_manipulate.rs:490-527), so an Int64 field 0 is never tested, even where its bits are a NaN double.
template <bool STALE_TEST = true>
__global__ void __launch_bounds__(kWarpsPerCta * 32) instant_fields_kernel(const __grid_constant__ FieldsInstantArgs fa) {
  const InstantArgs& a = fa.g;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t total_warps = gridDim.x * kWarpsPerCta;
  for (uint32_t s = blockIdx.x * kWarpsPerCta + warp; s < a.n_series; s += total_warps) {
    const uint64_t row0 = a.offsets[s], row1 = a.offsets[s + 1];
    const uint64_t n = row1 - row0;
    const size_t cell0 = (size_t)s * (size_t)a.T;
    uint32_t* vw_s = a.valid + (size_t)s * a.Tw;
    const int64_t* ts = a.ts + row0;
    int64_t k_lo = a.T, k_hi = -1;
    if (n > 0) {
      const int64_t first_ts = ts[0] + a.offset, last_ts = ts[n - 1] + a.offset;
      const int64_t last_useful = a.lookback > 0 ? last_ts + a.lookback - 1 : last_ts;
      const int64_t max_start = first_ts > a.start ? first_ts : a.start;
      const int64_t min_end = last_useful < a.end ? last_useful : a.end;
      const int64_t aligned_start = a.start + (max_start - a.start) / a.interval * a.interval;
      const int64_t aligned_end = a.end - (a.end - min_end) / a.interval * a.interval;
      if (aligned_start <= aligned_end) {
        k_lo = (aligned_start - a.start) / a.interval;
        k_hi = floor_div(aligned_end - a.start, a.interval);
      }
    }
    for (int64_t kb = 0; kb < a.T; kb += 32) {
      const int64_t k = kb + lane;
      bool ok = false;
      uint64_t row = 0;  // the chosen row (global index) when ok
      if (k < a.T && k >= k_lo && k <= k_hi) {
        const int64_t te = a.start + k * a.interval;
        uint64_t lo = 0, hi = n;
        while (lo < hi) {
          const uint64_t mid = (lo + hi) >> 1;
          if (ts[mid] + a.offset <= te) lo = mid + 1; else hi = mid;
        }
        if (lo > 0) {
          uint64_t j = lo - 1;
          const int64_t t = ts[j] + a.offset;
          if (t == te)
            while (j > 0 && ts[j - 1] + a.offset == te) --j;
          const bool fresh = (a.lookback > 0) ? (t + a.lookback > te) : (t == te);
          if (fresh && !(STALE_TEST && isnan(fa.vals[0][row0 + j]))) {  // the staleness test reads field 0 alone
            ok = true;
            row = row0 + j;
          }
        }
      }
      if (k < a.T)
        for (int f = 0; f < fa.F; ++f) fa.outs[f][cell0 + k] = ok ? fa.vals[f][row] : 0.0;
      const uint32_t word = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) vw_s[kb >> 5] = word;
    }
  }
}

// ---- K18 --------------------------------------------------------------------------------------------------------
struct ValidAndArgs {
  int F;
  const uint32_t* in[kMaxFields];  // [rows x Tw] per field; out may be one of them
  uint32_t* out;                   // [rows x Tw]
  uint64_t n_words;                // rows x Tw
  uint32_t Tw;
  uint64_t T;
};

// thread per validity word
__global__ void __launch_bounds__(256) valid_and_kernel(const __grid_constant__ ValidAndArgs a) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n_words; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t w = grid_mask(a.Tw, (uint32_t)(i % a.Tw), a.T);
    for (int f = 0; f < a.F && w; ++f) w &= __ldg(a.in[f] + i);
    a.out[i] = w;
  }
}

}  // namespace b2p
