// b2p_subquery.cuh — PromQL subquery `fn(<expr>[range:step])` (K13): a child's dense [rows x T'] grid on the inner eval
// steps t'_k = start' + k * interval' becomes the per-series sample rows the range tiers read (b2p_range_eval_dev's
// layout: ts / val columns, row offsets), with no host round trip:
//   subquery_count_kernel    one warp per row: its valid cells, by popcounts of its validity words, into offsets[row]
//   (CUB DeviceScan::ExclusiveSum over offsets[rows + 1], in place: the first sample of every row, and the total)
//   subquery_scatter_kernel  one warp per row, a validity word at a time, lane = step: each valid cell k to
//                            ts = start' + k * interval' and val = the cell, at offsets[row] + its rank among the row's
//                            valid cells
// The range call then runs the existing tiers over these rows; none of the range functions is evaluated here.
//
// The reference plans the inner expression on its own grid (start' = start - range + interval', the outer end) and puts
// RangeManipulate(start, end, interval, range) directly over it, with no SeriesNormalize in between
// (prom_subquery_expr_to_plan, src/query/src/promql/planner.rs:292-332).  So a child cell is a sample whatever its
// value: NaN is not filtered, and the value is a bit copy (NaN payloads and -0.0 survive).  A row with every cell valid
// is exactly regular, with cadence interval'.
#pragma once
#include <cstdint>

#include "b2p_cells.cuh"

namespace b2p {

constexpr uint64_t kSqBatchCells = 1ull << 27;  // grid cells of one batch of rows: 16 B each of scratch, 2.1 GB

struct SubqueryArgs {
  const double* vals;             // [rows x T] (the batch's first row)
  const uint32_t* valid;          // [rows x Tw]
  uint64_t T;
  uint32_t Tw, rows;
  int64_t start, interval;        // the inner grid: step k is start + k * interval
  unsigned long long* offsets;    // [rows + 1]: the counts, then (scanned) each row's first sample and the total
  int64_t* ts;                    // [total] sample rows, in row order
  double* val;
};

// bits of validity word w that are steps of the grid (a word past T's last step may carry stray bits)
__device__ __forceinline__ uint32_t sq_word(const SubqueryArgs& a, uint64_t row, uint32_t w) {
  return grid_word(a.valid, row, a.Tw, w, a.T);
}

__global__ void __launch_bounds__(256) subquery_count_kernel(const SubqueryArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  if (warp0 == 0 && lane == 0) a.offsets[a.rows] = 0ull;
  for (uint64_t r = warp0; r < a.rows; r += n_warps) {
    uint32_t n = 0;
    for (uint32_t w = lane; w < a.Tw; w += 32) n += __popc(sq_word(a, r, w));
    n = __reduce_add_sync(0xffffffffu, n);
    if (lane == 0) a.offsets[r] = n;
  }
}

__global__ void __launch_bounds__(256) subquery_scatter_kernel(const SubqueryArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t below = (1u << lane) - 1u;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t r = warp0; r < a.rows; r += n_warps) {
    unsigned long long base = a.offsets[r];
    const long long* row = reinterpret_cast<const long long*>(a.vals) + r * a.T;
    for (uint32_t w = 0; w < a.Tw; ++w) {
      const uint32_t word = sq_word(a, r, w);
      const uint64_t k = (uint64_t)w * 32 + lane;
      if ((word >> lane) & 1u) {
        const unsigned long long pos = base + __popc(word & below);
        a.ts[pos] = a.start + (int64_t)k * a.interval;
        reinterpret_cast<long long*>(a.val)[pos] = __ldcs(row + k);  // the cell's bits
      }
      base += __popc(word);
    }
  }
}

}  // namespace b2p
