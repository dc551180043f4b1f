// b2p_sort.cuh — PromQL sort / sort_desc (K14): the valid cells of a dense [rows x T] grid in value order, as the
// reference's Sort(value ASC | DESC, NULLS FIRST) over the child's rows orders them (planner.rs:1060-1089).
//   (K13's count kernel and CUB's exclusive scan: each row's first position among the valid cells, and the total)
//   sort_scatter_kernel  one warp per row, a validity word at a time, lane = step: each valid cell k of row r to
//                        (key, r * T + k) at the row's first position + its rank among the row's valid cells
//   (CUB DeviceRadixSort::SortPairs over the (key, cell) pairs, all 64 key bits)
// The key is the cell's f64 total-order key as an unsigned integer, total_key(v) ^ 2^63 (-NaN < -inf < .. < -0.0 <
// +0.0 < .. < +inf < +NaN, every bit pattern its own key), and its bitwise NOT for sort_desc.  The pairs enter the
// radix sort in row-major order and the sort is stable, so equal values keep the child's row, then step, order in
// both directions.  CUB's floating-point key mode is not used: it ranks -0.0 and +0.0 equal and does not put negative
// NaNs where total_cmp does.  An Int64 grid (b2p_sort_cells_i64) keys on its bits ^ 2^63 instead: the kernels take the
// key as a template parameter (F64Key / I64Key, b2p_window.cuh).
// Several fields (sort over a multi-field node: Sort(f0, f1, .. each ASC | DESC NULLS FIRST), planner.rs:2743-2749)
// sort least significant key first: the scatter keys on the last field, and for each earlier field
//   sort_rekey_kernel    one thread per pair: the pair's key reloaded from that field at its cell
// precedes one more stable radix sort.  Stability makes the order lexicographic over the fields.
#pragma once
#include <cstdint>

#include "b2p_cells.cuh"
#include "b2p_window.cuh"

namespace b2p {

struct SortArgs {
  const double* vals;                   // [rows x T]
  const uint32_t* valid;                // [rows x Tw]
  uint64_t T;
  uint32_t Tw, rows;
  int desc;
  const unsigned long long* offsets;    // [rows + 1]: each row's first position (scanned counts)
  unsigned long long* keys;             // [total]
  unsigned long long* cells;            // [total]
};

template <class Key = F64Key>
__global__ void __launch_bounds__(256) sort_scatter_kernel(const SortArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t below = (1u << lane) - 1u;
  const unsigned long long flip = a.desc ? ~0ull : 0ull;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t r = warp0; r < a.rows; r += n_warps) {
    unsigned long long base = a.offsets[r];
    const double* row = a.vals + r * a.T;
    for (uint32_t w = 0; w < a.Tw; ++w) {
      const uint32_t word = grid_word(a.valid, r, a.Tw, w, a.T);
      const uint64_t k = (uint64_t)w * 32 + lane;
      if ((word >> lane) & 1u) {
        const unsigned long long pos = base + __popc(word & below);
        a.keys[pos] = Key::key(__ldcs(row + k)) ^ flip;
        a.cells[pos] = r * a.T + k;
      }
      base += __popc(word);
    }
  }
}

template <class Key = F64Key>
__global__ void __launch_bounds__(256) sort_rekey_kernel(const double* __restrict__ vals,
                                                         const unsigned long long* __restrict__ cells,
                                                         unsigned long long* __restrict__ keys, uint64_t n, int desc) {
  const unsigned long long flip = desc ? ~0ull : 0ull;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    keys[i] = Key::key(__ldg(vals + cells[i])) ^ flip;
}

}  // namespace b2p
