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

#include "../../include/b200promql.h"
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

// ---- sort over rows sharded across ranks (b2p_sort_cells_allgather_dev) -------------------------------------------
// Every rank runs K14 over its own rows; the pack turns its run into one block of n entries,
//   [field 0 keys: n u64] .. [field F-1 keys: n u64][global cells: n u64],
// the key already flipped for desc and the cell row_id[r] * T + k.  Inside a rank K14 is stable in local row-major
// order, which with increasing row ids is the order of (key tuple, global cell); the merge orders every rank's entries
// by that same strict total order, so the result does not depend on which rank holds a row.
//   sort_shard_rows_kernel   row_id strictly increasing, else *bad = 1 (read back with K14's count)
//   sort_shard_pack_kernel   one thread per entry, in place over the cells K14 wrote into the block's last section
//   sort_shard_merge_kernel  one round of pairwise merge-path merges of runs, a tile of output positions per CTA
__global__ void __launch_bounds__(256) sort_shard_rows_kernel(const uint32_t* __restrict__ row_id, uint32_t n_rows,
                                                              uint32_t* bad) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x + 1; i < n_rows; i += stride)
    if (row_id[i] <= row_id[i - 1]) *bad = 1u;
}

struct SortPackArgs {
  const double* vals[B2P_MAX_FIELDS];
  int F;
  const uint32_t* row_id;
  uint64_t T, n;
  unsigned long long flip;
  unsigned long long* block;            // [F x n keys][n cells]; the cells section holds K14's local cells on entry
};

template <class Key = F64Key>
__global__ void __launch_bounds__(256) sort_shard_pack_kernel(const SortPackArgs a) {
  unsigned long long* cells = a.block + (uint64_t)a.F * a.n;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    const unsigned long long c = cells[i];
    for (int f = 0; f < a.F; ++f) a.block[(uint64_t)f * a.n + i] = Key::key(__ldg(a.vals[f] + c)) ^ a.flip;
    const uint64_t r = c / a.T;
    cells[i] = (unsigned long long)__ldg(a.row_id + r) * a.T + (c - r * a.T);
  }
}

// A sorted run of entries: field f's key i at base[f * stride + i], its cell at base[F * stride + i]
struct SortRun {
  const unsigned long long* base;
  uint64_t stride, len;
};
// One merge of a round: runs a and b (b may be empty) into output positions [out, out + a.len + b.len); its tiles are
// the round's tiles tile0 .. the next pair's tile0
struct SortPair {
  SortRun a, b;
  uint64_t out, tile0;
};
struct SortMergeArgs {
  const SortPair* pairs;
  uint32_t n_pairs;
  int F;
  uint32_t cap;                         // output positions per CTA: 256 x items
  // a round before the last: keys and cells to obase (field f's key at obase[f * ostride + p], the cell at F * ostride)
  unsigned long long* obase;
  uint64_t ostride;
  // the last round: the cells and the values decoded from the keys
  unsigned long long* out_cells;
  double* out_vals[B2P_MAX_FIELDS];
  unsigned long long flip;
};

// (key tuple, cell) of x < that of y; kOne: one field, no loop
template <bool kOne>
__device__ __forceinline__ bool shard_less(const unsigned long long* xb, uint64_t xs, uint64_t x,
                                           const unsigned long long* yb, uint64_t ys, uint64_t y, int F) {
  if constexpr (kOne) {
    const unsigned long long kx = xb[x], ky = yb[y];
    if (kx != ky) return kx < ky;
    return xb[xs + x] < yb[ys + y];
  } else {
    for (int f = 0; f < F; ++f) {
      const unsigned long long kx = xb[(uint64_t)f * xs + x], ky = yb[(uint64_t)f * ys + y];
      if (kx != ky) return kx < ky;
    }
    return xb[(uint64_t)F * xs + x] < yb[(uint64_t)F * ys + y];
  }
}

// Merge path: how many of the first d merged entries come from a (entries are distinct, so the split is unique)
template <bool kOne>
__device__ __forceinline__ uint64_t shard_corank(uint64_t d, const unsigned long long* ab, uint64_t as, uint64_t al,
                                                 const unsigned long long* bb, uint64_t bs, uint64_t bl, int F) {
  uint64_t lo = d > bl ? d - bl : 0, hi = d < al ? d : al;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (shard_less<kOne>(ab, as, mid, bb, bs, d - mid - 1, F)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Dynamic shared memory: keys [F x cap] and cells [cap] u64 of the tile's inputs (a's part, then b's), then the merged
// order as input slots [cap] u32.
template <bool kOne, bool kLast, class Key = F64Key>
__global__ void __launch_bounds__(256) sort_shard_merge_kernel(const SortMergeArgs a) {
  extern __shared__ unsigned long long sm[];
  const int F = kOne ? 1 : a.F;
  const uint32_t cap = a.cap;
  uint32_t* src = reinterpret_cast<uint32_t*>(sm + (uint64_t)(F + 1) * cap);
  __shared__ uint64_t s_corank[2];
  // this CTA's pair: the last one whose first tile is at or before blockIdx.x
  uint32_t lo = 0, hi = a.n_pairs - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (a.pairs[mid].tile0 <= blockIdx.x) lo = mid;
    else hi = mid - 1;
  }
  const SortPair p = a.pairs[lo];
  const uint64_t total = p.a.len + p.b.len;
  const uint64_t s = (uint64_t)(blockIdx.x - p.tile0) * cap;
  const uint64_t e = s + cap < total ? s + cap : total;
  if (threadIdx.x < 2)
    s_corank[threadIdx.x] = shard_corank<kOne>(threadIdx.x ? e : s, p.a.base, p.a.stride, p.a.len, p.b.base,
                                               p.b.stride, p.b.len, F);
  __syncthreads();
  const uint64_t i0 = s_corank[0], i1 = s_corank[1];
  const uint32_t na = (uint32_t)(i1 - i0), n = (uint32_t)(e - s), nb = n - na;
  const uint64_t j0 = s - i0;
  for (uint32_t q = threadIdx.x; q < n; q += blockDim.x) {
    const bool in_a = q < na;
    const unsigned long long* b = in_a ? p.a.base : p.b.base;
    const uint64_t st = in_a ? p.a.stride : p.b.stride, x = in_a ? i0 + q : j0 + (q - na);
    for (int f = 0; f <= F; ++f) sm[(uint64_t)f * cap + q] = b[(uint64_t)f * st + x];
  }
  __syncthreads();
  // each thread merges `items` consecutive outputs of the tile from the staged inputs: a's part at [0, na), b's after
  const uint32_t items = cap / blockDim.x;
  const uint32_t d = threadIdx.x * items < n ? threadIdx.x * items : n;
  const uint32_t d1 = d + items < n ? d + items : n;
  uint32_t x = (uint32_t)shard_corank<kOne>(d, sm, cap, na, sm + na, cap, nb, F);
  uint32_t y = d - x;
  for (uint32_t q = d; q < d1; ++q) {
    const bool take_a = y >= nb || (x < na && shard_less<kOne>(sm, cap, x, sm + na, cap, y, F));
    src[q] = take_a ? x++ : na + y++;
  }
  __syncthreads();
  for (uint32_t q = threadIdx.x; q < n; q += blockDim.x) {
    const uint32_t from = src[q];
    const uint64_t o = p.out + s + q;
    if constexpr (kLast) {
      a.out_cells[o] = sm[(uint64_t)F * cap + from];
      for (int f = 0; f < F; ++f) a.out_vals[f][o] = Key::value(sm[(uint64_t)f * cap + from] ^ a.flip);
    } else {
      for (int f = 0; f <= F; ++f) a.obase[(uint64_t)f * a.ostride + o] = sm[(uint64_t)f * cap + from];
    }
  }
}

}  // namespace b2p
