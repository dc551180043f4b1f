// b2p_count_values.cuh — PromQL `count_values("label", v)` over a dense [rows x T] grid whose rows are grouped by a
// b2p_group_index (K12):
//   count_values_scatter_kernel  per (32 member positions, 32-step tile) of a batch: each in-group cell's 64-bit
//                                total-order key into its (group, step) segment (an invalid cell writes the largest
//                                key), and the segment's valid-cell count (one integer atomic per group and warp)
//   (CUB DeviceSegmentedSort over the segments)
//   count_values_head_kernel     per sorted position: 1 where a distinct key starts, within the segment's valid prefix
//   (CUB DeviceScan::InclusiveSum over the flags, in place: the rank of every distinct key)
//   count_values_rank_kernel     per sorted position that starts a distinct key: its value into out_val, its position
//                                in the segment into the start table
//   count_values_count_kernel    per output cell: the run length from two starts, or count 0 past the distinct values
//
// The reference plans Aggregate(groupBy = [group labels.., ts, value], count(value)) and sorts by (group labels, ts,
// value) (planner.rs:402-445).  DataFusion groups a Float64 by its bits (so -0.0 and +0.0, or two NaN payloads, are two
// values) and arrow sorts it in the f64 total order; the 64-bit key u = total_key(v) ^ 2^63 is both: two cells share a
// key iff they share their bits, and keys order as the total order does.  The result per (group, step) is its distinct
// keys ascending with their multiplicities (an Int64 grid, b2p_count_values_i64, keys on its bits ^ 2^63 instead, I64Key:
// the two kernels that read or write values take the key as a template parameter): row goff[g] + j of out_val / out_cnt holds the j-th, out_cnt 0 past the
// last.  A group has at most as many distinct values at a step as members, so the output is the input's size.
//
// A segment is the (group, step) column of a batch's key buffer: the group's cells at a step, one per member position
// (member-major within the step), so the buffer needs no count pass or scan before the scatter.  A batch is a run of
// groups over a window of steps whose cells fit kCvBatchCells; position i of a batch lies in the segment of the group
// of member position m0 + i / W (W the window's width), which every kernel reads back from the member -> group table.
#pragma once
#include <cstdint>

#include "b2p_quantile.cuh"  // (and through it F64Key / I64Key: the unsigned order keys and their inverses)

namespace b2p {

constexpr uint64_t kCvBatchCells = 1ull << 27;  // cells of one batch: 20 B each of scratch, 2.7 GB
constexpr uint32_t kCvNone = 0xFFFFFFFFu;

struct CvArgs {
  const double* vals;       // [rows x T]
  const uint32_t* valid;    // [rows x Tw]
  const uint32_t* members;  // [n_series] CSR member order -> row
  const uint32_t* goff;     // [G + 1]
  const uint32_t* mgroup;   // [member position] its group (positions < goff[G])
  uint64_t T;
  uint32_t Tw;
  // the batch: groups [g0, g1), member positions [m0, m1) = [goff[g0], goff[g1]), steps [k0, k0 + W)
  uint32_t g0, g1, m0, m1, k0, W;
  uint32_t cells;           // (m1 - m0) * W
  uint32_t* seg_off;        // [(g1 - g0) * W + 1] segment (g, kk) = (g - g0) * W + kk starts here
  uint32_t* seg_n;          // [(g1 - g0) * W] valid cells of the segment
  unsigned long long* keys; // [cells] the scatter's output, the sort's input
  const unsigned long long* sorted;  // [cells]
  uint32_t* rank;           // [cells] head flags, then (scanned in place) the inclusive count of distinct keys
  uint32_t* start;          // [cells] member-major (position - m0) * W + kk: where distinct key j starts in its segment
  double* out_val;          // [rows x T]
  uint32_t* out_cnt;        // [rows x T]
};

// Segment offsets of the batch and zero counts: one thread per segment
__global__ void __launch_bounds__(256) count_values_segments_kernel(const CvArgs a) {
  const uint32_t n_seg = (a.g1 - a.g0) * a.W;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x) {
    const uint32_t g = a.g0 + s / a.W, kk = s % a.W;
    const uint32_t b = __ldg(a.goff + g), n = __ldg(a.goff + g + 1) - b;
    a.seg_off[s] = (b - a.m0) * a.W + kk * n;
    a.seg_n[s] = 0u;
    if (s == n_seg - 1) a.seg_off[n_seg] = a.cells;
  }
}

// One block of 32 x 8 threads per (32 member positions, 32-step tile) of the batch: the tile's values are read a
// member row at a time (32 steps, one coalesced load per warp and member; the member ids and validity words are read
// once per member), transposed through shared memory and written a step at a time (32 consecutive member positions of
// one group are 32 consecutive keys of the segment).
template <class Key = F64Key>
__global__ void __launch_bounds__(256) count_values_scatter_kernel(const CvArgs a) {
  __shared__ unsigned long long sk[32][33];
  __shared__ uint32_t son[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t mt_n = (a.m1 - a.m0 + 31) / 32, kt_n = (a.W + 31) / 32;
  const uint64_t units = (uint64_t)mt_n * kt_n;
  const uint32_t kend = a.k0 + a.W;  // <= T
  for (uint64_t u = blockIdx.x; u < units; u += gridDim.x) {
    const uint32_t mt = (uint32_t)(u / kt_n), kt = (uint32_t)(u - (uint64_t)mt * kt_n);
    const uint32_t mbase = a.m0 + mt * 32, kbase = a.k0 + kt * 32, tile = kbase / 32;
    // read: warp w takes members w, w + 8, .., lane = step
    const uint32_t k = kbase + lane;
    const bool live = k < kend;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t ml = warp + 8 * q, m = mbase + ml;
      bool on = false;
      unsigned long long key = ~0ull;
      if (m < a.m1) {
        const uint32_t row = __ldg(a.members + m);
        const uint32_t w = __ldg(a.valid + (uint64_t)row * a.Tw + tile);
        on = live && ((w >> lane) & 1u);
        if (on) key = Key::key(__ldg(a.vals + (uint64_t)row * a.T + k));
      }
      sk[ml][lane] = key;
      const uint32_t bits = __ballot_sync(0xFFFFFFFFu, on);
      if (lane == 0) son[ml] = bits;
    }
    __syncthreads();
    // write: lane = member position, warp w takes steps w, w + 8, ..
    const uint32_t m = mbase + lane;
    const bool in = m < a.m1;
    const uint32_t g = in ? __ldg(a.mgroup + m) : kCvNone;
    const uint32_t b = in ? __ldg(a.goff + g) : 0u, n = in ? __ldg(a.goff + g + 1) - b : 0u;
    const uint32_t on_bits = son[lane];
    const uint32_t same = __match_any_sync(0xFFFFFFFFu, g);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t kl = warp + 8 * q, kk = kbase + kl - a.k0;
      if (kbase + kl >= kend) break;  // warp-uniform
      const bool on = in && ((on_bits >> kl) & 1u);
      if (in) a.keys[(uint64_t)(b - a.m0) * a.W + (uint64_t)kk * n + (m - b)] = sk[lane][kl];
      const uint32_t mine = same & __ballot_sync(0xFFFFFFFFu, on);
      if (on && lane == __ffs(mine) - 1) atomicAdd(a.seg_n + (g - a.g0) * a.W + kk, (uint32_t)__popc(mine));
    }
    __syncthreads();
  }
}

// Position i of the batch: its group g, step kk of the window, segment s and place j in the segment.  True when i
// starts a distinct key within the segment's valid prefix (the invalid cells' keys sort after every valid one, or tie
// with it and are identical).
__device__ __forceinline__ bool cv_head(const CvArgs& a, uint32_t i, uint32_t& g, uint32_t& kk, uint32_t& j, uint32_t& s) {
  g = __ldg(a.mgroup + a.m0 + i / a.W);
  const uint32_t b = __ldg(a.goff + g), n = __ldg(a.goff + g + 1) - b;
  const uint32_t rel = i - (b - a.m0) * a.W;
  kk = rel / n;
  j = rel - kk * n;
  s = (g - a.g0) * a.W + kk;
  return j < a.seg_n[s] && (j == 0 || a.sorted[i] != a.sorted[i - 1]);
}

__global__ void __launch_bounds__(256) count_values_head_kernel(const CvArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += gridDim.x * blockDim.x) {
    uint32_t g, kk, j, s;
    a.rank[i] = cv_head(a, i, g, kk, j, s) ? 1u : 0u;
  }
}

// distinct keys of segment s before its first position (the scan is over the whole batch)
__device__ __forceinline__ uint32_t cv_before(const CvArgs& a, uint32_t s) {
  const uint32_t o = a.seg_off[s];
  return o ? a.rank[o - 1] : 0u;
}

template <class Key = F64Key>
__global__ void __launch_bounds__(256) count_values_rank_kernel(const CvArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += gridDim.x * blockDim.x) {
    uint32_t g, kk, j, s;
    if (!cv_head(a, i, g, kk, j, s)) continue;
    const uint32_t r = a.rank[i] - cv_before(a, s) - 1;  // the distinct key's rank in its segment
    const uint32_t row = __ldg(a.goff + g) + r;
    a.out_val[(uint64_t)row * a.T + a.k0 + kk] = Key::value(a.sorted[i]);
    a.start[(uint64_t)(row - a.m0) * a.W + kk] = j;
  }
}

// One thread per output cell (member position, step) of the batch, member-major like the start table
__global__ void __launch_bounds__(256) count_values_count_kernel(const CvArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += gridDim.x * blockDim.x) {
    const uint32_t row = a.m0 + i / a.W, kk = i % a.W;
    const uint32_t g = __ldg(a.mgroup + row);
    const uint32_t j = row - __ldg(a.goff + g), s = (g - a.g0) * a.W + kk;
    const uint32_t n = a.seg_n[s];
    const uint32_t d = n ? a.rank[a.seg_off[s] + n - 1] - cv_before(a, s) : 0u;  // distinct keys at this step
    const uint64_t o = (uint64_t)row * a.T + a.k0 + kk;
    if (j < d) {
      const uint32_t next = j + 1 < d ? a.start[i + a.W] : n;
      a.out_cnt[o] = next - a.start[i];
    } else {
      a.out_val[o] = 0.0;
      a.out_cnt[o] = 0u;
    }
  }
}

// member position -> group, for the positions of in-range rows
__global__ void __launch_bounds__(256) count_values_member_group_kernel(const uint32_t* gid, const uint32_t* members,
                                                                         uint32_t n, uint32_t* mgroup) {
  for (uint32_t m = blockIdx.x * blockDim.x + threadIdx.x; m < n; m += gridDim.x * blockDim.x)
    mgroup[m] = __ldg(gid + __ldg(members + m));
}

}  // namespace b2p
