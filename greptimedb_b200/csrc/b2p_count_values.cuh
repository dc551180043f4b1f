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

// ---- sharded count_values: every rank's distinct values and counts, merged ---------------------------------------
// A rank's K12 output fills each group's rows as a prefix at every step, so its first h_r(g) rows (h_r(g) = the most
// distinct values the group has at one step) hold every (key, count) it has.  Per batch of whole groups [g0, g0 + ng)
// over steps [k0, k0 + W), a rank's block is those rows' cells as (key u64, count u32) entries, segment-major: segment
// (q, kk) of group g0 + q and step k0 + kk starts at W * hoff(q) + kk * h(q), hoff the prefix of the rank's heights
// over the batch.  The merge lays every rank's entries of segment (q, kk) side by side (U(q) = sum over ranks of h) at
// W * uoff(q) + kk * U(q), sorts each segment by key with its counts, and writes each run of equal keys with the sum of
// its counts.  A cell past a rank's distinct values is packed as key ~0 with count 0: it sorts into the last run of
// its segment, and a run whose counts add up to 0 is no value.  The count decides, not the position: ~0 is also the key
// of the largest positive NaN (and of INT64_MAX), whose entries may land anywhere in that run.
struct CvShardArgs {
  uint64_t T;
  uint32_t k0, W, g0, ng;
  const uint32_t* off;        // [ng + 1] per-step entry offsets of the batch's groups: hoff (pack) or uoff (merge)
  // pack: this rank's K12 output [rows x T] (rows in member order) and its index's goff
  const double* vals;
  const uint32_t* cnt;
  const uint32_t* goff;
  unsigned long long* bkeys;  // [P] the block: keys, then counts
  uint32_t* bcnt;
  // merge: the gathered blocks, [keys of rank 0 .. R-1][counts of rank 0 .. R-1], each rank's block P entries
  uint32_t n_ranks;
  uint64_t P;
  const unsigned long long* gkeys;
  const uint32_t* gcnt;
  const uint32_t* hpre;       // [ng x (R + 1)] the prefix over ranks of h_r(g0 + q): rank r's entries of a segment
  const uint32_t* hoffs;      // [ng x R] hoff of rank r at group q
  uint32_t cells;             // W * uoff[ng]
  uint32_t* seg_off;          // [ng * W + 1]
  unsigned long long* keys;   // [cells] arranged, the sort's input
  uint32_t* kcnt;
  const unsigned long long* sorted;  // [cells] after the sort, and their counts
  const uint32_t* scnt;
  uint32_t* rank;             // [cells] head flags, then (scanned in place) the inclusive count of runs
  uint32_t* csum;             // [cells] inclusive u32 sum of the sorted counts (wrapping: only differences within a
                              // run are read, and a run's sum is at most its group's member count)
  uint32_t* start;            // [cells] (uoff(q) + j) * W + kk: where run j of segment (q, kk) starts in the batch
  double* out_val;            // [out rows x T], the batch's rows from out_row0
  uint32_t* out_cnt;
  uint32_t out_row0;
};

// the group q of the batch whose rows [off[q], off[q + 1]) hold row position p < off[ng]
__device__ __forceinline__ uint32_t cv_shard_group(const uint32_t* off, uint32_t ng, uint32_t p) {
  uint32_t lo = 0, hi = ng;  // off[lo] <= p < off[hi]
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (__ldg(off + mid) <= p) lo = mid; else hi = mid;
  }
  return lo;
}

// h_r(g) of this rank: 1 + the largest place in its group of a row with a count at some step.  One warp per row of the
// K12 output (member position m < in_rows); heights zeroed by the caller.
__global__ void __launch_bounds__(256) count_values_heights_kernel(const uint32_t* cnt, const uint32_t* gid,
                                                                    const uint32_t* members, const uint32_t* goff,
                                                                    uint32_t in_rows, uint64_t T, uint32_t* heights) {
  const int lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
  for (uint64_t m = (uint64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; m < in_rows; m += warps) {
    const uint32_t* row = cnt + m * T;
    bool any = false;
    for (uint64_t k = lane; k < T && !any; k += 32) any = __ldg(row + k) != 0u;
    if (__any_sync(0xFFFFFFFFu, any) && lane == 0) {
      const uint32_t g = __ldg(gid + __ldg(members + m));
      atomicMax(heights + g, (uint32_t)m - __ldg(goff + g) + 1u);
    }
  }
}

// Pack: one thread per (row p of the rank's block, step kk), kk fastest (the K12 output is read a row at a time)
template <class Key = F64Key>
__global__ void __launch_bounds__(256) count_values_pack_kernel(const CvShardArgs a) {
  const uint64_t n = (uint64_t)__ldg(a.off + a.ng) * a.W;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t p = (uint32_t)(i / a.W), kk = (uint32_t)(i - (uint64_t)p * a.W);
    const uint32_t q = cv_shard_group(a.off, a.ng, p);
    const uint32_t o = __ldg(a.off + q), h = __ldg(a.off + q + 1) - o, j = p - o;
    const uint64_t cell = (uint64_t)(__ldg(a.goff + a.g0 + q) + j) * a.T + a.k0 + kk;
    const uint32_t c = __ldg(a.cnt + cell);
    const uint64_t e = (uint64_t)o * a.W + (uint64_t)kk * h + j;
    a.bkeys[e] = c ? Key::key(__ldg(a.vals + cell)) : ~0ull;
    a.bcnt[e] = c;
  }
}

// Merge, 1: segment offsets (one thread per segment)
__global__ void __launch_bounds__(256) count_values_merge_segments_kernel(const CvShardArgs a) {
  const uint32_t n_seg = a.ng * a.W;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x) {
    const uint32_t q = s / a.W, kk = s - q * a.W;
    const uint32_t o = __ldg(a.off + q), u = __ldg(a.off + q + 1) - o;
    a.seg_off[s] = o * a.W + kk * u;
    if (s == n_seg - 1) a.seg_off[n_seg] = a.cells;
  }
}

// Merged entry i of the batch: its group q, step kk and place j in segment (q, kk) of U entries
__device__ __forceinline__ void cv_merge_place(const CvShardArgs& a, uint32_t i, uint32_t& q, uint32_t& kk, uint32_t& j,
                                               uint32_t& u) {
  q = cv_shard_group(a.off, a.ng, i / a.W);
  const uint32_t o = __ldg(a.off + q);
  u = __ldg(a.off + q + 1) - o;
  const uint32_t rel = i - o * a.W;
  kk = rel / u;
  j = rel - kk * u;
}

// Merge, 2: every rank's entries of a segment side by side, rank by rank (one thread per merged entry)
__global__ void __launch_bounds__(256) count_values_merge_arrange_kernel(const CvShardArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += gridDim.x * blockDim.x) {
    uint32_t q, kk, j, u;
    cv_merge_place(a, i, q, kk, j, u);
    const uint32_t* pre = a.hpre + (uint64_t)q * (a.n_ranks + 1);
    uint32_t r = 0;
    while (__ldg(pre + r + 1) <= j) ++r;  // the rank whose entries hold place j
    const uint32_t jr = j - __ldg(pre + r), h = __ldg(pre + r + 1) - __ldg(pre + r);
    const uint64_t src = (uint64_t)r * a.P + (uint64_t)__ldg(a.hoffs + (uint64_t)q * a.n_ranks + r) * a.W +
                         (uint64_t)kk * h + jr;
    a.keys[i] = __ldg(a.gkeys + src);
    a.kcnt[i] = __ldg(a.gcnt + src);
  }
}

// Merge, 3 (after the segmented sort): 1 where a run of equal keys starts in its segment
__global__ void __launch_bounds__(256) count_values_merge_head_kernel(const CvShardArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += gridDim.x * blockDim.x) {
    uint32_t q, kk, j, u;
    cv_merge_place(a, i, q, kk, j, u);
    a.rank[i] = (j == 0 || a.sorted[i] != a.sorted[i - 1]) ? 1u : 0u;
  }
}

// runs of the batch before segment s (the scan is over the whole batch)
__device__ __forceinline__ uint32_t cv_merge_before(const CvShardArgs& a, uint32_t s) {
  const uint32_t o = a.seg_off[s];
  return o ? a.rank[o - 1] : 0u;
}

// Merge, 4 (after the scans): where each run starts
__global__ void __launch_bounds__(256) count_values_merge_rank_kernel(const CvShardArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += gridDim.x * blockDim.x) {
    uint32_t q, kk, j, u;
    cv_merge_place(a, i, q, kk, j, u);
    if (!(j == 0 || a.sorted[i] != a.sorted[i - 1])) continue;
    const uint32_t r = a.rank[i] - cv_merge_before(a, q * a.W + kk) - 1;  // the run's place in its segment
    a.start[(uint64_t)(__ldg(a.off + q) + r) * a.W + kk] = i;
  }
}

// the sum of the sorted counts over entries [b, e) of the batch, e > b
__device__ __forceinline__ uint32_t cv_merge_sum(const CvShardArgs& a, uint32_t b, uint32_t e) {
  return a.csum[e - 1] - (b ? a.csum[b - 1] : 0u);
}

// Merge, 5: one thread per output cell (merged row p of the batch, step kk), row-major like the start table: the j-th
// run's key and count sum, or 0 / 0 past the runs (and in place of a last run whose counts add up to 0)
template <class Key = F64Key>
__global__ void __launch_bounds__(256) count_values_merge_count_kernel(const CvShardArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += gridDim.x * blockDim.x) {
    const uint32_t p = i / a.W, kk = i - p * a.W;
    const uint32_t q = cv_shard_group(a.off, a.ng, p);
    const uint32_t o = __ldg(a.off + q), j = p - o, s = q * a.W + kk;
    const uint32_t e = a.seg_off[s + 1];  // the segment is not empty: its group has row p
    const uint32_t runs = a.rank[e - 1] - cv_merge_before(a, s);
    const uint32_t last = a.start[(uint64_t)(o + runs - 1) * a.W + kk];
    const uint32_t d = cv_merge_sum(a, last, e) ? runs : runs - 1;  // distinct values at this step
    const uint64_t out = (uint64_t)(a.out_row0 + p) * a.T + a.k0 + kk;
    if (j < d) {
      const uint32_t st = a.start[i];
      const uint32_t next = j + 1 < runs ? a.start[i + a.W] : e;
      a.out_val[out] = Key::value(a.sorted[st]);
      a.out_cnt[out] = cv_merge_sum(a, st, next);
    } else {
      a.out_val[out] = 0.0;
      a.out_cnt[out] = 0u;
    }
  }
}

}  // namespace b2p
