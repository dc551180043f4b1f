// b2p_setop.cuh — PromQL set operators `and`, `or`, `unless` over dense [rows x T] grids:
//   K8 setop_mask_kernel    per key, the OR of the validity words of one side's rows with that key -> mask [n_keys x Tw]
//      setop_dedupe_kernel  `or`, rhs rows: the steps no lhs row and no earlier rhs row of the same key claims
//      setop_copy_kernel    per (row, step tile): the output word of the row, and its value where the bit is set
//      setop_key_check_kernel  a key >= n_keys (other than B2P_NO_KEY) sets a status bit
//
// The reference plans `and` / `unless` as `left.distinct()` LeftSemi- / LeftAnti-joined to the right on (key columns,
// time index), src/query/src/promql/planner.rs:3549-3703, and `or` as UnionDistinctOn (planner.rs:3707-3906,
// src/promql/src/extension_plan/union_distinct_on.rs:338-577).  All three work per cell (key, step), so with the label
// match done on the host (b2p_plan.cpp: one dense key id per row) only validity words need work: every output cell is a
// copy of an input cell or 0.0 (invalid).
//   * and:     lv & mask_rhs[key]; a row without key (B2P_NO_KEY) has no cell
//   * unless:  lv & ~mask_rhs[key]; a row without key keeps every cell
//   * or:      the lhs rows unchanged, then per rhs row rv & ~(mask_lhs[key] | rv of every earlier rhs row of the key):
//              the reference keeps the first rhs row per hash and removes the keys the lhs has (HashedData::new,
//              update_map).  "Earlier" is row order.
// The rhs values of `and` / `unless` are never read.  A row whose key is out of range is written invalid and nothing is
// read through its key; setop_key_check_kernel reports it (bit 3 of the status word's k0_errors -> B2P_E_INVALID).
//
// Work units: the mask and dedupe kernels take one warp per (key, 32 validity words), one word per lane, and walk the
// key's members (a CSR built by the group index's radix sort, so members come in row order) serially.  The copy kernel
// takes one warp per (row, 32-step tile), with K7's 128-bit variant (64 steps, two words) when T is even.  HBM traffic of
// `and` / `unless` per (lhs row, step): 8 B read, 8 B written and about 3 bits; the rhs adds 1 bit per (row, step).
#pragma once
#include <cstdint>

#include "b2p_status.cuh"
#include "b2p_window.cuh"

namespace b2p {

enum SetOp { kSetAnd = 0, kSetOr = 1, kSetUnless = 2 };
// what setop_copy_kernel does with a row's validity word lv (the word of its own row) and the per-key word m
enum SetCopyMode {
  kCopyAnd = 0,     // lv & m; no key -> 0
  kCopyUnless = 1,  // lv & ~m; no key -> lv
  kCopyKeep = 2,    // lv (the lhs rows of `or`)
  kCopyWords = 3,   // the row's word of `words` (the dedupe's result); no key -> lv
};
constexpr uint32_t kSetNoKey = 0xFFFFFFFFu;

__global__ void __launch_bounds__(256) setop_key_check_kernel(const uint32_t* key, uint64_t n, uint32_t n_keys,
                                                              Status* status) {
  bool bad = false;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t k = key[i];
    bad |= k >= n_keys && k != kSetNoKey;
  }
  if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(&status->k0_errors, kSetKeyError);
}

// mask[g * Tw + w] = OR over the members m of key g of valid[members[m] * Tw + w]
__global__ void __launch_bounds__(256) setop_mask_kernel(const uint32_t* __restrict__ valid,
                                                         const uint32_t* __restrict__ goff,
                                                         const uint32_t* __restrict__ members, uint32_t n_keys,
                                                         uint32_t Tw, uint32_t* __restrict__ mask) {
  const int lane = threadIdx.x & 31;
  const uint64_t tiles = (Tw + 31) / 32;
  const uint64_t units = (uint64_t)n_keys * tiles;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t u = warp0; u < units; u += n_warps) {
    const uint64_t g = u / tiles;
    const uint32_t w = (uint32_t)((u - g * tiles) * 32) + lane;
    if (w >= Tw) continue;
    uint32_t acc = 0;
    for (uint32_t m = goff[g], e = goff[g + 1]; m < e; ++m) acc |= __ldg(valid + (uint64_t)members[m] * Tw + w);
    mask[g * Tw + w] = acc;
  }
}

// `or`: for every rhs key g (members in row order), running = lmask[g] (zero without lhs rows); per member
// words[row] = rv & ~running, then running |= rv.  Eight members' words are loaded ahead of the (serial) bit chain.
__global__ void __launch_bounds__(256) setop_dedupe_kernel(const uint32_t* __restrict__ rvalid,
                                                           const uint32_t* __restrict__ goff,
                                                           const uint32_t* __restrict__ members,
                                                           const uint32_t* __restrict__ lmask, uint32_t n_keys,
                                                           uint32_t Tw, uint32_t* __restrict__ words) {
  constexpr uint32_t kAhead = 8;
  const int lane = threadIdx.x & 31;
  const uint64_t tiles = (Tw + 31) / 32;
  const uint64_t units = (uint64_t)n_keys * tiles;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t u = warp0; u < units; u += n_warps) {
    const uint64_t g = u / tiles;
    const uint32_t w = (uint32_t)((u - g * tiles) * 32) + lane;
    if (w >= Tw) continue;
    uint32_t running = lmask ? lmask[g * Tw + w] : 0u;
    const uint32_t e = goff[g + 1];
    for (uint32_t m0 = goff[g]; m0 < e; m0 += kAhead) {
      uint64_t row[kAhead];
      uint32_t rv[kAhead];
#pragma unroll
      for (uint32_t i = 0; i < kAhead; ++i) {
        row[i] = m0 + i < e ? (uint64_t)__ldg(members + m0 + i) : 0;
        rv[i] = m0 + i < e ? __ldg(rvalid + row[i] * Tw + w) : 0u;
      }
#pragma unroll
      for (uint32_t i = 0; i < kAhead; ++i) {
        if (m0 + i >= e) break;
        words[row[i] * Tw + w] = rv[i] & ~running;
        running |= rv[i];
      }
    }
  }
}

struct SetCopyArgs {
  const double* src;        // [n_rows x T]
  const uint32_t* svalid;   // [n_rows x Tw]
  const uint32_t* key;      // [n_rows]
  uint64_t n_rows;
  uint32_t n_keys;
  const uint32_t* mask;     // [n_keys x Tw] (kCopyAnd / kCopyUnless)
  const uint32_t* words;    // [n_rows x Tw] (kCopyWords; may be out_valid)
  uint64_t T;
  uint32_t Tw;
  double* out;              // [n_rows x T]; may be src
  uint32_t* out_valid;      // [n_rows x Tw]; may be svalid
};

// the output word w of row r (key k): see SetCopyMode; a key out of range gives 0, and no bit at or beyond step T is set
template <int MODE>
__device__ __forceinline__ uint32_t setop_word(const SetCopyArgs& a, uint64_t r, uint32_t k, uint32_t w) {
  if (k != kSetNoKey && k >= a.n_keys) return 0u;
  const uint64_t left = a.T - (uint64_t)w * 32;
  const uint32_t live = left >= 32 ? 0xFFFFFFFFu : (1u << left) - 1u;
  const uint32_t lv = a.svalid[r * a.Tw + w] & live;
  if (MODE == kCopyKeep) return lv;
  if (MODE == kCopyWords) return k == kSetNoKey ? lv : (a.words[r * a.Tw + w] & live);
  if (k == kSetNoKey) return MODE == kCopyAnd ? 0u : lv;
  const uint32_t m = a.mask[(uint64_t)k * a.Tw + w];
  return MODE == kCopyAnd ? (lv & m) : (lv & ~m);
}

// One warp per (row, tile of 32 steps, or 64 with VEC: T even, two steps per lane in one 128-bit access).  Every lane
// reads what it needs before any lane writes, so out / out_valid may be src / svalid (and words may be out_valid).
template <int MODE, bool VEC>
__global__ void __launch_bounds__(256) setop_copy_kernel(const SetCopyArgs a) {
  constexpr uint32_t kSteps = VEC ? 64 : 32;
  const int lane = threadIdx.x & 31;
  const uint64_t T = a.T;
  const uint64_t tiles = (T + kSteps - 1) / kSteps;
  const uint64_t units = a.n_rows * tiles;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t u = warp0; u < units; u += n_warps) {
    const uint64_t r = u / tiles;
    const uint64_t k0 = (u - r * tiles) * kSteps;
    const uint32_t key = a.key ? a.key[r] : kSetNoKey;
    double* orow = a.out + r * T;
    const double* srow = a.src + r * T;
    const uint32_t w0 = (uint32_t)(k0 >> 5);
    if (!VEC) {
      const uint64_t k = k0 + lane;
      const bool inside = k < T;
      const uint32_t word = setop_word<MODE>(a, r, key, w0);
      const double x = inside ? srow[k] : 0.0;
      __syncwarp();
      if (inside) orow[k] = ((word >> lane) & 1u) ? x : 0.0;
      if (lane == 0) a.out_valid[r * a.Tw + w0] = word;
    } else {
      // lane owns steps k0 + 2*lane and k0 + 2*lane + 1; T is even, so both exist or neither does
      const uint64_t k = k0 + 2 * (uint64_t)lane;
      const bool inside = k < T;
      const uint32_t wi = w0 + (uint32_t)(lane >> 4);  // validity word holding this lane's two steps
      const uint32_t word = inside ? setop_word<MODE>(a, r, key, wi) : 0u;
      const uint32_t bits = (word >> ((2 * lane) & 31)) & 3u;
      double2 x = make_double2(0.0, 0.0);
      if (inside) x = *reinterpret_cast<const double2*>(srow + k);
      __syncwarp();
      if (inside) *reinterpret_cast<double2*>(orow + k) = make_double2(bits & 1u ? x.x : 0.0, bits & 2u ? x.y : 0.0);
      if ((lane & 15) == 0 && inside) a.out_valid[r * a.Tw + wi] = word;
    }
  }
}

}  // namespace b2p
