// b2p_kernels.cuh — CUDA kernels (sm_90a) of the PromQL range-query path.
//
//  K0 series_offsets_kernel   SeriesDivide: series boundaries from the sorted u32 id column
//  K2L range_lean_kernel<FN>  (b2p_kernel_lean.cuh) first tier of the same fused stage: regular series only,
//                             everything else is handed to K2 through RangeArgs::w_list
//  K2 range_fast_kernel<FN>   SeriesNormalize + RangeManipulate + prom_* UDF + IS NOT NULL, fused:
//                             one warp per series, samples streamed with 128-bit coalesced loads
//                             into a per-warp shared-memory ring, lanes own consecutive eval steps
//     range_slow_kernel<FN>   exact fallback (literal calculate_range cursor walk) for the rare
//                             series the fast kernel defers (ring overflow, cursor-overshoot quirk)
//     range_udf_kernel<FN>    one prom_* UDF call over an explicit RangeArray (thread per window)
//  K4 instant_kernel          InstantManipulate
//
// HBM traffic per input sample: K0 reads 4 B (sid); K2 reads 16 B (ts, val) and writes 8 B + 1 bit
// per (series, step).  Window re-use (each sample is in ~range/interval windows) is served from the
// shared-memory ring, never from HBM.
#pragma once
#include <cstdint>

#include "b2p_status.cuh"
#include "b2p_window.cuh"

namespace b2p {

constexpr int kWarpsPerCta = 8;
#ifndef B2P_FAST_MIN_BLOCKS
#define B2P_FAST_MIN_BLOCKS 3  // resident CTAs per SM the fused kernel is register-budgeted for
#endif

__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) {  // b > 0
  int64_t q = a / b;
  return (a % b < 0) ? q - 1 : q;
}
__device__ __forceinline__ int64_t rem_euclid(int64_t a, int64_t b) {
  int64_t r = a % b;
  return r < 0 ? r + b : r;
}

// ---------------------------------------------------------------------------------------------
// K0: series offsets.  offsets[s] = first row with sid >= s (lower bound), offsets[n_series] = n.
// Replaces find_first_diff_row's row-by-row tag compare (series_divide.rs:622-670); ids must be
// non-decreasing (the reference requires the same ordering, series_divide.rs:410-440).
// ---------------------------------------------------------------------------------------------
// One id of the scalar scan (row r holds id `cur`, the row before it `prev`).
__device__ __forceinline__ void offsets_scan_one(uint32_t cur, uint32_t prev, uint64_t r, uint64_t n_rows,
                                                 uint32_t n_series, uint64_t* __restrict__ offsets, Status* status) {
  if (cur >= n_series) {
    atomicOr(&status->k0_errors, 2u);
  } else if (r == 0) {
    for (uint32_t s = 0; s <= cur; ++s) offsets[s] = 0;
  } else if (cur != prev) {
    if (cur < prev)
      atomicOr(&status->k0_errors, 1u);
    else
      for (uint32_t s = prev + 1; s <= cur; ++s) offsets[s] = r;
  }
  if (r == n_rows - 1 && cur < n_series)
    for (uint32_t s = cur + 1; s <= n_series; ++s) offsets[s] = n_rows;
}

__global__ void __launch_bounds__(256) series_offsets_kernel(const uint32_t* __restrict__ sid, uint64_t n_rows,
                                                             uint32_t n_series, uint32_t sid_base,
                                                             uint64_t* __restrict__ offsets, Status* status) {
  // A warp covers 512 consecutive ids per iteration: four independent 128-bit loads (4 ids each) per lane.
  // The id before a lane's quad comes from its neighbour by shuffle (lane 0: from lane 31's previous quad, or
  // one scalar read for the first).  Almost every quad lies inside one series: a branch-free XOR/OR test skips
  // it; only quads that contain a change (or the first / last row) take the scalar scan.
  constexpr int U = 4;
  const int lane = threadIdx.x & 31;
  const uint64_t nq = (n_rows + 3) / 4;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t base = warp0 * (32 * U); base < nq; base += n_warps * (32 * U)) {
    uint32_t v[U][4];
    int cnt[U];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint64_t r0 = (base + (uint64_t)j * 32 + lane) * 4;
      v[j][0] = v[j][1] = v[j][2] = v[j][3] = 0u;
      cnt[j] = 0;
      if (r0 + 3 < n_rows) {
        const uint4 x = __ldcs(reinterpret_cast<const uint4*>(sid + r0));
        v[j][0] = x.x; v[j][1] = x.y; v[j][2] = x.z; v[j][3] = x.w;
        cnt[j] = 4;
      } else if (r0 < n_rows) {
        cnt[j] = (int)(n_rows - r0);
#pragma unroll
        for (int i = 0; i < 3; ++i)
          if (i < cnt[j]) v[j][i] = sid[r0 + i];
      }
    }
    uint32_t carry = 0u;  // lane 31's last id of the previous quad row
    {
      const uint64_t r0 = base * 4;
      if (lane == 0 && r0 > 0 && r0 < n_rows) carry = sid[r0 - 1];
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint64_t r0 = (base + (uint64_t)j * 32 + lane) * 4;
      uint32_t prev_raw = __shfl_up_sync(0xffffffffu, v[j][3], 1);
      const uint32_t last = __shfl_sync(0xffffffffu, v[j][3], 31);
      if (lane == 0) prev_raw = (r0 == 0) ? v[j][0] : carry;
      carry = last;
      if (cnt[j] == 0) continue;
      uint32_t diff = prev_raw ^ v[j][0];
#pragma unroll
      for (int i = 1; i < 4; ++i) diff |= (i < cnt[j]) ? (v[j][i - 1] ^ v[j][i]) : 0u;
      const bool edge = (r0 == 0) || (r0 + 4 >= n_rows);
      const bool in_range = (v[j][0] - sid_base) < n_series;  // no change => one check covers the quad
      if (diff == 0u && !edge && in_range) continue;
      uint32_t prev = prev_raw - sid_base;  // ids below sid_base wrap to >= n_series and are flagged
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t cur = v[j][i] - sid_base;
        // only the row where the id changes (or the first / last row of the column) has anything to do; an id
        // equal to its predecessor was range-checked where it first appeared
        if (i < cnt[j] && (cur != prev || r0 + i == 0 || r0 + i == n_rows - 1))
          offsets_scan_one(cur, prev, r0 + i, n_rows, n_series, offsets, status);
        prev = cur;
      }
    }
  }
  if (n_rows == 0 && blockIdx.x == 0)
    for (uint32_t s = threadIdx.x; s <= n_series; s += blockDim.x) offsets[s] = 0;
}

// Launched after K0, in its stream: once a column has been flagged (bit 0 or 1; the higher bits belong to other
// operators), K0 has left offsets unwritten (past the last in-range id) or in the order of racing writes (after a
// decrease).  Every series is made empty, so the kernels queued before b2p_sync reads the verdict read no row.
__global__ void __launch_bounds__(256) series_offsets_clear_kernel(uint64_t* __restrict__ offsets, uint32_t n_series,
                                                                   const Status* __restrict__ status) {
  if ((status->k0_errors & 3u) == 0) return;
  for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= n_series; s += (uint64_t)gridDim.x * blockDim.x)
    offsets[s] = 0;
}

// ---------------------------------------------------------------------------------------------
// K2 fast path.
//
// One warp owns one series at a time.  Per 64-row block: 128-bit coalesced loads (prefetched one
// block ahead in registers) -> SeriesNormalize (NaN rows dropped by ballot compaction, offset added)
// -> append to the warp's shared-memory ring (ordinal = index after filtering) -> reset/change bits
// of the new ordinals by ballot -> every eval step whose window can no longer change is evaluated,
// one step per lane: window end/start by guess-and-walk on the ring, range function from the ring.
//
// TS32: the ring keeps timestamps as uint32 "ms since (start - range)", clamped to [0, span+1].
// A sample at or before start-range can never be inside a window (windows are (t-range, t] with
// t >= start) and a sample after `end` can never be either, so clamped samples only ever act as
// "before everything" / "after everything" sentinels; all in-window arithmetic is exact.  The host
// selects TS32 when end - start + range < 2^31 ms (24.8 days), else the int64 ring.
// ---------------------------------------------------------------------------------------------
struct BlockRegs {  // one lane's share (2 rows) of a 64-row block
  int64_t t0, t1;
  double v0, v1;
  bool in0, in1;
};

// rel = index (relative to the series' first row, may be -1 for the alignment row) of this lane's first
// row in the block; n = rows of the series; tail = rows from the series start to the end of the column
// (saturated to 32 bits).  p_ts / p_val already point at this lane's pair.
__device__ __forceinline__ BlockRegs load_block(const int64_t* p_ts, const double* p_val, int32_t rel, uint32_t n,
                                                uint32_t tail) {
  BlockRegs b;
  b.in0 = (uint32_t)rel < n;        // unsigned compare also rejects rel == -1
  b.in1 = (uint32_t)(rel + 1) < n;
  b.t0 = b.t1 = 0;
  b.v0 = b.v1 = 0.0;
  if (b.in0 || b.in1) {
    if ((uint32_t)(rel + 1) < tail) {  // both rows inside the allocation: one 128-bit load per column
      const longlong2 tt = __ldcs(reinterpret_cast<const longlong2*>(p_ts));
      const double2 vv = __ldcs(reinterpret_cast<const double2*>(p_val));
      b.t0 = tt.x; b.t1 = tt.y;
      b.v0 = vv.x; b.v1 = vv.y;
    } else {  // very last row of an odd-length column
      b.t0 = p_ts[0];
      b.v0 = p_val[0];
    }
  }
  return b;
}

__device__ __forceinline__ int64_t shfl_i64(int64_t v, int src) {
  const int lo = __shfl_sync(0xffffffffu, (int)(v & 0xffffffffll), src);
  const int hi = __shfl_sync(0xffffffffu, (int)(v >> 32), src);
  return ((int64_t)hi << 32) | (uint32_t)lo;
}

struct SeriesState {  // warp-uniform
  uint32_t j_cnt;    // samples inserted so far (ordinal space after NaN filtering)
  uint32_t base_lo;  // lower bound of every future window start
  int32_t base_hi;   // lower bound (index) of every future window end
  int32_t stride_lo, stride_hi;
  int32_t k_next;    // next global step to evaluate
  int32_t kf;        // first step the reference evaluates for this series (T = none)
  uint32_t vword;    // validity bits of the current aligned 32-step group
  uint32_t lrs;      // calculate_range's last_range_start (for the overshoot check)
  uint32_t max_c0;   // max cursor start (range_start_index + start_delta) feeding a non-empty window
  uint32_t carry_c0; // c0 of the last step of the previous group
  uint32_t last_flag;  // ordinal of the newest set reset/change bit (0 = none yet)
  bool any_nonempty;
  int32_t k_skip;      // fused by-label partials: steps below this were already added by an earlier tier
  // fused by-label partials only: the number of samples SeriesNormalize keeps (counted up front), so that the
  // cursor-overshoot quirk is recognised before a group's values are added (they cannot be taken back), and the flag
  // that stops the series there
  uint32_t m_total;
  bool quirk;
};

template <bool TS32>
struct TimeDom;
template <>
struct TimeDom<true> {
  using type = uint32_t;
  // ms since (start - range), clamped to [0, rel_max]
  static __device__ __forceinline__ uint32_t conv(int64_t t_abs, const RangeArgs& a) {
    const int64_t d = t_abs - a.tb;
    const int32_t dh = (int32_t)(d >> 32);
    const uint32_t dl = (uint32_t)d;
    const uint32_t in = dl < a.rel_max ? dl : a.rel_max;  // high word 0: plain 32-bit clamp
    return dh == 0 ? in : (dh < 0 ? 0u : a.rel_max);
  }
  static __device__ __forceinline__ uint32_t tlo(const RangeArgs& a, int32_t k) { return (uint32_t)k * (uint32_t)a.interval; }
  static __device__ __forceinline__ uint32_t range(const RangeArgs& a) { return (uint32_t)a.range; }
};
template <>
struct TimeDom<false> {
  using type = int64_t;
  static __device__ __forceinline__ int64_t conv(int64_t t_abs, const RangeArgs&) { return t_abs; }
  static __device__ __forceinline__ int64_t tlo(const RangeArgs& a, int32_t k) { return a.start + (int64_t)k * a.interval - a.range; }
  static __device__ __forceinline__ int64_t range(const RangeArgs& a) { return a.range; }
};

// Evaluate global steps [k_a, k_b) (inside one aligned group of 32); lane = k & 31.
// out_grp / vw_grp point at this lane's slot of the group and at the group's validity word.
template <int FN, int RING, bool TS32>
__device__ __forceinline__ void process_steps(const RangeArgs& a, SeriesState& st, RingAcc<RING, TS32>& acc,
                                              double* out_grp, uint32_t* vw_grp, int32_t k_a, int32_t k_b, int32_t kl,
                                              int lane) {
  using TD = TimeDom<TS32>;
  using time_type = typename TD::type;
  const int32_t k = (k_a & ~31) + lane;
  const bool active = (k >= k_a) && (k < k_b);
  const int idx = k - k_a;
  const int n_act = k_b - k_a;
  const time_type tlo = TD::tlo(a, k);
  const time_type rng = TD::range(a);
  const time_type te = tlo + rng;
  int32_t hi = st.base_hi;
  uint32_t lo = st.base_lo;
  acc.set_window((int32_t)st.base_lo - 16);
  if (st.j_cnt > 0) {
    // Window end = last ordinal with ts <= te, window start = first ordinal with ts > te - range.
    // Guess both from the previous group's stride and verify with four predicated ring reads; only when
    // some lane's guess is wrong does the whole warp take the (divergence-free to enter) walk.
    const int32_t top = (int32_t)st.j_cnt - 1;
    int32_t g = st.base_hi + (idx + 1) * st.stride_hi;
    g = g > top ? top : g;
    uint32_t q = st.base_lo + (uint32_t)((idx + 1) * st.stride_lo);
    q = q > (uint32_t)(g + 1) ? (uint32_t)(g + 1) : q;
    bool good = true;
    if (active) {
      const bool has_g = g > st.base_hi, has_g1 = g < top;
      const bool has_q = (int32_t)q <= g, has_qm = q > st.base_lo;
      const time_type tg = has_g ? acc.t((uint32_t)g) : (time_type)0;
      const time_type tg1 = has_g1 ? acc.t((uint32_t)(g + 1)) : (time_type)0;
      const time_type tq = has_q ? acc.t(q) : (time_type)0;
      const time_type tqm = has_qm ? acc.t(q - 1) : (time_type)0;
      good = (!has_g || tg <= te) && (!has_g1 || tg1 > te) && (!has_q || tq > tlo) && (!has_qm || tqm <= tlo);
    }
    if (!__all_sync(0xffffffffu, good)) {
      if (active) {
        while (g < top && acc.t((uint32_t)(g + 1)) <= te) ++g;
        while (g > st.base_hi && acc.t((uint32_t)g) > te) --g;
        const uint32_t qtop = (uint32_t)(g + 1);
        q = q > qtop ? qtop : q;
        while (q > st.base_lo && acc.t(q - 1) > tlo) --q;
        while (q < qtop && acc.t(q) <= tlo) ++q;
      }
    }
    if (active) {
      hi = g;
      lo = q;
    }
  }
  const uint32_t l = (active && (int32_t)lo <= hi) ? (uint32_t)(hi + 1 - (int32_t)lo) : 0u;
  const bool in_grid = active && (k >= st.kf) && (k <= kl);
  acc.no_flags = st.last_flag <= st.base_lo;  // warp-uniform: no reset/change bit can be inside any window
  double r = 0.0;
  bool ok = false;
  if (in_grid) ok = eval_window<FN>(acc, lo, l, te, rng, a.p0, a.p1, a.rcp_rs, r);
  if (!ok) r = 0.0;

  // --- calculate_range cursor-overshoot watch (DESIGN.md C-13) -----------------------------------
  // The reference's cursor for step k+1 starts at c0 = range_start_index_k + start_delta_k; when
  // c0 >= m (#samples) it reports an EMPTY window even if samples are inside.  Record the largest c0
  // whose following step has a non-empty true window; compared with m at the end of the series.
  const bool nonempty = in_grid && l > 0;
  const uint32_t ne_mask = __ballot_sync(0xffffffffu, nonempty);
  const int last = (k_b - 1) & 31;
  const int32_t nhi = __shfl_sync(0xffffffffu, hi, last);
  const uint32_t nlo = __shfl_sync(0xffffffffu, lo, last);
  if (ne_mask) {
    const uint32_t act_mask = (n_act == 32) ? 0xffffffffu : (((1u << n_act) - 1u) << (k_a & 31));
    const bool brk = (hi + 1 < (int32_t)st.j_cnt);  // a sample newer than the window end exists
    const uint32_t rsi = (brk && lo > 0) ? lo - 1 : lo;
    uint32_t c0, watch;
    if (ne_mask == act_mask) {  // common: every step of the group has a non-empty window
      uint32_t prev_lo = __shfl_up_sync(0xffffffffu, lo, 1);
      if (idx == 0) prev_lo = st.lrs;
      c0 = active ? rsi + (lo - prev_lo) : 0u;
      watch = (lane < last) ? c0 : 0u;           // my successor (lane+1) is non-empty
      if (idx == 0) watch = max(watch, st.carry_c0);
      st.lrs = nlo;
    } else {
      const uint32_t before = ne_mask & ((1u << lane) - 1u);
      const int src = before ? (31 - __clz(before)) : 0;
      const uint32_t lo_src = __shfl_sync(0xffffffffu, lo, src);
      const uint32_t my_lrs = before ? lo_src : st.lrs;
      c0 = nonempty ? (rsi + (lo - my_lrs)) : 0u;  // empty window => start_delta = 0 < m
      const bool next_ne = (ne_mask >> ((lane + 1) & 31)) & 1u;
      watch = (lane < last && next_ne) ? c0 : 0u;
      if (idx == 0 && nonempty) watch = max(watch, st.carry_c0);
      st.lrs = __shfl_sync(0xffffffffu, lo, 31 - __clz(ne_mask));
    }
    // only a cursor start at or beyond the samples seen so far can ever reach m (m >= j_cnt)
    if (__any_sync(0xffffffffu, watch >= st.j_cnt)) st.max_c0 = max(st.max_c0, __reduce_max_sync(0xffffffffu, watch));
    st.carry_c0 = __shfl_sync(0xffffffffu, c0, last);
    st.any_nonempty = true;
  } else {
    st.carry_c0 = 0;
  }

  // --- outputs -------------------------------------------------------------------------------------
  if (a.gsum && st.max_c0 >= st.m_total) {  // cursor-overshoot quirk inside this group: the exact slow path decides
    st.quirk = true;
    return;
  }
  if (a.gsum) {  // fused by-label partials: this tier adds with atomics (out_grp / vw_grp point into gsum / gcnt)
    if (ok && k >= st.k_skip) {
      atomicAdd(out_grp, r);
      atomicAdd(vw_grp + lane, 1u);
    }
  } else {
    if (active) *out_grp = r;
    st.vword |= __ballot_sync(0xffffffffu, ok);
    if ((k_b & 31) == 0 || k_b == (int32_t)a.T) {
      if (lane == 0) *vw_grp = st.vword;
      st.vword = 0;
    }
  }

  // --- advance the warp-uniform search bases ------------------------------------------------------
  if (st.j_cnt > 0) {
    const int sh = (n_act == 32) ? 5 : (32 - __clz(n_act));  // divide by >= n_act: the stride is only a guess
    st.stride_hi = (nhi - st.base_hi + (n_act >> 1)) >> sh;
    st.stride_lo = ((int32_t)(nlo - st.base_lo) + (n_act >> 1)) >> sh;
    st.base_hi = nhi;
    st.base_lo = nlo;
  }
}

// Steady-state variant of process_steps: a whole aligned group of 32 steps, every step inside the
// series' evaluated grid [kf, kl], ring non-empty.  No per-lane activity predicates; when consecutive
// steps advance both window edges by exactly one sample (stride 1: step == scrape interval) each lane
// reads ONE timestamp per edge and gets its neighbour's through a shuffle.
template <int FN, int RING, bool TS32>
__device__ __forceinline__ void process_group_full(const RangeArgs& a, SeriesState& st, RingAcc<RING, TS32>& acc,
                                                   double* out_grp, uint32_t* vw_grp, int32_t k_a, int lane) {
  using TD = TimeDom<TS32>;
  using time_type = typename TD::type;
  using TR = FnTraits<FN>;
  const int32_t k = k_a + lane;
  const time_type tlo = TD::tlo(a, k);
  const time_type rng = TD::range(a);
  const time_type te = tlo + rng;
  const int32_t top = (int32_t)st.j_cnt - 1;
  int32_t g;
  uint32_t q;
  time_type t_hi = 0, t_lo = 0;  // ts[g], ts[q] when the guess verified
  bool good;
  acc.set_window((int32_t)st.base_lo - 16);
  const bool unit_stride = st.stride_hi == 1 && st.stride_lo == 1 && st.base_hi >= 0 && st.base_hi + 33 <= top &&
                           (int32_t)st.base_lo + 32 <= top;
  if (unit_stride) {
    g = st.base_hi + 1 + lane;
    q = st.base_lo + 1 + (uint32_t)lane;
    t_hi = acc.t((uint32_t)g);
    time_type t_hi_next = __shfl_down_sync(0xffffffffu, t_hi, 1);
    if (lane == 31) t_hi_next = acc.t((uint32_t)(g + 1));
    const time_type t_lo_prev = acc.t(q - 1);
    t_lo = __shfl_down_sync(0xffffffffu, t_lo_prev, 1);
    if (lane == 31) t_lo = acc.t(q);
    good = (t_hi <= te) && (t_hi_next > te) && (t_lo_prev <= tlo) && (t_lo > tlo) && ((int32_t)q <= g);
  } else {
    g = st.base_hi + (lane + 1) * st.stride_hi;
    g = g > top ? top : g;
    q = st.base_lo + (uint32_t)((lane + 1) * st.stride_lo);
    q = q > (uint32_t)(g + 1) ? (uint32_t)(g + 1) : q;
    const bool has_g = g > st.base_hi, has_g1 = g < top;
    const bool has_q = (int32_t)q <= g, has_qm = q > st.base_lo;
    const time_type tg = has_g ? acc.t((uint32_t)g) : (time_type)0;
    const time_type tg1 = has_g1 ? acc.t((uint32_t)(g + 1)) : (time_type)0;
    const time_type tq = has_q ? acc.t(q) : (time_type)0;
    const time_type tqm = has_qm ? acc.t(q - 1) : (time_type)0;
    good = has_g && has_q && (tg <= te) && (!has_g1 || tg1 > te) && (tq > tlo) && (!has_qm || tqm <= tlo);
    t_hi = tg;
    t_lo = tq;
  }
  const bool all_good = __all_sync(0xffffffffu, good);
  if (!all_good) {  // some guess missed: every lane walks (zero steps where it was right)
    while (g < top && acc.t((uint32_t)(g + 1)) <= te) ++g;
    while (g > st.base_hi && acc.t((uint32_t)g) > te) --g;
    const uint32_t qtop = (uint32_t)(g + 1);
    q = q > qtop ? qtop : q;
    while (q > st.base_lo && acc.t(q - 1) > tlo) --q;
    while (q < qtop && acc.t(q) <= tlo) ++q;
    if (g >= 0) t_hi = acc.t((uint32_t)g);
    t_lo = acc.t(q);
  }
  const int32_t hi = g;
  const uint32_t lo = q;
  const uint32_t l = ((int32_t)lo <= hi) ? (uint32_t)(hi + 1 - (int32_t)lo) : 0u;
  acc.no_flags = st.last_flag <= st.base_lo;
  double r = 0.0;
  bool ok;
  if constexpr (TR::kExtrapolated) {
    ok = l >= 2;
    if (ok) r = extrapolated_value<FN>(acc, lo, l, t_lo, t_hi, te, rng, a.range_secs, a.rcp_rs);
  } else {
    ok = eval_window<FN>(acc, lo, l, te, rng, a.p0, a.p1, a.rcp_rs, r);
    if (!ok) r = 0.0;
  }

  // cursor-overshoot watch (see process_steps)
  const int32_t nhi = __shfl_sync(0xffffffffu, hi, 31);
  const uint32_t nlo = __shfl_sync(0xffffffffu, lo, 31);
  const bool nonempty = l > 0;
  uint32_t ne_mask = 0xffffffffu;
  if (unit_stride && all_good) {
    // every window is non-empty, followed by a sample, and starts one ordinal after its predecessor's:
    // c0 = (lo-1) + 1 = lo < j_cnt for every lane, so only the carried c0 of the previous group can matter
    if (st.carry_c0 >= st.j_cnt) st.max_c0 = max(st.max_c0, st.carry_c0);
    st.carry_c0 = nlo;
    st.lrs = nlo;
    st.any_nonempty = true;
  } else if ((ne_mask = __ballot_sync(0xffffffffu, nonempty)) == 0xffffffffu) {
    const bool brk = (hi + 1 < (int32_t)st.j_cnt);
    const uint32_t rsi = (brk && lo > 0) ? lo - 1 : lo;
    uint32_t prev_lo = __shfl_up_sync(0xffffffffu, lo, 1);
    if (lane == 0) prev_lo = st.lrs;
    const uint32_t c0 = rsi + (lo - prev_lo);
    uint32_t watch = (lane < 31) ? c0 : 0u;
    if (lane == 0) watch = max(watch, st.carry_c0);
    if (__any_sync(0xffffffffu, watch >= st.j_cnt)) st.max_c0 = max(st.max_c0, __reduce_max_sync(0xffffffffu, watch));
    st.carry_c0 = __shfl_sync(0xffffffffu, c0, 31);
    st.lrs = nlo;
    st.any_nonempty = true;
  } else if (ne_mask) {
    const bool brk = (hi + 1 < (int32_t)st.j_cnt);
    const uint32_t rsi = (brk && lo > 0) ? lo - 1 : lo;
    const uint32_t before = ne_mask & ((1u << lane) - 1u);
    const int src = before ? (31 - __clz(before)) : 0;
    const uint32_t lo_src = __shfl_sync(0xffffffffu, lo, src);
    const uint32_t my_lrs = before ? lo_src : st.lrs;
    const uint32_t c0 = nonempty ? (rsi + (lo - my_lrs)) : 0u;
    const bool next_ne = (ne_mask >> ((lane + 1) & 31)) & 1u;
    uint32_t watch = (lane < 31 && next_ne) ? c0 : 0u;
    if (lane == 0 && nonempty) watch = max(watch, st.carry_c0);
    if (__any_sync(0xffffffffu, watch >= st.j_cnt)) st.max_c0 = max(st.max_c0, __reduce_max_sync(0xffffffffu, watch));
    st.carry_c0 = __shfl_sync(0xffffffffu, c0, 31);
    st.lrs = __shfl_sync(0xffffffffu, lo, 31 - __clz(ne_mask));
    st.any_nonempty = true;
  } else {
    st.carry_c0 = 0;
  }

  if (a.gsum && st.max_c0 >= st.m_total) {
    st.quirk = true;
    return;
  }
  if (a.gsum) {
    if (ok && k >= st.k_skip) {
      atomicAdd(out_grp, r);
      atomicAdd(vw_grp + lane, 1u);
    }
  } else {
    *out_grp = r;
    const uint32_t vw = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) *vw_grp = vw;
  }

  st.stride_hi = (nhi - st.base_hi + 16) >> 5;
  st.stride_lo = ((int32_t)(nlo - st.base_lo) + 16) >> 5;
  st.base_hi = nhi;
  st.base_lo = nlo;
}

// BIG: the long-window instantiation (RING = 1024, one CTA per SM): runs over b_list, hands what even that ring
// cannot hold to the slow kernel.  The standard instantiation hands ring pressure to b_list when the host enabled
// it (a.b_list != nullptr), else to the slow kernel like the cursor-overshoot quirk.
template <int FN, int RING, bool TS32>
__global__ void __launch_bounds__(kWarpsPerCta * 32, (RING > 256 ? 1 : B2P_FAST_MIN_BLOCKS)) range_fast_kernel(const RangeArgs a) {
  using TD = TimeDom<TS32>;
  using time_type = typename TD::type;
  constexpr int FW = RING / 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // smem: [warps][2*RING] val f64 | [warps][2*RING] ts | [kRcpTable] f64 | [warps][FW] flag words
  double* rval = reinterpret_cast<double*>(smem_raw) + warp * (2 * RING);
  time_type* rts = reinterpret_cast<time_type*>(smem_raw + (size_t)kWarpsPerCta * 2 * RING * 8) + warp * (2 * RING);
  double* rcp_tab = reinterpret_cast<double*>(smem_raw + (size_t)kWarpsPerCta * 2 * RING * (8 + sizeof(time_type)));
  uint32_t* rfl = reinterpret_cast<uint32_t*>(rcp_tab + kRcpTable) + warp * FW;
  for (int i = threadIdx.x; i < kRcpTable; i += blockDim.x) rcp_tab[i] = (i > 0) ? 1.0 / (double)i : 0.0;
  __syncthreads();
  RingAcc<RING, TS32> acc;
  acc.init(rts, rval, rfl, rcp_tab);
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t total_warps = gridDim.x * kWarpsPerCta;
  const int32_t T = (int32_t)a.T;

  const uint32_t n_work = a.use_w_list == 2 ? a.status->b_count : (a.use_w_list ? a.status->w_count : a.n_series);
  for (uint32_t wi = blockIdx.x * kWarpsPerCta + warp; wi < n_work; wi += total_warps) {
    const uint32_t s = a.use_w_list == 2 ? a.b_list[wi] : (a.use_w_list ? a.w_list[wi] : wi);
    const uint64_t row0 = a.offsets[s], row1 = a.offsets[s + 1];
    // (fused by-label partials: the "row" of the series is its group's row of gsum / gcnt, one count per step)
    double* const out_s = a.gsum ? a.gsum + (size_t)a.gid[s] * (size_t)T : a.out + (size_t)s * (size_t)T;
    uint32_t* const vw_s = a.gsum ? a.gcnt + (size_t)a.gid[s] * (size_t)T : a.valid + (size_t)s * a.Tw;
    const int vw_step = a.gsum ? 32 : 1;
    const int32_t k_skip = !a.gsum ? 0 : (a.use_w_list == 2 ? (int32_t)a.b_skip[wi] : (a.use_w_list ? (int32_t)a.w_skip[wi] : 0));
    double* out_grp = out_s + lane;  // this lane's slot in the current aligned 32-step group
    uint32_t* vw_grp = vw_s;         // validity word of the current group
    SeriesState st;
    st.j_cnt = 0; st.base_lo = 0; st.base_hi = -1; st.stride_lo = 1; st.stride_hi = 1;
    st.k_next = 0; st.kf = T; st.vword = 0; st.lrs = 0; st.max_c0 = 0; st.carry_c0 = 0; st.last_flag = 0;
    st.any_nonempty = false;
    st.k_skip = k_skip;
    st.m_total = 0xffffffffu;
    st.quirk = false;
    int64_t last_ts = 0;  // exact (absolute, offset applied) timestamp of the newest surviving sample
    int32_t k_fin = 0;    // steps [0, k_fin) can be evaluated with what is in the ring
    bool defer = false;
    bool defer_ring = false;  // the reason is ring pressure (a longer ring can take the series)

    // evaluate [k_next, upto) in aligned groups of 32; advances the output cursors
#define B2P_RUN_STEPS(UPTO, KL)                                                                      \
    do {                                                                                              \
      const int32_t upto__ = (UPTO);                                                                  \
      while (st.k_next < upto__) {                                                                    \
        if (st.j_cnt - st.base_lo > (uint32_t)(RING - 32)) { defer = true; defer_ring = true; break; } \
        int32_t g_end = (st.k_next | 31) + 1;                                                         \
        if (g_end > upto__) g_end = upto__;                                                           \
        if (g_end - st.k_next == 32 && st.k_next >= st.kf && g_end - 1 <= (KL) && st.j_cnt > 0)       \
          process_group_full<FN, RING, TS32>(a, st, acc, out_grp, vw_grp, st.k_next, lane);           \
        else                                                                                          \
          process_steps<FN, RING, TS32>(a, st, acc, out_grp, vw_grp, st.k_next, g_end, (KL), lane);   \
        if (st.quirk) { defer = true; break; }                                                        \
        st.k_next = g_end;                                                                            \
        if ((g_end & 31) == 0) {                                                                      \
          out_grp += 32;                                                                              \
          vw_grp += vw_step;                                                                          \
        }                                                                                             \
      }                                                                                               \
    } while (0)

    // rows are walked in 64-row blocks starting at the 16-byte aligned pair boundary at or before row0;
    // everything inside the series is 32-bit relative to row0 (a series has < 2^32 rows, like the
    // reference's RangeTuple = (u32, u32), range_array.rs:24)
    const uint32_t n_ser = (uint32_t)(row1 - row0);
    const uint32_t lead = (uint32_t)(row0 & 1ull);
    const uint64_t tail64 = a.n_rows - row0;
    const uint32_t tail = tail64 > 0xffffffffull ? 0xffffffffu : (uint32_t)tail64;
    const int64_t* p_ts = a.ts + (row0 - lead) + 2 * lane;
    const double* p_val = a.val + (row0 - lead) + 2 * lane;
    int32_t rel = 2 * lane - (int32_t)lead;    // this lane's first row of the current block, relative to row0
    const uint32_t n_blk = n_ser + lead;       // rows the blocks have to cover, counted from the aligned start
    uint32_t done = 0;                         // rows covered by completed blocks
    if (a.gsum) {
      uint32_t dropped = 0;
      if (a.filter_nan)
        for (uint32_t j = lane; j < n_ser; j += 32) dropped += isnan(a.val[row0 + j]) ? 1u : 0u;
      st.m_total = n_ser - __reduce_add_sync(0xffffffffu, dropped);
    }
    BlockRegs nxt = load_block(p_ts, p_val, rel, n_ser, tail);
    while (done < n_blk && !defer) {
      const BlockRegs cur = nxt;
      done += 64;
      const bool more = done < n_blk;
      if (more) {
        p_ts += 64;
        p_val += 64;
        rel += 64;
        nxt = load_block(p_ts, p_val, rel, n_ser, tail);
      }

      // ---- SeriesNormalize: drop NaN rows, bias timestamps; append survivors to the ring ----------
      const bool k0 = cur.in0 && !(a.filter_nan && isnan(cur.v0));
      const bool k1 = cur.in1 && !(a.filter_nan && isnan(cur.v1));
      const uint32_t b0 = __ballot_sync(0xffffffffu, k0), b1 = __ballot_sync(0xffffffffu, k1);
      const uint32_t any = b0 | b1;
      if (any) {
        const int64_t t0 = cur.t0 + a.offset, t1 = cur.t1 + a.offset;
        const uint32_t j0 = st.j_cnt;
        const uint32_t pos0 = j0 + __popc(b0 & lt) + __popc(b1 & lt);
        const uint32_t pos1 = pos0 + (k0 ? 1u : 0u);
        if (k0) acc.put(pos0, TD::conv(t0, a), cur.v0);
        if (k1) acc.put(pos1, TD::conv(t1, a), cur.v1);
        st.j_cnt = j0 + __popc(b0) + __popc(b1);
        last_ts = shfl_i64(k1 ? t1 : t0, 31 - __clz(any));
        __syncwarp();
        if constexpr (FnTraits<FN>::kUsesFlags) {
          // Does any new sample reset/change against its predecessor?  Each lane tests its own one or two
          // survivors (predecessor = ring[pos0-1], or its own first sample): one LDS, one ballot.
          const double prev0 = (pos0 > 0) ? acc.vm(pos0 - 1) : cur.v0;
          const bool f0 = k0 && pos0 > 0 && flag_pred<FN>(cur.v0, prev0);
          const bool f1 = k1 && pos1 > 0 && flag_pred<FN>(cur.v1, k0 ? cur.v0 : prev0);
          if (__any_sync(0xffffffffu, f0 || f1)) {
            // rebuild the bit words of the new ordinals, one aligned 32-bit word per ballot
            for (uint32_t wb = j0 & ~31u; wb < st.j_cnt; wb += 32) {
              const uint32_t j = wb + lane;
              bool f = false;
              if (j >= 1 && j < st.j_cnt) f = flag_pred<FN>(acc.vm(j), acc.vm(j - 1));
              const uint32_t word = __ballot_sync(0xffffffffu, f);
              if (lane == 0) rfl[(wb >> 5) & (FW - 1)] = word;
              if (word) st.last_flag = wb + 31 - __clz(word);
            }
          } else {
            // no set bit among the new ordinals: clear the words they start (a partially filled word
            // already holds zeros above the previous j_cnt)
            const uint32_t w_first = (j0 + 31) >> 5, w_last = (st.j_cnt - 1) >> 5;
            if (lane < 3 && w_first + (uint32_t)lane <= w_last) rfl[(w_first + lane) & (FW - 1)] = 0u;
          }
          __syncwarp();
        }
        if (j0 == 0) {  // first surviving sample: RangeManipulate start trimming (range_manipulate.rs:714-725)
          const int64_t first_ts = shfl_i64(k0 ? t0 : t1, __ffs(any) - 1);
          const int64_t rem = rem_euclid(first_ts - a.start, a.interval);
          const int64_t first_aligned = rem == 0 ? first_ts : first_ts + (a.interval - rem);
          const int64_t s2 = a.start > first_aligned ? a.start : first_aligned;
          const int64_t kf = (s2 - a.start) / a.interval;
          st.kf = kf < (int64_t)T ? (int32_t)kf : T;
        }
        // steps whose window can no longer change and that the end-trim cannot remove:
        // t_k <= ts_cur - interval  <=>  k < floor((ts_cur - start) / interval)
        if constexpr (TS32) {
          // floor((rel - range) / interval) by reciprocal multiply + one correction step (exact for the
          // < 2^31 operands of the 32-bit time domain: the double product is within 1 of the quotient)
          const uint32_t rel = TD::conv(last_ts, a);
          if (rel >= (uint32_t)a.range) {
            const uint32_t x = rel - (uint32_t)a.range, d = (uint32_t)a.interval;
            uint32_t q = (uint32_t)__double2uint_rz((double)x * a.rcp_interval);
            const uint32_t back = q * d;
            if (back > x) --q; else if (x - back >= d) ++q;
            k_fin = (int32_t)q;
          } else {
            k_fin = 0;
          }
        } else {
          const int64_t kk = floor_div(last_ts - a.start, a.interval);
          k_fin = kk < 0 ? 0 : (kk > (int64_t)T ? T : (int32_t)kk);
        }
        k_fin = k_fin > T ? T : k_fin;
        // steady state: whole aligned groups only (a partial group waits for the next block)
        B2P_RUN_STEPS(k_fin & ~31, T - 1);
      }
      // ---- ring pressure: evaluate what is final, drop samples no future window can reach -----------
      if (!defer && more && st.j_cnt + 64u - st.base_lo > (uint32_t)(RING - 32)) {
        B2P_RUN_STEPS(k_fin, T - 1);  // partial group: frees the ring up to its last window start
        if (!defer) {
          const time_type tlo_next = TD::tlo(a, st.k_next < T ? st.k_next : T - 1);
          while (st.base_lo < st.j_cnt) {
            const uint32_t j = st.base_lo + lane;
            const bool dead = (j < st.j_cnt) && (acc.tm(j) <= tlo_next);
            const uint32_t m = __ballot_sync(0xffffffffu, dead);
            const uint32_t adv = (m == 0xffffffffu) ? 32u : (uint32_t)(__ffs(~m) - 1);
            st.base_lo += adv;
            if (adv < 32u) break;
          }
          if ((int32_t)st.base_lo - 1 > st.base_hi) st.base_hi = (int32_t)st.base_lo - 1;
          if (st.j_cnt + 64u - st.base_lo > (uint32_t)(RING - 32)) { defer = true; defer_ring = true; }
        }
      }
    }

    if (!defer) {
      // ---- end of stream: RangeManipulate end trimming (range_manipulate.rs:722-728) --------------
      int32_t kl = -1;
      if (st.j_cnt > 0 && st.kf < T) {
        const int64_t last_aligned = ((last_ts + a.range) / a.interval) * a.interval;
        const int64_t e2 = a.end < last_aligned ? a.end : last_aligned;
        const int64_t s2 = a.start + (int64_t)st.kf * a.interval;
        if (e2 >= s2) {
          const int64_t kk = floor_div(e2 - a.start, a.interval);
          kl = kk >= (int64_t)T ? T - 1 : (int32_t)kk;
        }
      }
      B2P_RUN_STEPS(T, kl);
      // cursor-overshoot quirk possible -> exact slow path decides
      if (!defer && st.j_cnt > 0 && st.max_c0 >= st.j_cnt) defer = true;
      // "ignore this if all ranges are empty" (range_manipulate.rs:641-643): only the functions that yield
      // Some on an empty window (absent_over_time, quantile_over_time, holt_winters) need the series-level veto.
      if (FnTraits<FN>::kSomeOnEmpty && !defer && !st.any_nonempty && !a.gsum) {
        for (int32_t k = lane; k < T; k += 32) out_s[k] = 0.0;
        for (uint32_t w = lane; w < a.Tw; w += 32) vw_s[w] = 0u;
      }
    }
    if (defer && lane == 0) {
      const uint32_t done = (uint32_t)(st.k_next > st.k_skip ? st.k_next : st.k_skip);  // steps already added
      if (RING <= 256 && defer_ring && a.b_list != nullptr) {
        const uint32_t i = atomicAdd(&a.status->b_count, 1u);
        a.b_list[i] = s;
        if (a.gsum) a.b_skip[i] = done;
      } else {
        const uint32_t i = atomicAdd(&a.status->slow_count, 1u);
        a.slow_list[i] = s;
        if (a.gsum) a.slow_skip[i] = done;
      }
    }
    __syncwarp();
  }
#undef B2P_RUN_STEPS
}

// ---------------------------------------------------------------------------------------------
// K2 slow path: exact restatement on the device.  One warp per deferred series: compact the series
// (SeriesNormalize) into a global arena, lane 0 runs the literal calculate_range cursor walk
// (range_manipulate.rs:730-769) into a per-warp window list, then lanes evaluate the windows.
// ---------------------------------------------------------------------------------------------
template <int FN>
__global__ void __launch_bounds__(128) range_slow_kernel(const RangeArgs a) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t total_warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t n_slow = a.status->slow_count;
  unsigned long long* wins = a.win_scratch + (size_t)warp_global * (size_t)a.T;
  const uint32_t lt = (1u << lane) - 1u;
  for (uint32_t w = warp_global; w < n_slow; w += total_warps) {
    const uint32_t s = a.slow_list[w];
    const uint64_t row0 = a.offsets[s], row1 = a.offsets[s + 1];
    const uint64_t n = row1 - row0;
    const bool fused = a.gsum != nullptr;  // by-label partials: add with atomics, nothing to clear
    const int64_t k_skip = fused ? (int64_t)a.slow_skip[w] : 0;
    if (k_skip >= a.T) continue;  // fused: every step was added already (also: finished by an earlier run of this kernel)
    double* out_s = fused ? a.gsum + (size_t)a.gid[s] * (size_t)a.T : a.out + (size_t)s * (size_t)a.T;
    uint32_t* vw_s = fused ? a.gcnt + (size_t)a.gid[s] * (size_t)a.T : a.valid + (size_t)s * a.Tw;
    if (!fused) {
      for (int64_t k = lane; k < a.T; k += 32) out_s[k] = 0.0;
      for (uint32_t q = lane; q < a.Tw; q += 32) vw_s[q] = 0u;
    }
    if (n == 0) continue;
    // every warp of this kernel owns one region of the arena and reuses it series after series; a series longer than
    // a region is reported (arena_needed = rows that make the regions large enough) and redone after b2p_sync grew it
    const unsigned long long region = a.arena_cap / total_warps;
    if (n > region) {
      if (lane == 0) {
        atomicMax(&a.status->arena_needed, (unsigned long long)n * total_warps);
        atomicExch(&a.status->arena_overflow, 1u);
      }
      continue;
    }
    int64_t* cts = a.arena_ts + (size_t)warp_global * region;
    double* cval = a.arena_val + (size_t)warp_global * region;
    uint32_t m = 0;
    for (uint64_t r = row0; r < row1; r += 32) {
      const uint64_t rr = r + lane;
      double v = 0.0;
      int64_t t = 0;
      bool keep = false;
      if (rr < row1) {
        v = a.val[rr];
        t = a.ts[rr] + a.offset;
        keep = !(a.filter_nan && isnan(v));
      }
      const uint32_t b = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const uint32_t p = m + __popc(b & lt);
        cts[p] = t;
        cval[p] = v;
      }
      m += __popc(b);
    }
    __syncwarp();
    if (m == 0) continue;
    // ---- literal calculate_range (lane 0) ------------------------------------------------------
    int64_t s2 = 0, e2 = -1;
    int64_t nwin = 0;
    if (lane == 0) {
      const int64_t first_ts = cts[0];
      const int64_t rem = rem_euclid(first_ts - a.start, a.interval);
      const int64_t first_aligned = rem == 0 ? first_ts : first_ts + (a.interval - rem);
      const int64_t last_ts = cts[m - 1];
      const int64_t last_aligned = ((last_ts + a.range) / a.interval) * a.interval;
      s2 = a.start > first_aligned ? a.start : first_aligned;
      e2 = a.end < last_aligned ? a.end : last_aligned;
      uint32_t rsi = 0, last_range_start = 0, start_delta = 0;
      for (int64_t curr = s2; curr <= e2; curr += a.interval) {
        const int64_t start_ts = curr - a.range;
        uint32_t range_start = m, range_end = 0;
        uint32_t cursor = rsi + start_delta;
        while (cursor < m && cts[cursor] > start_ts && cursor > 0) --cursor;
        while (cursor < m) {
          const int64_t t = cts[cursor];
          if (range_start > cursor && t > start_ts) {
            range_start = cursor;
            rsi = range_start;
          }
          if (t <= curr) {
            range_end = range_end > cursor ? range_end : cursor;
          } else {
            rsi = rsi > 0 ? rsi - 1 : 0;
            break;
          }
          ++cursor;
        }
        const int64_t k = (curr - a.start) / a.interval;
        unsigned long long packed = 0;
        if (range_start > range_end) {
          start_delta = 0;
        } else {
          packed = (unsigned long long)range_start | ((unsigned long long)(range_end + 1 - range_start) << 32);
          start_delta = range_start - last_range_start;
          last_range_start = range_start;
        }
        if (k >= 0 && k < a.T) wins[k] = packed;
        ++nwin;
      }
    }
    s2 = __shfl_sync(0xffffffffu, s2, 0);
    e2 = __shfl_sync(0xffffffffu, e2, 0);
    __syncwarp();
    if (s2 > e2) continue;
    const int64_t kf = (s2 - a.start) / a.interval;
    const int64_t kl = floor_div(e2 - a.start, a.interval);
    // all-empty veto (range_manipulate.rs:641-643)
    bool any = false;
    for (int64_t k = kf + lane; k <= kl; k += 32) any |= ((wins[k] >> 32) != 0ull);
    if (!__any_sync(0xffffffffu, any)) continue;
    const GlobalAcc acc{cts, cval};
    for (int64_t kb = kf & ~31ll; kb <= kl; kb += 32) {
      const int64_t k = kb + lane;
      bool ok = false;
      double r = 0.0;
      if (k >= kf && k <= kl) {
        const unsigned long long pk = wins[k];
        ok = eval_window<FN>(acc, (uint32_t)(pk & 0xffffffffull), (uint32_t)(pk >> 32), a.start + k * a.interval,
                             a.range, a.p0, a.p1, 0.0, r);
        if (ok && !fused) out_s[k] = r;
        if (ok && fused && k >= k_skip) {
          atomicAdd(out_s + k, r);
          atomicAdd(vw_s + k, 1u);
        }
      }
      const uint32_t word = __ballot_sync(0xffffffffu, ok);
      if (lane == 0 && !fused) vw_s[kb >> 5] = word;
    }
    // fused: the series is done; a repeat of this kernel (after an arena overflow elsewhere) must not add it again
    if (fused && lane == 0) a.slow_skip[w] = 0xffffffffu;
  }
}

// ---------------------------------------------------------------------------------------------
// UDF-level kernel: one prom_* ScalarUDF invocation over a RangeArray (range_array.rs:247-254:
// key = offset | len<<32).  Thread per window.
// ---------------------------------------------------------------------------------------------
template <int FN>
__global__ void __launch_bounds__(128) range_udf_kernel(const int64_t* __restrict__ ts, const double* __restrict__ val,
                                                        const int64_t* __restrict__ packed,
                                                        const int64_t* __restrict__ eval_ts, uint64_t n_win,
                                                        int64_t range_length, double p0, double p1,
                                                        double* __restrict__ out, uint8_t* __restrict__ valid) {
  const GlobalAcc acc{ts, val};
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_win; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long pk = (unsigned long long)packed[i];
    const int64_t te = eval_ts ? eval_ts[i] : 0;
    double r = 0.0;
    const bool ok =
        eval_window<FN>(acc, (uint32_t)(pk & 0xffffffffull), (uint32_t)(pk >> 32), te, range_length, p0, p1, 0.0, r);
    out[i] = ok ? r : 0.0;
    valid[i] = ok ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------------------
// K4: InstantManipulate (instant_manipulate.rs:473-585).  Warp per series, lane per eval step:
// newest sample with t - lookback < ts <= t; a NaN newest sample is a stale marker -> no row.
// (lookback == 0 selects ts == t only, matching the reference's cursor walk.)
// TIMESTAMP: timestamp(<selector>), where the reference projects ts / 1000 into the value column before
// InstantManipulate (planner.rs:905-909, 951-965): the chosen row's shifted timestamp (ts + offset) as
// (double)t / 1000.0, no value read and no stale-NaN test (a selected stale-NaN sample is kept).
// ---------------------------------------------------------------------------------------------
struct InstantArgs {
  int64_t start, end, interval, lookback, offset;
  int64_t T;
  uint32_t Tw;
  const int64_t* ts;
  const double* val;
  const uint64_t* offsets;
  uint32_t n_series;
  double* out;
  uint32_t* valid;
};

template <bool TIMESTAMP>
__global__ void __launch_bounds__(kWarpsPerCta * 32) instant_kernel(const InstantArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t total_warps = gridDim.x * kWarpsPerCta;
  for (uint32_t s = blockIdx.x * kWarpsPerCta + warp; s < a.n_series; s += total_warps) {
    const uint64_t row0 = a.offsets[s], row1 = a.offsets[s + 1];
    const uint64_t n = row1 - row0;
    double* out_s = a.out + (size_t)s * (size_t)a.T;
    uint32_t* vw_s = a.valid + (size_t)s * a.Tw;
    const int64_t* ts = a.ts + row0;
    const double* val = a.val + row0;  // (not read in TIMESTAMP mode)
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
      double r = 0.0;
      if (k < a.T && k >= k_lo && k <= k_hi) {
        const int64_t te = a.start + k * a.interval;
        // last row with ts + offset <= te  (binary search over the series in global memory)
        uint64_t lo = 0, hi = n;
        while (lo < hi) {
          const uint64_t mid = (lo + hi) >> 1;
          if (ts[mid] + a.offset <= te) lo = mid + 1; else hi = mid;
        }
        if (lo > 0) {
          uint64_t j = lo - 1;
          const int64_t t = ts[j] + a.offset;
          // rows that share the eval timestamp: the reference's cursor stops at the FIRST of them
          // (instant_manipulate.rs:523-541: `curr == expected` breaks without advancing)
          if (t == te)
            while (j > 0 && ts[j - 1] + a.offset == te) --j;
          const bool fresh = (a.lookback > 0) ? (t + a.lookback > te) : (t == te);
          if (fresh) {
            if constexpr (TIMESTAMP) {
              ok = true;
              r = (double)t / 1000.0;
            } else {
              const double v = val[j];
              if (!isnan(v)) { ok = true; r = v; }
            }
          }
        }
      }
      if (k < a.T) out_s[k] = r;
      const uint32_t word = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) vw_s[kb >> 5] = word;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Timestamp column of a batch whose series are all equally spaced (host path: b2p_host_scan_series found
// ts[i] == t0 + i * cadence for every row, so only the descriptors crossed PCIe): warp per series.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ts_expand_kernel(const uint64_t* __restrict__ offsets, const int64_t* __restrict__ t0,
                                                        const int64_t* __restrict__ cadence, uint32_t n_series,
                                                        int64_t* __restrict__ ts) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < n_series; s += warps) {
    const uint64_t r0 = offsets[s], r1 = offsets[s + 1];
    const int64_t first = t0[s], step = cadence[s];
    for (uint64_t i = lane; r0 + i < r1; i += 32) ts[r0 + i] = first + (int64_t)i * step;
  }
}

// ---------------------------------------------------------------------------------------------
// Synthetic workload generator (bench/test utility).  Same integer/f64 arithmetic as
// oracle/promql_oracle.c:orc_synth_fill.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__global__ void __launch_bounds__(256) synth_fill_kernel(uint64_t series_begin, uint64_t n_series, uint32_t n_samples,
                                                         int64_t t0, int64_t scrape_ms, uint32_t jitter_ms,
                                                         int with_resets, uint64_t seed, int64_t* __restrict__ ts,
                                                         double* __restrict__ val, uint32_t* __restrict__ sid) {
  const uint64_t total = n_series * (uint64_t)n_samples;
  for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < total;
       row += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t ls = row / n_samples;
    const uint32_t i = (uint32_t)(row - ls * n_samples);
    const uint64_t s = series_begin + ls;
    const uint64_t h = mix64(seed ^ mix64(s * 0x100000001B3ull + i));
    const int64_t jit = jitter_ms ? (int64_t)(h % jitter_ms) : 0;
    ts[row] = t0 + (int64_t)i * scrape_ms + jit;
    const double scale = (double)(1 + s % 13);
    double v;
    if (!with_resets) {
      const uint32_t q = (i + 1) / 7, r = (i + 1) % 7;
      v = (double)q * 12.25 + (double)r + 0.25 * (double)(r * (r - 1) / 2);
      if (r == 0) v = (double)q * 12.25;
    } else {
      const uint32_t ph = (uint32_t)((i + s) % 37);
      const bool has = (i >= ph) && (i - ph) > 0;
      const uint32_t j0 = has ? (i - ph) + 1 : 0;
      v = has ? 1.0 : 0.0;
      for (uint32_t j = j0; j <= i; ++j) v += 1.0 + (double)(j % 5) * 0.5;
    }
    val[row] = v * scale;
    if (sid) sid[row] = (uint32_t)ls;
  }
}

}  // namespace b2p
