// b2p_kernel_lean.cuh — K2L: the lean first tier of the fused range kernel (18 of the 21 range functions).
//
// Same contract as range_fast_kernel (SeriesNormalize -> RangeManipulate -> prom_* UDF -> IS NOT NULL for every
// series of the batch, one warp per series, samples streamed into a per-warp shared-memory ring, one eval step
// per lane), but it only keeps the work the common series needs and hands every series that needs more to
// range_fast_kernel through RangeArgs::w_list (which in turn hands the cursor-overshoot / long-window cases to
// range_slow_kernel).  A series stays on this tier while
//   * no sample is dropped by SeriesNormalize (normalize.rs:417-426: NaN values with filter_nan),
//   * no counter reset occurs (plain variant of rate / increase: extrapolate_rate.rs:226-233 would add a
//     correction; the FLAGS variant carries the reset / change bit words and keeps such series),
//   * every window and the 64-row block behind it fit the ring,
//   * the windows of the evaluated steps are empty only before the first and after the last non-empty one,
//   * calculate_range's cursor start (range_manipulate.rs:741, DESIGN.md C-13) stays below the number of
//     samples of the series wherever the next window is non-empty (the overshoot quirk needs the slow kernel).
// What it does evaluate is bit-identical to the second tier: window edges are the definitional ones
// (verified guesses, else a walk), the arithmetic is the same extrapolate_parts / eval_window.
//
// Differences that make it cheap:
//   * sentinels instead of bounds: ring slot -1 holds (ts 0, -inf) and, after the last row, slot m holds
//     ts 0xFFFFFFFF, so neither the verification reads nor the walks need index guards;
//   * readiness without division: a group of 32 steps is evaluated as soon as the window end of its last
//     step is older than the newest sample (te31 < t_new), tracked incrementally;
//   * proportional edge guesses (lane+1)*d/32 from the previous group's total advance, verified by four
//     ring reads; when they hold, the next bases follow without shuffles; two groups (64 steps) per vote
//     whenever two are ready;
//   * rows arrive through cp.async into a per-warp staging area (no prefetch registers), the next series'
//     offsets and first block are fetched while the current one evaluates its last groups;
//   * the hot shared-memory reads / stores use 32-bit shared-space addresses (ld.shared / st.shared);
//   * the end trim (range_manipulate.rs:722-728) is applied to the tail groups only — every step
//     evaluated before the end of the stream is below the trimmed end when range >= interval (host gate);
//   * UNI instantiation (rate / increase / delta, plain): where the samples are exactly one eval interval apart the
//     window edges of 64 steps follow from the previous step's without verification reads, ExtrapolatedRate::calc's
//     value-independent tail is evaluated once per window shape, and in the steady state (one uniform pair per full
//     regular block) the block epilogue is skipped altogether — see lean_pair.  cadence_probe_kernel picks the
//     instantiation per call on the device.
#pragma once
#include "b2p_kernels.cuh"

namespace b2p {

// Warps per CTA of the first tier and resident CTAs per SM, tuned together with the register budget: ONE CTA of 24
// warps per SM (80 registers; 172 KB of shared memory in the uniform-cadence variant, 196 KB with the fused by-label
// counters, within the H100's 227 KB per block).  The warps of a CTA work on ADJACENT series, so with one CTA the SM's
// concurrent streams (ts, val, out) each stay inside one contiguous 192 KB region instead of several regions megabytes
// apart (H100 timings of the alternatives: DESIGN.md section 5).  (B2P_LEAN_CONTIG = 1 additionally
// gives every CTA one contiguous range of series over time: no measurable difference, off.)
#ifndef B2P_LEAN_MIN_BLOCKS
#define B2P_LEAN_MIN_BLOCKS 1
#endif
constexpr int kLeanRing = 256;
#ifndef B2P_LEAN_CONTIG
#define B2P_LEAN_CONTIG 0
#endif
#ifndef B2P_LEAN_WARPS
#define B2P_LEAN_WARPS 24
#endif
constexpr int kLeanWarps = B2P_LEAN_WARPS;
// 64-row blocks of a warp's staging area: the block being consumed plus kLeanDepth - 1 in flight (cp.async groups)
#ifndef B2P_LEAN_DEPTH
#define B2P_LEAN_DEPTH 2
#endif
constexpr int kLeanDepth = B2P_LEAN_DEPTH;
// ... of the uniform-cadence kernel: with its steady form it is no longer issue bound and a third block in flight pays
#ifndef B2P_LEAN_DEPTH_UNI
#define B2P_LEAN_DEPTH_UNI 3
#endif
constexpr int kLeanDepthUni = B2P_LEAN_DEPTH_UNI;
// dynamic shared memory of one CTA: value ring + mirrored timestamp ring + reciprocal table + staging (two 64-row
// blocks per warp and column) + bit words + per-warp window-shape cache of the uniform-cadence path (32 B)
// GROUPED (fused by-label partials): per-warp counters "members of the current group whose 32-step word k/32 was valid
// throughout" — the by far most common word; they are added to the count row when the warp leaves the group, so the
// hot path updates the per-step counts in global memory only for the few partially valid words
constexpr int kLeanFullWords = 256;  // => T <= 8192 eval steps on the fused path (host gate)
__host__ __device__ constexpr size_t lean_smem_bytes(bool uni = false) {
  return (size_t)kLeanWarps * kLeanRing * 16 + kRcpTable * 8 + (size_t)kLeanWarps * (uni ? kLeanDepthUni : kLeanDepth) * 64 * 16 +
         (size_t)kLeanWarps * (kLeanRing / 32) * 4 + (size_t)kLeanWarps * 32;
}

// The per-warp sample ring of this tier.  Timestamps (uint32 ms since start - range) are stored twice, slot p
// and slot p + RING, so the edge reads around an index need no wrap handling after set_window(); values are
// stored once and read through a mask (two reads per step).
template <bool FLAGS>
struct LeanRingT {
  using time_type = uint32_t;
  static constexpr int RING = kLeanRing;
  // FLAGS: the ring also carries the reset / change bit of every sample (8 words per warp), like the second tier's.
  // Without them a series with a counter reset leaves the tier.
  static constexpr bool kHasFlags = FLAGS;
  static constexpr bool kHasRcp = true;
  uint32_t* ts;            // [2*RING]
  double* val;             // [RING]
  const double* rcp_tab;   // [kRcpTable] RN(1/n)
  // the same three arrays as 32-bit shared-space byte addresses: the hot reads go through ld.shared with a plain
  // register base (a generic pointer makes the compiler rebuild the shared window base around every use)
  uint32_t ts_sa, val_sa, rcp_sa;
  uint32_t flags_sa;       // [RING/32] bit words (FLAGS only)
  bool no_flags;           // warp-uniform hint: no set bit can lie inside any window of this group
  uint32_t lin_sa;         // ts_sa + 4 * ((j0 & (RING-1)) - j0)
  // uniform-cadence path: {f64 factor; u32 to_end, to_start, length, far} of the window shape last seen by this warp
  uint32_t shape_sa;
  __device__ __forceinline__ void init_addresses() {
    ts_sa = (uint32_t)__cvta_generic_to_shared(ts);
    val_sa = (uint32_t)__cvta_generic_to_shared(val);
    rcp_sa = (uint32_t)__cvta_generic_to_shared(rcp_tab);
    lin_sa = ts_sa;
  }
  static __device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t x;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x) : "r"(addr) : "memory");
    return x;
  }
  static __device__ __forceinline__ double lds64(uint32_t addr) {
    double x;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(x) : "r"(addr) : "memory");
    return x;
  }
  __device__ __forceinline__ void set_window(int32_t j0) { lin_sa = ts_sa + (uint32_t)(((j0 & (RING - 1)) - j0) << 2); }
  __device__ __forceinline__ void put(uint32_t j, uint32_t t, double v) {
    const uint32_t p = j & (RING - 1);
    ts[p] = t;
    ts[p + RING] = t;
    val[p] = v;
  }
  __device__ __forceinline__ uint32_t t(uint32_t j) const { return lds32(lin_sa + (j << 2)); }
  __device__ __forceinline__ uint32_t tm(uint32_t j) const { return lds32(ts_sa + ((j & (RING - 1)) << 2)); }
  __device__ __forceinline__ double v(uint32_t j) const { return lds64(val_sa + ((j & (RING - 1)) << 3)); }
  __device__ __forceinline__ double rcp(uint32_t n) const { return lds64(rcp_sa + (n << 3)); }
  __device__ __forceinline__ uint32_t fw(uint32_t w) const {
    if constexpr (FLAGS) return lds32(flags_sa + ((w & (uint32_t)(RING / 32 - 1)) << 2));
    else return 0u;
  }
};

// Range functions this tier evaluates: everything that is null on an empty window (absent_over_time,
// quantile_over_time and holt_winters yield a value there, which needs the series-level veto of
// range_manipulate.rs:641-643 that the second tier implements).  resets() / changes() run the FLAGS variant;
// rate / increase run the plain one and switch to FLAGS when most series of a call had counter resets.
template <int FN>
struct LeanTraits {
  static constexpr bool kSupported = !FnTraits<FN>::kSomeOnEmpty;
  static constexpr bool kNeedsFlags = (FN == B2P_FN_RESETS || FN == B2P_FN_CHANGES);  // only the FLAGS variant
  static constexpr bool kHasFlagsVariant = FnTraits<FN>::kUsesFlags;                  // rate / increase too
};

// 8-byte asynchronous global -> shared copy (LDGSTS): the next block's rows land in a per-warp staging area
// without passing through registers.
__device__ __forceinline__ void cp_async8(uint32_t smem_dst_sa, const void* gmem_src) {  // shared-space address
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_dst_sa), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t sa, uint32_t x) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(sa), "r"(x) : "memory"); }
__device__ __forceinline__ void sts64(uint32_t sa, double x) { asm volatile("st.shared.f64 [%0], %1;" ::"r"(sa), "d"(x) : "memory"); }
__device__ __forceinline__ long long lds_s64(uint32_t sa) {
  long long x;
  asm volatile("ld.shared.s64 %0, [%1];" : "=l"(x) : "r"(sa) : "memory");
  return x;
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct LeanState {  // warp-uniform
  uint32_t j_cnt;    // samples in the ring's ordinal space (== rows consumed: nothing is filtered on this tier)
  uint32_t base_lo;  // window start of the last evaluated step (in phase 1 also calculate_range's last_range_start)
  int32_t base_hi;   // window end (index) of the last evaluated step
  uint32_t d_lo, d_hi;  // advance of both edges over the previous group (32 steps)
  // 0 = no non-empty window yet (last_range_start is still 0), 1 = inside the run of non-empty windows,
  // 2 = after it, 3 = like 1 but the cursor start handed to the next step is >= m: a non-empty window there
  // would hit the overshoot quirk
  uint32_t phase;
  uint32_t last_flag;  // FLAGS variant: ordinal of the newest set reset / change bit (0 = none yet)
  // samples [reg_from, j_cnt) are exactly one eval interval apart from each other (tracked block by block while they
  // are appended): windows over them all have the same shape, see lean_pair
  uint32_t reg_from;
};

// The value of one step whose window [q, g] (both edge timestamps known) is already established.
template <int FN, bool FLAGS>
__device__ __forceinline__ double lean_value(const RangeArgs& a, const LeanRingT<FLAGS>& acc, int32_t g, uint32_t q,
                                             uint32_t t_lo, uint32_t t_hi, uint32_t te, bool& ok) {
  const uint32_t l = (uint32_t)(g + 1) - q;  // 0 for an empty window (q == g + 1)
  double r = 0.0;
  if constexpr (FnTraits<FN>::kExtrapolated) {
    ok = (int32_t)l >= 2;
    if (ok) {
      const double first_value = acc.v(q);
      const double last_value = acc.v((uint32_t)g);
      // counters add the reset correction: from the bit words (FLAGS), else 0.0 — no series with a reset stays on
      // the plain variant (adding 0.0 keeps the sign of a zero difference identical)
      double result_value = last_value - first_value;
      if constexpr (FnTraits<FN>::kCounter) result_value += FLAGS ? reset_correction(acc, q, (uint32_t)g) : 0.0;
      r = extrapolate_parts<FN, uint32_t, true>(result_value, first_value, t_lo, t_hi, l, te, (uint32_t)a.range,
                                                acc.rcp(l - 1u), a.range_secs, a.rcp_rs);
    }
  } else {
    ok = eval_window<FN>(acc, q, l, te, (uint32_t)a.range, a.p0, a.p1, a.rcp_rs, r);
    if (!ok) r = 0.0;
  }
  return r;
}

// One aligned group of 32 steps; lane's step is k (window end te, start tlo = te - range, both in the 32-bit
// domain).  Returns 0, or the reason (> 0) why the series has to go to the second tier.
// GROUPED (fused by-label partials): out_p / vw_p point at this lane's slot of the group's gsum / gcnt row and are
// updated by read-modify-write — the rows of a group belong to this warp for the whole kernel.
template <int FN, bool TAIL, bool FLAGS, bool GROUPED = false>
__device__ __forceinline__ int lean_group(const RangeArgs& a, LeanState& st, LeanRingT<FLAGS>& acc,
                                           uint32_t m, uint32_t te, int32_t k, int32_t kl, double* out_p,
                                           uint32_t* vw_p, int lane, uint32_t* full_p = nullptr) {
  const uint32_t rng = (uint32_t)a.range;
  const uint32_t tlo = te - rng;
  const int32_t top = (int32_t)st.j_cnt - 1;
  const uint32_t lane1 = (uint32_t)lane + 1u;
  acc.set_window((int32_t)st.base_lo - 1);
  if constexpr (FLAGS) acc.no_flags = st.last_flag <= st.base_lo;  // no bit can lie inside a window of this group
  int32_t g = st.base_hi + (int32_t)((lane1 * st.d_hi) >> 5);
  uint32_t q = st.base_lo + ((lane1 * st.d_lo) >> 5);
  // before the end of the stream the newest sample is younger than every window end of the group, so a
  // window ends below it; afterwards slot top+1 holds the end sentinel.  Either way g+1 and q stay on
  // written slots.
  const int32_t gmax = TAIL ? top : top - 1;
  g = g > gmax ? gmax : g;
  q = q > (uint32_t)(g + 1) ? (uint32_t)(g + 1) : q;
  uint32_t t_hi = acc.t((uint32_t)g);
  const uint32_t t_hi1 = acc.t((uint32_t)(g + 1));
  const uint32_t t_lo1 = acc.t(q - 1u);
  uint32_t t_lo = acc.t(q);
  // steps past the trimmed end (tail groups only) are never visited by calculate_range: their guesses need not hold
  const bool real = !TAIL || k <= kl;
  const bool good = !real || ((t_hi <= te) && (t_hi1 > te) && (t_lo1 <= tlo) && (t_lo > tlo) && ((int32_t)q <= g));
  // uniform: the previous step had a non-empty window and no cursor start of this group can reach the end of
  // the series.  A cursor start is lo - 1 + (advance of lo) while a younger sample follows the window: before
  // the end of the stream, with at most one sample of advance per step (d_lo <= 32), that is at most
  // lo <= hi <= top - 1, so verified guesses imply it; otherwise bound it by base_lo + d_lo + ceil(d_lo/32).
  bool uni = st.phase == 1u;
  if (TAIL) {
    // only the steps up to the trimmed end count: the largest window start among them plus one step's advance
    const int32_t n_real = kl - (k - lane) + 1;  // steps of this group that calculate_range visits
    const uint32_t nr = n_real < 0 ? 0u : (n_real > 32 ? 32u : (uint32_t)n_real);
    uni = uni && (st.base_lo + ((nr * st.d_lo) >> 5) + ((st.d_lo + 31u) >> 5) < m);
  } else if (st.d_lo > 32u) {
    uni = uni && (st.base_lo + st.d_lo + ((st.d_lo + 31u) >> 5) < m);
  }
  if (uni && __all_sync(0xffffffffu, good)) {
    st.base_hi += (int32_t)st.d_hi;
    st.base_lo += st.d_lo;
  } else {
    const bool lead = st.phase == 0u;
    // some guess missed (or the state is not the steady one): every lane walks to the definitional edges;
    // the sentinels bound all four walks
    while (acc.t((uint32_t)(g + 1)) <= te) ++g;
    while (acc.t((uint32_t)g) > te) --g;
    q = q > (uint32_t)(g + 1) ? (uint32_t)(g + 1) : q;
    while (acc.t(q - 1u) > tlo) --q;
    while (acc.t(q) <= tlo) ++q;
    t_hi = acc.t((uint32_t)g);
    t_lo = acc.t(q);
    // steps past the trimmed end (and past the grid) are never visited by calculate_range: for the cursor
    // bookkeeping they count as empty
    const bool ne = ((int32_t)q <= g) && (!TAIL || k <= kl);
    // Short form for the usual miss (a sample exactly on a window edge shifts a few guesses by one): inside the
    // run of non-empty windows, before the end of the stream, every window non-empty and no window start more
    // than two samples past its predecessor's.  A cursor start is then lo - 1 + advance <= lo + 1 <= hi + 1 <=
    // top < m (hi <= top - 1 before the end of the stream), so the exact bookkeeping below cannot object.
    bool short_form = false;
    if (!TAIL && st.phase == 1u) {
      uint32_t prev_q = __shfl_up_sync(0xffffffffu, q, 1);
      if (lane == 0) prev_q = st.base_lo;
      short_form = __all_sync(0xffffffffu, ne && (q - prev_q <= 2u));
    }
    const uint32_t ne_mask = short_form ? 0u : __ballot_sync(0xffffffffu, ne);
    // empty windows are only tolerated before the first and after the last non-empty one
    if (short_form) {
      // phase stays 1: the cursor start handed to the next group is below m as well
    } else if (ne_mask) {
      const int first = __ffs(ne_mask) - 1, last = 31 - __clz(ne_mask);
      const bool contiguous = (ne_mask >> first) == (0xffffffffu >> (31 - (last - first)));
      if (!contiguous || st.phase == 2u || (st.phase == 1u && first != 0)) return 1;
      if (st.phase == 3u) return 2;
      // exact cursor start after each non-empty step (range_manipulate.rs:741,757,765-768)
      const bool brk = g < top;
      const uint32_t rsi = (brk && q > 0u) ? q - 1u : q;
      uint32_t prev = __shfl_up_sync(0xffffffffu, q, 1);
      if (lane == first) prev = (st.phase == 1u) ? st.base_lo : 0u;  // last_range_start
      const uint32_t c0 = ne ? rsi + (q - prev) : 0u;
      const bool next_ne = (lane < 31) && ((ne_mask >> (lane + 1)) & 1u);
      if (__any_sync(0xffffffffu, next_ne && c0 >= m)) return 2;
      const uint32_t carry = __shfl_sync(0xffffffffu, c0, 31);  // 0 when lane 31's window is empty
      st.phase = (last == 31) ? (carry >= m ? 3u : 1u) : 2u;
    } else if (st.phase == 1u || st.phase == 3u) {
      st.phase = 2u;
    }
    const int32_t nhi = __shfl_sync(0xffffffffu, g, 31);
    const uint32_t nlo = __shfl_sync(0xffffffffu, q, 31);
    st.d_hi = (uint32_t)(nhi - st.base_hi);
    // the group that holds the first non-empty window ramps up (its window starts do not move until a window is
    // full): in the steady state that follows both edges advance at the same rate, so guess that instead
    st.d_lo = lead ? st.d_hi : nlo - st.base_lo;
    st.base_hi = nhi;
    st.base_lo = nlo;
  }
  bool ok;
  double r = lean_value<FN, FLAGS>(a, acc, g, q, t_lo, t_hi, te, ok);
  if (TAIL && k > kl) {  // trimmed by RangeManipulate's end alignment
    ok = false;
    r = 0.0;
  }
  if constexpr (GROUPED) {
    const uint32_t vw = __ballot_sync(0xffffffffu, ok);
    if (ok) *out_p = *out_p + r;  // (ok implies k < T: steps past the grid are trimmed)
    if (vw == 0xffffffffu) {
      if (lane == 0) *full_p += 1u;
    } else if (ok) {
      vw_p[lane] = vw_p[lane] + 1u;
    }
  } else {
    if (!TAIL || k < (int32_t)a.T) *out_p = r;
    const uint32_t vw = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) *vw_p = vw;
  }
  return 0;
}


#ifndef B2P_LEAN_PAIR
#define B2P_LEAN_PAIR 1
#endif
#ifndef B2P_LEAN_UNIFORM
#define B2P_LEAN_UNIFORM 1
#endif
#ifndef B2P_LEAN_STEADY
#define B2P_LEAN_STEADY 1
#endif

// The uniform-cadence path is compiled into the plain variants of the extrapolated functions (rate / increase / delta):
// there the per-step arithmetic it removes dominates.  (With the reset bit words the correction scan dominates, and the
// *_over_time functions walk their windows anyway: no gain.)
// It is a kernel variant of its own (template parameter UNI) — compiled into the general kernel it costs the jittered
// case time through register pressure — and cadence_probe_kernel picks one of the two per call on the device.
template <int FN, bool FLAGS>
constexpr bool kLeanUniform = B2P_LEAN_UNIFORM && !FLAGS && FnTraits<FN>::kExtrapolated;

// The window shape of a run of equally spaced samples evaluated at a step equal to their spacing: every window is the
// previous one moved on by one sample, so its length and the distances of its edge samples to the window edges repeat.
struct LeanShape {
  uint32_t to_end, to_start, len;  // te - t[hi], t[lo] - (te - range), hi - lo + 1
  bool far;                        // (t[hi] - t[lo]) >= to_start, the value-independent half of extrapolate_parts' shortcut
  double factor;                   // extrapolate_factor of the shape with to_start unchanged (extrapolated functions)
};

// A step of such a run.  Extrapolated functions: whenever ExtrapolatedRate::calc leaves to_start alone (no counter, no
// positive increase, or the zero crossing provably outside the window: the same exact shortcut as extrapolate_parts)
// the value is result * factor with the factor of the shape — the identical sequence of operations on identical
// operands, evaluated once per shape instead of once per step; any other step takes extrapolate_parts itself.
template <int FN, bool FLAGS>
__device__ __forceinline__ double lean_value_shape(const RangeArgs& a, const LeanRingT<FLAGS>& acc, int32_t g, uint32_t q,
                                                   uint32_t te, const LeanShape& sh, bool& ok) {
  using TR = FnTraits<FN>;
  const uint32_t t_hi = te - sh.to_end, t_lo = te - (uint32_t)a.range + sh.to_start;
  if constexpr (TR::kExtrapolated) {
    ok = sh.len >= 2u;
    double r = 0.0;
    if (ok) {
      const double first_value = acc.v(q);
      const double last_value = acc.v((uint32_t)g);
      double result_value = last_value - first_value;
      if constexpr (TR::kCounter) result_value += FLAGS ? reset_correction(acc, q, (uint32_t)g) : 0.0;
      bool plain = true;
      if constexpr (TR::kCounter)
        plain = !(result_value > 0.0 && first_value >= 0.0) || (B2P_LEAN_FAR && sh.far && first_value >= result_value);
      if (plain)
        r = result_value * sh.factor;
      else
        r = extrapolate_parts<FN, uint32_t, true>(result_value, first_value, t_lo, t_hi, sh.len, te, (uint32_t)a.range,
                                                  acc.rcp(sh.len - 1u), a.range_secs, a.rcp_rs);
    }
    return r;
  } else {
    return lean_value<FN, FLAGS>(a, acc, g, q, t_lo, t_hi, te, ok);
  }
}

// Two consecutive groups (64 steps) in one go, steady state only: before the end of the stream, previous step
// non-empty, at most one sample of advance per step (so no cursor start can reach m, see lean_group), and every
// one of the 64 proportional guesses verified by one vote.  Returns 0 without side effects when any of that
// does not hold; the caller then takes the groups one at a time.
//
// Uniform cadence (B2P_LEAN_UNIFORM): when every sample from the one before the previous step's window up to the one
// after the last of these 64 windows is exactly one eval interval after its predecessor (LeanState::reg_from, checked
// once per sample while the block is appended), step k's window is step k-1's moved on by one sample:
//   t[lo-1] <= tlo < t[lo] and t[hi] <= te < t[hi+1]   =>   t[lo] <= tlo + iv < t[lo+1] and t[hi+1] <= te + iv < t[hi+2].
// The edges of all 64 windows follow from the previous step's without a single verification read, all windows have
// the previous one's shape, and the cursor start of calculate_range is lo - 1 + 1 <= hi < m.  This is the layout of
// aligned scrapes (Prometheus aligns scrape timestamps to the schedule; the BASELINE generator without jitter).
//
// STEADY (uniform-cadence kernel): the block appended last is a full one without a break in the cadence and the block
// before it was followed by exactly one uniform pair.  Then everything the gates and the shape look-up would compute
// is what it was one block ago moved on by 64 samples / 64 steps (te31 + step32 < t_new, the run still covers the
// windows, base_hi + 65 <= top, the same shape in the warp's cache slot): the pair is evaluated without any of it.
// Returns 0 (nothing done), 1 (pair evaluated on verified guesses) or 2 (uniform pair).
template <int FN, bool FLAGS, bool GROUPED = false, bool UNI = false, bool STEADY = false>
__device__ __forceinline__ int lean_pair(const RangeArgs& a, LeanState& st, LeanRingT<FLAGS>& acc, uint32_t te,
                                         uint32_t step32, double* out_p, uint32_t* vw_p, int lane,
                                         uint32_t* full_p = nullptr) {
  using TR = FnTraits<FN>;
  static_assert(!STEADY || (UNI && TR::kExtrapolated), "the steady form belongs to the uniform-cadence kernel");
  const int32_t top = (int32_t)st.j_cnt - 1;
  if (!STEADY && st.phase != 1u) return 0;
  const uint32_t rng = (uint32_t)a.range;
  const uint32_t lane1 = (uint32_t)lane + 1u;
  const uint32_t te_b = te + step32;
  if constexpr (FLAGS) acc.no_flags = st.last_flag <= st.base_lo;  // no bit can lie inside a window of this group
  int32_t g_a, g_b;
  uint32_t q_a, q_b;
  bool ok_a, ok_b;
  double r_a, r_b;
  [[maybe_unused]] double s_a = 0.0, s_b = 0.0;
  // (reg_from < base_lo: the sample before the previous window is part of the run; base_hi + 65 <= top: so is the one
  // after the last window, and all of them have been appended)
  const bool uniform = STEADY || (UNI && st.reg_from < st.base_lo && st.base_hi + 65 <= top);
  if (uniform) {
    LeanShape sh;
    sh.far = false;
    sh.factor = 0.0;
    if constexpr (STEADY) {
      uint32_t k3;
      asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(sh.to_end), "=r"(sh.to_start), "=r"(sh.len), "=r"(k3) : "r"(acc.shape_sa + 16u) : "memory");
      sh.factor = LeanRingT<FLAGS>::lds64(acc.shape_sa);
      sh.far = k3 != 0u;
    } else {
    const uint32_t te_prev = te - lane1 * (uint32_t)a.interval;  // window end of the previous step
    const uint32_t t_hi_p = acc.tm((uint32_t)st.base_hi), t_lo_p = acc.tm(st.base_lo);
    sh.to_end = te_prev - t_hi_p;
    sh.to_start = t_lo_p - (te_prev - rng);
    sh.len = (uint32_t)st.base_hi - st.base_lo + 1u;
    if constexpr (TR::kExtrapolated) {
      // factor of this shape: per-warp cache of the last shape (a series keeps one shape over its run)
      uint32_t k0, k1, k2, k3;
      asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(k0), "=r"(k1), "=r"(k2), "=r"(k3) : "r"(acc.shape_sa + 16u) : "memory");
      if (k0 == sh.to_end && k1 == sh.to_start && k2 == sh.len) {
        sh.factor = LeanRingT<FLAGS>::lds64(acc.shape_sa);
        sh.far = k3 != 0u;
      } else {
        const uint32_t sampled_i = t_hi_p - t_lo_p;
        sh.far = sampled_i >= sh.to_start;
        if (sh.len >= 2u) {
          const double sampled = (double)sampled_i;
          const double average = div_by_rcp(sampled, (double)(sh.len - 1u), acc.rcp(sh.len - 1u));
          sh.factor = extrapolate_factor<FN, true>(sampled, average, (double)sh.to_start, (double)sh.to_end, a.range_secs, a.rcp_rs);
        }
        __syncwarp();
        if (lane == 0) {
          sts64(acc.shape_sa, sh.factor);
          sts32(acc.shape_sa + 16u, sh.to_end);
          sts32(acc.shape_sa + 20u, sh.to_start);
          sts32(acc.shape_sa + 24u, sh.len);
          sts32(acc.shape_sa + 28u, sh.far ? 1u : 0u);
        }
        __syncwarp();
      }
    }
    }
    g_a = st.base_hi + (int32_t)lane1;
    g_b = g_a + 32;
    q_a = st.base_lo + lane1;
    q_b = q_a + 32u;
    st.base_hi += 64;
    st.base_lo += 64u;
    st.d_hi = 32u;
    st.d_lo = 32u;
    if constexpr (GROUPED) { s_a = out_p[0]; s_b = out_p[32]; }  // the running partials are requested before the values
    r_a = lean_value_shape<FN, FLAGS>(a, acc, g_a, q_a, te, sh, ok_a);
    if constexpr (!GROUPED) out_p[0] = r_a;
    r_b = lean_value_shape<FN, FLAGS>(a, acc, g_b, q_b, te_b, sh, ok_b);
    if constexpr (!GROUPED) out_p[32] = r_b;
  } else {
    // uniform gates; the last two keep every read below the newest sample (slot top), i.e. on written slots
    if (st.d_lo > 32u || st.base_hi + 2 * (int32_t)st.d_hi >= top || st.base_lo + 2u * st.d_lo > (uint32_t)top) return 0;
    const uint32_t tlo_a = te - rng, tlo_b = te_b - rng;
    acc.set_window((int32_t)st.base_lo - 1);
    g_a = st.base_hi + (int32_t)((lane1 * st.d_hi) >> 5);
    g_b = g_a + (int32_t)st.d_hi;
    q_a = st.base_lo + ((lane1 * st.d_lo) >> 5);
    q_b = q_a + st.d_lo;
    uint32_t t_hi_a = acc.t((uint32_t)g_a);
    const uint32_t t_hi1_a = acc.t((uint32_t)(g_a + 1));
    const uint32_t t_lo1_a = acc.t(q_a - 1u);
    uint32_t t_lo_a = acc.t(q_a);
    uint32_t t_hi_b = acc.t((uint32_t)g_b);
    const uint32_t t_hi1_b = acc.t((uint32_t)(g_b + 1));
    const uint32_t t_lo1_b = acc.t(q_b - 1u);
    uint32_t t_lo_b = acc.t(q_b);
    const bool good = (t_hi_a <= te) && (t_hi1_a > te) && (t_lo1_a <= tlo_a) && (t_lo_a > tlo_a) && ((int32_t)q_a <= g_a) &&
                      (t_hi_b <= te_b) && (t_hi1_b > te_b) && (t_lo1_b <= tlo_b) && (t_lo_b > tlo_b) && ((int32_t)q_b <= g_b);
    if (__all_sync(0xffffffffu, good)) {
      st.base_hi += 2 * (int32_t)st.d_hi;
      st.base_lo += 2u * st.d_lo;
    } else {
      // Repair in place (the usual miss: a sample exactly on a window edge shifts a few guesses by one): every lane
      // walks both steps to their definitional edges — the newest sample is younger than both window ends and slot
      // base_lo - 1 / the -1 sentinel bound the walks — and the pair goes on if the short form of lean_group holds
      // for all 64 steps (non-empty windows, at most two samples of advance per step => every cursor start is
      // <= lo + 1 <= top < m).  Nothing of the warp state has been touched yet, so "false" still means "one at a time".
      while (acc.t((uint32_t)(g_a + 1)) <= te) ++g_a;
      while (acc.t((uint32_t)g_a) > te) --g_a;
      q_a = q_a > (uint32_t)(g_a + 1) ? (uint32_t)(g_a + 1) : q_a;
      while (acc.t(q_a - 1u) > tlo_a) --q_a;
      while (acc.t(q_a) <= tlo_a) ++q_a;
      while (acc.t((uint32_t)(g_b + 1)) <= te_b) ++g_b;
      while (acc.t((uint32_t)g_b) > te_b) --g_b;
      q_b = q_b > (uint32_t)(g_b + 1) ? (uint32_t)(g_b + 1) : q_b;
      while (acc.t(q_b - 1u) > tlo_b) --q_b;
      while (acc.t(q_b) <= tlo_b) ++q_b;
      uint32_t prev_a = __shfl_up_sync(0xffffffffu, q_a, 1);
      uint32_t prev_b = __shfl_up_sync(0xffffffffu, q_b, 1);
      const uint32_t last_a = __shfl_sync(0xffffffffu, q_a, 31);
      if (lane == 0) {
        prev_a = st.base_lo;
        prev_b = last_a;
      }
      const bool fine = ((int32_t)q_a <= g_a) && ((int32_t)q_b <= g_b) && (q_a - prev_a <= 2u) && (q_b - prev_b <= 2u);
      if (!__all_sync(0xffffffffu, fine)) return 0;
      t_hi_a = acc.t((uint32_t)g_a);
      t_lo_a = acc.t(q_a);
      t_hi_b = acc.t((uint32_t)g_b);
      t_lo_b = acc.t(q_b);
      const int32_t nhi = __shfl_sync(0xffffffffu, g_b, 31);
      const uint32_t nlo = __shfl_sync(0xffffffffu, q_b, 31);
      st.d_hi = (uint32_t)(nhi - st.base_hi + 1) >> 1;  // advance per group over the 64 steps
      st.d_lo = (nlo - st.base_lo + 1u) >> 1;
      st.base_hi = nhi;
      st.base_lo = nlo;
    }
    if constexpr (GROUPED) { s_a = out_p[0]; s_b = out_p[32]; }  // the running partials are requested before the values
    r_a = lean_value<FN, FLAGS>(a, acc, g_a, q_a, t_lo_a, t_hi_a, te, ok_a);
    if constexpr (!GROUPED) out_p[0] = r_a;
    r_b = lean_value<FN, FLAGS>(a, acc, g_b, q_b, t_lo_b, t_hi_b, te_b, ok_b);
    if constexpr (!GROUPED) out_p[32] = r_b;
  }
  uint32_t vw_a, vw_b;
  if (TR::kExtrapolated && uniform) {  // one shape: every step of the pair is valid, or none is
    vw_a = ok_a ? 0xffffffffu : 0u;
    vw_b = vw_a;
  } else {
    vw_a = __ballot_sync(0xffffffffu, ok_a);
    vw_b = __ballot_sync(0xffffffffu, ok_b);
  }
  if constexpr (GROUPED) {
    if (ok_a) out_p[0] = s_a + r_a;
    if (ok_b) out_p[32] = s_b + r_b;
    if ((vw_a & vw_b) == 0xffffffffu) {  // both words valid throughout: two per-warp counters instead of 64 counts
      if (lane == 0) {
        full_p[0] += 1u;
        full_p[1] += 1u;
      }
    } else {
      if (vw_a == 0xffffffffu) {
        if (lane == 0) full_p[0] += 1u;
      } else if (ok_a) {
        vw_p[lane] = vw_p[lane] + 1u;
      }
      if (vw_b == 0xffffffffu) {
        if (lane == 0) full_p[1] += 1u;
      } else if (ok_b) {
        vw_p[lane + 32] = vw_p[lane + 32] + 1u;
      }
    }
  } else {
    if (lane == 0) {
      vw_p[0] = vw_a;
      vw_p[1] = vw_b;
    }
  }
  return uniform ? 2 : 1;
}

template <int FN, bool FLAGS, bool GROUPED = false, bool UNI = false>
__global__ void __launch_bounds__(kLeanWarps * 32, B2P_LEAN_MIN_BLOCKS) range_lean_kernel(const RangeArgs a) {
  static_assert(!UNI || kLeanUniform<FN, FLAGS>, "no uniform-cadence variant of this instantiation");
  // functions with a uniform-cadence variant: the call launches both kernels, the probe's verdict keeps one
  if constexpr (kLeanUniform<FN, FLAGS>) {
    if ((a.status->uniform != 0u) != UNI) return;
  }
  using LeanRing = LeanRingT<FLAGS>;
  constexpr int RING = kLeanRing;
  using TR = FnTraits<FN>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // smem: [warps][RING] val f64 | [warps][2*RING] ts u32 | [kRcpTable] f64 | [warps][2][64] ts i64 |
  //       [warps][2][64] val f64 (staging of the block being fetched and the block being consumed) |
  //       [warps][RING/32] reset / change bit words (FLAGS variant) | [warps] 32 B window-shape cache
  double* rval = reinterpret_cast<double*>(smem_raw) + warp * RING;
  uint32_t* rts = reinterpret_cast<uint32_t*>(smem_raw + (size_t)kLeanWarps * RING * 8) + warp * (2 * RING);
  double* rcp_tab = reinterpret_cast<double*>(smem_raw + (size_t)kLeanWarps * RING * 16);
  // staging slots of this lane (shared-space byte addresses): [2 halves][64] per warp and column, 8 B elements
  constexpr int kDepth = UNI ? kLeanDepthUni : kLeanDepth;
  const uint32_t stage_t = (uint32_t)__cvta_generic_to_shared(rcp_tab + kRcpTable) + (uint32_t)(warp * (64 * kDepth) + lane) * 8u;
  const uint32_t stage_v = stage_t + (uint32_t)kLeanWarps * (64u * kDepth) * 8u;
  constexpr uint32_t kStageBytes = 512u * kDepth;  // per warp and column
  for (int i = threadIdx.x; i < kRcpTable; i += blockDim.x) rcp_tab[i] = (i > 0) ? 1.0 / (double)i : 0.0;
  __syncthreads();
  LeanRing acc;
  acc.ts = rts;
  acc.val = rval;
  acc.rcp_tab = rcp_tab;
  acc.init_addresses();
  acc.flags_sa = (uint32_t)__cvta_generic_to_shared(rcp_tab + kRcpTable + kLeanWarps * 128 * kDepth) + (uint32_t)warp * (RING / 32) * 4u;
  acc.no_flags = true;
  acc.shape_sa = acc.flags_sa - (uint32_t)warp * (RING / 32) * 4u + (uint32_t)kLeanWarps * (RING / 32) * 4u + (uint32_t)warp * 32u;
  if (lane == 0) sts32(acc.shape_sa + 24u, 0xffffffffu);  // no shape cached yet (a window length never is 2^32 - 1)
  // GROUPED: per-warp "valid throughout" counters of the current group, one per 32-step word (behind everything else)
  uint32_t* const full_w = reinterpret_cast<uint32_t*>(smem_raw + lean_smem_bytes(UNI)) + warp * kLeanFullWords;
  if constexpr (GROUPED) {
    for (int i = lane; i < kLeanFullWords; i += 32) full_w[i] = 0u;
    __syncwarp();
  }
  const uint32_t total_warps = gridDim.x * kLeanWarps;
  const int32_t T = (int32_t)a.T;
  const long long tb_off = a.tb - a.offset;  // rel = ts + offset - tb
  const uint32_t step32 = 32u * (uint32_t)a.interval;
  const uint32_t te_lane0 = (uint32_t)a.range + (uint32_t)lane * (uint32_t)a.interval;
  const uint32_t te31_minus_tlo0 = (uint32_t)a.range + 31u * (uint32_t)a.interval;  // te of step k+31 minus tlo of step k

  // Block 0 of a series is put in flight (into staging half 0) before the series starts: for the first series
  // right here, for every later one while its predecessor still evaluates its last groups; the offsets of the
  // next series are loaded at the start of the current one.
  auto issue_block0 = [&](uint64_t r0, uint64_t r1) {
    const uint64_t rows = r1 - r0;
    const uint32_t cnt = rows > 0xfffffff0ull ? 0u : (uint32_t)rows;  // oversize series are not evaluated here
    const long long* pt0 = reinterpret_cast<const long long*>(a.ts + r0) + lane;
    const double* pv0 = a.val + r0 + lane;
#pragma unroll
    for (int d = 0; d < kDepth - 1; ++d) {  // blocks 0 .. depth-2, one commit group each (empty past the end)
      const uint32_t o = 512u * d, r = 64u * d + (uint32_t)lane;
      if (r < cnt) { cp_async8(stage_t + o, pt0 + 64 * d); cp_async8(stage_v + o, pv0 + 64 * d); }
      if (r + 32u < cnt) { cp_async8(stage_t + o + 256u, pt0 + 64 * d + 32); cp_async8(stage_v + o + 256u, pv0 + 64 * d + 32); }
      cp_async_commit();
    }
  };
  // GROUPED: the warp walks whole groups, each group's member series in CSR order; groups are dealt out dynamically
  // (one atomic counter per launch) so that CTAs which start late — the all-reduce of the previous tile may hold a few
  // SMs — simply take fewer groups.  (grp, m, m_end) is the position of the current series, the *_n copies that of
  // the next one.
  uint32_t grp = 0, m = 0, m_end = 0, grp_n = 0, m_n = 0, m_end_n = 0;
  auto group_first = [&](uint32_t& g_o, uint32_t& m_o, uint32_t& e_o) {  // next non-empty group from the counter
    uint32_t g = a.g_hi, lo = 0, hi = 0;
    for (;;) {
      uint32_t t = 0;
      if (lane == 0) t = atomicAdd(&a.status->g_next, 1u);
      t = __shfl_sync(0xffffffffu, t, 0);
      g = a.g_lo + t;
      if (g >= a.g_hi || t >= a.g_hi) { g = a.g_hi; break; }
      lo = a.g_off[g];
      hi = a.g_off[g + 1];
      if (hi > lo) break;
    }
    g_o = g; m_o = lo; e_o = hi;
    return g < a.g_hi;
  };
#if B2P_LEAN_CONTIG
  // every CTA owns one contiguous range of series and its warps sweep it side by side: the SM's streams (ts, val, out)
  // stay inside a few 2 MB pages at any time and move on together
  const uint32_t per_cta = (a.n_series + gridDim.x - 1) / gridDim.x;
  const uint32_t s_end = min(a.n_series, (blockIdx.x + 1u) * per_cta);
  uint32_t s = blockIdx.x * per_cta + warp;
  bool have = s < s_end;
#else
  const uint32_t s_end = a.n_series;
  uint32_t s = blockIdx.x * kLeanWarps + warp;
  bool have = s < a.n_series;
#endif
  if constexpr (GROUPED) {
    have = group_first(grp, m, m_end);
    if (have) s = a.g_members[m];
  }
  uint64_t row0 = 0, row1 = 0;
  if (have) {
    row0 = a.offsets[s];
    row1 = a.offsets[s + 1];
    issue_block0(row0, row1);
  }
  while (have) {
#if B2P_LEAN_CONTIG
    uint32_t s_next = s + kLeanWarps;
#else
    uint32_t s_next = s + total_warps;
#endif
    bool have_next = s_next < s_end;
    if constexpr (GROUPED) {
      if (m + 1u < m_end) {
        grp_n = grp; m_n = m + 1u; m_end_n = m_end;
        have_next = true;
      } else {
        have_next = group_first(grp_n, m_n, m_end_n);
      }
      if (have_next) s_next = a.g_members[m_n];
    }
    uint64_t nrow0 = 0, nrow1 = 0;
    if (have_next) {
      nrow0 = a.offsets[s_next];
      nrow1 = a.offsets[s_next + 1];
    }
    bool next_issued = false;
    const uint32_t n = (uint32_t)(row1 - row0);
    int defer = ((n == 0u) || (row1 - row0 > 0xfffffff0ull)) ? 3 : 0;  // reason code, 0 = stays on this tier
    uint32_t k_done = 0;  // GROUPED: steps of this series already added to the partials when it leaves the tier
    if (!defer) {
      const int64_t* ts_s = a.ts + row0;
      const double* val_s = a.val + row0;
      double* out_p = GROUPED ? a.gsum + (size_t)grp * (size_t)T + lane : a.out + (size_t)s * (size_t)T + lane;
      uint32_t* vw_p = GROUPED ? a.gcnt + (size_t)grp * (size_t)T : a.valid + (size_t)s * a.Tw;
      constexpr int kVwGroup = GROUPED ? 32 : 1;  // advance of vw_p per 32-step group (counts vs validity words)
      uint32_t* full_p = full_w;
      double* const out_p0 = out_p;
      LeanState st;
      st.j_cnt = 0; st.base_lo = 0; st.base_hi = -1; st.d_lo = 0; st.d_hi = 32; st.phase = 0; st.last_flag = 0;
      st.reg_from = 0;
      uint32_t te = te_lane0;                                      // window end of step k_next + lane
      uint32_t te31 = (uint32_t)a.range + 31u * (uint32_t)a.interval;  // ... of step k_next + 31
      __syncwarp();
      if (lane == 0) acc.put(0xffffffffu, 0u, -__longlong_as_double(0x7ff0000000000000ll));  // slot -1: (0, -inf)

      // rows in 64-row blocks, lane owns rows j+lane and j+32+lane; the block after the one being consumed is
      // in flight into the other half of the staging area (cp.async, one commit group per block)
      const long long* p_t = reinterpret_cast<const long long*>(ts_s) + lane;
      const double* p_v = val_s + lane;
      // uniform-cadence kernel: the previous block was followed by exactly one uniform pair and nothing else (see
      // lean_pair's STEADY form)
      [[maybe_unused]] bool steady = false;
      uint32_t half = 0;                              // staging slot (byte offset) of the block being consumed
      uint32_t ahead = 512u * (kDepth - 1);       // ... of the block put in flight next
      while (st.j_cnt < n) {
        const uint32_t j0 = st.j_cnt;  // multiple of 64
        const uint32_t left = n - j0;
        const bool in0 = (uint32_t)lane < left, in1 = (uint32_t)lane + 32u < left;
        {
          constexpr uint32_t kA = 64u * (kDepth - 1);  // rows ahead
          if ((uint32_t)lane + kA < left) { cp_async8(stage_t + ahead, p_t + kA); cp_async8(stage_v + ahead, p_v + kA); }
          if ((uint32_t)lane + kA + 32u < left) { cp_async8(stage_t + ahead + 256u, p_t + kA + 32); cp_async8(stage_v + ahead + 256u, p_v + kA + 32); }
          cp_async_commit();
          p_t += 64;
          p_v += 64;
          ahead = ahead + 512u == kStageBytes ? 0u : ahead + 512u;
        }
        cp_async_wait<kDepth - 1>();  // everything but the newest depth-1 groups: the block to consume has landed
        const long long c_t0 = lds_s64(stage_t + half), c_t1 = lds_s64(stage_t + half + 256u);
        const double c_v0 = LeanRing::lds64(stage_v + half), c_v1 = LeanRing::lds64(stage_v + half + 256u);
        half = half + 512u == kStageBytes ? 0u : half + 512u;
        // SeriesNormalize (offset bias) + 32-bit time domain, append to the ring: the block occupies slots
        // (j0 mod RING) + [0, 64), which never wrap, and their mirrors RING further
        const uint32_t slot = (j0 & (uint32_t)(RING - 1)) + (uint32_t)lane;
        const uint32_t pt = acc.ts_sa + slot * 4u;  // shared-space addresses of the lane's first row
        const uint32_t pv = acc.val_sa + slot * 8u;
        uint32_t r0, r1;
        {
          const long long d = c_t0 - tb_off;
          const int32_t dh = (int32_t)(d >> 32);
          const uint32_t dl = (uint32_t)d;
          const uint32_t in = dl < a.rel_max ? dl : a.rel_max;
          r0 = dh == 0 ? in : (dh < 0 ? 0u : a.rel_max);
          if (in0) { sts32(pt, r0); sts32(pt + RING * 4u, r0); sts64(pv, c_v0); }
        }
        {
          const long long d = c_t1 - tb_off;
          const int32_t dh = (int32_t)(d >> 32);
          const uint32_t dl = (uint32_t)d;
          const uint32_t in = dl < a.rel_max ? dl : a.rel_max;
          r1 = dh == 0 ? in : (dh < 0 ? 0u : a.rel_max);
          if (in1) { sts32(pt + 128u, r1); sts32(pt + 128u + RING * 4u, r1); sts64(pv + 256u, c_v1); }
        }
        __syncwarp();
        bool bad = (a.filter_nan != 0) & ((in0 & isnan(c_v0)) | (in1 & isnan(c_v1)));
        // uniform cadence: is every new sample exactly one eval interval after its predecessor (the mirror of slot - 1
        // and slot + 31; the first sample of a series has none)?  A break behind a sample clamped to 0 (history before
        // start - range) only restarts the run; any other break gives the series up for this path (reg_from = ~0), so
        // jittered series pay for one block's check only.
        bool odd = false, hard = false;
        if constexpr (UNI) {
          if (st.reg_from != 0xffffffffu) {
            const uint32_t pr0 = LeanRing::lds32(pt + RING * 4u - 4u), pr1 = LeanRing::lds32(pt + 124u);
            const bool o0 = in0 & ((j0 | (uint32_t)lane) != 0u) & (r0 - pr0 != (uint32_t)a.interval);
            const bool o1 = in1 & (r1 - pr1 != (uint32_t)a.interval);
            odd = o0 | o1;
            hard = (o0 & (pr0 != 0u)) | (o1 & (pr1 != 0u));
          }
        }
        if constexpr (FLAGS) {
          // reset / change bit of every new sample against its predecessor (slot -1 of a series holds -inf, so
          // its first sample is never a reset; for changes() it is masked explicitly): the block is 64-aligned,
          // so its two ballots are exactly two bit words
          const double p0 = LeanRing::lds64(acc.val_sa + (((slot - 1u) & (uint32_t)(RING - 1)) << 3));
          const double p1 = LeanRing::lds64(pv + 248u);
          bool f0 = in0 & flag_pred<FN>(c_v0, p0);
          const bool f1 = in1 & flag_pred<FN>(c_v1, p1);
          if constexpr (TR::kFlagChange) f0 = f0 & ((j0 | (uint32_t)lane) != 0u);
          const uint32_t b0 = __ballot_sync(0xffffffffu, f0), b1 = __ballot_sync(0xffffffffu, f1);
          if (lane == 0) {
            sts32(acc.flags_sa + (((j0 >> 5) & (uint32_t)(RING / 32 - 1)) << 2), b0);
            sts32(acc.flags_sa + ((((j0 >> 5) + 1u) & (uint32_t)(RING / 32 - 1)) << 2), b1);
          }
          if (b1) st.last_flag = j0 + 63u - (uint32_t)__clz(b1);
          else if (b0) st.last_flag = j0 + 31u - (uint32_t)__clz(b0);
        } else if constexpr (TR::kCounter) {
          // slot -1 of a series holds -inf, so its first sample never counts as a reset
          const double p0 = LeanRing::lds64(acc.val_sa + (((slot - 1u) & (uint32_t)(RING - 1)) << 3));
          const double p1 = LeanRing::lds64(pv + 248u);
          bad = bad | (in0 & (c_v0 < p0)) | (in1 & (c_v1 < p1));
        }
        [[maybe_unused]] bool broken = false;  // (uniform-cadence kernel) a break in the cadence inside this block
        if (__any_sync(0xffffffffu, bad | odd)) {
          if (__any_sync(0xffffffffu, bad)) { defer = 4; break; }
          if constexpr (UNI) broken = true;
          // the run of equally spaced samples restarts at the newest one, or the series is not one of those
          st.reg_from = __any_sync(0xffffffffu, hard) ? 0xffffffffu : j0 + (left < 64u ? left : 64u) - 1u;
        }
        if constexpr (FLAGS) __syncwarp();  // the bit words are read by every lane below
        st.j_cnt = j0 + (left < 64u ? left : 64u);
        const uint32_t t_new = acc.tm(st.j_cnt - 1u);
        if constexpr (UNI) {
          // (the uniform-cadence kernel's copy of the block epilogue below: the steady form in front, and the bookkeeping
          // that arms it; kept apart so that the general kernel's code is exactly what it was)
          auto past_the_grid = [&]() {
            if (t_new < a.rel_max) return false;
            if (a.filter_nan) {
              bool nan_left = false;
              for (uint32_t j = st.j_cnt + (uint32_t)lane; j < n; j += 32u) nan_left = nan_left | isnan(val_s[j]);
              if (__any_sync(0xffffffffu, nan_left)) defer = 6;
            }
            return true;
          };
          if (B2P_LEAN_STEADY && steady && !broken && left >= 64u) {
            lean_pair<FN, FLAGS, GROUPED, UNI, true>(a, st, acc, te, step32, out_p, vw_p, lane, full_p);
            te += 2u * step32;
            te31 += 2u * step32;
            out_p += 64;
            vw_p += 2 * kVwGroup;
            full_p += 2;
            if (past_the_grid()) break;
            continue;  // (the ring holds what it held one block ago, moved on by 64 samples: room for the next block)
          }
          uint32_t n_pairs = 0, n_groups = 0;
          int last_pair = 0;
          while (te31 < t_new) {
            if (B2P_LEAN_PAIR && te31 + step32 < t_new && (last_pair = lean_pair<FN, FLAGS, GROUPED, UNI>(a, st, acc, te, step32, out_p, vw_p, lane, full_p)) != 0) {
              te += 2u * step32;
              te31 += 2u * step32;
              out_p += 64;
              vw_p += 2 * kVwGroup;
              full_p += 2;
              ++n_pairs;
              continue;
            }
            ++n_groups;
            if ((defer = lean_group<FN, false, FLAGS, GROUPED>(a, st, acc, GROUPED ? st.j_cnt : n, te, 0, 0, out_p, vw_p, lane, full_p))) break;
            te += step32;
            te31 += step32;
            out_p += 32;
            vw_p += kVwGroup;
            full_p += 1;
          }
          if (defer) break;
          steady = n_pairs == 1u && n_groups == 0u && last_pair == 2;
          if (past_the_grid()) break;
        } else {
        // every group whose last window end is older than the newest sample is final
        while (te31 < t_new) {
          if (B2P_LEAN_PAIR && te31 + step32 < t_new && lean_pair<FN, FLAGS, GROUPED, UNI>(a, st, acc, te, step32, out_p, vw_p, lane, full_p)) {
            te += 2u * step32;
            te31 += 2u * step32;
            out_p += 64;
            vw_p += 2 * kVwGroup;
            full_p += 2;
            continue;
          }
          // GROUPED: what is added cannot be taken back if a NaN shows up later in the series and lowers the sample
          // count m the cursor starts are compared with — compare with the samples seen so far instead (m >= j_cnt;
          // at worst a series is handed on that could have stayed)
          if ((defer = lean_group<FN, false, FLAGS, GROUPED>(a, st, acc, GROUPED ? st.j_cnt : n, te, 0, 0, out_p, vw_p, lane, full_p))) break;
          te += step32;
          te31 += step32;
          out_p += 32;
          vw_p += kVwGroup;
          full_p += 1;
        }
        if (defer) break;
        // a sample past the last window end: every remaining step is final and the rest of the series cannot
        // reach a window any more; it still has to be free of NaN samples (SeriesNormalize would drop them and
        // change the sample count m the cursor starts were compared with)
        if (t_new >= a.rel_max) {
          if (a.filter_nan) {
            bool nan_left = false;
            for (uint32_t j = st.j_cnt + (uint32_t)lane; j < n; j += 32u) nan_left = nan_left | isnan(val_s[j]);
            if (__any_sync(0xffffffffu, nan_left)) defer = 6;
          }
          break;
        }
        }
        // nothing seen so far can be inside a window that is still to come (history before the query): restart
        // both edges behind it.  Only before the first non-empty window, where last_range_start is still 0.
        if (st.phase == 0u && t_new <= te31 - te31_minus_tlo0) {
          st.base_lo = st.j_cnt;
          st.base_hi = (int32_t)st.j_cnt - 1;
        }
        // room for the next block (and the end sentinel) behind the oldest sample a window may still need
        if (st.j_cnt + 66u - st.base_lo > (uint32_t)RING) { defer = 5; break; }
      }
      if (!defer) {
        // ---- end of stream: sentinel, end trim (range_manipulate.rs:722-728), remaining groups -------
        cp_async_wait<0>();  // (an early finish leaves a block in flight) the staging area is free from here on
        issue_block0(nrow0, nrow1);
        next_issued = true;
        __syncwarp();  // lanes past the end of the last block have read (and ignored) the slot the sentinel takes
        if (lane == 0) acc.put(st.j_cnt, 0xffffffffu, 0.0);
        __syncwarp();
        int32_t kl = T - 1;
        {
          const int64_t d = ts_s[n - 1u] - tb_off;  // newest sample, ms since start - range
          if (d < 0) {
            kl = -1;  // every sample is older than every window
          } else if (d < (int64_t)a.rel_max) {
            // last_aligned = trunc((last_ts + range) / interval) * interval, aligned to 0 (not to start);
            // last_ts + range = start + d, so (last_ts + range) mod interval = (start_mod + d) mod interval
            // both quotients by reciprocal multiply + one correction step (operands < 2^32: the double product
            // is within 1 of the quotient)
            const uint32_t iv = (uint32_t)a.interval;
            const uint32_t x = a.start_mod + (uint32_t)d;
            uint32_t qx = (uint32_t)__double2uint_rz((double)x * a.rcp_interval);
            if ((unsigned long long)qx * iv > x) --qx; else if (x - qx * iv >= iv) ++qx;  // 64-bit: qx*iv < x + iv
            const uint32_t xm = x - qx * iv;  // x mod iv
            if ((uint32_t)d >= xm) {
              const uint32_t y = (uint32_t)d - xm;  // a multiple of iv away from start: last_aligned - start
              uint32_t qy = (uint32_t)__double2uint_rz((double)y * a.rcp_interval);
              if ((unsigned long long)qy * iv > y) --qy; else if (y - qy * iv >= iv) ++qy;
              kl = (int32_t)qy;
            } else {
              kl = -1;
            }
            kl = kl > T - 1 ? T - 1 : kl;
          }
        }
        for (int32_t k_next = (int32_t)(out_p - out_p0); k_next < T; k_next += 32) {
          if ((defer = lean_group<FN, true, FLAGS, GROUPED>(a, st, acc, n, te, k_next + lane, kl, out_p, vw_p, lane, full_p))) break;
          te += step32;
          out_p += 32;
          vw_p += kVwGroup;
          full_p += 1;
        }
      }
      k_done = (uint32_t)(out_p - out_p0);
    }
    if (defer && lane == 0) {
#ifdef B2P_LEAN_DEBUG
      printf("lean: series %u leaves the tier, reason %d\n", s, defer);
#endif
      const uint32_t i = atomicAdd(&a.status->w_count, 1u);
      a.w_list[i] = s;
      if constexpr (GROUPED) a.w_skip[i] = k_done;
    }
    if (!next_issued) {  // the series left the tier before its end of stream
      cp_async_wait<0>();
      issue_block0(nrow0, nrow1);
    }
    row0 = nrow0;
    row1 = nrow1;
    s = s_next;
    have = have_next;
    if constexpr (GROUPED) {
      if (!have_next || grp_n != grp) {
        // leaving the group: its "valid throughout" counters join the count row (coalesced, one word at a time)
        __syncwarp();
        uint32_t* gc = a.gcnt + (size_t)grp * (size_t)T + lane;
        for (uint32_t w = 0; w < a.Tw; ++w) {
          const uint32_t c = full_w[w];
          if (c != 0u && (int32_t)(w * 32u + (uint32_t)lane) < T) gc[w * 32u] += c;
        }
        __syncwarp();
        for (uint32_t w = lane; w < a.Tw; w += 32) full_w[w] = 0u;
      }
      grp = grp_n; m = m_n; m_end = m_end_n;
    }
    __syncwarp();
  }
  cp_async_wait<0>();
}

__host__ __device__ constexpr size_t lean_grouped_smem_bytes(bool uni = false) { return lean_smem_bytes(uni) + (size_t)kLeanWarps * kLeanFullWords * 4; }

// Which first-tier variant a call runs (rate / increase / delta, plain): one CTA looks at up to 1024 series spread over
// the call and counts those of at least 256 samples whose first 8 timestamp deltas all equal the eval interval; when at least half of
// them do, Status::uniform is set and the uniform-cadence kernel runs, else the general one.  Only a performance choice:
// both kernels check what they rely on sample by sample and produce the same bits.
constexpr int kProbeThreads = 1024;
__global__ void __launch_bounds__(kProbeThreads) cadence_probe_kernel(const RangeArgs a) {
  __shared__ uint32_t cnt[2];
  if (threadIdx.x < 2) cnt[threadIdx.x] = 0u;
  __syncthreads();
  const uint32_t k = a.n_series < (uint32_t)kProbeThreads ? a.n_series : (uint32_t)kProbeThreads;
  if (threadIdx.x < k) {
    const uint32_t s = (uint32_t)(((uint64_t)threadIdx.x * a.n_series) / k);
    const uint64_t r0 = a.offsets[s], r1 = a.offsets[s + 1];
    if (r1 - r0 >= 2ull) {
      const uint64_t m = r1 - r0 < 9ull ? r1 - r0 : 9ull;
      int64_t t[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) t[i] = (uint64_t)i < m ? a.ts[r0 + i] : 0;  // (independent loads, one round trip)
      // (short series spend their steps in the head / tail groups, which the uniform-cadence path does not cover, and
      // never reach its steady form: config 4's 128-sample series are slower on it)
      bool regular = r1 - r0 >= 256ull;
#pragma unroll
      for (int i = 1; i < 9; ++i) regular = regular && ((uint64_t)i >= m || t[i] - t[i - 1] == a.interval);
      atomicAdd(&cnt[0], 1u);
      if (regular) atomicAdd(&cnt[1], 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) a.status->uniform = (cnt[0] > 0u && cnt[1] * 2u >= cnt[0]) ? 1u : 0u;
}

}  // namespace b2p
