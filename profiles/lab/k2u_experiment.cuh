// k2u_experiment.cuh — K2U, an EXPERIMENT that is not part of the library: a ring-free first tier for series sampled
// exactly at the eval interval (rate / increase / delta).  Bit-identical to the shipped kernels and parity-green when it
// was wired in, but no faster than the uniform-cadence variant of range_lean_kernel when it was measured (stream_test.cu
// gives the bound of its access pattern), so the library keeps one kernel.  Build:
// k2l_lab.cu with -DLAB_K2U -I profiles/lab.
//
// Same contract as range_lean_kernel (SeriesNormalize -> RangeManipulate -> prom_* UDF -> IS NOT NULL, one warp per
// series, one eval step per lane, dense [S x T] values + validity words), for the series whose timestamps are
// ts[i] = ts[0] + i * interval: aligned scrapes evaluated at the scrape interval (Prometheus aligns scrape timestamps
// to the schedule; the BASELINE generator without jitter).  On such a series RangeManipulate's windows
// (range_manipulate.rs:700-770) need no search: with
//     g0 = floor((start - ts[0]) / interval)               index of the last sample <= the first window end
//     q0 = floor((start - range - ts[0]) / interval) + 1   index of the first sample > the first window start
// step k's window is samples [max(q0 + k, 0), min(g0 + k, n - 1)], so the lane that holds sample i = g0 + k evaluates
// step k: its own value is the window's last one, the first one is a second (cache-resident) read of the column
// L - 1 rows back, and no shared-memory ring, staging or edge verification is needed — the kernel is a 24 B / sample
// stream.  Every window that is cut by neither end of the series has the same shape (length, distances of its edge
// samples to the window edges), so ExtrapolatedRate::calc's factor (extrapolate_rate.rs:240-284) is computed once per
// shape (extrapolate_factor) and a step costs one subtraction, the to_start test and one multiplication; steps whose
// window is cut, or whose zero crossing may fall inside the window, take extrapolate_parts itself.  Both are the
// identical sequence of IEEE operations the other tiers run, so the results are the same bits.
//
// What is checked, sample by sample, while the series streams through: the timestamp is exactly ts[0] + i * interval,
// the value is not NaN (SeriesNormalize would drop it, normalize.rs:417-426) and, for counters, not below its
// predecessor (no reset correction on this tier).  A series that fails — or whose first non-empty window would hit
// calculate_range's cursor-start quirk (DESIGN.md C-13), or whose start lies more than 2^31 ms from the query — is
// handed to range_fast_kernel through RangeArgs::w_list, exactly like a series leaving range_lean_kernel; what has
// been written for it by then is overwritten.
//
// Whether a call runs this kernel or range_lean_kernel is cadence_probe_kernel's verdict (Status::uniform): both are
// launched, one returns at once.
#pragma once
#include "b2p_kernel_lean.cuh"

namespace b2p {

#ifndef B2P_UNI_WARPS
#define B2P_UNI_WARPS 8
#endif
#ifndef B2P_UNI_MIN_BLOCKS
#define B2P_UNI_MIN_BLOCKS 4
#endif
#ifndef B2P_UNI_UNROLL
#define B2P_UNI_UNROLL 4
#endif
constexpr int kUniWarps = B2P_UNI_WARPS;
// 32-step chunks a warp fetches in one go: kUniUnroll * 256 contiguous bytes of each column requested back to back keep
// DRAM rows open, and they are the bytes in flight per warp (profiles/lab/stream_test.cu measures this access pattern
// for 1 - 8 chunks; cp.async staging queues of 4 - 16 chunks in shared memory were slower)
constexpr int kUniUnroll = B2P_UNI_UNROLL;
#ifndef B2P_UNI_SHUF
#define B2P_UNI_SHUF 1
#endif
#ifndef B2P_UNI_STREAM_INLINE
#define B2P_UNI_STREAM_INLINE __noinline__
#endif
#ifndef B2P_UNI_FULL_INLINE
#define B2P_UNI_FULL_INLINE __noinline__
#endif
#ifndef B2P_UNI_VWACC
#define B2P_UNI_VWACC 1
#endif
#ifndef B2P_UNI_PREFETCH
#define B2P_UNI_PREFETCH 1
#endif

template <int FN>
constexpr bool kHasUniformKernel = B2P_LEAN_UNIFORM && FnTraits<FN>::kExtrapolated;

// floor(x / iv) for |x| < 2^32 by reciprocal multiply and one correction step (the double product is within 1 of the
// quotient), iv > 0
__device__ __forceinline__ int64_t floor_div_small(int64_t x, uint32_t iv, double rcp_iv) {
  const bool neg = x < 0;
  const uint64_t ax = neg ? (uint64_t)(-x) : (uint64_t)x;
  uint64_t q = (uint64_t)__double2ull_rz((double)ax * rcp_iv);
  if (q * iv > ax) --q; else if (ax - q * iv >= iv) ++q;
  return neg ? -(int64_t)(q + (q * iv != ax ? 1u : 0u)) : (int64_t)q;
}

// Last eval step RangeManipulate visits for a series whose newest sample lies d ms after start - range: the end is
// trimmed to trunc((last_ts + range) / interval) * interval, aligned to 0 and not to start (range_manipulate.rs:722-728).
// -1: none.
__device__ __forceinline__ int32_t end_trim_last_step(const RangeArgs& a, int64_t d, int32_t T) {
  if (d < 0) return -1;  // every sample is older than every window
  if (d >= (int64_t)a.rel_max) return T - 1;
  // last_ts + range = start + d, so (last_ts + range) mod interval = (start_mod + d) mod interval; both quotients by
  // reciprocal multiply + one correction step (operands < 2^32: the double product is within 1 of the quotient)
  const uint32_t iv = (uint32_t)a.interval;
  const uint32_t x = a.start_mod + (uint32_t)d;
  uint32_t qx = (uint32_t)__double2uint_rz((double)x * a.rcp_interval);
  if ((unsigned long long)qx * iv > x) --qx; else if (x - qx * iv >= iv) ++qx;  // 64-bit: qx*iv < x + iv
  const uint32_t xm = x - qx * iv;  // x mod iv
  if ((uint32_t)d < xm) return -1;
  const uint32_t y = (uint32_t)d - xm;  // a multiple of iv away from start: last_aligned - start
  uint32_t qy = (uint32_t)__double2uint_rz((double)y * a.rcp_interval);
  if ((unsigned long long)qy * iv > y) --qy; else if (y - qy * iv >= iv) ++qy;
  const int32_t kl = (int32_t)qy;
  return kl > T - 1 ? T - 1 : kl;
}

// The steps that cannot use the shape's factor (window cut by an end of the series, zero crossing possibly inside the
// window) are few: ExtrapolatedRate::calc in full, out of line so that it does not weigh on the streaming loop's registers.
template <int FN>
__device__ B2P_UNI_FULL_INLINE double uni_full_value(double result_value, double first_value, uint32_t t_lo, uint32_t t_hi, uint32_t l,
                                              uint32_t te, uint32_t range, double range_secs, double rcp_rs) {
  return extrapolate_parts<FN, uint32_t, true>(result_value, first_value, t_lo, t_hi, l, te, range, 1.0 / (double)(l - 1u),
                                               range_secs, rcp_rs);
}

// What a series needs on this tier (warp-uniform).
struct UniSeries {
  const int64_t* ts_s;
  const double* val_s;
  double* out_s;
  uint32_t* vw_s;
  int64_t ts0, d0;     // first timestamp; the same in ms after start - range (may be negative: history)
  int32_t n, g0, q0, kl, T;
  // shape of the windows cut by neither end of the series
  uint32_t len;
  bool far;
  double factor;
};

// kUniUnroll aligned chunks of 32 steps in the middle of a series (the streaming loop of the kernel): every lane holds
// a sample (i = g0 + k >= 1), every step is on the grid and before the trimmed end, no window is cut.  The chunks'
// loads are in flight together.  The window's first value (back samples back) and the sample's predecessor come out
// of the warp's registers by shuffle when the window spans at most 33 samples (SHUF; `carry` = the lane's value one
// chunk before the unit), else they are second reads of lines the value stream has just brought in.  A step whose
// to_start may move (extrapolate_parts' zero crossing) is recomputed in full afterwards.
// Returns true when a sample breaks the tier's conditions.
template <int FN, bool SHUF>
__device__ B2P_UNI_STREAM_INLINE bool uni_unit_interior(const RangeArgs& a, const UniSeries& S, int32_t kb, int lane, double& carry) {
  using TR = FnTraits<FN>;
  constexpr int U = kUniUnroll;
  const int32_t i0 = kb + S.g0 + lane;
  const long long* p_t = reinterpret_cast<const long long*>(S.ts_s) + i0;
  const double* p_v = S.val_s + i0;
  double* p_o = S.out_s + kb + lane;
  const int32_t back = (int32_t)S.len - 1;
  long long t[U];
  double v[U], first[U];
  [[maybe_unused]] double prev[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    t[u] = p_t[32 * u];
    v[u] = p_v[32 * u];
  }
  if constexpr (!SHUF) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      first[u] = p_v[32 * u - back];
      if constexpr (TR::kCounter) prev[u] = p_v[32 * u - 1];
    }
  }
  // SHUF: the lane that is asked provides the right chunk: lane s serves lane (s + back) & 31, which is in the same
  // chunk iff s + back < 32; the predecessor of lane 0 is lane 31 of the chunk before
  const int src_f = (lane - back) & 31, src_p = (lane - 1) & 31;
  const bool same_f = lane + back < 32;
  const long long t_exp = S.ts0 + (long long)i0 * (long long)a.interval;
  const long long chunk_ms = 32ll * (long long)a.interval;
  bool bad = false;
  uint32_t redo = 0u;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    if constexpr (SHUF) {
      const double before = u == 0 ? carry : v[u - 1];
      first[u] = __shfl_sync(0xffffffffu, same_f ? v[u] : before, src_f);
      if constexpr (TR::kCounter) prev[u] = __shfl_sync(0xffffffffu, lane == 31 ? before : v[u], src_p);
    }
    bad = bad || (t[u] != t_exp + (long long)u * chunk_ms) || (a.filter_nan != 0 && isnan(v[u]));
    if constexpr (TR::kCounter) bad = bad || (v[u] < prev[u]);
    const double result_value = v[u] - first[u];
    if constexpr (TR::kCounter) {
      const bool plain = !(result_value > 0.0 && first[u] >= 0.0) || (B2P_LEAN_FAR && S.far && first[u] >= result_value);
      if (!plain) redo |= 1u << u;
    }
    p_o[32 * u] = result_value * S.factor;
  }
  carry = v[U - 1];
  if constexpr (TR::kCounter) {
    if (__any_sync(0xffffffffu, redo != 0u)) {
      for (int u = 0; u < U; ++u) {  // (not unrolled: the rare steps that need ExtrapolatedRate::calc in full)
        if ((redo >> u) & 1u) {
          const int32_t g = i0 + 32 * u, q = g - back, k = kb + 32 * u + lane;
          const double first_value = S.val_s[q];
          const double result_value = S.val_s[g] - first_value;
          const uint32_t t_hi = (uint32_t)(S.d0 + (int64_t)g * a.interval), t_lo = (uint32_t)(S.d0 + (int64_t)q * a.interval);
          S.out_s[k] = uni_full_value<FN>(result_value, first_value, t_lo, t_hi, S.len, (uint32_t)a.range + (uint32_t)k * (uint32_t)a.interval,
                                          (uint32_t)a.range, a.range_secs, a.rcp_rs);
        }
      }
    }
  }
  return bad;
}

// kUniUnroll aligned chunks anywhere: steps off the grid, lanes without a sample, windows cut by either end of the
// series, steps past the trimmed end — the first and the last unit of a series.  Loads in flight together like the
// interior unit's; `words` receives the validity word of every chunk.
template <int FN>
__device__ B2P_UNI_STREAM_INLINE bool uni_unit_general(const RangeArgs& a, const UniSeries& S, int32_t kb, int lane, double& carry,
                                                       uint32_t (&words)[kUniUnroll]) {
  using TR = FnTraits<FN>;
  constexpr int U = kUniUnroll;
  const uint32_t iv = (uint32_t)a.interval, rng = (uint32_t)a.range;
  const int32_t i0 = kb + S.g0 + lane;
  const int32_t back = (int32_t)S.len - 1;
  long long t[U];
  double v[U], first[U];
  [[maybe_unused]] double prev[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int32_t i = i0 + 32 * u;
    const bool has = i >= 0 && i < S.n;
    t[u] = has ? S.ts_s[i] : 0;
    v[u] = has ? S.val_s[i] : 0.0;
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int32_t i = i0 + 32 * u;
    first[u] = (i >= back && i < S.n) ? S.val_s[i - back] : 0.0;
    if constexpr (TR::kCounter) prev[u] = (i >= 1 && i < S.n) ? S.val_s[i - 1] : 0.0;
  }
  bool bad = false;
  uint32_t redo = 0u, okm = 0u;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int32_t i = i0 + 32 * u, k = kb + 32 * u + lane;
    const bool has = i >= 0 && i < S.n;
    bad = bad || (has && ((t[u] != S.ts0 + (int64_t)i * (int64_t)iv) || (a.filter_nan != 0 && isnan(v[u]))));
    if constexpr (TR::kCounter) bad = bad || (has && i >= 1 && v[u] < prev[u]);
    const bool grid = k >= 0 && k < S.T && k <= S.kl;
    // uncut window over a sample of its own: the shape at hand
    bool fast = grid && has && i >= back && S.len >= 2u;
    const double result_value = v[u] - first[u];
    if constexpr (TR::kCounter)
      fast = fast && (!(result_value > 0.0 && first[u] >= 0.0) || (B2P_LEAN_FAR && S.far && first[u] >= result_value));
    if (k >= 0 && k < S.T) S.out_s[k] = fast ? result_value * S.factor : 0.0;
    if (fast) okm |= 1u << u;
    else if (grid) redo |= 1u << u;
  }
  carry = v[U - 1];
  for (int u = 0; u < U; ++u) {  // (not unrolled) every other step on the grid: its window as calculate_range cuts it
    const int32_t kc = kb + 32 * u;
    if (kc >= 0 && kc < S.T) {  // (warp-uniform)
      if ((redo >> u) & 1u) {
        const int32_t k = kc + lane, i = k + S.g0;
        const int32_t g = i < S.n ? i : S.n - 1;
        const int32_t qq = S.q0 + k;
        const int32_t q = qq < 0 ? 0 : qq;
        const int32_t l = g - q + 1;
        if (g >= 0 && l >= 2) {
          const double first_value = S.val_s[q];
          const double result_value = S.val_s[g] - first_value;
          const uint32_t t_hi = (uint32_t)(S.d0 + (int64_t)g * (int64_t)iv), t_lo = (uint32_t)(S.d0 + (int64_t)q * (int64_t)iv);
          S.out_s[k] = uni_full_value<FN>(result_value, first_value, t_lo, t_hi, (uint32_t)l, rng + (uint32_t)k * iv, rng, a.range_secs, a.rcp_rs);
          okm |= 1u << u;
        }
      }
      words[u] = __ballot_sync(0xffffffffu, (okm >> u) & 1u);
    }
  }
  return bad;
}

template <int FN>
__global__ void __launch_bounds__(kUniWarps * 32, B2P_UNI_MIN_BLOCKS) range_uniform_kernel(const RangeArgs a) {
  using TR = FnTraits<FN>;
  static_assert(TR::kExtrapolated, "rate / increase / delta only");
  if (a.status->uniform == 0u) return;  // the probe chose the general first tier
  constexpr int U = kUniUnroll;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t total_warps = gridDim.x * kUniWarps;
  const uint32_t iv = (uint32_t)a.interval, rng = (uint32_t)a.range;
  const long long tb_off = a.tb - a.offset;  // rel = ts + offset - tb
  // the shape whose factor is at hand (kept across series: a batch usually has one)
  uint32_t sh_end = 0xffffffffu, sh_start = 0;
  UniSeries S;
  S.T = (int32_t)a.T;
  S.len = 0; S.far = false; S.factor = 0.0;

  // the rows and the first timestamp of a series are fetched while its predecessor streams: per warp a series is a
  // chain of dependent round trips (rows -> first timestamp -> unit after unit), and with a fixed number of warps the
  // length of that chain is what the kernel's time is made of
  uint32_t s = blockIdx.x * kUniWarps + warp;
  uint64_t row0 = 0, row1 = 0;
  int64_t ts0 = 0;
  if (s < a.n_series) {
    row0 = a.offsets[s];
    row1 = a.offsets[s + 1];
    if (row1 > row0) ts0 = a.ts[row0];
  }
  while (s < a.n_series) {
    const uint32_t s_next = s + total_warps;
    uint64_t nrow0 = 0, nrow1 = 0;
    int64_t nts0 = 0;
    if (s_next < a.n_series) {
      nrow0 = a.offsets[s_next];
      nrow1 = a.offsets[s_next + 1];
    }
    bool next_ts_loaded = false;
    const uint64_t n64 = row1 - row0;
    bool defer = (n64 == 0ull) || (n64 > 0x7ffffff0ull);
    S.n = defer ? 1 : (int32_t)n64;
    S.ts_s = a.ts + row0;
    S.val_s = a.val + row0;
    S.ts0 = ts0;
    S.d0 = ts0 - tb_off;  // first sample, ms after start - range
    defer = defer || S.d0 <= -2147483648ll || S.d0 >= 2147483648ll;
    if (!defer) {
      S.g0 = (int32_t)floor_div_small((int64_t)rng - S.d0, iv, a.rcp_interval);
      S.q0 = (int32_t)floor_div_small(-S.d0, iv, a.rcp_interval) + 1;
      // the newest sample of a series on the grid (any other series leaves the tier below, whatever this says)
      S.kl = end_trim_last_step(a, S.d0 + (int64_t)(S.n - 1) * (int64_t)iv, S.T);
      // calculate_range's cursor start after the first non-empty step (last_range_start is still 0 there,
      // range_manipulate.rs:741,757,765-768): if it reaches the sample count while the next window is non-empty the
      // reference's windows differ from the definitional ones (C-13) — the slow path reproduces that
      const int32_t kf = S.g0 < 0 ? -S.g0 : 0;
      if (kf <= S.kl) {
        const int32_t gf = min(S.g0 + kf, S.n - 1), qf = max(S.q0 + kf, 0);
        if (qf <= gf) {
          const int32_t rsi = (gf < S.n - 1 && qf > 0) ? qf - 1 : qf;
          const int32_t gn = min(S.g0 + kf + 1, S.n - 1), qn = max(S.q0 + kf + 1, 0);
          if (kf + 1 <= S.kl && qn <= gn && rsi + qf >= S.n) defer = true;
        }
      }
    }
    if (!defer) {
      const uint32_t len = (uint32_t)(S.g0 - S.q0 + 1);
      const uint32_t to_end = (uint32_t)((int64_t)rng - S.d0 - (int64_t)S.g0 * (int64_t)iv);    // te - t[hi], in [0, iv)
      const uint32_t to_start = (uint32_t)(S.d0 + (int64_t)S.q0 * (int64_t)iv);                 // t[lo] - (te - range), in (0, iv]
      if (to_end != sh_end || to_start != sh_start || len != S.len) {
        sh_end = to_end; sh_start = to_start; S.len = len;
        const uint32_t sampled_i = (len - 1u) * iv;
        S.far = sampled_i >= to_start;
        S.factor = 0.0;
        if (len >= 2u) {
          const double sampled = (double)sampled_i;
          const double average = div_by_rcp(sampled, (double)(len - 1u), 1.0 / (double)(len - 1u));
          S.factor = extrapolate_factor<FN, true>(sampled, average, (double)to_start, (double)to_end, a.range_secs, a.rcp_rs);
        }
      }
      S.out_s = a.out + (size_t)s * (size_t)S.T;
      S.vw_s = a.valid + (size_t)s * a.Tw;
      // steps [0, T) and samples [0, n) (sample i sits at step i - g0), in units of U aligned chunks of 32 steps from
      // k_lo on; [f_lo, f_hi): the steps with uncut windows over samples >= 1, on the grid, before the trimmed end
      const int32_t k_lo = S.g0 > 0 ? -(int32_t)(((uint32_t)S.g0 + 31u) & ~31u) : 0;
      const int32_t k_hi = max(S.T, S.n - S.g0);
      const int32_t f_lo = max(max(0, 1 - S.g0), -S.q0);
      const int32_t f_hi = len >= 2u ? min(min(S.T, S.kl + 1), S.n - S.g0) : f_lo;
      const bool shuf = B2P_UNI_SHUF && len <= 33u;
      // validity words: lane w & 31 keeps word w, 32 words leave as one 128-byte store
      uint32_t vw_acc = 0u;
      auto put_word = [&](int32_t kc, uint32_t w) {  // kc in [0, T), a multiple of 32
        const int32_t wi = kc >> 5;
        if (lane == (wi & 31)) vw_acc = w;
        if ((wi & 31) == 31) S.vw_s[(wi & ~31) + lane] = vw_acc;
      };
      bool bad = false;
      double carry = 0.0;
      for (int32_t kb = k_lo; kb < k_hi && !bad; kb += 32 * U) {
        if (kb >= f_lo && kb + 32 * U <= f_hi) {
          bad = shuf ? uni_unit_interior<FN, true>(a, S, kb, lane, carry) : uni_unit_interior<FN, false>(a, S, kb, lane, carry);
#pragma unroll
          for (int u = 0; u < U; ++u) put_word(kb + 32 * u, 0xffffffffu);
        } else {
          uint32_t words[U];
          bad = uni_unit_general<FN>(a, S, kb, lane, carry, words);
#pragma unroll
          for (int u = 0; u < U; ++u)
            if (kb + 32 * u >= 0 && kb + 32 * u < S.T) put_word(kb + 32 * u, words[u]);
        }
        bad = __any_sync(0xffffffffu, bad);
#if B2P_UNI_PREFETCH
        if (!next_ts_loaded) {
          if (nrow1 > nrow0) nts0 = a.ts[nrow0];
          next_ts_loaded = true;
        }
#endif
      }
      // the words of the last, partial block of 32
      if (!bad && (a.Tw & 31u) != 0u && (uint32_t)lane < (a.Tw & 31u)) S.vw_s[(a.Tw & ~31u) + lane] = vw_acc;
      defer = bad;
    }
    if (defer && lane == 0) a.w_list[atomicAdd(&a.status->w_count, 1u)] = s;
    if (!next_ts_loaded && nrow1 > nrow0) nts0 = a.ts[nrow0];
    row0 = nrow0; row1 = nrow1; ts0 = nts0;
    s = s_next;
  }
}

}  // namespace b2p
