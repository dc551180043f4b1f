// b2p_instant.cuh — PromQL instant-vector math functions and scalar() over dense [rows x T] grids:
//   K9 instant_fn_kernel<FN, VEC>   fn(v) per cell: abs ceil floor sqrt exp ln log2 log10, the trigonometric and
//                                    hyperbolic functions, round, deg, rad, sgn, clamp (clamp_min / clamp_max are
//                                    clamp with one bound at ∓f64::MAX, chosen by the caller), and unary minus
//                                    (the sign bit flipped: -0.0 from 0.0 and a NaN's sign, as Rust's f64 Neg)
//      scalar_reduce_kernel          scalar(): live rows, their min / max series key, live cells on B2P_NO_KEY rows
//      scalar_write_kernel           scalar(): the one series' cells, or NaN at every step
//      i64_to_f64_kernel             an Int64 grid read as Float64 ((double)i64, round to nearest): what DataFusion's
//                                    coercion does before a Float64 projection, aggregate or filter of an Int64 column
//
// The reference projects the function over the value column and then filters `value IS NOT NULL`
// (src/query/src/promql/planner.rs:1012-1101, 1063).  A function of a non-null f64 is never null, so validity never
// changes: an invalid cell stays invalid and holds 0.0, a NaN or ±inf result is a row.
//   * abs ceil floor sqrt deg rad sgn clamp and round are exact: `-fmad=false` and the _rn intrinsics give what Rust's
//     f64 methods give.  deg / rad are one multiplication by the f64 constant 180/π / π/180, like Rust's to_degrees /
//     to_radians; round is `n == 0 ? round(a) : round(a / n) * n` with round half away from zero
//     (src/promql/src/functions/round.rs:52-105); sgn is 0.0 for ±0, else ±1.0 by the sign, NaN stays NaN; clamp is
//     `v < lo ? lo : v > hi ? hi : v` with IEEE comparisons (clamp.rs:75-224), so a NaN value passes through with its
//     bits and a NaN bound never binds.
//   * the transcendental functions are CUDA's; DESIGN.md section 2 states their measured ulp bound against glibc (which
//     Rust's std calls).  log2 of a power of two is its exponent, exact as glibc's.
//
// scalar(v) is ScalarCalculate (src/promql/src/extension_plan/scalar_calculate.rs:532-637): over the whole query, not
// per step.  When every live row (a row with at least one cell) carries one series key, the output is that series'
// cells; when there are no live rows, or live rows of two or more keys, it is NaN at every step.  A row whose labels
// include a NULL carries B2P_NO_KEY: the reference compares a NULL label as None against the "" it recorded for it, so
// such a series counts as one series only while it has a single cell (DESIGN.md, quirks).  Two rows of one key with a
// cell at the same step cannot be one dense row: bit 5 of the status word (-> B2P_E_INVALID).  A key >= n_rows other
// than B2P_NO_KEY is bit 4.
//
// Work unit of K9: one warp per (row, 32-step tile) like K7's scalar form; with T even, each lane handles two steps with
// one 128-bit access (64-step tiles).  Validity words are copied out of place and left alone in place: no ballots.
// HBM traffic per (row, step): 8 B read, 8 B written, plus the validity bit.
#pragma once
#include <cstdint>

#include "b2p_status.cuh"
#include "b2p_window.cuh"

namespace b2p {

enum InstantFn {
  kFnAbs = 0, kFnCeil, kFnFloor, kFnSqrt, kFnExp, kFnLn, kFnLog2, kFnLog10, kFnSin, kFnCos, kFnTan, kFnAsin, kFnAcos,
  kFnAtan, kFnSinh, kFnCosh, kFnTanh, kFnAsinh, kFnAcosh, kFnAtanh, kFnRound, kFnDeg, kFnRad, kFnSgn, kFnClamp,
  kFnNeg,         // B2P_IFN_NEG
  kFnKernelCount  // clamp_min / clamp_max (ids kFnClamp + 1, + 2) run as kFnClamp
};
constexpr uint32_t kScalarNoKey = 0xFFFFFFFFu;

struct InstantFnArgs {
  const double* vals;       // [n_rows x T]
  const uint32_t* valid;    // [n_rows x Tw]
  uint64_t n_rows;
  uint64_t T;
  uint32_t Tw;
  double arg0, arg1;        // round: to_nearest; clamp: lo, hi
  double* out;              // may be vals
  uint32_t* out_valid;      // may be valid (then it is not written)
};

// log2 of a power of two (subnormals included) is its exponent, exactly, as glibc gives it; CUDA's log2 can be an ulp
// off there (log2(8) = 2.9999999999999996, log2(2^-1012) = -1011.9999999999999).  Every other operand is CUDA's.
__device__ __forceinline__ double log2_pow2_exact(double v) {
  const long long b = __double_as_longlong(v);
  const long long e = b >> 52, m = b & 0x000FFFFFFFFFFFFFll;  // (negative and NaN bit patterns fail both tests)
  if (e > 0 && e < 0x7FF && m == 0) return (double)(e - 1023);
  if (e == 0 && m != 0 && (m & (m - 1)) == 0) return (double)(-1074 + 63 - __clzll(m));
  return log2(v);
}

template <int FN>
__device__ __forceinline__ double instant_fn(double v, double a0, double a1) {
  // the sign bit cleared, a NaN's too, as Rust's f64::abs does; PTX abs.f64 leaves a NaN's sign unspecified (it kept
  // -NaN), and the sign of a NaN decides where it falls in the total order that comparisons and sort use
  if (FN == kFnAbs) return __longlong_as_double(__double_as_longlong(v) & 0x7FFFFFFFFFFFFFFFll);
  if (FN == kFnCeil) return ceil(v);
  if (FN == kFnFloor) return floor(v);
  if (FN == kFnSqrt) return __dsqrt_rn(v);
  if (FN == kFnExp) return exp(v);
  if (FN == kFnLn) return log(v);
  if (FN == kFnLog2) return log2_pow2_exact(v);
  if (FN == kFnLog10) return log10(v);
  if (FN == kFnSin) return sin(v);
  if (FN == kFnCos) return cos(v);
  if (FN == kFnTan) return tan(v);
  if (FN == kFnAsin) return asin(v);
  if (FN == kFnAcos) return acos(v);
  if (FN == kFnAtan) return atan(v);
  if (FN == kFnSinh) return sinh(v);
  if (FN == kFnCosh) return cosh(v);
  if (FN == kFnTanh) return tanh(v);
  if (FN == kFnAsinh) return asinh(v);
  if (FN == kFnAcosh) return acosh(v);
  if (FN == kFnAtanh) return atanh(v);
  if (FN == kFnRound) return a0 == 0.0 ? round(v) : __dmul_rn(round(__ddiv_rn(v, a0)), a0);
  if (FN == kFnDeg) return __dmul_rn(v, 57.29577951308232);       // 180.0 / π in f64 (Rust's to_degrees constant)
  if (FN == kFnRad) return __dmul_rn(v, 0.017453292519943295);    // π / 180.0 in f64 (Rust's to_radians)
  if (FN == kFnSgn) return v == 0.0 ? 0.0 : v != v ? v : (v < 0.0 ? -1.0 : 1.0);
  if (FN == kFnNeg) return __longlong_as_double(__double_as_longlong(v) ^ (long long)0x8000000000000000ull);
  return v < a0 ? a0 : v > a1 ? a1 : v;  // kFnClamp
}

template <int FN, bool VEC>
__global__ void __launch_bounds__(256) instant_fn_kernel(const InstantFnArgs a) {
  constexpr uint32_t kSteps = VEC ? 64 : 32;
  const int lane = threadIdx.x & 31;
  const uint64_t T = a.T;
  const uint64_t tiles = (T + kSteps - 1) / kSteps;
  const uint64_t units = a.n_rows * tiles;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  const bool copy_words = a.out_valid != a.valid;
  for (uint64_t u = warp0; u < units; u += n_warps) {
    const uint64_t r = u / tiles;
    const uint64_t k0 = (u - r * tiles) * kSteps;
    const double* srow = a.vals + r * T;
    double* orow = a.out + r * T;
    const uint32_t w0 = (uint32_t)(k0 >> 5);
    if (!VEC) {
      const uint64_t k = k0 + lane;
      const uint32_t word = a.valid[r * a.Tw + w0];
      if (k < T) orow[k] = ((word >> lane) & 1u) ? instant_fn<FN>(srow[k], a.arg0, a.arg1) : 0.0;
      if (copy_words && lane == 0) a.out_valid[r * a.Tw + w0] = word;
    } else {
      // lane owns steps k0 + 2*lane and k0 + 2*lane + 1; T is even, so both exist or neither does
      const uint64_t k = k0 + 2 * (uint64_t)lane;
      if (k < T) {
        const uint32_t wi = w0 + (uint32_t)(lane >> 4);  // validity word holding this lane's two steps
        const uint32_t word = a.valid[r * a.Tw + wi];
        const uint32_t bits = (word >> ((2 * lane) & 31)) & 3u;
        const double2 x = *reinterpret_cast<const double2*>(srow + k);
        *reinterpret_cast<double2*>(orow + k) = make_double2(bits & 1u ? instant_fn<FN>(x.x, a.arg0, a.arg1) : 0.0,
                                                             bits & 2u ? instant_fn<FN>(x.y, a.arg0, a.arg1) : 0.0);
        if (copy_words && (lane & 15) == 0) a.out_valid[r * a.Tw + wi] = word;
      }
    }
  }
}

// ---- scalar() --------------------------------------------------------------------------------------------------
struct ScalarState {
  uint32_t min_key;      // over live rows (init 0xFFFFFFFF)
  uint32_t first_live;   // lowest live row index (init 0xFFFFFFFF)
  uint32_t max_key;      // over live rows (init 0)
  uint32_t last_live;    // highest live row index (init 0)
  uint32_t live_rows;    // (init 0)
  uint32_t null_cells;   // cells on live B2P_NO_KEY rows (init 0; each warp adds at most 2: only 0 / 1 / more matter)
};

struct ScalarArgs {
  const double* vals;     // [n_rows x T]
  const uint32_t* valid;  // [n_rows x Tw]
  const uint32_t* key;    // [n_rows]
  uint32_t n_rows;
  uint64_t T;
  uint32_t Tw;
  double* out;            // [T]
  uint32_t* out_valid;    // [Tw]
  ScalarState* state;
  Status* status;
};

// bits of validity word w that are steps < T (the bits past T of a row's last word are undefined)
__device__ __forceinline__ uint32_t step_mask(uint64_t T, uint64_t w) {
  const uint64_t left = T - w * 32;
  return left >= 32 ? 0xFFFFFFFFu : (1u << left) - 1u;
}

// one warp per row: the OR and the population count of its validity words (steps < T).  Each warp folds its rows into
// registers and adds them to the state with one set of atomics when it is done.
__global__ void __launch_bounds__(256) scalar_reduce_kernel(const ScalarArgs a) {
  const int lane = threadIdx.x & 31;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  uint32_t min_key = 0xFFFFFFFFu, max_key = 0u, first = 0xFFFFFFFFu, last = 0u, live_rows = 0u, null_cells = 0u;
  bool bad_key = false;
  for (uint64_t r = warp0; r < a.n_rows; r += n_warps) {
    uint32_t any = 0, cells = 0;
    for (uint32_t w = lane; w < a.Tw; w += 32) {
      const uint32_t v = a.valid[r * a.Tw + w] & step_mask(a.T, w);
      any |= v;
      cells += __popc(v);
    }
    any = __reduce_or_sync(0xFFFFFFFFu, any);
    cells = __reduce_add_sync(0xFFFFFFFFu, cells);
    const uint32_t k = a.key[r];
    if (k != kScalarNoKey && k >= a.n_rows) {
      bad_key = true;
      continue;
    }
    if (!any) continue;
    min_key = min(min_key, k);
    max_key = max(max_key, k);
    first = min(first, (uint32_t)r);
    last = max(last, (uint32_t)r);
    ++live_rows;
    if (k == kScalarNoKey) null_cells = min(null_cells + min(cells, 2u), 2u);
  }
  if (lane != 0) return;
  if (bad_key) atomicOr(&a.status->k0_errors, kScalarKeyError);
  if (!live_rows) return;
  atomicMin(&a.state->min_key, min_key);
  atomicMax(&a.state->max_key, max_key);
  atomicMin(&a.state->first_live, first);
  atomicMax(&a.state->last_live, last);
  atomicAdd(&a.state->live_rows, live_rows);
  if (null_cells) atomicAdd(&a.state->null_cells, null_cells);
}

// one warp per 32-step output word: either the OR of the live rows' cells (all of one key), values copied bit for bit,
// or NaN at every step with every bit valid
__global__ void __launch_bounds__(256) scalar_write_kernel(const ScalarArgs a) {
  const int lane = threadIdx.x & 31;
  const ScalarState s = *a.state;
  const bool one_series =
      s.live_rows > 0 && s.min_key == s.max_key && (s.min_key != kScalarNoKey || s.null_cells == 1);
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t w = warp0; w < a.Tw; w += n_warps) {
    const uint64_t k = w * 32 + lane;
    const uint32_t live = step_mask(a.T, w);
    uint32_t word = 0;
    double x = 0.0;
    if (!one_series) {
      word = live;
      x = __longlong_as_double(0x7FF8000000000000ll);  // f64::NAN
    } else {
      bool overlap = false;
      for (uint64_t r = s.first_live; r <= s.last_live; ++r) {
        if (a.key[r] != s.min_key) continue;  // (a row with a bad key is not live)
        const uint32_t v = a.valid[r * a.Tw + w] & live;  // (so no value past the row's end is read)
        if (!v) continue;
        overlap |= (word & v) != 0;
        if (((v & ~word) >> lane) & 1u) x = a.vals[r * a.T + k];
        word |= v;
      }
      if (overlap && lane == 0) atomicOr(&a.status->k0_errors, kScalarOverlapError);
    }
    if (k < a.T) a.out[k] = ((word >> lane) & 1u) ? x : 0.0;
    if (lane == 0) a.out_valid[w] = word;
  }
}

// thread per cell; out may be vals
__global__ void __launch_bounds__(256) i64_to_f64_kernel(const long long* vals, uint64_t n, double* out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    out[i] = __ll2double_rn(vals[i]);
}

}  // namespace b2p
