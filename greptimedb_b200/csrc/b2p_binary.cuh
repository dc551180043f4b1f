// b2p_binary.cuh — PromQL binary operators over dense [rows x T] grids:
//   K7 binary_op_kernel<OP, MODE, FORM, VEC>  arithmetic (+ - * / % ^ atan2) and comparisons (== != > < >= <=) of
//                             two node results matched into (lhs row, rhs row) pairs, or of one result and a number.
//                             The reference plans these as ProjectionExec / FilterExec over a HashJoinExec on
//                             (tag columns, time index), src/query/src/promql/planner.rs:556-777, 3436-3546; the join
//                             becomes a host-side series match (b2p_plan.cpp) and this kernel the per-step pass.
//      count_valid_kernel     cnt (== 0 <=> no row) of a by-label aggregate -> validity words
//
// Semantics (restated from the reference, not improved on):
//   * both operands are Float64; `/` and `%` are IEEE (x / 0 = ±inf or NaN, `%` is fmod), `^` is pow, atan2(lhs, rhs)
//   * comparisons order floats by the IEEE 754 totalOrder predicate, which is what arrow-rs' cmp kernels do for f64:
//     -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN, and equal bit patterns compare equal (NaN == NaN)
//   * MODE kArith / kBool: valid iff both sides are valid; kBool stores 1.0 / 0.0.  kFilter (comparison without `bool`)
//     additionally drops the cell when the comparison is false, and a kept cell holds the vector operand's value (the lhs
//     of a vector-vector pair).  An invalid cell holds 0.0.
//   * `-fmad=false` and IEEE div: + - * / % and every comparison are bit-identical to the CPU; pow / atan2 are CUDA's
//     (DESIGN.md section 2 states the bound against glibc), except pow's cases where glibc is exact (pow_exact_cases).
//
// Work unit: one warp per (pair, 32-step tile) — one AND of the two validity words and one ballot per output word.  With
// T even every row starts 16-byte aligned, and the VEC variant has each lane load two steps with one 128-bit access (a
// unit is then 64 steps = two output words).  HBM traffic per (pair, step): 16 B read, 8 B + 1 bit written (the scalar
// form: 8 B read).  Row indices out of range set bit 2 of the status word's k0_errors (b2p_sync -> B2P_E_INVALID) and
// the pair's cells are written invalid; nothing is read out of bounds.
#pragma once
#include <cstdint>

#include "b2p_status.cuh"
#include "b2p_window.cuh"

namespace b2p {

enum BinOp { kOpAdd = 0, kOpSub, kOpMul, kOpDiv, kOpMod, kOpPow, kOpAtan2, kOpEq, kOpNe, kOpGt, kOpLt, kOpGe, kOpLe, kOpCount };
enum BinMode { kArith = 0, kFilter = 1, kBool = 2 };
enum BinForm { kVecVec = 0, kScalarLeft = 1, kScalarRight = 2 };

struct BinaryArgs {
  const double* lhs;        // vector-vector: lhs grid; scalar forms: the vector operand
  const uint32_t* lvalid;
  const uint32_t* lrow;     // [n_pairs] (vector-vector only)
  uint32_t n_lhs;
  const double* rhs;
  const uint32_t* rvalid;
  const uint32_t* rrow;
  uint32_t n_rhs;
  double scalar;
  uint64_t n_pairs;         // output rows
  uint64_t T;
  uint32_t Tw;
  double* out;              // [n_pairs x T]; may alias lhs in the scalar forms
  uint32_t* out_valid;      // [n_pairs x Tw]
  Status* status;
};

// comparisons on f64::total_cmp's key (b2p_window.cuh): the bit pattern as i64, low 63 bits flipped for negative values
template <int OP>
__device__ __forceinline__ bool bin_cmp(double a, double b) {
  const long long ka = total_key(a), kb = total_key(b);
  if (OP == kOpEq) return ka == kb;
  if (OP == kOpNe) return ka != kb;
  if (OP == kOpGt) return ka > kb;
  if (OP == kOpLt) return ka < kb;
  if (OP == kOpGe) return ka >= kb;
  return ka <= kb;
}

__device__ __forceinline__ bool is_snan(double x) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(x);
  return (u & 0x7FF8000000000000ull) == 0x7FF0000000000000ull && (u & 0x000FFFFFFFFFFFFFull) != 0;
}

// pow where glibc's is exact and CUDA's can be an ulp off (pow(19, 2) = 361.00000000000006, pow(2, -1012), 10^17):
// x^1, x^2 and x^-1 are one IEEE operation, x^0.5 of a positive x is sqrt, 2^k is built from its bits (k < -1074
// rounds to 0, k > 1023 to inf, as glibc's does), and an integer x to an integer y in [3, 64] is multiplied out when
// every product is exact (fma(p, q, -pq) == 0; integers cannot underflow).  Every other pair is CUDA's pow.
__device__ __forceinline__ double pow_exact_cases(double x, double y) {
  if (y == 1.0) return x;
  if (y == 2.0) return __dmul_rn(x, x);
  if (y == -1.0) return __ddiv_rn(1.0, x);
  if (y == 0.5 && x > 0.0) return __dsqrt_rn(x);
  const bool y_int = y == rint(y) && fabs(y) <= 2048.0;
  if (x == 2.0 && y_int) {
    const int k = (int)y;
    if (k > 1023) return __longlong_as_double(0x7FF0000000000000ll);
    if (k >= -1022) return __longlong_as_double((long long)(k + 1023) << 52);
    return k >= -1074 ? __longlong_as_double(1ll << (k + 1074)) : 0.0;
  }
  if (y_int && y >= 3.0 && y <= 64.0 && x == rint(x) && x != 0.0 && fabs(x) < 9007199254740992.0) {
    double r = 1.0, p = x;
    bool exact = true;
    for (int n = (int)y;;) {
      if (n & 1) {
        const double q = __dmul_rn(r, p);
        exact = exact && __fma_rn(r, p, -q) == 0.0 && fabs(q) <= 1.7976931348623157e308;
        r = q;
      }
      n >>= 1;
      if (!n || !exact) break;
      const double q = __dmul_rn(p, p);
      exact = exact && __fma_rn(p, p, -q) == 0.0 && fabs(q) <= 1.7976931348623157e308;
      p = q;
    }
    if (exact) return r;
  }
  return pow(x, y);
}

template <int OP>
__device__ __forceinline__ double bin_arith(double a, double b) {
  if (OP == kOpAdd) return __dadd_rn(a, b);
  if (OP == kOpSub) return __dsub_rn(a, b);
  if (OP == kOpMul) return __dmul_rn(a, b);
  if (OP == kOpDiv) return __ddiv_rn(a, b);
  if (OP == kOpMod) return fmod(a, b);  // exact, like Rust's `%` on f64
  if (OP == kOpPow) {
    // glibc's pow (what f64::powf calls) returns NaN when an operand is a signaling NaN, pow(sNaN, 0) and pow(1, sNaN)
    // included, where CUDA's follows C99 Annex F and returns 1
    if (is_snan(a) || is_snan(b)) return __dadd_rn(a, b);
    return pow_exact_cases(a, b);
  }
  return atan2(a, b);
}

// One cell: a / b are the lhs / rhs operand values, v their joint validity.  Returns the validity; *o the value.
template <int OP, int MODE, int FORM>
__device__ __forceinline__ bool bin_cell(double a, double b, bool v, double* o) {
  if (MODE == kArith) {
    *o = v ? bin_arith<OP>(a, b) : 0.0;
    return v;
  }
  const bool c = bin_cmp<OP>(a, b);
  if (MODE == kBool) {
    *o = v ? (c ? 1.0 : 0.0) : 0.0;
    return v;
  }
  const bool keep = v && c;
  *o = keep ? (FORM == kScalarLeft ? b : a) : 0.0;  // the vector operand's value
  return keep;
}

// spreads the low 16 bits of x to the even bit positions
__device__ __forceinline__ uint32_t spread16(uint32_t x) {
  x &= 0xFFFFu;
  x = (x | (x << 8)) & 0x00FF00FFu;
  x = (x | (x << 4)) & 0x0F0F0F0Fu;
  x = (x | (x << 2)) & 0x33333333u;
  x = (x | (x << 1)) & 0x55555555u;
  return x;
}

template <int OP, int MODE, int FORM, bool VEC>
__global__ void __launch_bounds__(256) binary_op_kernel(const BinaryArgs a) {
  constexpr uint32_t kSteps = VEC ? 64 : 32;
  const int lane = threadIdx.x & 31;
  const uint64_t T = a.T;
  const uint64_t tiles = (T + kSteps - 1) / kSteps;
  const uint64_t units = a.n_pairs * tiles;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t u = warp0; u < units; u += n_warps) {
    const uint64_t p = u / tiles;
    const uint64_t k0 = (u - p * tiles) * kSteps;
    uint64_t lr = p, rr = p;
    bool in_range = true;
    if (FORM == kVecVec) {
      lr = a.lrow[p];
      rr = a.rrow[p];
      in_range = lr < a.n_lhs && rr < a.n_rhs;
      if (!in_range && lane == 0) atomicOr(&a.status->k0_errors, kBinRowError);
    }
    double* orow = a.out + p * T;
    uint32_t* ovw = a.out_valid + p * a.Tw;
    const uint32_t w0 = (uint32_t)(k0 >> 5);
    if (!VEC) {
      const uint64_t k = k0 + lane;
      const bool inside = k < T;
      double x = 0.0, y = 0.0;
      bool v = false;
      if (in_range) {
        uint32_t bw = a.lvalid[lr * a.Tw + w0];
        if (FORM == kVecVec) bw &= a.rvalid[rr * a.Tw + w0];
        v = inside && ((bw >> lane) & 1u);
        if (inside) {
          const double vv = a.lhs[lr * T + k];
          if (FORM == kVecVec) {
            x = vv;
            y = a.rhs[rr * T + k];
          } else if (FORM == kScalarLeft) {
            x = a.scalar;
            y = vv;
          } else {
            x = vv;
            y = a.scalar;
          }
        }
      }
      double o;
      const bool ov = bin_cell<OP, MODE, FORM>(x, y, v, &o);
      const uint32_t word = __ballot_sync(0xFFFFFFFFu, ov);
      if (inside) orow[k] = o;
      if (lane == 0) ovw[w0] = word;
    } else {
      // lane owns steps k0 + 2*lane and k0 + 2*lane + 1; T is even, so both exist or neither does
      const uint64_t k = k0 + 2 * (uint64_t)lane;
      const bool inside = k < T;
      const uint32_t wi = w0 + (uint32_t)(lane >> 4);  // validity word holding this lane's two steps
      const int sh = (2 * lane) & 31;
      double2 x = make_double2(0.0, 0.0), y = make_double2(0.0, 0.0);
      uint32_t bits = 0;
      if (in_range && inside) {
        uint32_t bw = a.lvalid[lr * a.Tw + wi];
        if (FORM == kVecVec) bw &= a.rvalid[rr * a.Tw + wi];
        bits = (bw >> sh) & 3u;
        const double2 vv = *reinterpret_cast<const double2*>(a.lhs + lr * T + k);
        if (FORM == kVecVec) {
          x = vv;
          y = *reinterpret_cast<const double2*>(a.rhs + rr * T + k);
        } else if (FORM == kScalarLeft) {
          x = make_double2(a.scalar, a.scalar);
          y = vv;
        } else {
          x = vv;
          y = make_double2(a.scalar, a.scalar);
        }
      }
      double2 o;
      const bool v0 = bin_cell<OP, MODE, FORM>(x.x, y.x, bits & 1u, &o.x);
      const bool v1 = bin_cell<OP, MODE, FORM>(x.y, y.y, (bits >> 1) & 1u, &o.y);
      const uint32_t b0 = __ballot_sync(0xFFFFFFFFu, v0), b1 = __ballot_sync(0xFFFFFFFFu, v1);
      if (inside) *reinterpret_cast<double2*>(orow + k) = o;
      if (lane == 0) ovw[w0] = spread16(b0) | (spread16(b1) << 1);
      if (lane == 1 && w0 + 1 < a.Tw) ovw[w0 + 1] = spread16(b0 >> 16) | (spread16(b1 >> 16) << 1);
    }
  }
}

// cnt [n_rows x T] (a by-label aggregate's counts) -> valid_words [n_rows x Tw]: bit k set iff cnt != 0.  One warp per
// (row, 32-step word).
__global__ void __launch_bounds__(256) count_valid_kernel(const uint32_t* cnt, uint64_t n_rows, uint64_t T, uint32_t Tw,
                                                          uint32_t* valid_words) {
  const int lane = threadIdx.x & 31;
  const uint64_t units = n_rows * Tw;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t u = warp0; u < units; u += n_warps) {
    const uint64_t r = u / Tw;
    const uint64_t w = u - r * Tw;
    const uint64_t k = w * 32 + lane;
    const bool v = k < T && cnt[r * T + k] != 0;
    const uint32_t word = __ballot_sync(0xFFFFFFFFu, v);
    if (lane == 0) valid_words[u] = word;
  }
}

}  // namespace b2p
