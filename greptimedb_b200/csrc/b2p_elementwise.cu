// b2p_elementwise.cu — per-cell entry points of the C ABI: binary operators, instant-vector functions, scalar(),
// absent() and the set operators `and` / `or` / `unless`.
#include <algorithm>
#include <cfloat>

#include "b2p_runtime.cuh"
#include "b2p_absent.cuh"
#include "b2p_binary.cuh"
#include "b2p_instant.cuh"
#include "b2p_setop.cuh"
#include "b2p_time.cuh"

using namespace b2p;

namespace {

// ---- binary operators: OP / MODE / FORM are template arguments, chosen here once per call ----------------------------
template <int OP, int MODE, int FORM>
int launch_binary(b2p_ctx* c, const BinaryArgs& a, bool vec) {
  const uint64_t steps = vec ? 64 : 32;
  // 8 warps per CTA, one unit each, grid-stride beyond the cap
  const unsigned blocks = capped_grid(c, a.n_pairs * ((a.T + steps - 1) / steps), 8, 16);
  if (blocks == 0) return B2P_OK;
  if (vec) binary_op_kernel<OP, MODE, FORM, true><<<blocks, 256, 0, c->stream>>>(a);
  else binary_op_kernel<OP, MODE, FORM, false><<<blocks, 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

template <int FORM>
int dispatch_binary(b2p_ctx* c, int op, bool return_bool, const BinaryArgs& a, bool vec) {
#define B2P_CMP_CASE(OPV)                                                                                \
  case OPV:                                                                                              \
    return return_bool ? launch_binary<OPV, kBool, FORM>(c, a, vec) : launch_binary<OPV, kFilter, FORM>(c, a, vec);
  switch (op) {
    case kOpAdd: return launch_binary<kOpAdd, kArith, FORM>(c, a, vec);
    case kOpSub: return launch_binary<kOpSub, kArith, FORM>(c, a, vec);
    case kOpMul: return launch_binary<kOpMul, kArith, FORM>(c, a, vec);
    case kOpDiv: return launch_binary<kOpDiv, kArith, FORM>(c, a, vec);
    case kOpMod: return launch_binary<kOpMod, kArith, FORM>(c, a, vec);
    case kOpPow: return launch_binary<kOpPow, kArith, FORM>(c, a, vec);
    case kOpAtan2: return launch_binary<kOpAtan2, kArith, FORM>(c, a, vec);
    B2P_CMP_CASE(kOpEq)
    B2P_CMP_CASE(kOpNe)
    B2P_CMP_CASE(kOpGt)
    B2P_CMP_CASE(kOpLt)
    B2P_CMP_CASE(kOpGe)
    B2P_CMP_CASE(kOpLe)
    default: return fail(B2P_E_INVALID, "unknown binary operator %d", op);
  }
#undef B2P_CMP_CASE
}

int check_binop(int32_t op, int32_t return_bool) {
  if (op < 0 || op >= kOpCount) return fail(B2P_E_INVALID, "unknown binary operator %d", op);
  if (return_bool && op < kOpEq) return fail(B2P_E_INVALID, "the bool modifier needs a comparison operator, got %d", op);
  return B2P_OK;
}

// clears `bit` (kBinRowError / kSetKeyError / the scalar() bits) of the status word after a synchronous call has read it; B2P_E_INVALID
// when it was set
int take_row_error(b2p_ctx* c, uint32_t bit) {
  CU(cudaMemcpyAsync(c->h_k0, c->d_k0, sizeof(Status), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  const uint32_t k0 = c->h_k0->k0_errors;
  if (!(k0 & bit)) return B2P_OK;
  const uint32_t rest = k0 & ~bit;
  CU(cudaMemcpy(&c->d_k0->k0_errors, &rest, sizeof rest, cudaMemcpyHostToDevice));
  return k0_fail(k0 & bit);
}

// clamp_min / clamp_max -> clamp with the other bound at ∓f64::MAX (ScalarValue::max / min of Float64, clamp.rs:258-271,
// 312-325); every bound check (`lo > hi`, IEEE: a NaN bound passes) happens here, once per call
int instant_fn_bounds(int32_t fn, double arg0, double arg1, int* kfn, double* lo, double* hi) {
  *kfn = fn;
  *lo = arg0;
  *hi = arg1;
  if (fn == B2P_IFN_CLAMP_MIN) *hi = DBL_MAX;
  if (fn == B2P_IFN_CLAMP_MAX) *lo = -DBL_MAX, *hi = arg0;
  if (fn == B2P_IFN_CLAMP_MIN || fn == B2P_IFN_CLAMP_MAX) *kfn = B2P_IFN_CLAMP;
  if (fn == B2P_IFN_NEG) *kfn = kFnNeg;
  if (fn < 0 || (fn >= B2P_IFN__COUNT && fn != B2P_IFN_NEG)) return fail(B2P_E_INVALID, "unknown instant function %d", fn);
  if (*kfn == B2P_IFN_CLAMP && *lo > *hi) return fail(B2P_E_INVALID, "clamp: min %.17g > max %.17g", *lo, *hi);
  return B2P_OK;
}
static_assert((int)B2P_IFN_CLAMP == (int)kFnClamp && (int)kFnNeg + 1 == (int)kFnKernelCount,
              "enum b2p_ifn and InstantFn disagree");
static_assert((int)B2P_STEP_TIME == (int)kPartTime && (int)B2P_STEP_DAYS_IN_MONTH == (int)kPartDaysInMonth &&
                  (int)B2P_STEP__COUNT == (int)kPartCount, "enum b2p_step_part and StepPart disagree");

// K19: one CTA per (W steps, slab of rows); at most 16 CTAs per SM, the rows grid-strided beyond that
int step_fn_run(b2p_ctx* c, int32_t part, const int64_t* eval_ts, const uint32_t* valid, uint64_t n_rows, uint64_t T,
                double* out) {
  StepFnArgs a{};
  a.eval_ts = eval_ts; a.valid = valid; a.n_rows = n_rows; a.T = T; a.Tw = (uint32_t)((T + 31) / 32); a.out = out;
  a.status = c->d_k0;
  a.W = step_fn_width(T);
  const uint64_t gx = (T + a.W - 1) / a.W, rows_per_pass = kStepThreads / a.W;
  const uint64_t cap = std::max<uint64_t>(1, (uint64_t)c->num_sms * 16 / gx);
  const uint64_t gy = std::min<uint64_t>(std::min<uint64_t>((n_rows + rows_per_pass - 1) / rows_per_pass, cap), 65535);
  if (gx > INT32_MAX) return fail(B2P_E_TOO_LARGE, "step function: %llu steps", (unsigned long long)T);
  const dim3 grid((unsigned)gx, (unsigned)gy);
  return with_id<kPartCount>(part, "step part", [&](auto k) {
    step_fn_kernel<decltype(k)::value><<<grid, kStepThreads, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
    return B2P_OK;
  });
}

// the scalar() reduction and write pass; the verdict stays on the device
int scalar_calculate_run(b2p_ctx* c, const ScalarArgs& a0) {
  int rc;
  if ((rc = c->sc_state.ensure(sizeof(ScalarState)))) return rc;
  ScalarArgs a = a0;
  a.state = c->sc_state.as<ScalarState>();
  a.status = c->d_k0;
  // min_key, first_live = 0xFFFFFFFF; the rest 0
  CU(cudaMemsetAsync(a.state, 0xFF, 2 * sizeof(uint32_t), c->stream));
  CU(cudaMemsetAsync(&a.state->max_key, 0, sizeof(ScalarState) - 2 * sizeof(uint32_t), c->stream));
  if (a.n_rows > 0) {
    scalar_reduce_kernel<<<capped_grid(c, a.n_rows, 8, 16), 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
  }
  scalar_write_kernel<<<capped_grid(c, a.Tw, 8, 16), 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// absent(): steps up to 32 * (2^32 - 1), so that a row's validity words are counted in 32 bits
int check_absent_shape(uint64_t T) {
  if (T > 32ull * UINT32_MAX) return fail(B2P_E_TOO_LARGE, "absent: %llu steps, at most 32 x (2^32 - 1)", (unsigned long long)T);
  return B2P_OK;
}

// K15: acc = 0, the OR pass over the rows' validity words (none without rows: every step is absent), the write pass.
// Scratch: 4 B per output word (ab_acc).
int absent_run(b2p_ctx* c, const uint32_t* valid, uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  AbsentArgs a{};
  a.valid = valid; a.rows = n_rows; a.T = T; a.Tw = (uint32_t)((T + 31) / 32); a.out = out; a.out_valid = out_valid;
  if (int rc = c->ab_acc.ensure((size_t)a.Tw * 4)) return rc;
  a.acc = c->ab_acc.as<uint32_t>();
  CU(cudaMemsetAsync(a.acc, 0, (size_t)a.Tw * 4, c->stream));
  if (n_rows > 0) {
    // at least 4 words per thread, at most 8 CTAs per SM; the kernel sweeps whole rows beyond that
    const unsigned grid = std::max(1u, capped_grid(c, (uint64_t)n_rows * a.Tw, kAbsentThreads * 4, 8));
    absent_or_kernel<<<grid, kAbsentThreads, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
  }
  absent_write_kernel<<<capped_grid(c, a.Tw, 8, 16), 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

int setop_key_check(b2p_ctx* c, const uint32_t* key, uint32_t n, uint32_t n_keys) {
  if (n == 0) return B2P_OK;
  setop_key_check_kernel<<<capped_grid(c, n, 256, 8), 256, 0, c->stream>>>(key, n, n_keys, c->d_k0);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// the rows of one side grouped by key (CSR s_goff[side] / s_members[side], members in row order: the sort is stable)
int setop_group(b2p_ctx* c, int side, const uint32_t* key, uint32_t n_rows, uint32_t n_keys) {
  int rc;
  if ((rc = c->s_goff[side].ensure(((size_t)n_keys + 1) * 4))) return rc;
  if ((rc = c->s_members[side].ensure((size_t)(n_rows ? n_rows : 1) * 4))) return rc;
  return build_group_csr(c, key, n_rows, n_keys, c->s_goff[side].as<uint32_t>(), c->s_members[side].as<uint32_t>());
}

// s_mask[g] = OR of the validity words of side `side`'s rows with key g
int setop_mask(b2p_ctx* c, int side, const uint32_t* valid, uint32_t n_keys, uint32_t Tw) {
  const unsigned grid = capped_grid(c, (uint64_t)n_keys * ((Tw + 31) / 32), 8, 16);
  if (grid == 0) return B2P_OK;
  setop_mask_kernel<<<grid, 256, 0, c->stream>>>(valid, c->s_goff[side].as<uint32_t>(), c->s_members[side].as<uint32_t>(),
                                                 n_keys, Tw, c->s_mask.as<uint32_t>());
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

template <int MODE>
int setop_copy(b2p_ctx* c, const SetCopyArgs& a, bool vec) {
  const uint64_t steps = vec ? 64 : 32;
  const unsigned grid = capped_grid(c, a.n_rows * ((a.T + steps - 1) / steps), 8, 16);
  if (grid == 0) return B2P_OK;
  if (vec) setop_copy_kernel<MODE, true><<<grid, 256, 0, c->stream>>>(a);
  else setop_copy_kernel<MODE, false><<<grid, 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

int setop_run(b2p_ctx* c, int32_t op, const double* lhs, const uint32_t* lhs_valid, const uint32_t* lhs_key,
              uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid, const uint32_t* rhs_key,
              uint32_t n_rhs_rows, uint32_t n_keys, uint64_t T, double* out, uint32_t* out_valid) {
  int rc;
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  if ((rc = setop_key_check(c, lhs_key, n_lhs_rows, n_keys)) || (rc = setop_key_check(c, rhs_key, n_rhs_rows, n_keys)))
    return rc;
  if (n_keys > 0 && (rc = c->s_mask.ensure((size_t)n_keys * Tw * 4))) return rc;
  const bool vec = (T % 2) == 0 && aligned16(lhs) && aligned16(out) && (op != kSetOr || aligned16(rhs));
  SetCopyArgs a{};
  a.src = lhs; a.svalid = lhs_valid; a.key = lhs_key; a.n_rows = n_lhs_rows; a.n_keys = n_keys;
  a.mask = c->s_mask.as<uint32_t>(); a.T = T; a.Tw = Tw; a.out = out; a.out_valid = out_valid;
  if (op != kSetOr) {
    if (n_keys > 0) {
      if ((rc = setop_group(c, 1, rhs_key, n_rhs_rows, n_keys)) || (rc = setop_mask(c, 1, rhs_valid, n_keys, Tw))) return rc;
    }
    return op == kSetAnd ? setop_copy<kCopyAnd>(c, a, vec) : setop_copy<kCopyUnless>(c, a, vec);
  }
  // or: the steps each key's lhs rows claim, then the rhs words deduplicated into the rhs part of out_valid
  uint32_t* rwords = out_valid + (size_t)n_lhs_rows * Tw;
  if (n_keys > 0) {
    if ((rc = setop_group(c, 0, lhs_key, n_lhs_rows, n_keys)) || (rc = setop_mask(c, 0, lhs_valid, n_keys, Tw)) ||
        (rc = setop_group(c, 1, rhs_key, n_rhs_rows, n_keys)))
      return rc;
    const unsigned grid = capped_grid(c, (uint64_t)n_keys * ((Tw + 31) / 32), 8, 16);
    setop_dedupe_kernel<<<grid, 256, 0, c->stream>>>(rhs_valid, c->s_goff[1].as<uint32_t>(), c->s_members[1].as<uint32_t>(),
                                                     c->s_mask.as<uint32_t>(), n_keys, Tw, rwords);
    c->launches++;
    CU(cudaGetLastError());
  }
  if ((rc = setop_copy<kCopyKeep>(c, a, vec))) return rc;
  SetCopyArgs b = a;
  b.src = rhs; b.svalid = rhs_valid; b.key = rhs_key; b.n_rows = n_rhs_rows; b.mask = nullptr; b.words = rwords;
  b.out = out + (size_t)n_lhs_rows * T; b.out_valid = rwords;
  return setop_copy<kCopyWords>(c, b, vec);
}

int check_setop_args(int32_t op, const double* lhs, const uint32_t* lhs_valid, const uint32_t* lhs_key, uint32_t n_lhs_rows,
                     const double* rhs, const uint32_t* rhs_valid, const uint32_t* rhs_key, uint32_t n_rhs_rows,
                     double* out, uint32_t* out_valid) {
  if (op < kSetAnd || op > kSetUnless) return fail(B2P_E_INVALID, "unknown set operator %d", op);
  const uint64_t n_out = op == kSetOr ? (uint64_t)n_lhs_rows + n_rhs_rows : n_lhs_rows;
  if (n_out > UINT32_MAX) return fail(B2P_E_INVALID, "set operator: more than 2^32 - 1 output rows");
  if ((n_lhs_rows && (!lhs || !lhs_valid || !lhs_key)) || (n_rhs_rows && (!rhs_valid || !rhs_key)) ||
      (n_rhs_rows && op == kSetOr && !rhs) || (n_out && (!out || !out_valid)))
    return fail(B2P_E_INVALID, "NULL argument");
  return B2P_OK;
}
}  // namespace

extern "C" {

/* ---- binary operators ---------------------------------------------------------------------------------------- */
int b2p_binary_op_dev(b2p_ctx* c, int32_t op, int32_t return_bool, const double* lhs, const uint32_t* lhs_valid,
                      const uint32_t* lhs_row, uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid,
                      const uint32_t* rhs_row, uint32_t n_rhs_rows, uint64_t n_pairs, uint64_t T, double* out,
                      uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int rc;
  if ((rc = check_binop(op, return_bool))) return rc;
  if (n_pairs == 0 || T == 0) return B2P_OK;
  if (!lhs_row || !rhs_row || !out || !out_valid || (n_lhs_rows && (!lhs || !lhs_valid)) ||
      (n_rhs_rows && (!rhs || !rhs_valid)))
    return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  BinaryArgs a{};
  a.lhs = lhs; a.lvalid = lhs_valid; a.lrow = lhs_row; a.n_lhs = n_lhs_rows;
  a.rhs = rhs; a.rvalid = rhs_valid; a.rrow = rhs_row; a.n_rhs = n_rhs_rows;
  a.n_pairs = n_pairs; a.T = T; a.Tw = (uint32_t)((T + 31) / 32); a.out = out; a.out_valid = out_valid; a.status = c->d_k0;
  const bool vec = (T % 2) == 0 && aligned16(lhs) && aligned16(rhs) && aligned16(out);
  stage_begin(c, 3);
  rc = dispatch_binary<kVecVec>(c, op, return_bool != 0, a, vec);
  stage_end(c, 3);
  return rc;
}

int b2p_scalar_op_dev(b2p_ctx* c, int32_t op, int32_t return_bool, int32_t scalar_on_left, double scalar,
                      const double* vals, const uint32_t* valid, uint64_t n_rows, uint64_t T, double* out,
                      uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int rc;
  if ((rc = check_binop(op, return_bool))) return rc;
  if (n_rows == 0 || T == 0) return B2P_OK;
  if (!vals || !valid || !out || !out_valid) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  BinaryArgs a{};
  a.lhs = vals; a.lvalid = valid; a.scalar = scalar;
  a.n_pairs = n_rows; a.T = T; a.Tw = (uint32_t)((T + 31) / 32); a.out = out; a.out_valid = out_valid; a.status = c->d_k0;
  const bool vec = (T % 2) == 0 && aligned16(vals) && aligned16(out);
  stage_begin(c, 3);
  rc = scalar_on_left ? dispatch_binary<kScalarLeft>(c, op, return_bool != 0, a, vec)
                      : dispatch_binary<kScalarRight>(c, op, return_bool != 0, a, vec);
  stage_end(c, 3);
  return rc;
}

int b2p_count_valid_words_dev(b2p_ctx* c, const uint32_t* cnt, uint64_t n_rows, uint64_t T, uint32_t* valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_rows == 0 || T == 0) return B2P_OK;
  if (!cnt || !valid_words) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  count_valid_kernel<<<capped_grid(c, n_rows * Tw, 8, 16), 256, 0, c->stream>>>(cnt, n_rows, T, Tw, valid_words);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

/* ---- Int64 -> Float64 ------------------------------------------------------------------------------------------ */

int b2p_i64_to_f64_dev(b2p_ctx* c, const int64_t* vals, uint64_t n, double* out) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n == 0) return B2P_OK;
  if (!vals || !out) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  i64_to_f64_kernel<<<capped_grid(c, n, 256, 16), 256, 0, c->stream>>>(reinterpret_cast<const long long*>(vals), n, out);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

/* ---- instant-vector functions and scalar() --------------------------------------------------------------------- */

int b2p_instant_fn_dev(b2p_ctx* c, int32_t fn, double arg0, double arg1, const double* vals, const uint32_t* valid,
                       uint64_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int rc, kfn;
  InstantFnArgs a{};
  if ((rc = instant_fn_bounds(fn, arg0, arg1, &kfn, &a.arg0, &a.arg1))) return rc;
  if (n_rows == 0 || T == 0) return B2P_OK;
  if (!vals || !valid || !out || !out_valid) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  a.vals = vals; a.valid = valid; a.n_rows = n_rows; a.T = T; a.Tw = (uint32_t)((T + 31) / 32);
  a.out = out; a.out_valid = out_valid;
  const bool vec = (T % 2) == 0 && aligned16(vals) && aligned16(out);
  const uint64_t steps = vec ? 64 : 32;
  // 8 warps per CTA, one unit each, grid-stride beyond the cap
  const unsigned blocks = capped_grid(c, n_rows * ((T + steps - 1) / steps), 8, 16);
  stage_begin(c, 3);
  rc = with_id<kFnKernelCount>(kfn, "instant function", [&](auto k) {
    constexpr int FN = decltype(k)::value;
    if (vec) instant_fn_kernel<FN, true><<<blocks, 256, 0, c->stream>>>(a);
    else instant_fn_kernel<FN, false><<<blocks, 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
    return B2P_OK;
  });
  stage_end(c, 3);
  return rc;
}

int b2p_scalar_calculate_dev(b2p_ctx* c, const double* vals, const uint32_t* valid, const uint32_t* row_key,
                             uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (T == 0) return B2P_OK;
  if ((n_rows && (!vals || !valid || !row_key)) || !out || !out_valid) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  ScalarArgs a{};
  a.vals = vals; a.valid = valid; a.key = row_key; a.n_rows = n_rows; a.T = T; a.Tw = (uint32_t)((T + 31) / 32);
  a.out = out; a.out_valid = out_valid;
  stage_begin(c, 3);
  const int rc = scalar_calculate_run(c, a);
  stage_end(c, 3);
  return rc;
}

int b2p_absent_dev(b2p_ctx* c, const uint32_t* valid, uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (int rc = check_absent_shape(T)) return rc;
  if ((n_rows && !valid) || (T && (!out || !out_valid))) return fail(B2P_E_INVALID, "NULL argument");
  if (T == 0) return B2P_OK;
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = absent_run(c, valid, n_rows, T, out, out_valid);
  stage_end(c, 3);
  return rc;
}

/* ---- functions of the eval step ------------------------------------------------------------------------------ */

int b2p_step_fn_dev(b2p_ctx* c, int32_t part, const int64_t* eval_ts, const uint32_t* valid, uint64_t n_rows,
                    uint64_t T, double* out) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (part < 0 || part >= kPartCount) return fail(B2P_E_INVALID, "unknown step part %d", part);
  if (n_rows == 0 || T == 0) return B2P_OK;
  if (!eval_ts || !valid || !out) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = step_fn_run(c, part, eval_ts, valid, n_rows, T, out);
  stage_end(c, 3);
  return rc;
}

/* ---- set operators ------------------------------------------------------------------------------------------- */

int b2p_setop_dev(b2p_ctx* c, int32_t op, const double* lhs, const uint32_t* lhs_valid, const uint32_t* lhs_key,
                  uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid, const uint32_t* rhs_key,
                  uint32_t n_rhs_rows, uint32_t n_keys, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int rc;
  if ((rc = check_setop_args(op, lhs, lhs_valid, lhs_key, n_lhs_rows, rhs, rhs_valid, rhs_key, n_rhs_rows, out,
                             out_valid)))
    return rc;
  if (T == 0) return B2P_OK;
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  rc = setop_run(c, op, lhs, lhs_valid, lhs_key, n_lhs_rows, rhs, rhs_valid, rhs_key, n_rhs_rows, n_keys, T, out,
                 out_valid);
  stage_end(c, 3);
  return rc;
}

/* ---- host-pointer API ------------------------------------------------------------------------ */

int b2p_binary_op(b2p_ctx* c, int32_t op, int32_t return_bool, const double* lhs, const uint32_t* lhs_valid,
                  const uint32_t* lhs_row, uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid,
                  const uint32_t* rhs_row, uint32_t n_rhs_rows, uint64_t n_pairs, uint64_t T, double* out,
                  uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (int rc = check_binop(op, return_bool)) return rc;
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  const size_t nl = n_lhs_rows, nr = n_rhs_rows, np = (size_t)n_pairs;
  Staging s{c};
  const double* d_lhs = s.in(lhs, nl * T * 8);
  const uint32_t* d_lhs_valid = s.in(lhs_valid, nl * Tw * 4);
  const uint32_t* d_lhs_row = s.in(lhs_row, np * 4);
  const double* d_rhs = s.in(rhs, nr * T * 8);
  const uint32_t* d_rhs_valid = s.in(rhs_valid, nr * Tw * 4);
  const uint32_t* d_rhs_row = s.in(rhs_row, np * 4);
  double* d_out = s.out(out, np * T * 8);
  uint32_t* d_out_valid = s.out(out_valid, np * Tw * 4);
  const int rc = s.end([&] {
    return b2p_binary_op_dev(c, op, return_bool, d_lhs, d_lhs_valid, d_lhs_row, n_lhs_rows, d_rhs, d_rhs_valid,
                             d_rhs_row, n_rhs_rows, n_pairs, T, d_out, d_out_valid);
  }, false);
  return rc ? rc : take_row_error(c, kBinRowError);  // (synchronises)
}

int b2p_scalar_op(b2p_ctx* c, int32_t op, int32_t return_bool, int32_t scalar_on_left, double scalar, const double* vals,
                  const uint32_t* valid, uint64_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (int rc = check_binop(op, return_bool)) return rc;
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  const size_t vb = (size_t)n_rows * T * 8, wb = (size_t)n_rows * Tw * 4;
  Staging s{c};
  double* d_vals = s.in(vals, vb);  // the operator runs in place
  uint32_t* d_valid = s.in(valid, wb);
  double* d_out = s.copy_back(out, d_vals, vb);
  uint32_t* d_out_valid = s.copy_back(out_valid, d_valid, wb);
  return s.end([&] {
    return b2p_scalar_op_dev(c, op, return_bool, scalar_on_left, scalar, d_vals, d_valid, n_rows, T, d_out, d_out_valid);
  });
}

int b2p_setop(b2p_ctx* c, int32_t op, const double* lhs, const uint32_t* lhs_valid, const uint32_t* lhs_key,
              uint32_t n_lhs_rows, const double* rhs, const uint32_t* rhs_valid, const uint32_t* rhs_key,
              uint32_t n_rhs_rows, uint32_t n_keys, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (int rc = check_setop_args(op, lhs, lhs_valid, lhs_key, n_lhs_rows, rhs, rhs_valid, rhs_key, n_rhs_rows, out,
                                out_valid))
    return rc;
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  const size_t nl = n_lhs_rows, nr = n_rhs_rows, no = op == kSetOr ? nl + nr : nl;
  Staging s{c};
  const double* d_lhs = s.in(lhs, nl * T * 8);
  const uint32_t* d_lhs_valid = s.in(lhs_valid, nl * Tw * 4);
  const uint32_t* d_lhs_key = s.in(lhs_key, nl * 4);
  const double* d_rhs = s.in(op == kSetOr ? rhs : nullptr, nr * T * 8);  // and / unless never read the rhs values
  const uint32_t* d_rhs_valid = s.in(rhs_valid, nr * Tw * 4);
  const uint32_t* d_rhs_key = s.in(rhs_key, nr * 4);
  double* d_out = s.out(out, no * T * 8);
  uint32_t* d_out_valid = s.out(out_valid, no * Tw * 4);
  const int rc = s.end([&] {
    return b2p_setop_dev(c, op, d_lhs, d_lhs_valid, d_lhs_key, n_lhs_rows, d_rhs, d_rhs_valid, d_rhs_key, n_rhs_rows,
                         n_keys, T, d_out, d_out_valid);
  }, false);
  return rc ? rc : take_row_error(c, kSetKeyError);  // (synchronises)
}

int b2p_instant_fn(b2p_ctx* c, int32_t fn, double arg0, double arg1, const double* vals, const uint32_t* valid,
                   uint64_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int kfn;
  double lo, hi;
  if (int rc = instant_fn_bounds(fn, arg0, arg1, &kfn, &lo, &hi)) return rc;
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  const size_t vb = (size_t)n_rows * T * 8, wb = (size_t)n_rows * Tw * 4;
  Staging s{c};
  double* d_vals = s.in(vals, vb);  // the function runs in place; validity is unchanged
  uint32_t* d_valid = s.in(valid, wb);
  double* d_out = s.copy_back(out, d_vals, vb);
  uint32_t* d_out_valid = out_valid == valid ? d_valid : s.copy_back(out_valid, d_valid, wb);
  return s.end([&] { return b2p_instant_fn_dev(c, fn, arg0, arg1, d_vals, d_valid, n_rows, T, d_out, d_out_valid); });
}

int b2p_step_fn(b2p_ctx* c, int32_t part, const int64_t* eval_ts, const uint32_t* valid, uint64_t n_rows, uint64_t T,
                double* out) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  Staging s{c};
  const int64_t* d_ts = s.in(eval_ts, (size_t)T * 8);
  const uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw * 4);
  double* d_out = s.out(out, (size_t)n_rows * T * 8);
  const int rc = s.end([&] { return b2p_step_fn_dev(c, part, d_ts, d_valid, n_rows, T, d_out); }, false);
  return rc ? rc : take_row_error(c, kStepRangeError);  // (synchronises)
}

int b2p_i64_to_f64(b2p_ctx* c, const int64_t* vals, uint64_t n, double* out) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  Staging s{c};
  int64_t* d = s.in(vals, (size_t)n * 8);
  double* d_out = s.copy_back(out, reinterpret_cast<double*>(d), (size_t)n * 8);  // in place
  return s.end([&] { return b2p_i64_to_f64_dev(c, d, n, d_out); });
}

int b2p_scalar_calculate(b2p_ctx* c, const double* vals, const uint32_t* valid, const uint32_t* row_key,
                         uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  Staging s{c};
  const double* d_vals = s.in(vals, (size_t)n_rows * T * 8);
  const uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw * 4);
  const uint32_t* d_key = s.in(row_key, (size_t)n_rows * 4);
  double* d_out = s.out(out, (size_t)T * 8);
  uint32_t* d_out_valid = s.out(out_valid, Tw * 4);
  const int rc =
      s.end([&] { return b2p_scalar_calculate_dev(c, d_vals, d_valid, d_key, n_rows, T, d_out, d_out_valid); }, false);
  return rc ? rc : take_row_error(c, kScalarKeyError | kScalarOverlapError);  // (synchronises)
}

int b2p_absent(b2p_ctx* c, const uint32_t* valid, uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (int rc = check_absent_shape(T)) return rc;
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  Staging s{c};
  const uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw * 4);
  double* d_out = s.out(out, (size_t)T * 8);
  uint32_t* d_out_valid = s.out(out_valid, Tw * 4);
  return s.end([&] { return b2p_absent_dev(c, d_valid, n_rows, T, d_out, d_out_valid); });
}

}  // extern "C"
