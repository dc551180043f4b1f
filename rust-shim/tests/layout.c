/* Compile-time check of every layout assumption rust-shim/src/ffi.rs makes about include/b200promql.h.
 *   gcc -std=c11 -fsyntax-only -I../../include layout.c        (tests/test_abi.py runs exactly this)
 * If a field of struct b2p_range_params moves, or an enum value changes, this file stops compiling — and
 * B2pRangeParams / B2pFn / B2pAgg / B2pBinOp / B2pIfn in ffi.rs have to follow. */
#include <stddef.h>
#include <stdint.h>

#include "b200promql.h"

#define SA(cond, name) _Static_assert(cond, name)

/* #[repr(C)] pub struct B2pRangeParams { fn_id: i32, filter_nan: i32, start, end, interval, range, offset: i64, param0, param1: f64 } */
SA(sizeof(b2p_range_params) == 64, "b2p_range_params is 64 bytes");
SA(_Alignof(b2p_range_params) == 8, "b2p_range_params is 8-aligned");
SA(offsetof(b2p_range_params, fn_id) == 0, "fn_id");
SA(offsetof(b2p_range_params, filter_nan) == 4, "filter_nan");
SA(offsetof(b2p_range_params, start) == 8, "start");
SA(offsetof(b2p_range_params, end) == 16, "end");
SA(offsetof(b2p_range_params, interval) == 24, "interval");
SA(offsetof(b2p_range_params, range) == 32, "range");
SA(offsetof(b2p_range_params, offset) == 40, "offset");
SA(offsetof(b2p_range_params, param0) == 48, "param0");
SA(offsetof(b2p_range_params, param1) == 56, "param1");

/* #[repr(i32)] enum B2pFn */
SA(B2P_FN_RATE == 0 && B2P_FN_INCREASE == 1 && B2P_FN_DELTA == 2 && B2P_FN_IRATE == 3 && B2P_FN_IDELTA == 4, "B2pFn 0-4");
SA(B2P_FN_RESETS == 5 && B2P_FN_CHANGES == 6 && B2P_FN_COUNT_OVER_TIME == 7 && B2P_FN_SUM_OVER_TIME == 8, "B2pFn 5-8");
SA(B2P_FN_AVG_OVER_TIME == 9 && B2P_FN_MIN_OVER_TIME == 10 && B2P_FN_MAX_OVER_TIME == 11 && B2P_FN_LAST_OVER_TIME == 12, "B2pFn 9-12");
SA(B2P_FN_PRESENT_OVER_TIME == 13 && B2P_FN_ABSENT_OVER_TIME == 14 && B2P_FN_STDVAR_OVER_TIME == 15, "B2pFn 13-15");
SA(B2P_FN_STDDEV_OVER_TIME == 16 && B2P_FN_DERIV == 17 && B2P_FN_PREDICT_LINEAR == 18, "B2pFn 16-18");
SA(B2P_FN_QUANTILE_OVER_TIME == 19 && B2P_FN_HOLT_WINTERS == 20 && B2P_FN__COUNT == 21, "B2pFn 19-21");
/* #[repr(i32)] enum B2pAgg */
SA(B2P_AGG_SUM == 0 && B2P_AGG_AVG == 1 && B2P_AGG_COUNT == 2 && B2P_AGG_MIN == 3 && B2P_AGG_MAX == 4, "B2pAgg 0-4");
SA(B2P_AGG_STDDEV == 5 && B2P_AGG_STDVAR == 6, "B2pAgg 5-6");
/* #[repr(i32)] enum B2pBinOp: arithmetic 0-6, comparisons 7-12 (B2pBinOp::is_comparison tests >= Eq) */
SA(B2P_OP_ADD == 0 && B2P_OP_SUB == 1 && B2P_OP_MUL == 2 && B2P_OP_DIV == 3 && B2P_OP_MOD == 4, "B2pBinOp 0-4");
SA(B2P_OP_POW == 5 && B2P_OP_ATAN2 == 6 && B2P_OP_EQ == 7 && B2P_OP_NE == 8 && B2P_OP_GT == 9, "B2pBinOp 5-9");
SA(B2P_OP_LT == 10 && B2P_OP_GE == 11 && B2P_OP_LE == 12, "B2pBinOp 10-12");
SA(sizeof(enum b2p_binop) == 4, "b2p_binop is passed as i32");
SA(B2P_SET_AND == 0 && B2P_SET_OR == 1 && B2P_SET_UNLESS == 2, "B2pSetOp");
SA(sizeof(enum b2p_setop) == 4, "b2p_setop is passed as i32");
SA(B2P_NO_KEY == 0xFFFFFFFFu, "B2P_NO_KEY");
/* #[repr(i32)] enum B2pIfn */
SA(B2P_IFN_ABS == 0 && B2P_IFN_CEIL == 1 && B2P_IFN_FLOOR == 2 && B2P_IFN_SQRT == 3 && B2P_IFN_EXP == 4, "B2pIfn 0-4");
SA(B2P_IFN_LN == 5 && B2P_IFN_LOG2 == 6 && B2P_IFN_LOG10 == 7 && B2P_IFN_SIN == 8 && B2P_IFN_COS == 9, "B2pIfn 5-9");
SA(B2P_IFN_TAN == 10 && B2P_IFN_ASIN == 11 && B2P_IFN_ACOS == 12 && B2P_IFN_ATAN == 13 && B2P_IFN_SINH == 14, "B2pIfn 10-14");
SA(B2P_IFN_COSH == 15 && B2P_IFN_TANH == 16 && B2P_IFN_ASINH == 17 && B2P_IFN_ACOSH == 18 && B2P_IFN_ATANH == 19, "B2pIfn 15-19");
SA(B2P_IFN_ROUND == 20 && B2P_IFN_DEG == 21 && B2P_IFN_RAD == 22 && B2P_IFN_SGN == 23 && B2P_IFN_CLAMP == 24, "B2pIfn 20-24");
SA(B2P_IFN_CLAMP_MIN == 25 && B2P_IFN_CLAMP_MAX == 26 && B2P_IFN__COUNT == 27, "B2pIfn 25-27");
SA(sizeof(enum b2p_ifn) == 4, "b2p_ifn is passed as i32");
/* status codes and sizes the shim hard-codes */
SA(B2P_OK == 0 && B2P_E_INVALID == -1 && B2P_E_CUDA == -2 && B2P_E_UNSORTED == -3 && B2P_E_NOMEM == -4 && B2P_E_TOO_LARGE == -5, "codes");
SA(B2P_COMM_ID_BYTES == 128, "communicator id");
/* arrow::ffi::FFI_ArrowArray / FFI_ArrowSchema are #[repr(C)] copies of these (LP64) */
SA(sizeof(struct ArrowArray) == 80 && sizeof(struct ArrowSchema) == 72, "Arrow C Data Interface structs");
SA(offsetof(struct ArrowArray, buffers) == 40 && offsetof(struct ArrowArray, release) == 64, "ArrowArray fields");
SA(offsetof(struct ArrowSchema, n_children) == 32 && offsetof(struct ArrowSchema, release) == 56, "ArrowSchema fields");
/* integer widths the signatures assume */
SA(sizeof(int) == 4 && sizeof(size_t) == 8 && sizeof(void*) == 8, "LP64");

int b2p_layout_check_translation_unit_is_not_empty;
