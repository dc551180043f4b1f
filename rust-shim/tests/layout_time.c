/* Compile-time check of the enums of the time functions as rust-shim/src/ffi.rs mirrors them (B2pIfn::Neg,
 * B2pStepPart, B2pEmptyMetricKind):  gcc -std=c11 -fsyntax-only -I../../include layout_time.c */
#include "b200promql.h"

#define SA(cond, name) _Static_assert(cond, name)

/* B2pIfn::Neg = 28; 27 stays B2P_IFN__COUNT, no function */
SA(B2P_IFN_NEG == 28 && B2P_IFN__COUNT == 27, "B2pIfn::Neg");
SA(sizeof(enum b2p_ifn) == 4, "b2p_ifn is passed as i32");
/* #[repr(i32)] enum B2pStepPart */
SA(B2P_STEP_TIME == 0 && B2P_STEP_MINUTE == 1 && B2P_STEP_HOUR == 2 && B2P_STEP_DAY_OF_MONTH == 3, "B2pStepPart 0-3");
SA(B2P_STEP_DAY_OF_WEEK == 4 && B2P_STEP_DAY_OF_YEAR == 5 && B2P_STEP_MONTH == 6 && B2P_STEP_YEAR == 7, "B2pStepPart 4-7");
SA(B2P_STEP_DAYS_IN_MONTH == 8 && B2P_STEP__COUNT == 9, "B2pStepPart 8");
SA(sizeof(enum b2p_step_part) == 4, "b2p_step_part is passed as i32");
/* #[repr(i32)] enum B2pEmptyMetricKind */
SA(B2P_EMPTY_NONE == 0 && B2P_EMPTY_TIME == 1 && B2P_EMPTY_LITERAL == 2, "B2pEmptyMetricKind");
SA(sizeof(enum b2p_empty_metric_kind) == 4, "b2p_empty_metric_kind is passed as i32");
