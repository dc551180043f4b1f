"""The ulp bounds the transcendental results are held to against glibc (DESIGN.md section 2), shared by every test of
them, and the distance they are measured in."""
import numpy as np

# max ulp distance from glibc per K9 function: the distance measured on an H100 over the 2^20 seeded operands of
# test_gpu_instant_fn.py::test_ulp_bound_over_a_million_operands and over the classes of tests/libm_cases.py
ULP_BOUND = {"exp": 1, "ln": 1, "log2": 1, "log10": 2, "sin": 1, "cos": 1, "tan": 2, "asin": 2, "acos": 1, "atan": 1,
             "sinh": 2, "cosh": 2, "tanh": 3, "asinh": 2, "acosh": 2, "atanh": 2}
# K7's `^` and `atan2`: the larger of the two distances measured the same way
POW_ATAN2_ULPS = 2
# classes of tests/libm_cases.py held to their own measured bound (DESIGN.md section 2): at 6381956970095103 * 2^797,
# the double nearest a multiple of π/2, the device's cos and tan are correctly rounded and glibc's are 8 and 14 ulps off
CLASS_ULPS = {("cos", "worst reduction"): 8, ("tan", "worst reduction"): 14}
# threshold classes where CUDA's exp / pow give +0 where glibc gives the smallest subnormal (1 ulp; DESIGN.md section 2)
UNDERFLOW_TO_ZERO = {("exp", "smallest subnormal"), ("pow", "subnormal by 2^y"), ("pow", "subnormal by 10^y"),
                     ("pow", "subnormal by 0.5^y"), ("pow", "subnormal by x^2")}


def ulp_distance(a, b):
    """|a - b| in units in the last place (0 when both are NaN or equal; inf when one is NaN)."""
    def ordered(x):   # the bit pattern as a monotone int64 (subtracted in integers: float64 cannot hold 2^63)
        i = np.ascontiguousarray(x, np.float64).view(np.int64)
        return np.where(i < 0, np.int64(-0x8000000000000000) - i, i)
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    with np.errstate(over="ignore"):
        d = np.abs(ordered(a) - ordered(b)).astype(np.float64)
    both_nan = np.isnan(a) & np.isnan(b)
    one_nan = np.isnan(a) ^ np.isnan(b)
    return np.where(both_nan, 0.0, np.where(one_nan, np.inf, d))
