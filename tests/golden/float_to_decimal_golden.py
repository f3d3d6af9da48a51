"""floatingPointToDecimal goldens: (name, values, output type id, precision, cudf scale, expected values with None for
a null row, whether some row fails).  Names starting with f32 are FLOAT32 inputs, the rest FLOAT64.

The first five are DecimalUtilsTest.floatingPointToDecimalTest of the reference (src/test/java/com/nvidia/spark/rapids/
jni/DecimalUtilsTest.java:668-708).  The rest were derived by hand from decimal_utils.cu:1193-1309 and cudf's
floating_conversion.hpp; the comment on each says which step decides it."""
DECIMAL32, DECIMAL64, DECIMAL128 = 25, 26, 27

CASES = [
    ("java_1", [3527.61953125], DECIMAL64, 12, -7, [35276195313], False),
    ("java_2", [9.95], DECIMAL32, 3, -1, [100], False),
    ("java_3", [10.3], DECIMAL128, 18, -1, [103], False),
    ("java_4", [-10000000.0, -100000.0, 1.0, 100.0, 1000.0], DECIMAL32, 4, -1, [None, None, 10, 1000, None], True),
    ("java_5", [-10000000.0, 1.0, float("nan"), -2.0, float("-inf")], DECIMAL64, 4, -1, [None, 10, None, -20, None], True),
    # 1.005 is 1.00499999999999989...; the half-bit added to a double that is not whole carries it to 1.01
    ("half_bit_1_005", [1.005, -1.005], DECIMAL64, 18, -2, [101, -101], False),
    # 0.125 is exact: the last digit rounds half up, away from zero
    ("tie_0_125", [0.125, -0.125], DECIMAL32, 9, -2, [13, -13], False),
    # a float gets no half-bit: 1.005f is 1.00499999523..., which rounds to 1.00
    ("f32_no_half_bit", [1.005], DECIMAL32, 9, -2, [100], False),
    # the bound is exclusive: 99.995 rounds to 10000 = 10^4 and fails at precision 4, scale 2; 99.99 fits
    ("bound_exclusive", [99.99, 99.995, -99.995], DECIMAL64, 4, -2, [9999, None, None], True),
    # zeros of either sign are 0; NaN and infinities are null without failing
    ("zeros_and_specials", [0.0, -0.0, float("nan"), float("inf")], DECIMAL128, 38, -10, [0, 0, None, None], False),
    # a legacy negative Spark scale (cudf scale 2): 12345.0 is 123 hundreds, 12355.0 rounds to 124
    ("legacy_scale", [12345.0, 12355.0], DECIMAL64, 10, 2, [123, 124], False),
    # 10^300 at DECIMAL64 scale 2: floor_pow10 is 285 and 10^285 mod 2^64 is 0, so the floored magnitude is a valid 0
    ("dec64_power_wraps_to_zero", [1e300], DECIMAL64, 18, -2, [0], False),
    # 2^63 at DECIMAL64 scale 2: the floored magnitude 922337203685477600000 wraps to 19200 in the cast to int64
    ("dec64_wrap_inside_bound", [2.0 ** 63], DECIMAL64, 18, -2, [19200], False),
]
