"""Arithmetic test data (data only): the cases of the reference's ArithmeticTest.java and src/main/cpp/tests/multiply.cpp.

MULTIPLY: (name, type, left, right, ansi, try, expected).  left / right are lists (None = null), or ("scalar", value) for a
scalar operand; expected is a list (None = null), or ("row", r) for an ExceptionWithRowIndex at row r, or "error" for an
argument error.
ROUND: (name, type, scale (cudf's: the value is unscaled * 10^scale), values, decimal_places, mode (0 HALF_UP,
1 HALF_EVEN), ansi, expected).  values and expected are lists (None = null; decimals as unscaled integers, the result at
scale -decimal_places), or ("row", r).
"""
INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, BOOL8, DECIMAL32 = "INT8", "INT16", "INT32", "INT64", "FLOAT32", "FLOAT64", "BOOL8", "DECIMAL32"
INT32_MAX, INT64_MAX, INT64_MIN = 2**31 - 1, 2**63 - 1, -2**63

MULTIPLY = [
    # ArithmeticTest.java
    ("multiplyAnsiOffWithOverflow", INT32, [0, 1, INT32_MAX], [0, 1, 2], False, False, [0, 1, -2]),
    ("multiplyAnsiOnWithOverflow", INT32, [0, 1, INT32_MAX], [0, 1, 2], True, False, ("row", 2)),
    ("multiplyTryOnWithOverflow", INT32, [0, 1, INT32_MAX], [0, 1, 2], False, True, [0, 1, None]),
    ("multiplyLongScalar", INT64, [0, 1, INT64_MAX], ("scalar", 2), False, True, [0, 2, None]),
    ("multiplyScalarInt", INT32, ("scalar", 2), [0, 1, INT32_MAX], False, False, [0, 2, -2]),
    ("multiplyScalarIntAnsi", INT32, ("scalar", 2), [0, 1, INT32_MAX], True, False, ("row", 2)),
    # multiply.cpp
    ("int8_try", INT8, [1, 127, 120], [1, 2, -2], False, True, [1, None, None]),
    ("int8_ansi", INT8, [1, 127, 120], [1, 2, -2], True, False, ("row", 1)),
    ("int16_try", INT16, [1, 2, 32767, -30000], [1, 2, 2, 2], False, True, [1, 4, None, None]),
    ("int16_ansi", INT16, [1, 2, 32767, -30000], [1, 2, 2, 2], True, False, ("row", 2)),
    ("int32_try", INT32, [None, 1, 2, 2147483647, None, 5, None, 2000000000], [5, 1, 2, 2, 4, None, None, -2], False, True,
     [None, 1, 4, None, None, None, None, None]),
    ("int32_ansi", INT32, [None, 1, 2, 2147483647, None, 5, None, 2000000000], [5, 1, 2, 2, 4, None, None, -2], True, False, ("row", 3)),
    ("int64_try", INT64, [1, 2, INT64_MIN, -1, INT64_MAX - 10, INT64_MAX - 10, INT64_MIN + 10, INT64_MIN + 10, -1, -1],
     [1, 2, -1, INT64_MIN, 2, -2, 2, -2, 2, 2], False, True, [1, 4, None, None, None, None, None, None, -2, -2]),
    ("int64_ansi", INT64, [1, 2, INT64_MIN, -1, INT64_MAX - 10, INT64_MAX - 10, INT64_MIN + 10, INT64_MIN + 10, -1, -1],
     [1, 2, -1, INT64_MIN, 2, -2, 2, -2, 2, 2], True, False, ("row", 2)),
    ("float_try", FLOAT32, [1.0, 2.0], [1.0, 2.0], False, True, [1.0, 4.0]),
    ("float_ansi", FLOAT32, [1.0, 2.0], [1.0, 2.0], True, False, [1.0, 4.0]),
    ("double_try", FLOAT64, [1.0, 2.0], [1.0, 2.0], False, True, [1.0, 4.0]),
    ("double_ansi", FLOAT64, [1.0, 2.0], [1.0, 2.0], True, False, [1.0, 4.0]),
    ("checkTypeEquals", (INT8, INT16), [1, 127], [1, 2], True, False, "error"),
    ("checkRows", INT8, [1, 2, 3], [1, 2], True, False, "error"),
    ("invalidType", (BOOL8, INT8), [1, 0], [1, 2], True, False, "error"),
    ("invalidMode", INT8, [1, 2], [1, 2], True, True, "error"),
]

ROUND = [
    ("roundFloatsHalfUp_0", FLOAT32, 0, [1.234, 25.66, None, 154.9, 2346.0], 0, 0, False, [1.0, 26.0, None, 155.0, 2346.0]),
    ("roundFloatsHalfUp_1", FLOAT32, 0, [1.234, 25.66, None, 154.9, 2346.0], 1, 0, False, [1.2, 25.7, None, 154.9, 2346.0]),
    ("roundFloatsHalfUp_m1", FLOAT32, 0, [1.234, 25.66, None, 154.9, 2346.0], -1, 0, False, [0.0, 30.0, None, 150.0, 2350.0]),
    ("roundFloatsHalfEven_0", FLOAT32, 0, [1.5, 2.5, 1.35, None, 1.25, 15.0, 25.0], 0, 1, False, [2.0, 2.0, 1.0, None, 1.0, 15.0, 25.0]),
    ("roundFloatsHalfEven_1", FLOAT32, 0, [1.5, 2.5, 1.35, None, 1.25, 15.0, 25.0], 1, 1, False, [1.5, 2.5, 1.4, None, 1.2, 15.0, 25.0]),
    ("roundFloatsHalfEven_m1", FLOAT32, 0, [1.5, 2.5, 1.35, None, 1.25, 15.0, 25.0], -1, 1, False, [0.0, 0.0, 0.0, None, 0.0, 20.0, 20.0]),
    ("roundIntsHalfUp_2", INT32, 0, [12, 135, 160, -1454, None, -1500, -140, -150], 2, 0, False, [12, 135, 160, -1454, None, -1500, -140, -150]),
    ("roundIntsHalfUp_m2", INT32, 0, [12, 135, 160, -1454, None, -1500, -140, -150], -2, 0, False, [0, 100, 200, -1500, None, -1500, -100, -200]),
    ("roundIntsHalfEven_2", INT32, 0, [12, 24, 135, 160, None, 1450, 1550, -1650], 2, 1, False, [12, 24, 135, 160, None, 1450, 1550, -1650]),
    ("roundIntsHalfEven_m2", INT32, 0, [12, 24, 135, 160, None, 1450, 1550, -1650], -2, 1, False, [0, 0, 100, 200, None, 1400, 1600, -1600]),
    ("roundDecimal_halfUp", DECIMAL32, 2, [14, 15, 16, 24, 25, 26], -3, 0, False, [1, 2, 2, 2, 3, 3]),
    ("roundDecimal_halfEven", DECIMAL32, 2, [14, 15, 16, 24, 25, 26], -3, 1, False, [1, 2, 2, 2, 2, 3]),
    ("roundDefault", FLOAT32, 0, [1.234, 25.66, None, 154.9, 2346.0], 0, 0, False, [1.0, 26.0, None, 155.0, 2346.0]),
    ("roundWithDecimalPlaces", FLOAT32, 0, [1.234, 25.66, None, 154.9, 2346.0], 2, 0, False, [1.23, 25.66, None, 154.9, 2346.0]),
    ("roundDoublesHalfUp_0", FLOAT64, 0, [1.234, 25.66, None, 154.9, 2346.0], 0, 0, False, [1.0, 26.0, None, 155.0, 2346.0]),
    ("roundDoublesHalfUp_1", FLOAT64, 0, [1.234, 25.66, None, 154.9, 2346.0], 1, 0, False, [1.2, 25.7, None, 154.9, 2346.0]),
    ("roundDoublesHalfUp_m1", FLOAT64, 0, [1.234, 25.66, None, 154.9, 2346.0], -1, 0, False, [0.0, 30.0, None, 150.0, 2350.0]),
    ("roundDoublesHalfEven_0", FLOAT64, 0, [1.5, 2.5, 1.35, None, 1.25, 15.0, 25.0], 0, 1, False, [2.0, 2.0, 1.0, None, 1.0, 15.0, 25.0]),
    ("roundDoublesHalfEven_1", FLOAT64, 0, [1.5, 2.5, 1.35, None, 1.25, 15.0, 25.0], 1, 1, False, [1.5, 2.5, 1.4, None, 1.2, 15.0, 25.0]),
    ("roundDoublesHalfEven_m1", FLOAT64, 0, [1.5, 2.5, 1.35, None, 1.25, 15.0, 25.0], -1, 1, False, [0.0, 0.0, 0.0, None, 0.0, 20.0, 20.0]),
    ("roundByteAnsiNoOverflow", INT8, 0, [10, 50, None, -50], -1, 0, True, [10, 50, None, -50]),
    ("roundByteAnsiWithOverflow", INT8, 0, [10, 50, 125], -1, 0, True, ("row", 2)),
    ("roundByteAnsiNegativeOverflow", INT8, 0, [10, -125], -1, 0, True, ("row", 1)),
    ("roundShortAnsiNoOverflow", INT16, 0, [10, 200, 32700], -2, 0, True, [0, 200, 32700]),
    ("roundShortAnsiWithOverflow", INT16, 0, [10, 100, 32760], -2, 0, True, ("row", 2)),
    ("roundShortAnsiNegativeOverflow", INT16, 0, [10, -32760], -2, 0, True, ("row", 1)),
    ("roundIntAnsiWithOverflow", INT32, 0, [10, 100, 2147483645], -1, 0, True, ("row", 2)),
    ("roundIntAnsiNoOverflow", INT32, 0, [12, 135, 160, None, -1454], -2, 0, True, [0, 100, 200, None, -1500]),
    ("roundLongAnsiWithOverflow", INT64, 0, [10, 100, 5000000000000000001], -19, 0, True, ("row", 2)),
    ("roundLongAnsiNoOverflow", INT64, 0, [10, 100, 4000000], -18, 0, True, [0, 0, 0]),
    ("roundPositiveDecimalPlacesNoOverflow", INT32, 0, [12, 135, None, 160], 2, 0, True, [12, 135, None, 160]),
    ("roundWithNulls", INT16, 0, [None, 100, None, 32760], -2, 0, True, ("row", 3)),
    ("roundHalfEvenAnsi", INT16, 0, [32750, 32755], -1, 1, True, [32750, 32760]),
    ("roundByteHalfEvenNoOverflow", INT8, 0, [125, 115, 105], -1, 1, True, [120, 120, 100]),
    ("roundByteHalfUpVsHalfEvenOverflow_up", INT8, 0, [125], -1, 0, True, ("row", 0)),
    ("roundByteHalfUpVsHalfEvenOverflow_even", INT8, 0, [125], -1, 1, True, [120]),
    ("roundByteHalfEvenOverflowAtCorrectThreshold", INT8, 0, [126], -1, 1, True, ("row", 0)),
    ("roundByteHalfEvenNegativeOverflow_ok", INT8, 0, [-125], -1, 1, True, [-120]),
    ("roundByteHalfEvenNegativeOverflow_bad", INT8, 0, [-126], -1, 1, True, ("row", 0)),
]
