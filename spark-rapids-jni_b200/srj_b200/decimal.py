"""com.nvidia.spark.rapids.jni.DecimalUtils (DecimalUtils.java) over the C ABI (include/srj_b200.h:
srj_decimal128_binary): the DECIMAL128 arithmetic Spark runs on every row of a batch when the exact intermediate value
can need more than 128 bits.

    t = DecimalUtils.multiply128(a, b, productScale, interimCast=True)   # Table [BOOL8 overflow, DECIMAL128(productScale)]
    t = DecimalUtils.divide128(a, b, quotientScale)                     # HALF_UP
    t = DecimalUtils.integerDivide128(a, b)                             # [BOOL8, INT64]
    t = DecimalUtils.remainder128(a, b, remainderScale)
    t = DecimalUtils.add128(a, b, targetScale) / subtract128(a, b, targetScale)

    r = DecimalUtils.floatingPointToDecimal(x, DType(DType.DECIMAL64, -2), 18)   # CAST(x AS DECIMAL(18, 2))
    r.result, r.failureRowId                                            # (srj_float_to_fixed_point)

Scales are cudf scales (the value is unscaled * 10^scale).  Both output columns carry the AND of the inputs' null masks
and its null count.  Java's IllegalArgumentException raises ValueError; errors of the native layer (a column that is not
DECIMAL128, differing row counts, an unsupported scale combination) raise CudfException; a null column raises TypeError.
floatingPointToDecimal's result carries a mask only when it has nulls; its failureRowId is the smallest failing row, or
-1.
"""
import ctypes as C

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, Table, _empty, _stream_ptr

MULTIPLY, DIVIDE, INTEGER_DIVIDE, REMAINDER, ADD, SUBTRACT = range(6)     # SRJ_DECIMAL_*


def _device(*cols):
    for c in cols:
        for t in (c.data, c.mask):
            if t is not None:
                return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _binary(op, a: ColumnView, b: ColumnView, scale: int, interim_cast: bool, what: str) -> Table:
    if a is None or b is None:
        raise TypeError(f"{what}: column is null")                                 # JNI_NULL_CHECK
    n = a.size
    dev = _device(a, b)
    with torch.cuda.device(dev):
        ovf = _empty(n, torch.uint8, dev)
        out = _empty(n * (8 if op == INTEGER_DIVIDE else 16), torch.uint8, dev)
        has_mask = a.mask is not None or b.mask is not None
        mask = _empty((n + 31) // 32, torch.int32, dev) if has_mask else None
        nulls = C.c_int64(0)
        N.check(N.lib().srj_decimal128_binary(op, C.byref(a._c()), C.byref(b._c()), int(scale), int(bool(interim_cast)),
                                              ovf.data_ptr() if n else None, out.data_ptr() if n else None,
                                              mask.data_ptr() if mask is not None and mask.numel() else None, C.byref(nulls),
                                              _stream_ptr()), what)
        out_type = DType(DType.INT64) if op == INTEGER_DIVIDE else DType(DType.DECIMAL128, scale)
        m2 = mask.clone() if mask is not None else None                             # each column owns its mask
        return Table(ColumnVector(DType.BOOL8, n, ovf, mask, null_count=nulls.value),
                     ColumnVector(out_type, n, out, m2, null_count=nulls.value))


def _check_scale_gap(a: ColumnView, b: ColumnView):
    if a is not None and b is not None and abs(a.getType().scale - b.getType().scale) > 77:     # DecimalUtils.java:152, 176
        raise ValueError("The intermediate scale for calculating the result exceeds 256-bit representation")


class CastFloatToDecimalResult:
    """DecimalUtils.CastFloatToDecimalResult: the cast's column and the smallest failing row (negative: none)."""

    def __init__(self, result: ColumnVector, failureRowId: int):
        self.result = result
        self.failureRowId = failureRowId


class DecimalUtils:
    @staticmethod
    def multiply128(a: ColumnView, b: ColumnView, productScale: int, interimCast: bool = True) -> Table:
        """a * b rounded HALF_UP to productScale; interimCast first rounds a product of more than 38 digits to 38
        (Spark before 3.4.2 / 3.5.1 / 4.0.0, SPARK-40129)."""
        return _binary(MULTIPLY, a, b, productScale, interimCast, "DecimalUtils.multiply128")

    @staticmethod
    def divide128(a: ColumnView, b: ColumnView, quotientScale: int) -> Table:
        """a / b rounded HALF_UP to quotientScale; a zero divisor overflows with value 0."""
        return _binary(DIVIDE, a, b, quotientScale, False, "DecimalUtils.divide128")

    @staticmethod
    def integerDivide128(a: ColumnView, b: ColumnView) -> Table:
        """a div b as INT64 (the low 64 bits); overflow is judged on the whole quotient."""
        return _binary(INTEGER_DIVIDE, a, b, 0, False, "DecimalUtils.integerDivide128")

    @staticmethod
    def remainder128(a: ColumnView, b: ColumnView, remainderScale: int) -> Table:
        """a - (a div b) * b at remainderScale, with the sign of a."""
        return _binary(REMAINDER, a, b, remainderScale, False, "DecimalUtils.remainder128")

    @staticmethod
    def add128(a: ColumnView, b: ColumnView, targetScale: int) -> Table:
        """a + b at the finer input scale, rounded HALF_UP to targetScale (Spark 3.4+)."""
        _check_scale_gap(a, b)
        return _binary(ADD, a, b, targetScale, False, "DecimalUtils.add128")

    @staticmethod
    def subtract128(a: ColumnView, b: ColumnView, targetScale: int) -> Table:
        """a - b at the finer input scale, rounded HALF_UP to targetScale (Spark 3.4+)."""
        _check_scale_gap(a, b)
        return _binary(SUBTRACT, a, b, targetScale, False, "DecimalUtils.subtract128")

    @staticmethod
    def floatingPointToDecimal(input: ColumnView, outputType: DType, precision: int) -> CastFloatToDecimalResult:
        """CAST(float / double AS DECIMAL(precision, -outputType.scale)) as Spark computes it: a null, NaN or infinite
        row is null; a value whose rounded result has more than `precision` digits is null and fails."""
        what = "DecimalUtils.floatingPointToDecimal"
        if input is None:
            raise TypeError(f"{what}: column is null")                                # JNI_NULL_CHECK
        n = input.size
        dev = _device(input)
        with torch.cuda.device(dev):
            out = _empty(n * max(outputType.size_in_bytes(), 1), torch.uint8, dev)
            mask = _empty((n + 31) // 32, torch.int32, dev)
            nulls, failure = C.c_int64(0), C.c_int64(-1)
            N.check(N.lib().srj_float_to_fixed_point(C.byref(input._c()), outputType.type_id, int(precision), outputType.scale,
                                                     out.data_ptr() if n else None, mask.data_ptr() if n else None,
                                                     C.byref(nulls), C.byref(failure), _stream_ptr()), what)
            col = ColumnVector(DType(outputType.type_id, outputType.scale), n, out, mask if nulls.value else None,
                               null_count=nulls.value)
            return CastFloatToDecimalResult(col, failure.value)
