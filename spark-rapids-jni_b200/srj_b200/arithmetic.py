"""com.nvidia.spark.rapids.jni.Arithmetic (Arithmetic.java:22-194) over the C ABI (include/srj_b200.h: srj_multiply,
srj_round).

    prod = Arithmetic.multiply(left, right, isAnsiMode, isTryMode)   # column * column, column * Scalar or Scalar * column
    r    = Arithmetic.round(col, decimalPlaces, RoundMode.HALF_EVEN)  # round(col, 2) / bround(col, 2)

multiply is Spark's `*` on byte, short, int, long, float and double: an integer overflow wraps by default, gives a null
row in try mode (try_multiply), and raises ExceptionWithRowIndex with the first overflowing row in ANSI mode.  round is
round / bround on integers, floats and decimals; in ANSI mode an integer whose rounded value leaves its type raises
ExceptionWithRowIndex.  Other errors of the native layer raise CudfException, as the reference's JNI layer does.
"""
import ctypes as C
import enum

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, _empty, _stream_ptr
from .bloom import Scalar


class RoundMode(enum.IntEnum):
    """com.nvidia.spark.rapids.jni.RoundMode: HALF_UP is round, HALF_EVEN is bround."""
    HALF_UP = 0
    HALF_EVEN = 1

    @property
    def nativeId(self) -> int:
        return int(self)


class ExceptionWithRowIndex(RuntimeError):
    """com.nvidia.spark.rapids.jni.ExceptionWithRowIndex: the first row whose result overflows in ANSI mode."""

    def __init__(self, rowIndex: int):
        super().__init__(f"overflow at row {rowIndex}")
        self.rowIndex = int(rowIndex)

    def getRowIndex(self) -> int:
        return self.rowIndex


def _device(*xs):
    for x in xs:
        if x is not None and x.data is not None:
            return x.data.device
    return torch.device("cuda", torch.cuda.current_device())


def _nullable(c: ColumnView) -> N.SrjColumn:
    """The descriptor of c, its mask dropped when it holds no null (the C ABI reads a mask as nulls)."""
    d = c._c()
    if c.mask is not None and c.getNullCount() == 0:
        d.null_mask = None
    return d


def _operand(x):
    """(descriptor, scalar validity pointer) of a column or a fixed-width Scalar."""
    if isinstance(x, Scalar):
        if x.dtype is None:
            raise TypeError("Arithmetic.multiply: a scalar operand must have a numeric type")
        d = N.SrjColumn()
        d.type_id, d.scale, d.size, d.data = x.dtype.type_id, x.dtype.scale, 1, x.data.data_ptr()
        return d, x.valid.data_ptr()
    return _nullable(x), None


class Arithmetic:
    @staticmethod
    def multiply(left, right, isAnsiMode: bool, isTryMode: bool) -> ColumnVector:
        """left * right with Spark's overflow handling; left and right are columns, or one of them a Scalar."""
        if left is None or right is None:
            raise TypeError("Arithmetic.multiply: " + ("left" if left is None else "right") + " input is null")
        dev = _device(left, right)
        with torch.cuda.device(dev):
            lib = N.lib()
            cl, lv = _operand(left)
            cr, rv = _operand(right)
            column = right if isinstance(left, Scalar) else left
            rows, dtype = column.size, column.dtype
            out = _empty(rows * dtype.size_in_bytes(), torch.uint8, dev)
            mask = _empty((rows + 31) // 32, torch.int32, dev)
            nulls, row = C.c_int64(0), C.c_int64(-1)
            N.check(lib.srj_multiply(C.byref(cl), lv, C.byref(cr), rv, int(bool(isAnsiMode)), int(bool(isTryMode)),
                                     out.data_ptr() if rows else None, mask.data_ptr() if rows else None, C.byref(nulls),
                                     C.byref(row), _stream_ptr()), "Arithmetic.multiply")
            if row.value >= 0:
                raise ExceptionWithRowIndex(row.value)
            return ColumnVector(dtype, rows, out, mask if nulls.value else None, null_count=nulls.value)

    @staticmethod
    def round(input: ColumnView, *args) -> ColumnVector:
        """round(input), round(input, decimalPlaces), round(input, mode), round(input, decimalPlaces, mode) and
        round(input, decimalPlaces, mode, isAnsiMode); decimalPlaces defaults to 0, mode to HALF_UP, isAnsiMode to false."""
        if len(args) == 1 and isinstance(args[0], RoundMode):
            args = (0, args[0])
        decimalPlaces, mode, isAnsiMode = (tuple(args) + (0, RoundMode.HALF_UP, False)[len(args):])[:3]
        if input is None:
            raise TypeError("Arithmetic.round: input is null")
        dev = _device(input)
        with torch.cuda.device(dev):
            lib = N.lib()
            cin = _nullable(input)
            rows = input.size
            # a decimal's result has scale -decimalPlaces; an empty input keeps its type, as the reference's empty_like
            dtype = DType(input.dtype.type_id, -int(decimalPlaces)) if rows and input.dtype.type_id in (
                DType.DECIMAL32, DType.DECIMAL64, DType.DECIMAL128) else input.dtype
            out = _empty(rows * max(dtype.size_in_bytes(), 1), torch.uint8, dev)
            has_mask = cin.null_mask is not None
            mask = _empty((rows + 31) // 32, torch.int32, dev) if has_mask and rows else None
            row = C.c_int64(-1)
            N.check(lib.srj_round(C.byref(cin), int(decimalPlaces), int(mode), int(bool(isAnsiMode)), out.data_ptr() if rows else None,
                                  mask.data_ptr() if mask is not None else None, C.byref(row), _stream_ptr()), "Arithmetic.round")
            if row.value >= 0:
                raise ExceptionWithRowIndex(row.value)
            return ColumnVector(dtype, rows, out, mask, null_count=input.getNullCount() if has_mask else 0)
