"""com.nvidia.spark.rapids.jni.NumberConverter (NumberConverter.java): Spark's conv(), over the C ABI (include/srj_b200.h:
srj_conv_sizes, srj_conv, srj_conv_overflow).

    s = NumberConverter.convertCvSS(strings, 10, 16)             # STRING column, bases 10 -> 16
    s = NumberConverter.convertSCvCv(Scalar.fromString("-127"), fromBases, toBases)
    NumberConverter.isConvertOverflowCvSS(strings, 10, 16)       # True when a row overflows under Spark's ANSI rule

The input is a STRING column (Cv) or a STRING Scalar (S); each base is an INT32 column (Cv) or an int (S).  The result
has the column arguments' rows; a row is null where its input or a base is null, a base is outside [2, 36] (|toBase|),
or the string is empty after trimming spaces.  It carries a mask only when it has nulls.  A null column or scalar
raises TypeError; errors of the native layer (wrong types, differing row counts, a null scalar input) raise
CudfException.  CastStrings' bin() and hex() casts are in srj_b200.cast.
"""
import ctypes as C

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, _empty, _stream_ptr
from .bloom import Scalar


def _device(*args):
    for a in args:
        for t in (getattr(a, "offsets", None), getattr(a, "data", None), getattr(a, "mask", None)):
            if isinstance(t, torch.Tensor):
                return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() else None


def strings_result(n, offsets, chars, mask, nulls) -> ColumnVector:
    """The STRING column of a radix cast: its mask dropped when it holds no null."""
    return ColumnVector(DType(DType.STRING), n, chars, mask if nulls else None, offsets, null_count=nulls)


def _conv_args(input, from_base, to_base, what):
    if input is None:
        raise TypeError(f"{what}: input column/scalar handle is null")                 # JNI_NULL_CHECK
    args = []
    if isinstance(input, Scalar):
        if input.dtype is None or input.dtype.type_id != DType.STRING:
            raise N.CudfException(f"{what}: Input scalar must be of type STRING")
        if input.valid is None or not bool(input.valid.cpu()[0]):
            raise N.CudfException(f"{what}: Input scalar must be valid")
        args += [None, _ptr(input.data), int(input.data.numel())]
    else:
        args += [C.byref(input._c()), None, 0]
    for b, name in ((from_base, "from_base"), (to_base, "to_base")):
        if isinstance(b, ColumnView):
            args += [C.byref(b._c()), 0]
        elif b is None:
            raise TypeError(f"{what}: {name} column handle is null")
        else:
            args += [None, int(b)]
    return args


def _convert(input, from_base, to_base) -> ColumnVector:
    what = "NumberConverter.convert"
    args = _conv_args(input, from_base, to_base, what)
    lead = next(a for a in (input, from_base, to_base) if isinstance(a, ColumnView))
    n = lead.size
    dev = _device(input, from_base, to_base)
    with torch.cuda.device(dev):
        lib, stream = N.lib(), _stream_ptr()
        offsets = _empty(n + 1, torch.int32, dev)
        mask = _empty(max((n + 31) // 32, 1), torch.int32, dev)
        ws = _empty(max(lib.srj_conv_workspace_bytes(n), 8), torch.uint8, dev)
        nulls, total = C.c_int64(0), C.c_int64(0)
        N.check(lib.srj_conv_sizes(*args, offsets.data_ptr(), mask.data_ptr(), C.byref(nulls), C.byref(total), ws.data_ptr(), stream), what)
        chars = _empty(total.value, torch.uint8, dev)
        N.check(lib.srj_conv(*args, offsets.data_ptr(), _ptr(chars), ws.data_ptr(), stream), what)
        return strings_result(n, offsets, chars, mask, nulls.value)


def _is_overflow(input, from_base, to_base) -> bool:
    what = "NumberConverter.isConvertOverflow"
    args = _conv_args(input, from_base, to_base, what)
    with torch.cuda.device(_device(input, from_base, to_base)):
        flag = C.c_int32(0)
        N.check(N.lib().srj_conv_overflow(*args, C.byref(flag), _stream_ptr()), what)
        return bool(flag.value)


class NumberConverter:
    """Spark's conv(input, fromBase, toBase): a number's digits in one base rewritten in another (toBase < 0: signed)."""

    @staticmethod
    def convertCvCvCv(input: ColumnView, fromBase: ColumnView, toBase: ColumnView) -> ColumnVector:
        return _convert(input, fromBase, toBase)

    @staticmethod
    def convertCvCvS(input: ColumnView, fromBase: ColumnView, toBase: int) -> ColumnVector:
        return _convert(input, fromBase, toBase)

    @staticmethod
    def convertCvSCv(input: ColumnView, fromBase: int, toBase: ColumnView) -> ColumnVector:
        return _convert(input, fromBase, toBase)

    @staticmethod
    def convertCvSS(input: ColumnView, fromBase: int, toBase: int) -> ColumnVector:
        return _convert(input, fromBase, toBase)

    @staticmethod
    def convertSCvCv(input: Scalar, fromBase: ColumnView, toBase: ColumnView) -> ColumnVector:
        return _convert(input, fromBase, toBase)

    @staticmethod
    def convertSCvS(input: Scalar, fromBase: ColumnView, toBase: int) -> ColumnVector:
        return _convert(input, fromBase, toBase)

    @staticmethod
    def convertSSCv(input: Scalar, fromBase: int, toBase: ColumnView) -> ColumnVector:
        return _convert(input, fromBase, toBase)

    @staticmethod
    def isConvertOverflowCvCvCv(input: ColumnView, fromBase: ColumnView, toBase: ColumnView) -> bool:
        return _is_overflow(input, fromBase, toBase)

    @staticmethod
    def isConvertOverflowCvCvS(input: ColumnView, fromBase: ColumnView, toBase: int) -> bool:
        return _is_overflow(input, fromBase, toBase)

    @staticmethod
    def isConvertOverflowCvSCv(input: ColumnView, fromBase: int, toBase: ColumnView) -> bool:
        return _is_overflow(input, fromBase, toBase)

    @staticmethod
    def isConvertOverflowCvSS(input: ColumnView, fromBase: int, toBase: int) -> bool:
        return _is_overflow(input, fromBase, toBase)

    @staticmethod
    def isConvertOverflowSCvCv(input: Scalar, fromBase: ColumnView, toBase: ColumnView) -> bool:
        return _is_overflow(input, fromBase, toBase)

    @staticmethod
    def isConvertOverflowSCvS(input: Scalar, fromBase: ColumnView, toBase: int) -> bool:
        return _is_overflow(input, fromBase, toBase)

    @staticmethod
    def isConvertOverflowSSCv(input: Scalar, fromBase: int, toBase: ColumnView) -> bool:
        return _is_overflow(input, fromBase, toBase)
