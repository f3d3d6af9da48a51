"""com.nvidia.spark.rapids.jni.DateTimeUtils (DateTimeUtils.java) over the C ABI (include/srj_b200.h: srj_datetime_*):
the calendar rebase Spark runs on every date / timestamp row read or written in LEGACY rebase mode, and the truncation
behind trunc(date, fmt) and date_trunc(fmt, ts).

    out = DateTimeUtils.rebaseGregorianToJulian(col)    # TIMESTAMP_DAYS or TIMESTAMP_MICROSECONDS, same type
    out = DateTimeUtils.rebaseJulianToGregorian(col)
    out = DateTimeUtils.truncate(col, "MONTH")          # a format string, or a STRING column of formats

The rebase keeps the input's null mask and null count.  A truncation's row is null where its datetime, its format or
the format's parse is; the result has a mask only when it has nulls.  A null column raises TypeError
(NullPointerException); errors of the native layer (a type that is not a timestamp of days or microseconds, a format
column that is not STRING, mismatched row counts) raise CudfException.
"""
import ctypes as C

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, _empty, _stream_ptr

GREGORIAN_TO_JULIAN, JULIAN_TO_GREGORIAN = 0, 1      # SRJ_DATETIME_*


def _device(*cols):
    for c in cols:
        for t in (c.data, c.offsets, c.mask):
            if t is not None:
                return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() else None


def _width(cv: ColumnView) -> int:
    return 4 if cv.dtype.type_id == DType.TIMESTAMP_DAYS else 8


def _rebase(direction: int, input: ColumnView, what: str) -> ColumnVector:
    if input is None:
        raise TypeError(f"{what}: input column is null")                         # JNI_NULL_CHECK
    n = input.size
    dev = _device(input)
    with torch.cuda.device(dev):
        out = _empty(n * _width(input), torch.uint8, dev)
        mask = _empty((n + 31) // 32, torch.int32, dev) if input.mask is not None else None
        N.check(N.lib().srj_datetime_rebase(direction, C.byref(input._c()), _ptr(out), _ptr(mask), _stream_ptr()), what)
        return ColumnVector(DType(input.dtype.type_id), n, out, mask, null_count=input.getNullCount())


class DateTimeUtils:
    @staticmethod
    def rebaseGregorianToJulian(input: ColumnView) -> ColumnVector:
        """Each day's (or timestamp's) proleptic Gregorian local date-time, read as a Julian one (UTC)."""
        return _rebase(GREGORIAN_TO_JULIAN, input, "DateTimeUtils.rebaseGregorianToJulian")

    @staticmethod
    def rebaseJulianToGregorian(input: ColumnView) -> ColumnVector:
        """Each day's (or timestamp's) Julian local date-time, read as a proleptic Gregorian one (UTC)."""
        return _rebase(JULIAN_TO_GREGORIAN, input, "DateTimeUtils.rebaseJulianToGregorian")

    @staticmethod
    def truncate(datetime: ColumnView, format) -> ColumnVector:
        """datetime truncated to format: a str (DateTimeUtils.truncate(ColumnView, String); None is an empty format) or a
        STRING ColumnView with one format per row, the datetime then having one row or as many as the format."""
        what = "DateTimeUtils.truncate"
        if datetime is None:
            raise TypeError(f"{what}: input datetime is null")                    # JNI_NULL_CHECK
        column = isinstance(format, ColumnView)
        if format is not None and not column and not isinstance(format, str):
            raise TypeError(f"{what}: format must be a str or a ColumnView")
        n = format.size if column else datetime.size
        dev = _device(datetime, format) if column else _device(datetime)
        with torch.cuda.device(dev):
            out = _empty(n * _width(datetime), torch.uint8, dev)
            mask = _empty((n + 31) // 32, torch.int32, dev)
            nulls = C.c_int64(0)
            fmt_c = format._c() if column else None
            fmt_s = None if column else (format or "").encode("utf-8")
            N.check(N.lib().srj_datetime_truncate(C.byref(datetime._c()), C.byref(fmt_c) if column else None, fmt_s,
                                                  len(fmt_s) if fmt_s is not None else 0, _ptr(out), _ptr(mask), C.byref(nulls),
                                                  _stream_ptr()), what)
            null_count = datetime.getNullCount() if nulls.value < 0 else nulls.value
            return ColumnVector(DType(datetime.dtype.type_id), n, out, mask if null_count else None, null_count=null_count)
