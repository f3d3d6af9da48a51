"""com.nvidia.spark.rapids.jni.iceberg.IcebergBucket, IcebergTruncate and IcebergDateTimeUtil (IcebergBucket.java,
IcebergTruncate.java, IcebergDateTimeUtil.java) over the C ABI (include/srj_b200.h: srj_iceberg_*): the bucket[N],
truncate[W] and year / month / day / hour partition transforms an Iceberg writer applies to every row.

    ids  = IcebergBucket.computeBucket(col, numBuckets)    # INT32: (murmur3_x86_32 & INT32_MAX) % numBuckets
    out  = IcebergTruncate.truncate(col, width)           # same type: integral floor to a multiple, string / binary prefix
    yrs  = IcebergDateTimeUtil.yearsFromEpoch(col)        # INT32; monthsFromEpoch, daysFromEpoch (TIMESTAMP_DAYS),
                                                          # hoursFromEpoch (TIMESTAMP_MICROSECONDS only)

Every result keeps the input's null mask and null count.  Argument errors Java reports as IllegalArgumentException raise
ValueError; errors of the native layer raise CudfException; a null column raises TypeError (NullPointerException).
"""
import ctypes as C

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, _empty, _stream_ptr

_INTEGRAL = (DType.INT32, DType.INT64, DType.DECIMAL32, DType.DECIMAL64, DType.DECIMAL128)
YEARS, MONTHS, DAYS, HOURS = 0, 1, 2, 3      # SRJ_ICEBERG_YEARS .. SRJ_ICEBERG_HOURS


def _device(cv: ColumnView):
    kid = cv.child.data if cv.child is not None else None
    for t in (cv.data, cv.offsets, cv.mask, kid):
        if t is not None:
            return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _not_null(cv: ColumnView, what: str):
    if cv is None:
        raise TypeError(f"{what}: input column is null")                         # JNI_NULL_CHECK


def _out_mask(cv: ColumnView, dev):
    return _empty((cv.size + 31) // 32, torch.int32, dev) if cv.mask is not None else None


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() else None


class IcebergBucket:
    @staticmethod
    def computeBucket(input: ColumnView, numBuckets: int) -> ColumnVector:
        """INT32 bucket ids of Iceberg's bucket[numBuckets] transform; 0 under a null row."""
        numBuckets = int(numBuckets)
        if numBuckets <= 0:                                                        # IcebergBucket.java
            raise ValueError(f"numBuckets must be positive, got: {numBuckets}")
        _not_null(input, "IcebergBucket.computeBucket")
        n = input.size
        dev = _device(input)
        with torch.cuda.device(dev):
            out = _empty(n, torch.int32, dev)
            mask = _out_mask(input, dev)
            N.check(N.lib().srj_iceberg_bucket(C.byref(input._c()), numBuckets, _ptr(out), _ptr(mask), _stream_ptr()),
                    "IcebergBucket.computeBucket")
            return ColumnVector(DType.INT32, n, out.view(torch.uint8), mask, null_count=input.getNullCount())


class IcebergTruncate:
    @staticmethod
    def truncate(input: ColumnView, width: int) -> ColumnVector:
        """Iceberg's truncate[width]: INT32 / INT64 / DECIMAL values floored to a multiple of width, STRING rows cut to
        their first width characters, binary (LIST<UINT8>) rows to their first width bytes."""
        _not_null(input, "IcebergTruncate.truncate")
        width = int(width)
        t = input.dtype.type_id
        if t not in _INTEGRAL and t not in (DType.STRING, DType.LIST):             # IcebergTruncateJni.cpp
            raise ValueError("Unsupported type for truncation")
        n = input.size
        dev = _device(input)
        with torch.cuda.device(dev):
            lib = N.lib()
            stream = _stream_ptr()
            mask = _out_mask(input, dev)
            nulls = input.getNullCount()
            cin = input._c()
            if t in _INTEGRAL:
                data = _empty(n * input.dtype.size_in_bytes(), torch.uint8, dev)
                out = ColumnVector(DType(t, input.dtype.scale), n, data, mask, null_count=nulls)
            else:                                                                  # STRING, LIST<UINT8>
                offsets = _empty(n + 1, torch.int32, dev)
                ws = _empty(max(lib.srj_iceberg_truncate_workspace_bytes(n), 8), torch.uint8, dev)
                total = C.c_int64(0)
                N.check(lib.srj_iceberg_truncate_sizes(C.byref(cin), width, offsets.data_ptr(), C.byref(total), ws.data_ptr(),
                                                       stream), "IcebergTruncate.truncate")
                data = _empty(total.value, torch.uint8, dev)
                if t == DType.STRING:
                    out = ColumnVector(DType.STRING, n, data, mask, offsets, null_count=nulls)
                else:
                    out = ColumnVector(DType.LIST, n, None, mask, offsets, ColumnVector(DType.UINT8, total.value, data, null_count=0),
                                       null_count=nulls)
            N.check(lib.srj_iceberg_truncate(C.byref(cin), width, C.byref(out._c()), stream), "IcebergTruncate.truncate")
            return out


class IcebergDateTimeUtil:
    @staticmethod
    def _transform(input: ColumnView, transform: int, what: str) -> ColumnVector:
        _not_null(input, what)
        t = input.dtype.type_id
        if transform == HOURS and t != DType.TIMESTAMP_MICROSECONDS:               # IcebergDateTimeUtil.java
            raise ValueError("Input column must be of type TIMESTAMP_MICROSECONDS")
        if t not in (DType.TIMESTAMP_MICROSECONDS, DType.TIMESTAMP_DAYS):
            raise ValueError("Input column must be of type TIMESTAMP_MICROSECONDS or TIMESTAMP_DAYS")
        n = input.size
        dev = _device(input)
        with torch.cuda.device(dev):
            out = _empty(n, torch.int32, dev)
            mask = _out_mask(input, dev)
            N.check(N.lib().srj_iceberg_datetime(transform, C.byref(input._c()), _ptr(out), _ptr(mask), _stream_ptr()), what)
            out_type = DType.TIMESTAMP_DAYS if transform == DAYS else DType.INT32
            return ColumnVector(out_type, n, out.view(torch.uint8), mask, null_count=input.getNullCount())

    @staticmethod
    def yearsFromEpoch(input: ColumnView) -> ColumnVector:
        """INT32 years since 1970 of a TIMESTAMP_DAYS or TIMESTAMP_MICROSECONDS column."""
        return IcebergDateTimeUtil._transform(input, YEARS, "IcebergDateTimeUtil.yearsFromEpoch")

    @staticmethod
    def monthsFromEpoch(input: ColumnView) -> ColumnVector:
        """INT32 months since 1970-01."""
        return IcebergDateTimeUtil._transform(input, MONTHS, "IcebergDateTimeUtil.monthsFromEpoch")

    @staticmethod
    def daysFromEpoch(input: ColumnView) -> ColumnVector:
        """TIMESTAMP_DAYS days since 1970-01-01 (floored for microseconds)."""
        return IcebergDateTimeUtil._transform(input, DAYS, "IcebergDateTimeUtil.daysFromEpoch")

    @staticmethod
    def hoursFromEpoch(input: ColumnView) -> ColumnVector:
        """INT32 hours since the epoch (floored) of a TIMESTAMP_MICROSECONDS column."""
        return IcebergDateTimeUtil._transform(input, HOURS, "IcebergDateTimeUtil.hoursFromEpoch")
