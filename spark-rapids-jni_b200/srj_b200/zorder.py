"""com.nvidia.spark.rapids.jni.ZOrder (ZOrder.java:24-88) over the C ABI (include/srj_b200.h: srj_interleave_bits*,
srj_hilbert_index).

    rows = ZOrder.interleaveBits(numRows, *columns)          # LIST<UINT8>: Delta Lake's InterleaveBits (ZORDER BY)
    idx  = ZOrder.hilbertIndex(numBits, numRows, *columns)   # INT64: Hilbert clustering over INT32 columns

With no columns both return numRows rows without calling the native layer, as ZOrder.java does: numRows empty lists,
numRows zeros.  Errors of the native layer raise CudfException.
"""
import ctypes as C

import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, _carray, _empty, _stream_ptr


def _device(columns):
    for c in columns:
        for t in (c.data, c.mask):
            if t is not None:
                return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _args(numRows: int, columns):
    cols = list(columns)
    for c in cols:
        if c is None:
            raise TypeError("ZOrder: input column is null")
    return int(numRows), cols


class ZOrder:
    @staticmethod
    def interleaveBits(numRows: int, *inputColumns: ColumnView) -> ColumnVector:
        """Row r: the N * W bytes of the columns' bits interleaved MSB first, column 0 first (no null mask)."""
        n, cols = _args(numRows, inputColumns)
        dev = _device(cols)
        with torch.cuda.device(dev):
            if not cols:
                offsets = torch.zeros(n + 1, dtype=torch.int32, device=dev)
                return ColumnVector(DType.LIST, n, None, None, offsets, ColumnVector(DType.UINT8, 0, _empty(0, torch.uint8, dev)),
                                    null_count=0)
            rows = cols[0].size
            lib = N.lib()
            carr = _carray(cols)
            total = C.c_int64(0)
            N.check(lib.srj_interleave_bits_sizes(carr, len(cols), rows, C.byref(total)), "ZOrder.interleaveBits")
            offsets = _empty(rows + 1, torch.int32, dev)
            data = _empty(total.value, torch.uint8, dev)
            N.check(lib.srj_interleave_bits(carr, len(cols), rows, offsets.data_ptr(), data.data_ptr() if total.value else None,
                                            _stream_ptr()), "ZOrder.interleaveBits")
            return ColumnVector(DType.LIST, rows, None, None, offsets, ColumnVector(DType.UINT8, total.value, data), null_count=0)

    @staticmethod
    def hilbertIndex(numBits: int, numRows: int, *inputColumns: ColumnView) -> ColumnVector:
        """INT64 Hilbert index of each row's point (the INT32 values' low numBits bits; nulls count as 0)."""
        n, cols = _args(numRows, inputColumns)
        dev = _device(cols)
        with torch.cuda.device(dev):
            if not cols:
                return ColumnVector(DType.INT64, n, torch.zeros(n, dtype=torch.int64, device=dev).view(torch.uint8), None,
                                    null_count=0)
            rows = cols[0].size
            out = _empty(rows, torch.int64, dev)
            N.check(N.lib().srj_hilbert_index(int(numBits), _carray(cols), len(cols), rows, out.data_ptr() if rows else None,
                                              _stream_ptr()), "ZOrder.hilbertIndex")
            return ColumnVector(DType.INT64, rows, out.view(torch.uint8), None, null_count=0)
