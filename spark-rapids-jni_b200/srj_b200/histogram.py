"""com.nvidia.spark.rapids.jni.Histogram (Histogram.java:23-76) over the C ABI (include/srj_b200.h: srj_histogram_*,
srj_percentile_*).

    hist = Histogram.createHistogramIfValid(values, frequencies, outputAsLists)   # STRUCT<value, freq> or LIST of it
    pct  = Histogram.percentileFromHistogram(histograms, [0.5], outputAsLists)    # FLOAT64, or LIST<FLOAT64>

Spark's percentile(col, p [, freq]) runs createHistogramIfValid on the update side and percentileFromHistogram on the
final side; median(col) is percentile(col, 0.5).  Errors of the native layer raise CudfException
(CudfColumnSizeOverflowException when rows * percentages exceeds INT32_MAX).
"""
import ctypes as C

import numpy as np
import torch

from . import _native as N
from . import ColumnVector, ColumnView, DType, _empty, _stream_ptr


def _device(*cols):
    for c in cols:
        if c is None:
            continue
        for t in (c.offsets, c.data, c.mask):
            if t is not None:
                return t.device
        for k in ([c.child] if c.child is not None else []) + list(c.children or []):
            d = _device(k)
            if d is not None:
                return d
    return torch.device("cuda", torch.cuda.current_device())


def _nullable(c: ColumnView) -> N.SrjColumn:
    """The descriptor of c, its mask dropped when it holds no null (the C ABI reads a mask as nulls)."""
    d = c._c()
    if c.mask is not None and c.getNullCount() == 0:
        d.null_mask = None
    return d


class Histogram:
    @staticmethod
    def createHistogramIfValid(values: ColumnView, frequencies: ColumnView, outputAsLists: bool) -> ColumnVector:
        """STRUCT<values, frequencies> (or each row as a one-element list) after checking the frequencies."""
        if values is None or frequencies is None:
            raise TypeError("Histogram.createHistogramIfValid: input column is null")
        dev = _device(values, frequencies)
        with torch.cuda.device(dev):
            lib = N.lib()
            stream = _stream_ptr()
            cv, cf = _nullable(values), _nullable(frequencies)
            rows = values.size
            ws = _empty(max(lib.srj_histogram_workspace_bytes(rows), 8), torch.uint8, dev)
            n_out, nulls = C.c_int64(0), C.c_int64(0)
            N.check(lib.srj_histogram_create_size(C.byref(cv), C.byref(cf), int(bool(outputAsLists)), C.byref(n_out), C.byref(nulls),
                                                  ws.data_ptr(), stream), "Histogram.createHistogramIfValid")
            n = n_out.value
            width = values.dtype.size_in_bytes()
            out_v = _empty(n * width, torch.uint8, dev)
            out_f = _empty(n, torch.int64, dev)
            has_mask = not outputAsLists or cv.null_mask is not None
            mask = _empty(max((n if outputAsLists else rows) + 31, 32) // 32, torch.int32, dev) if has_mask else None
            offsets = torch.zeros(rows + 1, dtype=torch.int32, device=dev) if outputAsLists else None
            N.check(lib.srj_histogram_create(C.byref(cv), C.byref(cf), int(bool(outputAsLists)), out_v.data_ptr() if n else None,
                                             mask.data_ptr() if mask is not None else None, out_f.data_ptr() if n else None,
                                             offsets.data_ptr() if offsets is not None else None, ws.data_ptr(), stream),
                    "Histogram.createHistogramIfValid")
            vcol = ColumnVector(values.dtype, n, out_v, mask if nulls.value else None, null_count=nulls.value)
            fcol = ColumnVector(DType.INT64, n, out_f.view(torch.uint8), None, null_count=0)
            st = ColumnVector(DType.STRUCT, n, None, None, None, None, null_count=0, children=[vcol, fcol])
            if not outputAsLists:
                return st
            return ColumnVector(DType.LIST, rows, None, None, offsets, st, null_count=0)

    @staticmethod
    def percentileFromHistogram(input: ColumnView, percentages, outputAsLists: bool) -> ColumnVector:
        """Per histogram row, the percentiles of its (value, count) elements: FLOAT64 rows * P, or LIST<FLOAT64>."""
        if input is None or percentages is None:
            raise TypeError("Histogram.percentileFromHistogram: input is null")
        pct = np.ascontiguousarray(np.asarray(percentages, dtype=np.float64).reshape(-1))
        P = int(pct.size)
        dev = _device(input)
        with torch.cuda.device(dev):
            lib = N.lib()
            stream = _stream_ptr()
            cin = input._c()
            kids = fields = None                 # the descriptors below must outlive both calls
            if input.dtype.type_id == DType.LIST and input.child is not None:
                # the struct child and the counts count as nullable only when they hold a null
                st = input.child
                kids = (N.SrjColumn * 1)(_nullable(st))
                if st.children:
                    fields = (N.SrjColumn * len(st.children))(*[f._c() if i == 0 else _nullable(f) for i, f in enumerate(st.children)])
                    kids[0].children = fields
                cin.children = kids
            rows = input.size
            elements = input.child.size if input.child is not None else 0
            ws = _empty(max(lib.srj_percentile_workspace_bytes(rows, elements, P), 8), torch.uint8, dev)
            valid, n_values = C.c_int64(0), C.c_int64(0)
            N.check(lib.srj_percentile_from_histogram_size(C.byref(cin), P, int(bool(outputAsLists)), C.byref(valid), C.byref(n_values),
                                                           ws.data_ptr(), stream), "Histogram.percentileFromHistogram")
            n_out = n_values.value
            out = _empty(n_out, torch.float64, dev)
            mask = _empty(max((rows if outputAsLists else n_out) + 31, 32) // 32, torch.int32, dev)   # a bit per row / per double
            offsets = torch.zeros(rows + 1, dtype=torch.int32, device=dev) if outputAsLists else None
            N.check(lib.srj_percentile_from_histogram(C.byref(cin), pct.ctypes.data_as(C.c_void_p) if P else None, P,
                                                      int(bool(outputAsLists)), out.data_ptr() if n_out else None, mask.data_ptr(),
                                                      offsets.data_ptr() if offsets is not None else None, ws.data_ptr(), stream),
                    "Histogram.percentileFromHistogram")
            nulls = rows - valid.value
            if not outputAsLists:                # rows * P doubles (rows when every row is null), each null where its row is
                return ColumnVector(DType.FLOAT64, n_out, out.view(torch.uint8), mask if nulls else None,
                                    null_count=nulls * (n_out // rows) if rows else 0)
            child = ColumnVector(DType.FLOAT64, n_out, out.view(torch.uint8), None, null_count=0)
            return ColumnVector(DType.LIST, rows, None, mask if nulls else None, offsets, child, null_count=nulls)

