"""Histogram.percentileFromHistogram and Histogram.createHistogramIfValid, restated in numpy.

Reference lines (src/main/cpp/src/ of the reference):
  - percentile_from_histogram: histogram.cu:46-249, 415-493.  Per row, the non-null values in ascending order (floats:
    every NaN equal and after +inf; -0.0 pinned before 0.0, where the reference's unstable sort may choose either;
    BOOL8: nonzero = true), acc = the inclusive running sum of their counts, and per percentage p:
        position = float64(acc[-1] - 1) * p, lower = floor(position), higher = ceil(position)
        lo / hi  = the first element with acc >= lower + 1 / higher + 1 (the last element when none has)
        result   = float64(lo) when higher == lower or lo == hi in T,
                   else (float64(higher) - position) * lo + (position - float64(lower)) * hi   (two rounded products)
    A row without a non-null value is null; with P == 0 or no element at all every row is null (histogram.cu:170).
  - create_histogram_if_valid: histogram.cu:274-413.

Columns are host numpy arrays: values (any numpy dtype), valid (bool per element, or None = all valid), counts int64.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np


def sort_keys(values: np.ndarray) -> np.ndarray:
    """uint64 keys in the order above (equal keys: equal values)."""
    v = np.asarray(values)
    if v.dtype == np.bool_:
        return v.astype(np.uint64)
    if v.dtype.kind == "f":
        bits, top = (v.astype(np.float64).view(np.uint64), np.uint64(1 << 63)) if v.dtype == np.float64 else \
            (v.view(np.uint32).astype(np.uint64), np.uint64(1 << 31))
        key = np.where(bits & top, ~bits & (top | (top - np.uint64(1))), bits | top)
        nan_key = np.uint64(0xfff8000000000000) if v.dtype == np.float64 else np.uint64(0xffc00000)
        return np.where(np.isnan(v), nan_key, key)
    if v.dtype.kind == "i":
        return v.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63)
    return v.astype(np.uint64)


def _as_double(x) -> np.float64:
    if isinstance(x, (np.integer, int)) and not isinstance(x, (bool, np.bool_)):
        return np.float64(int(x))
    return np.float64(x)


def percentile_row(values: np.ndarray, counts: np.ndarray, percentages: Sequence[float]) -> Optional[np.ndarray]:
    """The P results of one histogram of non-null values, or None when it has none."""
    if len(values) == 0:
        return None
    order = np.argsort(sort_keys(values), kind="stable")
    vals = np.asarray(values)[order]
    acc = np.cumsum(np.asarray(counts, dtype=np.int64)[order])
    is_float = vals.dtype.kind == "f"
    last = int(acc[-1])
    out = np.empty(len(percentages), np.float64)
    for q, p in enumerate(percentages):
        position = np.float64(last - 1) * np.float64(p)
        lower, higher = int(np.floor(position)), int(np.ceil(position))
        lo = vals[min(int(np.searchsorted(acc, lower + 1, side="left")), len(vals) - 1)]
        if higher == lower:
            out[q] = _as_double(lo)
            continue
        hi = vals[min(int(np.searchsorted(acc, higher + 1, side="left")), len(vals) - 1)]
        if (np.float64(lo) == np.float64(hi)) if is_float else (lo == hi):
            out[q] = _as_double(lo)
            continue
        out[q] = (np.float64(higher) - position) * _as_double(lo) + (position - np.float64(lower)) * _as_double(hi)
    return out


def percentile_from_histogram(offsets: np.ndarray, values: np.ndarray, valid: Optional[np.ndarray], counts: np.ndarray,
                              percentages: Sequence[float]) -> Tuple[np.ndarray, np.ndarray]:
    """-> (out float64 [rows, P] (0.0 under null rows), row_valid bool [rows])."""
    offsets = np.asarray(offsets, dtype=np.int64)
    rows, P = len(offsets) - 1, len(percentages)
    out = np.zeros((rows, P), np.float64)
    ok = np.zeros(rows, bool)
    if P == 0 or offsets[-1] == offsets[0]:
        return out, ok
    values, counts = np.asarray(values), np.asarray(counts)
    for r in range(rows):
        idx = np.arange(offsets[r], offsets[r + 1])
        if valid is not None:
            idx = idx[np.asarray(valid, bool)[idx]]
        res = percentile_row(values[idx], counts[idx], percentages)
        if res is not None:
            out[r], ok[r] = res, True
    return out, ok


def create_histogram_if_valid(values: np.ndarray, valid: Optional[np.ndarray], freqs: np.ndarray, output_as_lists: bool):
    """STRUCT: (values, value_valid, freqs).  LISTS: (offsets, values, value_valid, freqs) of the child.
    ValueError for a negative frequency (histogram.cu:324-326)."""
    values = np.asarray(values)
    freqs = np.asarray(freqs, dtype=np.int64)
    n = len(values)
    valid = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    if (freqs < 0).any():
        raise ValueError("The input frequencies must not contain negative values.")
    if output_as_lists:
        keep = freqs > 0
        offsets = np.concatenate([[0], np.cumsum(keep)]).astype(np.int32)
        return offsets, values[keep], valid[keep], freqs[keep]
    if not (freqs == 0).any():
        return values.copy(), valid.copy(), freqs.copy()
    out_valid = valid & (freqs != 0)
    return values.copy(), out_valid, np.where(out_valid, freqs, 1)
