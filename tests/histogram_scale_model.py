"""percentileFromHistogram over every row at once, in numpy, for inputs of millions of rows.

oracle/histogram.py answers one row at a time in Python; this model sorts, sums and searches all rows with a handful of
whole-array operations, so a million-row column is checked in seconds.  It restates the definition in
oracle/histogram.py's docstring and shares no code with it:

  * every non-null element is ordered by (row, key) with one np.lexsort, where the key keeps Spark's order:
      signed integers: the sign bit flipped;  unsigned: the value;  BOOL8: != 0;
      floats: the IEEE total order, every NaN one key above +inf (NaNs are equal), -0.0 before 0.0;
  * one running sum of the counts over all rows; a row's ranks lower + 1 and higher + 1 become the global targets
    base + lower + 1 and base + higher + 1 (base: the running sum before the row), each found by np.searchsorted (the
    higher one only where the element found for the lower one falls short of it);
  * the found index is clamped to the row's [start, end - 1]: a row whose total count is 0 puts rank 0 at base, which
    the search would resolve into an earlier row, and a rank past the row's total reads the row's last element;
  * (higher - position) * lo + (position - lower) * hi with each product rounded to float64 on its own.

The global running sum must stay below 2^63 (asserted), and counts are non-negative, as createHistogramIfValid makes them.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

_TOP64 = np.uint64(1 << 63)


def sort_keys(values: np.ndarray, bool8: bool = False) -> np.ndarray:
    """uint64 keys in Spark's order: equal keys for equal values (every NaN one key)."""
    v = np.asarray(values)
    if bool8 or v.dtype == np.bool_:
        return (v != 0).astype(np.uint64)
    if v.dtype.kind == "f":
        def bits(x):                                                  # float32 in the high half: one sign bit for both
            return x.view(np.uint64) if x.dtype == np.float64 else x.view(np.uint32).astype(np.uint64) << np.uint64(32)
        b = bits(v)
        key = np.where(b & _TOP64, ~b, b | _TOP64)                    # negatives reversed below the positives
        inf_key = bits(np.array([np.inf], v.dtype))[0] | _TOP64
        return np.where(np.isnan(v), inf_key + np.uint64(1), key)
    if v.dtype.kind == "i":
        return v.astype(np.int64).view(np.uint64) ^ _TOP64
    return v.astype(np.uint64)


def percentile(offsets: np.ndarray, values: np.ndarray, valid: Optional[np.ndarray], counts: np.ndarray,
               percentages: Sequence[float], bool8: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """-> (out float64 [rows, P], 0.0 under null rows; row_valid bool [rows]).  offsets may start above 0 (a slice);
    bool8: the values are BOOL8 bytes (any nonzero byte is true)."""
    offsets = np.asarray(offsets, np.int64)
    rows, P = len(offsets) - 1, len(percentages)
    out = np.zeros((rows, P), np.float64)
    ok = np.zeros(rows, bool)
    if P == 0 or offsets[-1] == offsets[0]:
        return out, ok
    s0, e0 = int(offsets[0]), int(offsets[-1])
    row = np.repeat(np.arange(rows, dtype=np.int64), np.diff(offsets))
    vals = np.asarray(values)[s0:e0]
    cnt = np.asarray(counts, np.int64)[s0:e0]
    if valid is not None:
        keep = np.asarray(valid, bool)[s0:e0]
        row, vals, cnt = row[keep], vals[keep], cnt[keep]
    assert (cnt >= 0).all(), "counts must be non-negative"
    assert cnt.astype(np.float64).sum() < 2.0**62, "the running sum over all rows must stay below 2^63"
    key = sort_keys(vals, bool8)
    order = np.lexsort((key, row))
    row, key, vals, cnt = row[order], key[order], vals[order], cnt[order]
    is_float = vals.dtype.kind == "f"
    with np.errstate(invalid="ignore"):                               # signalling NaN payloads widen quietly
        dv = key.astype(np.float64) if (bool8 or vals.dtype == np.bool_) else vals.astype(np.float64)

    nv = np.bincount(row, minlength=rows)
    ok = nv > 0
    end = np.cumsum(nv)[ok]
    start = end - nv[ok]
    cum = np.cumsum(cnt)
    base = np.where(start > 0, cum[np.maximum(start - 1, 0)], 0)
    total = cum[end - 1] - base

    def find(target):
        return np.clip(np.searchsorted(cum, target, side="left"), start, end - 1)

    last = (total - 1).astype(np.float64)
    res = np.empty((len(start), P), np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        for q, p in enumerate(percentages):
            position = last * np.float64(p)
            lower = np.floor(position)
            higher = np.ceil(position)
            lo = find(base + lower.astype(np.int64) + 1)
            t_hi = base + higher.astype(np.int64) + 1
            hi = lo.copy()                                      # lo already reaches the higher rank, unless:
            short = cum[lo] < t_hi
            hi[short] = np.clip(np.searchsorted(cum, t_hi[short], side="left"), start[short], end[short] - 1)
            vlo, vhi = dv.take(lo), dv.take(hi)
            equal = (vlo == vhi) if is_float else (key.take(lo) == key.take(hi))  # equal in T
            mix = (higher - position) * vlo + (position - lower) * vhi
            res[:, q] = np.where((higher == lower) | equal, vlo, mix)
    out[ok] = res
    return out, ok
