"""ZOrder.interleaveBits and ZOrder.hilbertIndex, restated in numpy (vectorised over rows).

Reference lines (src/main/cpp/src/ of the reference unless noted):
  - interleave_bits: zorder.cu:137-216 and the "source of truth from deltalake" of InterleaveBitsTest.java:31-137.
    N >= 1 columns of one fixed-width type id; a value is its W little-endian bytes read as an unsigned 8W-bit integer,
    a null row counts as 0.  Row r is N * W bytes; stream position i (i = 0 is bit 7 of byte 0) holds bit
    8W - 1 - i // N of column i % N.  Offsets r * N * W, no null mask.
  - hilbert_index: zorder.cu:218-267, ZOrder.java:57-83.  INT32 columns, value = uint32 bits masked to num_bits, a null
    counts as 0.  Skilling, "Programming the Hilbert curve" (2004): AxesToTranspose with Gray encoding; then the
    transposed coordinates read out with the same stream rule (num_bits in place of 8W) as one integer.
Columns are (data, mask) pairs of host numpy arrays: data = the raw little-endian bytes (uint8, rows * W) or any numpy
array viewed as such, mask = cudf bitmask words (uint32) or None.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

INT32_MAX = 2**31 - 1
_CHUNK = 1 << 20            # rows per vectorised block (bounds the bit matrix at 8 * N * W bytes per row)


def _valid(mask: Optional[np.ndarray], rows: int) -> np.ndarray:
    if mask is None:
        return np.ones(rows, dtype=bool)
    return np.unpackbits(np.ascontiguousarray(mask).view(np.uint8), bitorder="little")[:rows].astype(bool)


def interleave_bits(cols: Sequence[Tuple[np.ndarray, Optional[np.ndarray]]], width: int, rows: int) -> Tuple[np.ndarray, np.ndarray]:
    """-> (offsets int32[rows + 1], bytes uint8[rows * N * W])."""
    n = len(cols)
    if n == 0:
        raise ValueError("The input table must have at least one column.")
    rb = n * width
    if rows * rb > INT32_MAX:
        raise ValueError("Input is too large to process")
    offsets = (np.arange(rows + 1, dtype=np.int64) * rb).astype(np.int32)
    out = np.empty(rows * rb, dtype=np.uint8)
    datas = [np.ascontiguousarray(d).view(np.uint8).reshape(-1)[: rows * width].reshape(rows, width) for d, _ in cols]
    valids = [_valid(m, rows) for _, m in cols]
    for s in range(0, rows, _CHUNK):
        e = min(rows, s + _CHUNK)
        bits = np.empty((e - s, 8 * width, n), dtype=np.uint8)
        for c in range(n):
            be = datas[c][s:e, ::-1] * valids[c][s:e, None]                 # big-endian bytes, nulls as 0
            bits[:, :, c] = np.unpackbits(be, axis=1)                         # MSB first
        out[s * rb:e * rb] = np.packbits(bits.reshape(e - s, -1), axis=1).reshape(-1)
    return offsets, out


def hilbert_index(num_bits: int, cols: Sequence[Tuple[np.ndarray, Optional[np.ndarray]]], rows: int) -> np.ndarray:
    """-> int64[rows]."""
    n = len(cols)
    if not 1 <= num_bits <= 32:
        raise ValueError("the number of bits must be >0 and <= 32.")
    if num_bits * n > 64:
        raise ValueError("we only support up to 64 bits of output right now.")
    if n == 0:
        raise ValueError("at least one column is required.")
    vmask = np.uint64((1 << num_bits) - 1)
    X = [np.ascontiguousarray(d).view(np.uint32)[:rows].astype(np.uint64) * _valid(m, rows) & vmask for d, m in cols]
    # AxesToTranspose: inverse undo
    for q in range(num_bits - 1, 0, -1):
        Q, P = np.uint64(1 << q), np.uint64((1 << q) - 1)
        for i in range(n):
            hit = (X[i] & Q) != 0
            t = np.where(hit, np.uint64(0), (X[0] ^ X[i]) & P)
            X[0] = np.where(hit, X[0] ^ P, X[0] ^ t)
            if i:
                X[i] = X[i] ^ t
    # Gray encode
    for i in range(1, n):
        X[i] = X[i] ^ X[i - 1]
    t = np.zeros(rows, dtype=np.uint64)
    for q in range(num_bits - 1, 0, -1):
        t = np.where((X[n - 1] & np.uint64(1 << q)) != 0, t ^ np.uint64((1 << q) - 1), t)
    X = [x ^ t for x in X]
    # interleave, column 0 taking the higher bit of each group
    out = np.zeros(rows, dtype=np.uint64)
    for q in range(num_bits - 1, -1, -1):
        for i in range(n):
            out = (out << np.uint64(1)) | ((X[i] >> np.uint64(q)) & np.uint64(1))
    return out.view(np.int64)
