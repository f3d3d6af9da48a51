"""An independent model of the JCUDF row format, in plain numpy.

Written from the format's definition: the RowConversion.java Javadoc (RowConversion.java:44-117), the layout rule of
compute_column_information (RC:1332-1371) and the batch cut of build_batches (RC:1466-1557).  It shares no code with
the C oracle (oracle/srj_oracle.c) or the product package, so a misreading of the format that both of those made would
show up as a difference here.

The format, as this model reads it:
  * a row is laid out like a C struct: each fixed-width field in schema order, aligned to its own size; a STRING column
    is a (uint32 offset, uint32 length) pair aligned to 4 bytes, the offset counted from the start of the row;
  * then one validity byte per 8 columns, no padding before it: bit c % 8 of byte c / 8 is set when column c is valid;
  * size_per_row ends there.  A fixed-width row is padded with zeros to a multiple of 8 bytes.  A row with STRING
    columns continues with the chars of its strings, back to back in column order and unpadded, from byte size_per_row;
    the whole row is then padded with zeros to a multiple of 8 bytes;
  * a null value's payload bytes are copied like any other; a null string keeps whatever length its offsets give it;
  * the rows go out in batches of at most INT32_MAX bytes, cut on 32-row boundaries.

Columns are duck-typed: anything with `type_id`, `size`, `data` (bytes of the values, or the chars), `mask` (uint32
words, or None = all valid) and `offsets` (STRING: int32[size + 1]) will do.  Everything is vectorised over rows; the
fixed section of a block of rows is held as an (rows, size_per_row) byte array and the chars are moved with index
arrays built from repeat / cumsum."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

# cudf type ids (cudf/types.hpp)
(INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8) = range(1, 12)
(TIMESTAMP_DAYS, TIMESTAMP_SECONDS, TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS, TIMESTAMP_NANOSECONDS) = range(12, 17)
(DURATION_DAYS, DURATION_SECONDS, DURATION_MILLISECONDS, DURATION_MICROSECONDS, DURATION_NANOSECONDS) = range(17, 22)
STRING, DECIMAL32, DECIMAL64, DECIMAL128 = 23, 25, 26, 27

SIZE = {INT8: 1, UINT8: 1, BOOL8: 1, INT16: 2, UINT16: 2, INT32: 4, UINT32: 4, FLOAT32: 4, TIMESTAMP_DAYS: 4,
        DURATION_DAYS: 4, DECIMAL32: 4, INT64: 8, UINT64: 8, FLOAT64: 8, TIMESTAMP_SECONDS: 8,
        TIMESTAMP_MILLISECONDS: 8, TIMESTAMP_MICROSECONDS: 8, TIMESTAMP_NANOSECONDS: 8, DURATION_SECONDS: 8,
        DURATION_MILLISECONDS: 8, DURATION_MICROSECONDS: 8, DURATION_NANOSECONDS: 8, DECIMAL64: 8, DECIMAL128: 16}

MAX_BATCH_BYTES = 2**31 - 1          # MAX_BATCH_SIZE: a LIST<INT8> column holds at most INT32_MAX bytes
STATUS_NON_CANONICAL = 1             # status word bit: some row does not place its chars where to_rows would
STATUS_CHARS_OVERFLOW = 2            # status word bit: a STRING column has more than INT32_MAX chars
_BLOCK_BYTES = 1 << 26               # fixed-section bytes handled at once (bounds the index arrays)


@dataclass
class Layout:
    starts: List[int]      # byte offset of each column's field in the row
    sizes: List[int]       # its size: the type's width, 8 for a STRING pair
    validity_offset: int
    size_per_row: int      # fixed fields + validity bytes
    fixed_row_size: int    # size_per_row rounded up to 8: the stride of a fixed-width table

    @property
    def num_columns(self) -> int:
        return len(self.starts)


def layout(types: Sequence[int]) -> Layout:
    off, starts, sizes = 0, [], []
    for t in types:
        if t == STRING:
            sz, align = 8, 4
        elif t in SIZE:
            sz = align = SIZE[t]
        else:
            raise NotImplementedError(f"type id {t} has no JCUDF row representation")
        off = (off + align - 1) // align * align
        starts.append(off)
        sizes.append(sz)
        off += sz
    voff = off
    spr = voff + (len(types) + 7) // 8
    return Layout(starts, sizes, voff, spr, (spr + 7) // 8 * 8)


def _valid(col, n: int) -> np.ndarray:
    if col.mask is None:
        return np.ones(n, bool)
    return np.unpackbits(np.ascontiguousarray(col.mask).view(np.uint8), bitorder="little")[:n].astype(bool)


def _pack_mask(valid: np.ndarray) -> np.ndarray:
    """uint32 words, bit r % 32 of word r / 32; the bits past the last row are zero."""
    n = len(valid)
    bits = np.zeros((n + 31) // 32 * 32, np.uint8)
    bits[:n] = valid
    return np.packbits(bits, bitorder="little").view(np.uint32)


def _str_lens(col, n: int) -> np.ndarray:
    return np.diff(np.asarray(col.offsets, dtype=np.int64)[: n + 1])


def _fixed_bytes(col, n: int) -> np.ndarray:
    sz = SIZE[col.type_id]
    return np.ascontiguousarray(col.data).view(np.uint8)[: n * sz].reshape(n, sz)


def row_sizes(cols) -> np.ndarray:
    """Bytes of each row: size_per_row + the chars of its strings, rounded up to 8."""
    n = cols[0].size if cols else 0
    lay = layout([c.type_id for c in cols])
    var = np.zeros(n, np.int64)
    for c in cols:
        if c.type_id == STRING:
            var += _str_lens(c, n)
    return ((lay.size_per_row + var + 7) // 8 * 8).astype(np.int64)


def build_batches(sizes: np.ndarray) -> List[int]:
    """Row boundaries of the batches.  From each batch start: the first row at which the running byte count (counted, as
    the reference's lower_bound counts it, from the row after the start) reaches INT32_MAX, rounded down to a multiple
    of 32 rows unless the table ends first; then 32 rows (or the odd remainder) at a time off the end until the batch
    really fits INT32_MAX bytes."""
    n = len(sizes)
    cum = np.cumsum(np.asarray(sizes, dtype=np.uint64))
    bounds, last = [0], 0
    while last < n:
        rel = cum[last:] - cum[last]
        lb = int(np.searchsorted(rel, MAX_BATCH_BYTES, side="left"))
        end = n if last + lb == n else last + lb // 32 * 32
        before = int(cum[last - 1]) if last else 0
        while True:
            if end <= last:
                raise OverflowError("a single row does not fit a 2 GiB batch")
            if int(cum[end - 1]) - before <= MAX_BATCH_BYTES:
                break
            m = end - last
            end -= m % 32 or 32
        bounds.append(end)
        last = end
    return bounds


def _fixed_section(cols, lay: Layout, r0: int, r1: int, pair_off: dict) -> np.ndarray:
    """(r1 - r0, size_per_row) bytes: the fields, the STRING pairs, the validity bytes, zero padding between fields."""
    m = r1 - r0
    F = np.zeros((m, lay.size_per_row), np.uint8)
    valid = np.zeros((m, (len(cols) + 7) // 8 * 8), bool)
    for c, col in enumerate(cols):
        st = lay.starts[c]
        if col.type_id == STRING:
            pair = np.empty((m, 2), np.uint32)
            pair[:, 0] = pair_off[c][r0:r1]
            pair[:, 1] = _str_lens(col, r1)[r0:r1]
            F[:, st:st + 8] = pair.view(np.uint8)
        else:
            F[:, st:st + lay.sizes[c]] = _fixed_bytes(col, r1)[r0:r1]
        valid[:, c] = _valid(col, r1)[r0:r1]
    F[:, lay.validity_offset:] = np.packbits(valid, axis=1, bitorder="little")
    return F


def to_rows(cols) -> List[tuple]:
    """-> [(offsets int32[rows + 1], data uint8[bytes])] per batch.  An empty table gives one empty batch."""
    n = cols[0].size if cols else 0
    lay = layout([c.type_id for c in cols])
    sizes = row_sizes(cols)
    strs = [c for c, col in enumerate(cols) if col.type_id == STRING]
    # pair offsets: size_per_row + the lengths of the STRING columns before this one in the row
    pair_off, run = {}, np.full(n, lay.size_per_row, np.int64)
    for c in strs:
        pair_off[c] = run.copy()
        run += _str_lens(cols[c], n)
    if n == 0:
        return [(np.zeros(1, np.int32), np.zeros(0, np.uint8))]
    bounds = build_batches(sizes)
    out = []
    for b0, b1 in zip(bounds[:-1], bounds[1:]):
        offs = np.zeros(b1 - b0 + 1, np.int64)
        np.cumsum(sizes[b0:b1], out=offs[1:])
        data = np.zeros(int(offs[-1]), np.uint8)
        block = max(1, _BLOCK_BYTES // max(lay.size_per_row, 1))
        for r0 in range(b0, b1, block):
            r1 = min(b1, r0 + block)
            F = _fixed_section(cols, lay, r0, r1, pair_off)
            if not strs:
                data.reshape(b1 - b0, lay.fixed_row_size)[r0 - b0:r1 - b0, :lay.size_per_row] = F
            else:
                idx = offs[r0 - b0:r1 - b0, None] + np.arange(lay.size_per_row)
                data[idx] = F
        for c in strs:
            col = cols[c]
            so = np.asarray(col.offsets, dtype=np.int64)
            lens = so[b0 + 1:b1 + 1] - so[b0:b1]
            src = np.ascontiguousarray(col.data).view(np.uint8)[so[b0]:so[b1]]
            # destination of chars byte j of row r: row start + pair offset + (j - first char of the row)
            shift = offs[:-1] + pair_off[c][b0:b1] - (so[b0:b1] - so[b0])
            data[np.repeat(shift, lens) + np.arange(len(src), dtype=np.int64)] = src
        out.append((offs.astype(np.int32), data))
    return out


@dataclass
class FromRows:
    data: list            # per column: values as uint8[n * size] (fixed width), chars uint8[total] (STRING)
    masks: list           # per column: uint32[ceil(n / 32)]
    offsets: list         # per column: int32[n + 1] (STRING) or None
    null_counts: np.ndarray
    char_totals: np.ndarray   # per column: chars of a STRING column, 0 otherwise
    status: int           # STATUS_* bits


def from_rows(data: np.ndarray, offsets: Optional[np.ndarray], n: int, types: Sequence[int]) -> FromRows:
    """Rows -> columns.  offsets=None: fixed-width rows at a stride of fixed_row_size.  STRING values follow the pairs
    stored in each row (chars at row start + pair offset, pair length bytes), whatever order the chars are in."""
    lay = layout(types)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    start = (np.arange(n, dtype=np.int64) * lay.fixed_row_size if offsets is None
             else np.asarray(offsets, dtype=np.int64)[:n])
    nc = len(types)

    def field(st: int, sz: int) -> np.ndarray:
        return data[start[:, None] + (st + np.arange(sz))]

    vbytes = field(lay.validity_offset, (nc + 7) // 8)
    res = FromRows([], [], [], np.zeros(nc, np.int64), np.zeros(nc, np.int64), 0)
    prev_end = np.full(n, lay.size_per_row, np.int64)
    for c, t in enumerate(types):
        valid = ((vbytes[:, c // 8] >> (c % 8)) & 1).astype(bool) if n else np.zeros(0, bool)
        res.masks.append(_pack_mask(valid))
        res.null_counts[c] = n - int(valid.sum())
        if t != STRING:
            res.data.append(field(lay.starts[c], SIZE[t]).reshape(-1))
            res.offsets.append(None)
            continue
        pair = field(lay.starts[c], 8).copy().view(np.uint32).astype(np.int64) if n else np.zeros((0, 2), np.int64)
        so, ln = pair[:, 0], pair[:, 1]
        if np.any(so != prev_end):
            res.status |= STATUS_NON_CANONICAL
        prev_end = so + ln
        cum = np.zeros(n + 1, np.int64)
        np.cumsum(ln, out=cum[1:])
        total = int(cum[-1])
        if total > MAX_BATCH_BYTES:
            res.status |= STATUS_CHARS_OVERFLOW
        res.char_totals[c] = total
        res.offsets.append(cum.astype(np.int32))
        res.data.append(data[np.repeat(start + so - cum[:-1], ln) + np.arange(total, dtype=np.int64)])
    return res
