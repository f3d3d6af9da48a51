"""CPU restatement of Apache Spark's UnsafeRow format -- TEST INFRASTRUCTURE ONLY (tests/, smoke(), bench cpu legs).

PARITY UNPINNED: the reference repository holds no vector of this format (the reference speaks JCUDF rows only,
RowConversion.java:44-117; the plugin adapts them with CudfUnsafeRow).  The format is Apache Spark's, restated from its
published sources (branch-3.5):
  sql/catalyst/src/main/java/org/apache/spark/sql/catalyst/expressions/UnsafeRow.java
      calculateBitSetWidthInBytes: ((numFields + 63) / 64) * 8;  getFieldOffset: base + bitSetWidth + ordinal * 8;
      isNullAt: bit `ordinal` of the bitset SET;  setNullAt also writes 0 into the slot
  .../expressions/codegen/UnsafeRowWriter.java
      write(ordinal, boolean/byte/short/int/float): zero the 8-byte slot, then write the value at its start
      write(ordinal, UTF8String / byte[]): bytes at the cursor, zero-padded to a multiple of 8,
          slot = (relativeOffset << 32) | size  (UnsafeWriter.setOffsetAndSize)
      write(ordinal, Decimal, precision, scale): precision <= 18 -> the unscaled long; else 16 bytes are always reserved
          and zeroed in the variable region, holding BigInteger.toByteArray() (big-endian two's complement, minimal
          length); slot = (offset << 32) | byte count; a NULL keeps the offset with size 0 and sets the null bit
Pinned by the hand-derived known answers in tests/test_oracle_unsafe_row.py.
"""
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import oracle as O

_LONG_DEC = (O.DECIMAL32, O.DECIMAL64)


def bitset_bytes(ncols: int) -> int:
    return ((ncols + 63) // 64) * 8


def _field_bytes(col: O.HCol, r: int) -> bytes:
    sz = O.size_of(col.type_id)
    return np.ascontiguousarray(col.data).view(np.uint8)[r * sz:(r + 1) * sz].tobytes()


def to_unsafe_rows(cols: Sequence[O.HCol]) -> Tuple[np.ndarray, np.ndarray]:
    """-> (int64 offsets[n + 1], uint8 row bytes)."""
    n = cols[0].size if cols else 0
    nf = len(cols)
    bs = bitset_bytes(nf)
    valids = [c.valid() for c in cols]
    out = bytearray()
    offsets = np.zeros(n + 1, dtype=np.int64)
    for r in range(n):
        row = bytearray(bs + 8 * nf)
        for f, c in enumerate(cols):
            slot_at = bs + 8 * f
            valid = bool(valids[f][r])
            if not valid:
                row[f // 64 * 8 + (f % 64) // 8] |= 1 << (f % 8)          # little-endian 64-bit words: byte (f%64)//8, bit f%8
            if c.type_id == O.STRING:
                if valid:
                    s = c.data[c.offsets[r]:c.offsets[r + 1]].tobytes()
                    cursor = len(row)
                    row[slot_at:slot_at + 8] = ((cursor << 32) | len(s)).to_bytes(8, "little")
                    row += s + b"\0" * (-len(s) % 8)
            elif c.type_id == O.DECIMAL128:
                cursor = len(row)
                payload = b""
                if valid:
                    v = int.from_bytes(_field_bytes(c, r), "little", signed=True)
                    payload = v.to_bytes((v if v >= 0 else ~v).bit_length() // 8 + 1, "big", signed=True)   # BigInteger.toByteArray: bitLength() / 8 + 1
                row[slot_at:slot_at + 8] = ((cursor << 32) | len(payload)).to_bytes(8, "little")
                row += payload + b"\0" * (16 - len(payload))
            elif valid:
                b = _field_bytes(c, r)
                if c.type_id in _LONG_DEC:
                    b = int.from_bytes(b, "little", signed=True).to_bytes(8, "little", signed=True)
                row[slot_at:slot_at + len(b)] = b
        assert len(row) % 8 == 0
        out += row
        offsets[r + 1] = len(out)
    return offsets, np.frombuffer(bytes(out), dtype=np.uint8).copy()


def from_unsafe_rows(data: np.ndarray, offsets: np.ndarray, types: Sequence[int]) -> List[O.HCol]:
    n = len(offsets) - 1
    nf = len(types)
    bs = bitset_bytes(nf)
    raw = data.tobytes()
    vals = [[] for _ in types]
    valid = np.ones((nf, n), dtype=bool)
    for r in range(n):
        row = raw[offsets[r]:offsets[r + 1]]
        for f, t in enumerate(types):
            isnull = (row[f // 64 * 8 + (f % 64) // 8] >> (f % 8)) & 1
            valid[f, r] = not isnull
            slot = int.from_bytes(row[bs + 8 * f: bs + 8 * f + 8], "little")
            if t == O.STRING:
                vals[f].append(b"" if isnull else row[slot >> 32:(slot >> 32) + (slot & 0xffffffff)])
            elif t == O.DECIMAL128:
                v = 0 if isnull else int.from_bytes(row[slot >> 32:(slot >> 32) + (slot & 0xffffffff)], "big", signed=True)
                vals[f].append(v.to_bytes(16, "little", signed=True))
            else:
                vals[f].append(row[bs + 8 * f: bs + 8 * f + O.size_of(t)])
    cols = []
    for f, t in enumerate(types):
        mask = None if valid[f].all() else O.pack_mask(valid[f])
        if t == O.STRING:
            offs = np.zeros(n + 1, dtype=np.int32)
            np.cumsum([len(v) for v in vals[f]], out=offs[1:])
            cols.append(O.HCol(O.STRING, np.frombuffer(b"".join(vals[f]), dtype=np.uint8).copy(), mask, offs, 0, n))
        else:
            cols.append(O.HCol(t, np.frombuffer(b"".join(vals[f]), dtype=np.uint8).copy(), mask, None, 0, n))
    return cols


def to_unsafe_rows_fixed(cols: Sequence[O.HCol]) -> np.ndarray:
    """Vectorised numpy form of to_unsafe_rows for tables of fixed-width columns (no STRING, no DECIMAL128): all rows have
    bitset + 8 * fields bytes.  -> uint8[n, row bytes].  (bench.py times it as the single-core CPU baseline.)"""
    n = cols[0].size if cols else 0
    nf = len(cols)
    bs = bitset_bytes(nf)
    rows = np.zeros((n, bs + 8 * nf), dtype=np.uint8)
    for f, c in enumerate(cols):
        assert c.type_id not in (O.STRING, O.DECIMAL128)
        valid = c.valid()
        rows[:, f // 64 * 8 + (f % 64) // 8] |= (~valid).astype(np.uint8) << (f % 8)
        sz = O.size_of(c.type_id)
        v = np.ascontiguousarray(c.data).view(np.uint8).reshape(n, sz)
        if c.type_id in _LONG_DEC and sz == 4:
            v = np.ascontiguousarray(c.data).view(np.int32).astype(np.int64).view(np.uint8).reshape(n, 8)
            sz = 8
        at = bs + 8 * f
        rows[:, at:at + sz] = np.where(valid[:, None], v, 0)
    return rows
