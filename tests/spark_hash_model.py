"""An independent model of Spark's row hashes (xxhash64, Murmur3_x86_32, HiveHash), one row at a time in plain Python
integers.

It is written from the Spark / Hive definitions rather than from the CUDA kernels or the C oracle, and imports neither:
XXH64 comes from the `xxhash` package, Murmur3 and the Hive fold are spelled out below.  Columns are read through the
attributes every host column of the test suite has (type_id, data, mask, offsets, size, children), as raw bytes.

Element rules (Spark's HashExpression, with the GPU plugin's choices where Spark leaves room):
  BOOL8 -> int 1 if the byte is nonzero else 0; INT8 / INT16 sign-extended, UINT8 / UINT16 zero-extended, to an int;
  4-byte integers and dates -> int; 8-byte integers, timestamps, durations, DECIMAL64 -> long; DECIMAL32 -> long of
  its value; DECIMAL128 -> the bytes of BigInteger.toByteArray() of the unscaled value; STRING -> its UTF-8 bytes.
  Floats: every NaN becomes the canonical quiet NaN; xxhash64 also folds -0.0 into 0.0, murmur3 and hive do not.
Row rules: xxhash64 / murmur3 chain the elements left to right with the running hash as the next seed, and a null
element leaves the hash unchanged; hive folds h = 31 * h + x with x = 0 for a null.
"""
from __future__ import annotations

import numpy as np
import xxhash

# cudf type ids
(INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8, TIMESTAMP_DAYS, TIMESTAMP_SECONDS,
 TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS, TIMESTAMP_NANOSECONDS, DURATION_DAYS, DURATION_SECONDS,
 DURATION_MILLISECONDS, DURATION_MICROSECONDS, DURATION_NANOSECONDS) = range(1, 22)
STRING, LIST, DECIMAL32, DECIMAL64, DECIMAL128, STRUCT = 23, 24, 25, 26, 27, 28

M32, M64 = (1 << 32) - 1, (1 << 64) - 1

_SIZE = {INT8: 1, UINT8: 1, BOOL8: 1, INT16: 2, UINT16: 2, DECIMAL128: 16}
_SIZE.update({t: 4 for t in (INT32, UINT32, FLOAT32, TIMESTAMP_DAYS, DURATION_DAYS, DECIMAL32)})
_SIZE.update({t: 8 for t in (INT64, UINT64, FLOAT64, TIMESTAMP_SECONDS, TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS,
                             TIMESTAMP_NANOSECONDS, DURATION_SECONDS, DURATION_MILLISECONDS, DURATION_MICROSECONDS,
                             DURATION_NANOSECONDS, DECIMAL64)})
_SIGNED = {INT8, INT16, INT32, INT64, DECIMAL32, DECIMAL64, DECIMAL128, TIMESTAMP_DAYS, TIMESTAMP_SECONDS,
           TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS, TIMESTAMP_NANOSECONDS, DURATION_DAYS, DURATION_SECONDS,
           DURATION_MILLISECONDS, DURATION_MICROSECONDS, DURATION_NANOSECONDS}
HIVE_TYPES = {BOOL8, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, TIMESTAMP_DAYS, TIMESTAMP_MICROSECONDS, STRING}


# ---------------------------------------------------------------- Murmur3_x86_32 (org.apache.spark.unsafe.hash)
def _rotl32(x: int, r: int) -> int:
    return ((x << r) | (x >> (32 - r))) & M32


def _mix_k1(k1: int) -> int:
    k1 = (k1 * 0xCC9E2D51) & M32
    return (_rotl32(k1, 15) * 0x1B873593) & M32


def _mix_h1(h1: int, k1: int) -> int:
    return (_rotl32(h1 ^ k1, 13) * 5 + 0xE6546B64) & M32


def _fmix(h1: int, length: int) -> int:
    h1 ^= length
    h1 ^= h1 >> 16
    h1 = (h1 * 0x85EBCA6B) & M32
    h1 ^= h1 >> 13
    h1 = (h1 * 0xC2B2AE35) & M32
    return h1 ^ (h1 >> 16)


def murmur_int(v: int, seed: int) -> int:
    """Murmur3_x86_32.hashInt"""
    return _fmix(_mix_h1(seed & M32, _mix_k1(v & M32)), 4)


def murmur_long(v: int, seed: int) -> int:
    """Murmur3_x86_32.hashLong: the low word, then the high word"""
    v &= M64
    h1 = _mix_h1(seed & M32, _mix_k1(v & M32))
    return _fmix(_mix_h1(h1, _mix_k1(v >> 32)), 8)


def murmur_bytes(b: bytes, seed: int) -> int:
    """Murmur3_x86_32.hashUnsafeBytes: whole little-endian words, then every tail byte on its own, sign-extended"""
    h1 = seed & M32
    n4 = len(b) // 4 * 4
    for i in range(0, n4, 4):
        h1 = _mix_h1(h1, _mix_k1(int.from_bytes(b[i:i + 4], "little")))
    for x in b[n4:]:
        h1 = _mix_h1(h1, _mix_k1((x - 256 if x >= 128 else x) & M32))
    return _fmix(h1, len(b))


# ---------------------------------------------------------------- XXH64 (the xxhash package)
def xx_bytes(b: bytes, seed: int) -> int:
    return xxhash.xxh64_intdigest(b, seed=seed & M64)


def xx_int(v: int, seed: int) -> int:
    return xx_bytes((v & M32).to_bytes(4, "little"), seed)


def xx_long(v: int, seed: int) -> int:
    return xx_bytes((v & M64).to_bytes(8, "little"), seed)


# ---------------------------------------------------------------- element decoding
def java_big_integer_bytes(v: int) -> bytes:
    """BigInteger.toByteArray(): minimal big-endian two's complement, bitLength() / 8 + 1 bytes.  Java's bitLength of
    a negative value is that of its complement (-128 -> 7 bits -> one byte 0x80), not of its magnitude."""
    bit_length = v.bit_length() if v >= 0 else (~v).bit_length()
    return v.to_bytes(bit_length // 8 + 1, "big", signed=True)


def _valid(col, i: int) -> bool:
    m = col.mask
    if m is None:
        return True
    w = np.asarray(m).view(np.uint32)
    return bool((int(w[i >> 5]) >> (i & 31)) & 1)


def _raw(col, i: int) -> int:
    sz = _SIZE[col.type_id]
    b = np.ascontiguousarray(col.data).view(np.uint8)[i * sz:(i + 1) * sz].tobytes()
    return int.from_bytes(b, "little", signed=col.type_id in _SIGNED)


def _str(col, i: int) -> bytes:
    o = col.offsets
    return np.ascontiguousarray(col.data).view(np.uint8)[int(o[i]):int(o[i + 1])].tobytes()


def _f32(bits: int, fold_zero: bool) -> int:
    if (bits & 0x7F800000) == 0x7F800000 and (bits & 0x007FFFFF):
        return 0x7FC00000                        # Float.NaN
    if fold_zero and bits == 0x80000000:
        return 0
    return bits


def _f64(bits: int, fold_zero: bool) -> int:
    if (bits & 0x7FF0000000000000) == 0x7FF0000000000000 and (bits & 0x000FFFFFFFFFFFFF):
        return 0x7FF8000000000000                # Double.NaN
    if fold_zero and bits == 0x8000000000000000:
        return 0
    return bits


def _element(col, i: int, fold_zero: bool):
    """-> ("int", v) | ("long", v) | ("bytes", b): what Spark hands to hashInt / hashLong / hashUnsafeBytes."""
    t = col.type_id
    if t == STRING:
        return "bytes", _str(col, i)
    v = _raw(col, i)
    if t == BOOL8:
        return "int", int(v != 0)
    if t in (INT8, INT16, UINT8, UINT16, INT32, UINT32, TIMESTAMP_DAYS, DURATION_DAYS):
        return "int", v
    if t == FLOAT32:
        return "int", _f32(v, fold_zero)
    if t == FLOAT64:
        return "long", _f64(v, fold_zero)
    if t == DECIMAL128:
        return "bytes", java_big_integer_bytes(v)
    if t in _SIZE:                               # DECIMAL32 (as a long), DECIMAL64, 8-byte integers / times
        return "long", v
    raise NotImplementedError(f"type id {t}")


def _hash_element(kind: str, col, i: int, h: int) -> int:
    form, v = _element(col, i, fold_zero=(kind == "xxhash64"))
    if kind == "xxhash64":
        return {"int": xx_int, "long": xx_long, "bytes": xx_bytes}[form](v, h)
    return {"int": murmur_int, "long": murmur_long, "bytes": murmur_bytes}[form](v, h)


def _hive_long(v: int) -> int:
    v &= M64
    return ((v >> 32) ^ v) & M32


def hive_element(col, i: int) -> int:
    """HiveHash of one non-null leaf value, as an unsigned 32-bit int."""
    t = col.type_id
    if t == STRING:
        h = 0
        for x in _str(col, i):
            h = (31 * h + (x - 256 if x >= 128 else x)) & M32
        return h
    if t not in HIVE_TYPES:
        raise NotImplementedError(f"hive: type id {t}")
    v = _raw(col, i)
    if t == BOOL8:
        return int(v != 0)
    if t in (INT8, INT16, INT32, TIMESTAMP_DAYS):
        return v & M32
    if t == INT64:
        return _hive_long(v)
    if t == FLOAT32:
        return _f32(v & M32, False)
    if t == FLOAT64:
        return _hive_long(_f64(v & M64, False))
    # TIMESTAMP_MICROSECONDS: seconds and nanoseconds with Java's truncating / and %, packed as (s << 30) | ns
    ts = abs(v) // 1_000_000 * (1 if v >= 0 else -1)
    tns = (v - ts * 1_000_000) * 1000
    return _hive_long((ts << 30) | tns)


# ---------------------------------------------------------------- rows, nesting
def _chain(kind: str, col, lo: int, hi: int, h: int) -> int:
    """xxhash64 / murmur3: every leaf value under elements [lo, hi) of col, depth first, chained into h.

    xxhash64 does not look at LIST or STRUCT level nulls: a null list still contributes the elements its offsets
    select, a null struct its fields.  murmur3 skips a null LIST or STRUCT element with everything under it (Spark's
    Murmur3Hash of a null struct or array is the seed)."""
    t = col.type_id
    if t == LIST:
        o = col.offsets
        if kind == "xxhash64":
            return _chain(kind, col.children[0], int(o[lo]), int(o[hi]), h)
        for i in range(lo, hi):
            if _valid(col, i):
                h = _chain(kind, col.children[0], int(o[i]), int(o[i + 1]), h)
        return h
    if t == STRUCT:
        for i in range(lo, hi):
            if kind == "xxhash64" or _valid(col, i):
                for f in col.children:
                    h = _chain(kind, f, i, i + 1, h)
        return h
    for i in range(lo, hi):
        if _valid(col, i):
            h = _hash_element(kind, col, i, h)
    return h


def _hive(col, i: int) -> int:
    """hive: a struct folds its fields, a list its elements; LIST / STRUCT level nulls are not looked at."""
    t = col.type_id
    if t == LIST:
        h = 0
        for e in range(int(col.offsets[i]), int(col.offsets[i + 1])):
            h = (31 * h + _hive(col.children[0], e)) & M32
        return h
    if t == STRUCT:
        h = 0
        for f in col.children:
            h = (31 * h + _hive(f, i)) & M32
        return h
    return hive_element(col, i) if _valid(col, i) else 0


def row_hash(kind: str, cols, row: int, seed: int = 0) -> int:
    """kind in {"xxhash64", "murmur3", "hive"}; the hash of one row as a signed int (int64 / int32)."""
    if kind == "hive":
        h = 0
        for c in cols:
            h = (31 * h + _hive(c, row)) & M32
        return h - (1 << 32) if h >> 31 else h
    h = seed & (M64 if kind == "xxhash64" else M32)
    for c in cols:
        h = _chain(kind, c, row, row + 1, h)
    bits = 64 if kind == "xxhash64" else 32
    return h - (1 << bits) if h >> (bits - 1) else h


def hash_rows(kind: str, cols, seed: int = 0, rows=None) -> np.ndarray:
    """The hashes of `rows` (default: every row) as int64 (xxhash64) or int32."""
    n = cols[0].size if cols else 0
    rows = range(n) if rows is None else rows
    dt = np.int64 if kind == "xxhash64" else np.int32
    return np.array([row_hash(kind, cols, int(r), seed) for r in rows], dtype=dt)


def pmod(h: int, n: int) -> int:
    """Spark's Pmod on an int: ((h % n) + n) % n with Java's truncating %."""
    r = abs(h) % n * (1 if h >= 0 else -1)
    return (r + n) % n
