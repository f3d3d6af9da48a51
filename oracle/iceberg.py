"""Iceberg's bucket, truncate and year / month / day / hour transforms, restated in numpy (vectorised over rows).

Reference lines (src/main/cpp/src/ of the reference unless noted):
  - bucket: iceberg/iceberg_bucket.cu:59-209 (the hash), 216-374 (per type), 388-457 (dispatch).  h = standard
    MurmurHash3_x86_32 (seed 0) of the value's bytes; result (h & INT32_MAX) % numBuckets, 0 under a null row.  INT32 /
    TIMESTAMP_DAYS are widened to int64 (hash_int, :86-90), INT64 / TIMESTAMP_MICROSECONDS hashed as 8 little-endian
    bytes (:75-79), decimals as their unscaled value's minimal big-endian two's complement (:132-208), STRING / binary as
    their bytes.
  - truncate: iceberg/iceberg_truncate.cu:52-66 (integral: v - (((v % W) + W) % W) in the storage type), :71-101
    (STRING: the first W characters; here the bytes before the (W+1)-th byte that is not 10xxxxxx, which is what cudf's
    string_view::substr gives for valid UTF-8), :103-127 (binary: min(len, W) bytes).  A null row holds 0 / no bytes.
  - year / month / day / hour: iceberg/iceberg_datetime_util.cu:48-135: floor division of microseconds by 86 400 000 000
    or 3 600 000 000 (hours cast to int32), proleptic Gregorian civil date of a day count (datetime_utils.cuh:81-94).
    Rows under nulls are computed like the others.
Columns are host numpy arrays: data = the raw little-endian bytes (uint8) or any numpy array viewed as such, mask = cudf
bitmask words (uint32) or None, offsets = int32[rows + 1] for STRING / LIST<UINT8>.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

INT32, INT64, TIMESTAMP_DAYS, TIMESTAMP_MICROSECONDS, STRING, LIST, DECIMAL32, DECIMAL64, DECIMAL128 = 3, 4, 12, 15, 23, 24, 25, 26, 27
INT32_MAX = 2**31 - 1
MICROS_PER_DAY = 86_400_000_000
MICROS_PER_HOUR = 3_600_000_000

_C1, _C2 = np.uint32(0xCC9E2D51), np.uint32(0x1B873593)


def valid_rows(mask: Optional[np.ndarray], rows: int) -> np.ndarray:
    if mask is None:
        return np.ones(rows, dtype=bool)
    return np.unpackbits(np.ascontiguousarray(mask).view(np.uint8), bitorder="little")[:rows].astype(bool)


def _rotl(x, r):
    return (x << np.uint32(r)) | (x >> np.uint32(32 - r))


def _scramble(k):
    return _rotl(k * _C1, 15) * _C2


def murmur3_rows(b: np.ndarray) -> np.ndarray:
    """Standard MurmurHash3_x86_32, seed 0, of each row of a uint8 matrix [rows, L] (every row L bytes) -> uint32[rows]."""
    rows, L = b.shape
    with np.errstate(over="ignore"):
        h = np.zeros(rows, dtype=np.uint32)
        nb = L // 4
        if nb:
            words = np.ascontiguousarray(b[:, : 4 * nb]).view("<u4").reshape(rows, nb)
            for i in range(nb):
                h ^= _scramble(words[:, i])
                h = _rotl(h, 13) * np.uint32(5) + np.uint32(0xE6546B64)
        if L & 3:
            k = np.zeros(rows, dtype=np.uint32)
            for j in range(L & 3):
                k |= b[:, 4 * nb + j].astype(np.uint32) << np.uint32(8 * j)
            h ^= _scramble(k)
        h ^= np.uint32(L)
        h ^= h >> np.uint32(16)
        h *= np.uint32(0x85EBCA6B)
        h ^= h >> np.uint32(13)
        h *= np.uint32(0xC2B2AE35)
        h ^= h >> np.uint32(16)
    return h


def _bucket_of(h: np.ndarray, n: int) -> np.ndarray:
    return ((h & np.uint32(INT32_MAX)).astype(np.int64) % n).astype(np.int32)


def _hash_var(chars: np.ndarray, starts: np.ndarray, lens: np.ndarray) -> np.ndarray:
    """murmur3 of chars[starts[i] : starts[i] + lens[i]], grouped by length"""
    out = np.zeros(len(starts), dtype=np.uint32)
    for L in np.unique(lens):
        sel = np.nonzero(lens == L)[0]
        L = int(L)
        idx = starts[sel][:, None] + np.arange(L, dtype=np.int64)[None, :]
        out[sel] = murmur3_rows(chars[idx] if L else np.zeros((len(sel), 0), np.uint8))
    return out


def decimal_java_bytes(v: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """BigInteger.toByteArray() of int64 or (lo, hi) int128 values: (big-endian bytes [rows, 16] right-aligned, lengths)"""
    if v.ndim == 1:                                                  # int32 / int64 unscaled values
        v64 = v.astype(np.int64)
        lo = v64.view(np.uint64)
        hi = (v64 >> 63).view(np.uint64)
    else:
        lo, hi = v[:, 0].view(np.uint64), v[:, 1].view(np.uint64)
    sign = (hi.view(np.int64) >> 63).view(np.uint64)
    xh, xl = hi ^ sign, lo ^ sign
    bits = np.zeros(len(lo), dtype=np.int64)
    for i in range(64):
        bits = np.where((xh >> np.uint64(i)) & np.uint64(1), 65 + i, bits)
    low_bits = np.zeros(len(lo), dtype=np.int64)
    for i in range(64):
        low_bits = np.where((xl >> np.uint64(i)) & np.uint64(1), 1 + i, low_bits)
    bits = np.where(xh != 0, bits, low_bits)                         # significant bits, sign bit excluded
    n = bits // 8 + 1
    le = np.stack([lo, hi], axis=1).copy().view(np.uint8).reshape(-1, 16)
    return le[:, ::-1].copy(), n                                      # big-endian 16 bytes


def bucket(type_id: int, data: Optional[np.ndarray], mask: Optional[np.ndarray], rows: int, num_buckets: int,
           offsets: Optional[np.ndarray] = None) -> np.ndarray:
    """int32[rows] bucket ids (0 under nulls)"""
    valid = valid_rows(mask, rows)
    out = np.zeros(rows, dtype=np.int32)
    if rows == 0:
        return out
    raw = np.ascontiguousarray(data).view(np.uint8) if data is not None else np.zeros(0, np.uint8)
    if type_id in (INT32, TIMESTAMP_DAYS, INT64, TIMESTAMP_MICROSECONDS):
        v = raw.view("<i4" if type_id in (INT32, TIMESTAMP_DAYS) else "<i8")[:rows].astype(np.int64)
        h = murmur3_rows(v.view(np.uint8).reshape(rows, 8))
    elif type_id in (DECIMAL32, DECIMAL64, DECIMAL128):
        v = {DECIMAL32: lambda: raw.view("<i4")[:rows], DECIMAL64: lambda: raw.view("<i8")[:rows],
             DECIMAL128: lambda: raw.view("<i8")[: 2 * rows].reshape(rows, 2)}[type_id]()
        be, n = decimal_java_bytes(v)
        flat = be.reshape(-1)
        h = _hash_var(flat, np.arange(rows, dtype=np.int64) * 16 + (16 - n), n)
    elif type_id in (STRING, LIST):
        off = np.asarray(offsets, dtype=np.int64)
        h = _hash_var(raw, off[:-1], off[1:] - off[:-1])
    else:
        raise ValueError(f"unsupported type {type_id}")
    out[valid] = _bucket_of(h[valid], num_buckets)
    return out


def _wrap(x, bits):
    m = 1 << bits
    return ((x + (m >> 1)) % m) - (m >> 1)


def truncate_integral(type_id: int, data: np.ndarray, mask: Optional[np.ndarray], rows: int, width: int) -> np.ndarray:
    """the output's raw bytes (uint8); v - (((v % W) + W) % W) with C's truncated % and wrapping + / -, 0 under nulls"""
    valid = valid_rows(mask, rows)
    raw = np.ascontiguousarray(data).view(np.uint8)
    if type_id in (INT32, DECIMAL32):
        v = raw.view("<i4")[:rows].astype(np.int64)
        r1 = np.fmod(v, width)                                        # exact in int64: |v| <= 2^31
        s = _wrap(r1 + width, 32)
        out = _wrap(v - np.fmod(s, width), 32).astype("<i4")
    elif type_id in (INT64, DECIMAL64):
        v = raw.view("<i8")[:rows]
        u = v.view(np.uint64)
        d = np.uint64(abs(width))
        w = np.uint64(width % 2**64)
        with np.errstate(over="ignore"):
            neg = v < 0
            ra = np.where(neg, np.uint64(0) - u, u) % d
            s = np.where(neg, np.uint64(0) - ra, ra) + w              # (v % W) + W, wrapping
            sneg = s.view(np.int64) < 0
            sa = np.where(sneg, np.uint64(0) - s, s) % d
            r2 = np.where(sneg, np.uint64(0) - sa, sa)
            out = (u - r2).view("<i8")
    else:                                                             # DECIMAL128 in Python integers
        lo = raw.view("<u8")[0: 2 * rows: 2]
        hi = raw.view("<i8")[1: 2 * rows: 2]
        res = np.zeros((rows, 2), dtype="<u8")
        for i in range(rows):
            x = (int(hi[i]) << 64) | int(lo[i])
            r1 = _c_rem(x, width)
            s = _wrap(r1 + width, 128)
            y = _wrap(x - _c_rem(s, width), 128) % 2**128
            res[i] = (y & (2**64 - 1), y >> 64)
        out = res
    out = np.ascontiguousarray(out).view(np.uint8).reshape(rows, -1).copy() if rows else np.zeros((0, 1), np.uint8)
    out[~valid] = 0
    return out.reshape(-1)


def _c_rem(x: int, w: int) -> int:
    r = abs(x) % abs(w)
    return -r if x < 0 else r


def truncate_bytes(type_id: int, chars: np.ndarray, offsets: np.ndarray, mask: Optional[np.ndarray], rows: int,
                   width: int) -> Tuple[np.ndarray, np.ndarray]:
    """(offsets int32[rows + 1], bytes uint8) of a truncated STRING / LIST<UINT8> column; null rows have zero length"""
    valid = valid_rows(mask, rows)
    off = np.asarray(offsets, dtype=np.int64)
    chars = np.ascontiguousarray(chars).view(np.uint8) if chars is not None else np.zeros(0, np.uint8)
    b, e = off[:-1], off[1:]
    lens = e - b
    if type_id == STRING:
        starts = (chars & 0xC0) != 0x80
        C = np.concatenate([[0], np.cumsum(starts, dtype=np.int64)])  # C[i] = character starts in chars[0:i]
        p = np.searchsorted(C, C[b] + width + 1, side="left") - 1     # the (width+1)-th start of the row, if inside it
        size = np.where(p < e, p - b, lens)
    else:
        size = np.minimum(lens, width)
    size = np.where(valid, size, 0)
    out_off = np.concatenate([[0], np.cumsum(size)]).astype(np.int32)
    total = int(out_off[-1])
    idx = np.repeat(b - out_off[:-1].astype(np.int64), size) + np.arange(total, dtype=np.int64)
    return out_off, chars[idx]


def _civil(days: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """proleptic Gregorian (year, month) of int64 day counts from 1970-01-01"""
    z = days + 719468
    era = np.floor_divide(z, 146097)
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    month = np.where(mp < 10, mp + 3, mp - 9)
    year = yoe + era * 400 + (month <= 2)
    return year, month


def datetime_transform(transform: str, type_id: int, data: np.ndarray, rows: int) -> np.ndarray:
    """int32[rows]: transform in years / months / days / hours; rows under nulls are computed from their bits"""
    raw = np.ascontiguousarray(data).view(np.uint8)
    if type_id == TIMESTAMP_DAYS:
        if transform == "hours":
            raise ValueError("hours needs TIMESTAMP_MICROSECONDS")
        days = raw.view("<i4")[:rows].astype(np.int64)
    else:
        t = raw.view("<i8")[:rows]
        if transform == "hours":
            return _wrap(np.floor_divide(t, MICROS_PER_HOUR), 32).astype(np.int32)
        days = np.floor_divide(t, MICROS_PER_DAY)
    if transform == "days":
        return days.astype(np.int32)
    year, month = _civil(days)
    if transform == "years":
        return (year - 1970).astype(np.int32)
    return ((year - 1970) * 12 + month - 1).astype(np.int32)
