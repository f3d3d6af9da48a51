"""Arithmetic.multiply and Arithmetic.round, restated in numpy.

Reference lines (src/main/cpp/src/ of the reference, and thirdparty/cudf/cpp/src/round/round.cu):
  - multiply: multiply.cu:38-131.  An integer row overflows when its exact product is outside the type: it wraps by
    default, is null in try mode, and in ANSI mode the smallest such row with both operands valid is the error row.
    Floats are IEEE products.  A null operand (a null scalar: every row) gives a null row; a null row holds 0.
  - round: round_float.cu:45-176, 306-341 and round.cu:77-298.  Floats: n = T(pow(10, |dp|)); dp == 0 round / rint;
    dp > 0 modf, then int_part + round(frac * n) / n; dp < 0 round(e / n) * n; every operation rounded to nearest in T.
    Integers: dp >= 0 copies; dp < 0 rounds to a multiple of 10^-dp (HALF_UP away from zero, HALF_EVEN to the even
    multiple), the exact result wrapped to the type; in ANSI mode the smallest valid row whose exact result is outside
    the type is the error row.  Decimals (storage integers; ANSI ignored): output scale -dp; the same scale copies; a
    larger input scale multiplies by 10^k wrapping; a scale movement above 9 / 18 / 38 digits gives zeros; else the
    storage integer is rounded and divided by 10^k exactly.  Values under null rows are computed from their bits.

Columns are host numpy arrays; `valid` is a bool array or None (all valid).  DECIMAL128 storage is an (n, 2) uint64
array of little-endian halves.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import numpy as np

HALF_UP, HALF_EVEN = 0, 1
_INTS = (np.int8, np.int16, np.int32, np.int64)


def _valid(valid, n: int) -> np.ndarray:
    return np.ones(n, bool) if valid is None else np.asarray(valid, bool).copy()


def _mul_overflow(a: np.ndarray, b: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(a * b wrapped, exact product outside the type)."""
    t = a.dtype.type
    if t in (np.int8, np.int16, np.int32):
        p = a.astype(np.int64) * b.astype(np.int64)
        info = np.iinfo(t)
        return p.astype(t), (p < info.min) | (p > info.max)
    with np.errstate(over="ignore"):
        p = (a.view(np.uint64) * b.view(np.uint64)).view(np.int64)
    lo = np.iinfo(np.int64).min
    special = ((a == -1) & (b == lo)) | ((b == -1) & (a == lo))
    d = np.where((a == 0) | special, 1, a)
    # no overflow: p is the exact product and p / a is b with no remainder; an overflow leaves p off by k * 2^64, k != 0
    ovf = (a != 0) & ~special & ((np.floor_divide(p, d) != b) | (np.remainder(p, d) != 0))
    return p, ovf | special


def multiply(a: np.ndarray, a_valid, b: np.ndarray, b_valid, ansi: bool, try_mode: bool,
             a_scalar: bool = False, b_scalar: bool = False) -> Tuple[np.ndarray, np.ndarray, int]:
    """-> (values, valid, error_row (-1 when none)).  A scalar operand is a one-element array, its validity a bool."""
    n = len(b) if a_scalar else len(a)
    a = np.broadcast_to(a, (n,)) if a_scalar else np.asarray(a)
    b = np.broadcast_to(b, (n,)) if b_scalar else np.asarray(b)
    va = np.full(n, bool(a_valid)) if a_scalar else _valid(a_valid, n)
    vb = np.full(n, bool(b_valid)) if b_scalar else _valid(b_valid, n)
    valid = va & vb
    if a.dtype.kind == "f":
        with np.errstate(all="ignore"):
            out = a * b
        ovf = np.zeros(n, bool)
    else:
        out, ovf = _mul_overflow(a, b)
    err = -1
    if ansi or try_mode:
        bad = ovf & valid
        if ansi and bad.any():
            err = int(np.argmax(bad))
        valid &= ~bad
    out = np.where(valid, out, out.dtype.type(0))
    return out, valid, err


# ---- round ------------------------------------------------------------------------------------------------------------
def _round_half_up(x: np.ndarray) -> np.ndarray:
    """C's round(): halves away from zero (x - trunc(x) is exact)."""
    t = np.trunc(x)
    return np.where(np.abs(x - t) >= 0.5, t + np.copysign(x.dtype.type(1), x), t).astype(x.dtype)


def _round_half(x: np.ndarray, mode: int) -> np.ndarray:
    return np.rint(x) if mode == HALF_EVEN else _round_half_up(x)


def pow10(k: int) -> float:
    """The C library's pow(10, k) in double, inf past the double range: the reference computes n = std::pow(10, |dp|) on
    the host.  That is not always the double nearest 10^k (glibc gives 10^23 one ulp high), and numpy's power need not
    agree with it (on some CPUs it differs at 10^301), so the oracle calls the same pow."""
    try:
        return math.pow(10.0, k)
    except OverflowError:
        return math.inf


def round_float(e: np.ndarray, dp: int, mode: int) -> np.ndarray:
    t = e.dtype.type
    with np.errstate(all="ignore"):
        n = t(pow10(abs(int(dp))))
        if dp == 0:
            return _round_half(e, mode)
        if dp > 0:
            frac, ip = np.modf(e)
            return (ip + _round_half(frac * n, mode) / n).astype(t)
        return (_round_half(e / n, mode) * n).astype(t)


def _round_mag(x: np.ndarray, d: int, mode: int) -> np.ndarray:
    """round(x / d) for uint64 magnitudes x, half up or half even."""
    d = np.uint64(d)
    q, r = x // d, x % d
    h = d - r
    bump = (r > h) | ((r == h) & ((mode == HALF_UP) | ((q & np.uint64(1)) == 1)))
    return q + bump.astype(np.uint64)


def _split(v: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(v < 0, |v| as uint64)."""
    neg = v < 0
    u = v.astype(np.int64).view(np.uint64)
    return neg, np.where(neg, np.uint64(0) - u, u)


def round_int(v: np.ndarray, valid, dp: int, mode: int, ansi: bool) -> Tuple[np.ndarray, int]:
    """-> (values, error_row)."""
    t = v.dtype.type
    if dp >= 0:
        return v.copy(), -1
    k = -int(dp)
    neg, x = _split(v)
    if k >= 20:                                        # 10^k > 2^64: every value rounds to 0
        return np.zeros_like(v), -1
    d = 10 ** k
    with np.errstate(over="ignore"):
        mag = _round_mag(x, d, mode) * np.uint64(d)    # exact: below 2^64
        wrapped = np.where(neg, np.uint64(0) - mag, mag).view(np.int64).astype(t)
    info = np.iinfo(t)
    ovf = np.where(neg, mag > np.uint64(-info.min), mag > np.uint64(info.max)) & _valid(valid, len(v))
    return wrapped, (int(np.argmax(ovf)) if ansi and ovf.any() else -1)


def _digits(t) -> int:
    return {np.int32: 9, np.int64: 18}[t]


def round_decimal(v: np.ndarray, scale: int, dp: int, mode: int) -> np.ndarray:
    """DECIMAL32 / DECIMAL64 storage (int32 / int64) at `scale` -> storage at scale -dp."""
    t = v.dtype.type
    k = -int(dp) - int(scale)
    bits = 8 * v.dtype.itemsize
    if k == 0:
        return v.copy()
    if k < 0:
        p = pow(10, -k, 1 << bits)
        with np.errstate(over="ignore"):
            return (v.astype(np.int64).view(np.uint64) * np.uint64(p)).view(np.int64).astype(t)
    if k > _digits(t):
        return np.zeros_like(v)
    neg, x = _split(v)
    q = _round_mag(x, 10 ** k, mode)
    with np.errstate(over="ignore"):
        return np.where(neg, np.uint64(0) - q, q).view(np.int64).astype(t)


def dec128_to_ints(a: np.ndarray) -> list:
    a = np.asarray(a, np.uint64).reshape(-1, 2)
    out = []
    for lo, hi in a.tolist():
        u = (hi << 64) | lo
        out.append(u - (1 << 128) if u >> 127 else u)
    return out


def ints_to_dec128(vals) -> np.ndarray:
    out = np.empty((len(vals), 2), np.uint64)
    for i, v in enumerate(vals):
        u = v % (1 << 128)
        out[i] = (u & ((1 << 64) - 1), u >> 64)
    return out


def round_decimal128(a: np.ndarray, scale: int, dp: int, mode: int) -> np.ndarray:
    """DECIMAL128 storage ((n, 2) uint64) at `scale` -> storage at scale -dp."""
    k = -int(dp) - int(scale)
    vals = dec128_to_ints(a)
    if k == 0:
        res = vals
    elif k < 0:
        p = pow(10, -k, 1 << 128)
        res = [v * p for v in vals]
    elif k > 38:
        res = [0] * len(vals)
    else:
        d = 10 ** k
        res = []
        for v in vals:
            q, r = divmod(abs(v), d)
            if r > d - r or (r == d - r and (mode == HALF_UP or q & 1)):
                q += 1
            res.append(-q if v < 0 else q)
    return ints_to_dec128(res)


def round_(v: np.ndarray, valid, dp: int, mode: int, ansi: bool, type_id: Optional[int] = None,
           scale: int = 0) -> Tuple[np.ndarray, int]:
    """round of any supported column: type_id 25 / 26 / 27 marks DECIMAL32 / 64 / 128 storage.  -> (values, error_row)."""
    if type_id in (25, 26):
        return round_decimal(v, scale, dp, mode), -1
    if type_id == 27:
        return round_decimal128(v, scale, dp, mode), -1
    if v.dtype.kind == "f":
        return round_float(v, dp, mode), -1
    return round_int(v, valid, dp, mode, ansi)
