"""DecimalUtils.floatingPointToDecimal restated step by step in Python integers (TEST INFRASTRUCTURE), with a ctypes
front-end of its C twin, oracle/float_to_decimal.c, which the GPU tests use for sweeps of 2^32 rows.

    vals, valid, failure_row = floating_point_to_decimal(values, valid, out_type, precision, scale)
    out, valid, failure_row = floating_point_to_decimal_c(values, mask_words, out_type, precision, scale)

Scales are cudf scales (the value is unscaled * 10^scale).
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np

from .decimal import M128, to_ints  # noqa: F401  (to_ints: DECIMAL128 output bytes -> Python ints, for callers)

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "float_to_decimal.c")
_SO = os.path.join(_HERE, "libf2d_oracle.so")
_lib = None


# decimal_utils.cu:1174-1417 (scaled_round :1193-1309, floating_point_to_decimal_fn :1311-1336, the bound :1372-1373,
# the mask :1412-1414) over cudf's fixed_point/detail/floating_conversion.hpp (FC below) and fixed_point.hpp:78-97
# (ipow).  The reference instantiates the shifting with FloatingType = double, so its constants are the double ones
# (FC:537-600): 128-bit shifting rep, 4 buffer bits, 18 digits / 60 bits per step.  Every value is a Python integer
# masked to the width of the C++ type that holds it at that step, so that the reference's wraps are kept.

F2D_DECIMAL32, F2D_DECIMAL64, F2D_DECIMAL128 = 25, 26, 27        # cudf type ids
F2D_WIDTH = {F2D_DECIMAL32: 32, F2D_DECIMAL64: 64, F2D_DECIMAL128: 128}
F2D_MAX_PRECISION = {F2D_DECIMAL32: 9, F2D_DECIMAL64: 18, F2D_DECIMAL128: 38}
F2D_MIN_SPARK_SCALE = -38


def _mask(bits):
    return (1 << bits) - 1


def ipow10(k, bits):                              # fixed_point.hpp:78-97 modulo 2^bits; k < 0 returns 10 (assert compiled out)
    if k == 0:
        return 1
    extra, square = 1, 10
    while k > 1:
        if k & 1:
            extra = extra * square & _mask(bits)
        k >>= 1
        square = square * square & _mask(bits)
    return square * extra & _mask(bits)


def _mul_pow10(v, k, rep_bits, t_bits):           # FC:402-472: the switch of the 32-bit helper is 0 outside 0..9
    if rep_bits == 32:
        return v * 10 ** k & _mask(t_bits) if 0 <= k <= 9 else 0
    return v * ipow10(k, rep_bits) & _mask(t_bits)


def _div_pow10(v, k, rep_bits, t_bits):           # FC:324-391, 487-498
    if rep_bits == 32:
        return v // 10 ** k if 0 <= k <= 9 else 0
    d = ipow10(k, rep_bits)
    if d == 0:                                    # 10^k = 0 mod 2^64 (k >= 64): undefined in C++; defined here as all ones
        return _mask(t_bits)
    return v // d


def _gls(v, s, bits):                             # FC:509-515 guarded_left_shift
    return v << s & _mask(bits) if s <= bits - 1 else _mask(bits)


def _grs(v, s, bits):                             # FC:526-531 guarded_right_shift
    return v >> s if s <= bits - 1 else 0


def _pospow(base2, pow2, p, ub):                  # FC:687-759 shift_to_decimal_pospow (pow2 > 0, p > 0)
    sr = base2
    if pow2 <= 70:                                # max_init_shift = 124 - 54
        return _div_pow10(sr << pow2 & M128, p, 128, 128) & _mask(ub)
    sr, pow2 = sr << 70 & M128, pow2 - 70
    while p > 18:
        sr, p = sr // 10 ** 18, p - 18
        if pow2 <= 60:
            return _div_pow10(sr << pow2 & M128, p, 128, 128) & _mask(ub)
        sr, pow2 = sr << 60 & M128, pow2 - 60
    sr = _div_pow10(sr, p, 64, 128)               # divide_power10_64bit
    return _gls(sr & _mask(ub), pow2, ub)


def _negpow(base2, pow2, p, ub):                  # FC:774-845 shift_to_decimal_negpow (pow2 < 0, p < 0)
    sr, p10, p2 = base2, -p, -pow2

    def final(sr, p10, p2):                       # multiply_power10_64bit, then a guarded right shift
        return _grs(sr * ipow10(p10, 64) & M128, p2, 128) & _mask(ub)

    if p10 <= 18:
        return final(sr, p10, p2)
    sr, p2 = sr << 14 & M128, p2 + 14             # num_init_bit_shift = (128 - 60) - 54
    while True:
        sr, p10 = sr * 10 ** 18 & M128, p10 - 18
        if p2 <= 60:
            return _mul_pow10((sr >> p2) & _mask(ub), p10, ub, ub)
        sr, p2 = sr >> 60, p2 - 60
        if p10 <= 18:
            return final(sr, p10, p2)


def _convert(base2, p, pow2, ub):                 # FC:860-898 convert_floating_to_integral_shifting, UnsignedRep of ub bits
    if p == 0:
        return _gls(base2 & _mask(ub), pow2, ub) if pow2 >= 0 else _grs(base2, -pow2, 64) & _mask(ub)
    if p > 0:
        if pow2 <= 0:
            return _div_pow10(_grs(base2, -pow2, 64), p, 64, 64) & _mask(ub)
        return _pospow(base2, pow2, p, ub)
    if pow2 >= 0:
        return _mul_pow10(_gls(base2 & _mask(ub), pow2, ub), -p, ub, ub)
    return _negpow(base2, pow2, p, ub)


def _ctrunc_div(a, b):                            # C++ integer division: truncates toward zero
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


_F2D_MAX_REP = {32: 2147483647.0, 64: 2.0 ** 63, 128: 2.0 ** 127}    # double(numeric_limits<IntType>::max())


def f2d_scale_factor(width, pow10):               # :1206-1207: double(multiply_power10<IntType>(1, -pow10))
    return float(_mul_pow10(1, -pow10, width, width))


def scaled_round(x, is_f32, width, pow10, scale_factor=None):
    """:1193-1309 for one finite x (a Python float holding the input's value), IntType of `width` bits and the cudf
    scale pow10; the signed IntType result."""
    if scale_factor is None:
        scale_factor = f2d_scale_factor(width, pow10)
    bits = int(np.float64(x).view(np.uint64))
    if bits & ~(1 << 63) == 0:
        return 0
    neg = bits >> 63
    mant, e = bits & _mask(52), (bits >> 52) & 0x7FF
    if e == 0:                                    # FC:187-200: a denormal lined up to the understood bit
        fp2 = 1 - 1023
        shift = 53 - mant.bit_length()
        mant, fp2 = mant << shift, fp2 - shift
    else:
        fp2, mant = e - 1023, mant | (1 << 52)
    pow2 = fp2 - 52
    uf = abs(x)
    rwo = 10.0 * uf * scale_factor < _F2D_MAX_REP[width]          # :1205-1210, in double
    can_round = rwo if width == 128 else True
    sp = pow10 - 1 if can_round else pow10
    whole = math.floor(x) == x
    base2 = (mant << 1) + (0 if is_f32 or whole else 1)           # :1223-1236
    pow2 -= 1
    ub = (32 if rwo else 64) if width == 32 else 128              # :1239-1253: the rep of the shifting
    tb = 64 if width == 32 else 128                               # the intermediate magnitude
    mag = _convert(base2, sp, pow2, ub)
    fp = _ctrunc_div(3 * pow2 - 10 * pow10 + (0 if is_f32 else 9 * (uf > 2.0 ** 63)), 10)    # :1259-1270
    if can_round:                                                 # :1273-1303
        if fp < 0:
            mag = ((mag + 5) & _mask(tb)) // 10
        else:
            if is_f32 or whole:
                mag = mag + _mul_pow10(5, fp, width, tb) & _mask(tb)
            mag = _mul_pow10(_div_pow10(mag, fp + 1, width, tb), fp, width, tb)
    elif fp > 0:
        mag = _mul_pow10(_div_pow10(mag, fp, width, tb), fp, width, tb)
    s = mag & _mask(width)                                        # :1307-1308: the cast and the negation wrap
    if neg:
        s = -s & _mask(width)
    return s - (1 << width) if s >> (width - 1) else s


def f2d_check(out_type, precision, scale):
    """The domain of the C ABI: DECIMAL32 / 64 / 128, precision 1 .. 9 / 18 / 38, and the cudf scale in
    [-precision, 38] (Spark scale -38 .. precision).  TypeError for another type, ValueError outside the domain."""
    if out_type not in F2D_WIDTH:
        raise TypeError(f"unsupported output type {out_type}")
    if not 1 <= precision <= F2D_MAX_PRECISION[out_type]:
        raise ValueError(f"precision {precision} outside 1..{F2D_MAX_PRECISION[out_type]}")
    if not -precision <= scale <= -F2D_MIN_SPARK_SCALE:
        raise ValueError(f"scale {scale} outside [{-precision}, {-F2D_MIN_SPARK_SCALE}]")


def floating_point_to_decimal(values, valid, out_type, precision, scale):
    """The whole cast: values a float32 or float64 numpy array, valid a bool array or None (all valid), out_type a
    DECIMAL type id, scale the cudf scale.  Returns (signed Python ints, validity bool array, failure row): a null,
    NaN or infinite row is null with value 0; a row outside (-10^precision, 10^precision) is null with value 0 and
    fails; the failure row is the smallest failing row, or -1."""
    f2d_check(out_type, precision, scale)
    width = F2D_WIDTH[out_type]
    is_f32 = np.asarray(values).dtype == np.float32
    sf = f2d_scale_factor(width, scale)
    bound = _mul_pow10(1, precision, width, width)
    n = len(values)
    ok = np.ones(n, bool) if valid is None else np.array(valid, bool)
    out, first = [0] * n, -1
    with np.errstate(invalid="ignore"):
        xs = np.asarray(values, np.float64).tolist()
    for i, x in enumerate(xs):
        if not ok[i] or not math.isfinite(x):
            ok[i] = False
            continue
        v = scaled_round(x, is_f32, width, scale, sf)
        if -bound >= v or v >= bound:
            ok[i] = False
            first = i if first < 0 else first
        else:
            out[i] = v
    return out, ok, first


def build(force: bool = False) -> str:
    """Compile float_to_decimal.c -> libf2d_oracle.so with the system gcc and OpenMP, when it is missing or older."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-shared",
                               "-o", _SO, _SRC])
    return _SO


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def floating_point_to_decimal_c(values, mask, out_type, precision, scale):
    """floating_point_to_decimal through float_to_decimal.c (OpenMP; for sweeps of 2^32 rows in chunks).  values a
    float32 or float64 numpy array, mask its uint32 null-mask words or None.  Returns (out numpy array: int32 / int64,
    or uint8 [n, 16] little-endian for DECIMAL128; validity bool array; failure row)."""
    f2d_check(out_type, precision, scale)
    values = np.ascontiguousarray(values)
    n = len(values)
    out = np.zeros(n, np.int32) if out_type == F2D_DECIMAL32 else np.zeros(n, np.int64) if out_type == F2D_DECIMAL64 \
        else np.zeros((n, 16), np.uint8)
    valid = np.zeros(n, np.uint8)
    first = C.c_int64(-1)
    m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint32)
    rc = lib().f2d_float_to_decimal(C.c_void_p(values.ctypes.data), C.c_int32(values.dtype == np.float32),
                                    None if m is None else C.c_void_p(m.ctypes.data), C.c_int64(n), C.c_int32(out_type),
                                    C.c_int32(precision), C.c_int32(scale), C.c_void_p(out.ctypes.data),
                                    C.c_void_p(valid.ctypes.data), C.byref(first))
    if rc != 0:
        raise RuntimeError(f"f2d_float_to_decimal: {rc}")
    return out, valid.astype(bool), first.value
