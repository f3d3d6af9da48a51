"""DecimalUtils' DECIMAL128 arithmetic restated step by step in Python integers (reference
src/main/cpp/src/decimal_utils.cu).  Values are 256-bit two's complement, masked so that every step wraps where the
reference's chunked256 wraps; line numbers cite that file.

    ovf, val = multiply(a, b, a_scale, b_scale, product_scale, interim_cast)
    ovf, val = divide(a, b, a_scale, b_scale, quotient_scale, integer_divide)
    ovf, val = remainder(a, b, a_scale, b_scale, remainder_scale)
    ovf, val = add(a, b, a_scale, b_scale, target_scale) / subtract(...)

a and b are the signed 128-bit unscaled values of one row; scales are cudf scales (the value is v * 10^scale).  ovf is
a bool; val is the signed 128-bit (64-bit for integer_divide) value the reference writes, or 0 where it writes nothing
(the multiply's early exit, which this library defines as 0).  The row functions raise ValueError where the reference
needs a power of ten it cannot represent (pow_ten's CUDF_UNREACHABLE, or a truncating as_128_bits of 10^k, k > 38);
the column functions (multiply_cols, ...) check that per call first, as the C ABI does.
"""
import numpy as np

M256 = (1 << 256) - 1
M128 = (1 << 128) - 1


def s256(x):
    x &= M256
    return x - (1 << 256) if x >> 255 else x


def s128(x):
    x &= M128
    return x - (1 << 128) if x >> 127 else x


def s64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def pow_ten(k):                                   # :240-503, 10^0 .. 10^76
    if not 0 <= k <= 76:
        raise ValueError(f"pow_ten({k}): exponent exceeds supported value")
    return 10 ** k


def pow_ten_128(k):                               # pow_ten(k).as_128_bits(): exact only for k <= 38
    if k > 38:
        raise ValueError(f"10^{k} does not fit the 128-bit divisor")
    return pow_ten(k)


def divide_unsigned(n, d):                        # :141-161 bit-serial; d is a 128-bit magnitude
    n &= M256
    d &= M128
    if d == 0:                                    # every step subtracts 0: all quotient bits set, r = n's low 128 bits
        return M256, n & M128
    return n // d, n % d


def _divide(n, d):                                # :163-183: n 256-bit signed, d 128-bit signed -> (q 256, r 128 signed)
    n, d = s256(n), s128(d)
    n_neg, d_neg = n < 0, d < 0
    abs_n = (-n) & M256 if n_neg else n
    abs_d = (-d) & M128 if d_neg else d           # -INT128_MIN wraps to itself; as an unsigned divisor that is 2^127
    q, r = divide_unsigned(abs_n, abs_d)
    if d_neg != n_neg:
        q = (-q) & M256
    r = s128(r)
    if n_neg:
        r = s128(-r)
    return s256(q), r


def round_from_remainder(q, r, n, d):             # :185-217, signed 128-bit remainder arithmetic as in the reference
    r, d = s128(r), s128(d)
    dr = s128(r << 1)
    abs_dr = s128(-dr) if dr < 0 else dr
    abs_d = s128(-d) if d < 0 else d
    need_inc = (dr >> 1) != r or abs_dr >= abs_d
    round_down = (s256(n) < 0) != (d < 0)
    return s256(q + ((-1 if round_down else 1) if need_inc else 0))


def divide_and_round(n, d):                       # :222-227 (HALF_UP)
    q, r = _divide(n, d)
    return round_from_remainder(q, r, n, d)


def integer_divide(n, d):                         # :233-238 (DOWN)
    return _divide(n, d)[0]


def precision10(v):                               # :512-527: smallest i in [0, 76] with 10^i >= |v|, else -1
    v = s256(v)
    a = (-v) & M256 if v < 0 else v
    for i in range(77):
        if 10 ** i >= a:
            return i
    return -1


def gt38(v):                                      # is_greater_than_decimal_38, :529-534
    v = s256(v)
    a = (-v) & M256 if v < 0 else v
    return a >= 10 ** 38


def mul(a, b):                                    # :119-139, low 256 bits
    return s256(a * b)


def set_scale_and_round(data, old, new):          # :536-551
    if old != new:
        if new < old:
            data = mul(data, pow_ten(old - new))
        else:
            data = divide_and_round(data, pow_ten_128(new - old))
    return data


def add_sub(a, b, a_scale, b_scale, target_scale, sub):   # :574-588, :613-646
    a, b = s256(s128(a)), s256(s128(b))
    inter = min(a_scale, b_scale)
    if a_scale != inter:
        a = set_scale_and_round(a, a_scale, inter)
    if b_scale != inter:
        b = set_scale_and_round(b, b_scale, inter)
    if sub:
        b = s256(-b)
    a = s256(a + b)
    if target_scale != inter:
        a = set_scale_and_round(a, inter, target_scale)
    return gt38(a), s128(a)


def add(a, b, a_scale, b_scale, target_scale):
    return add_sub(a, b, a_scale, b_scale, target_scale, False)


def subtract(a, b, a_scale, b_scale, target_scale):
    return add_sub(a, b, a_scale, b_scale, target_scale, True)


def multiply(a, b, a_scale, b_scale, product_scale, interim_cast=True):   # :667-714
    p = mul(s128(a), s128(b))
    mult_scale = a_scale + b_scale
    if interim_cast:
        k = precision10(p) - 38
        if k > 0:
            p = divide_and_round(p, pow_ten_128(k))
            mult_scale += k
    exponent = product_scale - mult_scale
    if exponent < 0:
        if precision10(p) - exponent > 38:
            return True, 0                        # the reference returns without writing the value (:697-701)
        p = mul(p, pow_ten(-exponent))
    else:
        d = pow_ten_128(exponent)
        if d != 1:
            p = divide_and_round(p, d)
    return gt38(p), s128(p)


def divide(a, b, a_scale, b_scale, quot_scale, integer_div=False):   # :754-833
    n, d = s256(s128(a)), s128(b)
    if d == 0:
        return True, 0
    x = quot_scale - (a_scale - b_scale)
    trunc = s64 if integer_div else s128
    if x > 0:
        q1 = _divide(n, d)[0]
        sd = pow_ten_128(x)
        res = integer_divide(q1, sd) if integer_div else divide_and_round(q1, sd)
        return gt38(res), trunc(res)
    if x < -38:
        n = mul(n, pow_ten(38))
        q1, r1 = _divide(n, d)
        m = pow_ten(-x - 38)
        res = mul(q1, m)
        sdr = mul(r1, m)
        q2, r2 = _divide(sdr, d)
        res = s256(res + q2)
        if not integer_div:
            res = round_from_remainder(res, r2, sdr, d)
        return gt38(res), trunc(res)
    if x < 0:
        n = mul(n, pow_ten(-x))
    res = integer_divide(n, d) if integer_div else divide_and_round(n, d)
    return gt38(res), trunc(res)


def remainder(a, b, a_scale, b_scale, rem_scale):  # :862-949
    n, d = s256(s128(a)), s128(b)
    if d == 0:
        return True, 0
    n_neg, d_neg = n < 0, d < 0
    d_shift = rem_scale - b_scale
    n_shift = rem_scale - a_scale
    abs_d = s128(-d) if d_neg else d
    if d_shift > 0:
        abs_d = s128(divide_and_round(s256(abs_d), pow_ten_128(d_shift)))
    else:
        n_shift -= d_shift
    abs_n = s256(-n) if n_neg else n
    if n_shift > 0:
        q1 = _divide(abs_n, abs_d)[0]
        idr = integer_divide(q1, pow_ten_128(n_shift))
    else:
        if n_shift < 0:
            abs_n = mul(abs_n, pow_ten(-n_shift))
        idr = integer_divide(abs_n, abs_d)
    less = mul(idr, s256(abs_d))
    if d_shift < 0:
        less = mul(less, pow_ten(-d_shift))
    abs_n = s256(abs_n - less)
    ovf = gt38(abs_n)
    res = s128(abs_n)
    if n_neg:
        res = s128(-res)
    return ovf, res


MULTIPLY, DIVIDE, INTEGER_DIVIDE, REMAINDER, ADD, SUBTRACT = range(6)     # SRJ_DECIMAL_*


def check_scales(op, a_scale, b_scale, out_scale):
    """Raise ValueError for the scale combinations whose rows would need a power of ten the reference cannot represent
    (or, for multiply, that its own check_scale_divisor rejects, :505-510).  Spark's type rules never produce them."""
    def bad(why):
        raise ValueError(f"scales ({a_scale}, {b_scale}) -> {out_scale}: {why}")
    if op == MULTIPLY:
        if out_scale - (a_scale + b_scale) > 38:
            bad("divisor too big")
    elif op in (DIVIDE, INTEGER_DIVIDE):
        x = out_scale - (a_scale - b_scale)
        if x > 38 or x < -38 - 76:
            bad("the quotient needs 10^k with k outside the supported range")
    elif op == REMAINDER:
        ds, ns = out_scale - b_scale, out_scale - a_scale
        if ds <= 0:
            ns -= ds
        if ds > 38 or ds < -76 or ns > 38 or ns < -76:
            bad("the remainder needs 10^k with k outside the supported range")
    elif op in (ADD, SUBTRACT):
        inter = min(a_scale, b_scale)
        if abs(a_scale - b_scale) > 76 or inter - out_scale > 76 or out_scale - inter > 38:
            bad("the intermediate scale needs 10^k with k outside the supported range")
    else:
        raise ValueError(f"unknown op {op}")


def row(op, a, b, a_scale, b_scale, out_scale, interim_cast=True):
    """(overflow, value) of one row of op."""
    if op == MULTIPLY:
        return multiply(a, b, a_scale, b_scale, out_scale, interim_cast)
    if op in (DIVIDE, INTEGER_DIVIDE):
        return divide(a, b, a_scale, b_scale, out_scale, op == INTEGER_DIVIDE)
    if op == REMAINDER:
        return remainder(a, b, a_scale, b_scale, out_scale)
    return add_sub(a, b, a_scale, b_scale, out_scale, op == SUBTRACT)


def to_ints(u8):
    """DECIMAL128 column bytes (little-endian, 16 per row) -> list of signed Python ints."""
    w = np.ascontiguousarray(u8).view(np.uint64).reshape(-1, 2)
    return [s128(int(lo) | (int(hi) << 64)) for lo, hi in w]


def from_ints(vals, width=16):
    """signed Python ints -> little-endian column bytes of `width` (16 or 8) bytes per row."""
    m = (1 << (8 * width)) - 1
    return np.frombuffer(b"".join((v & m).to_bytes(width, "little") for v in vals), dtype=np.uint8).copy()


def binary(op, a_u8, b_u8, a_scale, b_scale, out_scale, interim_cast=True):
    """Both output columns of op over DECIMAL128 column bytes: (overflow uint8 [n], value bytes [n * 16], or [n * 8]
    for INTEGER_DIVIDE).  Every row is computed from its bits, null or not."""
    check_scales(op, a_scale, b_scale, out_scale)
    res = [row(op, x, y, a_scale, b_scale, out_scale, interim_cast) for x, y in zip(to_ints(a_u8), to_ints(b_u8))]
    ovf = np.array([r[0] for r in res], dtype=np.uint8)
    return ovf, from_ints([r[1] for r in res], 8 if op == INTEGER_DIVIDE else 16)


def mask_and(ma, mb, n):
    """The outputs' null mask (uint32 words) and null count: the AND of the input masks (None = all valid)."""
    words = (n + 31) // 32
    out = np.full(words, 0xFFFFFFFF, dtype=np.uint32)
    for m in (ma, mb):
        if m is not None:
            out &= np.asarray(m, dtype=np.uint32)[:words]
    if ma is None and mb is None:
        return None, 0
    bits = np.unpackbits(out.view(np.uint8), bitorder="little")[:n]
    return out, int(n - bits.sum())
