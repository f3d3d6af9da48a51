"""An independent model of DecimalUtils in Python's decimal module (200 digits, ROUND_HALF_UP / ROUND_DOWN), following
Spark's semantics rather than the reference's steps: the exact result rounded once to the output scale, overflow when
|result| >= 10^38.  It agrees with oracle/decimal.py except on the reference's quirks, which quirk() names:
  interim     multiply with the interim cast rounds twice when the product has more than 38 digits
  pow10       precision10 takes an exact power of ten 10^k as k digits (the multiply's early exit and interim cast)
(Integral divide keeps the low 64 bits of a quotient that needs more, and every overflowing row the low 128 bits of its
value: the tests compare the model's exact value truncated the same way, so those rows need no exemption.)
  wrap        a 256-bit intermediate of the reference wraps
"""
from decimal import ROUND_DOWN, ROUND_HALF_UP, Context, Decimal

CTX = Context(prec=200)
MAX = 10 ** 38


def _val(v, scale):
    return CTX.multiply(Decimal(v), CTX.power(Decimal(10), scale))


def _at(x, scale, rounding):
    """x at cudf scale `scale` as an unscaled integer"""
    q = CTX.divide(x, CTX.power(Decimal(10), scale))
    return int(q.to_integral_value(rounding=rounding, context=CTX))


def model(op, a, b, sa, sb, so, interim_cast=True):
    """(overflow, unscaled result) of Spark's arithmetic; op codes as oracle/decimal.py"""
    x, y = _val(a, sa), _val(b, sb)
    if op in (1, 2, 3) and b == 0:
        return True, 0
    if op == 0:
        r = _at(CTX.multiply(x, y), so, ROUND_HALF_UP)
    elif op == 1:
        r = _at(CTX.divide(x, y), so, ROUND_HALF_UP)
    elif op == 2:
        r = _at(CTX.divide(x, y), so, ROUND_DOWN)
        return abs(r) >= MAX, r
    elif op == 3:
        q = CTX.divide(x, y).to_integral_value(rounding=ROUND_DOWN, context=CTX)
        r = _at(CTX.subtract(x, CTX.multiply(q, y)), so, ROUND_HALF_UP)
    else:
        r = _at(CTX.add(x, y) if op == 4 else CTX.subtract(x, y), so, ROUND_HALF_UP)
    return abs(r) >= MAX, r


def quirk(op, a, b, sa, sb, so, interim_cast=True):
    """the name of the reference quirk this row may hit, or None when oracle and model must agree exactly"""
    if op == 0:
        p = abs(a * b)
        if interim_cast and p > 10 ** 38:                                # precision10 > 38: rounded twice
            return "interim"
        if any(p == 10 ** k for k in range(77)):
            return "pow10"
        if so < sa + sb and p * 10 ** (sa + sb - so) >= MAX:
            return "pow10"            # the early exit leaves 0 where the model has the exact (overflowing) value
    if op in (1, 2) and b != 0 and so - (sa - sb) < -38 and abs(a) * 10 ** (sa - sb - so) >= 2 ** 255:
        return "wrap"
    if op == 3 and b != 0 and so > sb and abs(b) * 2 < 10 ** (so - sb):
        return "wrap"                 # the divisor rounds to 0 at the remainder's scale
    return None
