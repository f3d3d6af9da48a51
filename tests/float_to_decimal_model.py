"""An independent model of what Spark means by CAST(float / double AS DECIMAL(p, s)): the value's shortest decimal
string (Java's Double.toString of x.toDouble, which Python's repr of the same double matches), as a BigDecimal, rounded
HALF_UP to s places, and null when it then has more than p digits.  It shares no step with the reference's binary
shifting, so tests/test_oracle_float_to_decimal.py can name every class of rows where the two differ."""
import decimal
import math

_CTX = decimal.Context(prec=1000, Emax=decimal.MAX_EMAX, Emin=decimal.MIN_EMIN)


def cast(x, precision, spark_scale):
    """The unscaled integer of x at spark_scale, or None for a null (NaN, infinite, or more than precision digits)."""
    x = float(x)
    if not math.isfinite(x):
        return None
    d = decimal.Decimal(repr(x))
    q = d.quantize(decimal.Decimal(1).scaleb(-spark_scale), rounding=decimal.ROUND_HALF_UP, context=_CTX)
    v = int(q.scaleb(spark_scale, context=_CTX))
    return v if abs(v) < 10 ** precision else None
