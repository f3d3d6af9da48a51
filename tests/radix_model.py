"""An independent model of the radix casts from Spark's documented intent, built on Python's int(), bin() and
format(x, "X"), for tests/test_oracle_radix.py.

conv(s, from, to) (Spark's NumberConverter, "convert a number in a string from one base to another"): trim spaces; an
empty string is null; an optional '-' and the longest prefix of digits valid in `from` are read with int() (no digits:
0).  The number is an unsigned 64-bit value: past 2^64 - 1 it saturates to all ones (non-ANSI) or is an overflow (ANSI).
A '-' negates it modulo 2^64 when `to` > 0, except that a value already read as negative (top bit set) gives all ones.
With `to` < 0 the result is signed: a value with the top bit set prints as '-' and its magnitude, and an input '-' is
kept in front.  Digits are upper case.

The model differs from oracle/radix.py on no class of rows: the prefix rule, the saturation and the sign rules give the
reference's results on every row the tests generate, the edges included.
"""
M64 = (1 << 64) - 1
DIGITS = "0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZ"


def to_base(u: int, base: int) -> str:
    if base == 2:
        return bin(u)[2:]
    if base == 16:
        return format(u, "X")
    if base == 8:
        return format(u, "o")
    if base == 10:
        return str(u)
    s = ""
    while True:
        s = DIGITS[u % base] + s
        u //= base
        if not u:
            return s


def conv(s: bytes, fb: int, tb: int, ansi: bool = False):
    """(result str or None, overflow)"""
    t = s.strip(b" ")
    if not t:
        return None, False
    neg = t[:1] == b"-"
    body = t[1:] if neg else t
    k = 0
    while k < len(body) and body[k] < 0x80 and chr(body[k]).isalnum() and int(chr(body[k]), 36) < fb:
        k += 1
    u = int(body[:k].decode(), fb) if k else 0
    overflow = u > M64
    if overflow:
        if ansi:
            return None, True
        u = M64
    if neg and tb > 0:
        u = M64 if u >> 63 else (-u) & M64
    if tb < 0:
        signed = u - (1 << 64) if u >> 63 else u
        return ("-" if neg or signed < 0 else "") + to_base(abs(signed), -tb), overflow
    return to_base(u, tb), overflow


def long_to_binary(v: int) -> str:
    return bin(v & M64)[2:]


def integer_to_string(v: int, bits: int, base: int) -> str:
    return str(v) if base == 10 else format(v & ((1 << bits) - 1), "X")


def bytes_to_hex(b: bytes) -> str:
    return "".join(format(x, "02X") for x in b)
