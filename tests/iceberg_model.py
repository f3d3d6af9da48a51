"""An independent per-row model of Iceberg's bucket / truncate / date-time transforms in Python integers, written from the
algorithms rather than from the reference: MurmurHash3_x86_32 from Appleby's description, decimals through
int.to_bytes(signed=True) (BigInteger.toByteArray), the calendar through datetime.date for years 1..9999 and whole
400-year cycles (146097 days) beyond."""
import datetime

M32 = 0xFFFFFFFF
INT32_MAX = 2**31 - 1
EPOCH = datetime.date(1970, 1, 1)


def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & M32


def murmur3_32(data: bytes, seed: int = 0) -> int:
    """signed 32-bit MurmurHash3_x86_32"""
    c1, c2 = 0xCC9E2D51, 0x1B873593
    h = seed & M32
    n = len(data)
    for i in range(0, n - n % 4, 4):
        k = int.from_bytes(data[i:i + 4], "little")
        k = (_rotl((k * c1) & M32, 15) * c2) & M32
        h = (_rotl(h ^ k, 13) * 5 + 0xE6546B64) & M32
    tail = data[n - n % 4:]
    if tail:
        k = int.from_bytes(tail, "little")
        h ^= (_rotl((k * c1) & M32, 15) * c2) & M32
    h ^= n
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    h ^= h >> 16
    return h - 2**32 if h >= 2**31 else h


def java_bytes(v: int) -> bytes:
    """BigInteger.valueOf(v).toByteArray(): the shortest big-endian two's complement"""
    n = 1
    while True:
        try:
            return v.to_bytes(n, "big", signed=True)
        except OverflowError:
            n += 1


def hash_long(v: int) -> int:
    return murmur3_32((v % 2**64).to_bytes(8, "little"))


def bucket_value(h: int, n: int) -> int:
    return (h & INT32_MAX) % n


def trunc_int(v: int, w: int, bits: int) -> int:
    """v - (((v % w) + w) % w) with C's truncated % and + / - wrapping at `bits`"""
    def wrap(x):
        return (x + 2**(bits - 1)) % 2**bits - 2**(bits - 1)

    def crem(a, b):
        r = abs(a) % abs(b)
        return -r if a < 0 else r
    return wrap(v - crem(wrap(crem(v, w) + w), w))


def trunc_utf8(b: bytes, width: int) -> bytes:
    """the bytes before the (width+1)-th byte that is not a continuation byte 10xxxxxx"""
    seen = 0
    for i, c in enumerate(b):
        if c & 0xC0 != 0x80:
            seen += 1
            if seen == width + 1:
                return b[:i]
    return b


def civil(days: int):
    """(year, month) of a day count from 1970-01-01, proleptic Gregorian"""
    cycles = 0
    # bring the day into datetime.date's range by whole 400-year cycles (the Gregorian calendar repeats every 146097 days)
    lo, hi = (datetime.date(1, 1, 1) - EPOCH).days, (datetime.date(9999, 12, 31) - EPOCH).days
    if days < lo or days > hi:
        cycles = (days - (-719162 + 146097 * 5)) // 146097
        days -= cycles * 146097
    d = EPOCH + datetime.timedelta(days=days)
    return d.year + 400 * cycles, d.month


def years(days: int) -> int:
    return civil(days)[0] - 1970


def months(days: int) -> int:
    y, m = civil(days)
    return (y - 1970) * 12 + m - 1


def floor_days(micros: int) -> int:
    return micros // 86_400_000_000


def hours(micros: int) -> int:
    h = micros // 3_600_000_000
    return (h + 2**31) % 2**32 - 2**31
