"""CPU oracle of DateTimeUtils' rebase and truncation (reference datetime_rebase.cu, datetime_truncate.cu), vectorised in
numpy.  Values are int32 days (TIMESTAMP_DAYS) or int64 microseconds (TIMESTAMP_MICROSECONDS) since 1970-01-01 UTC.

Dates go through y/m/d with the year reduced to int16 (two's complement), as the reference's cuda::std::chrono::year
stores it; results wrap to the storage type.  Day counts above INT32_MAX - 719468 (where the reference's int conversion
overflows) and WEEK rows within 4 of INT32_MAX are defined by exact arithmetic here.
"""
import numpy as np

TIMESTAMP_DAYS, TIMESTAMP_MICROSECONDS = 12, 15
GREGORIAN_TO_JULIAN, JULIAN_TO_GREGORIAN = 0, 1
US_PER_DAY = 86_400_000_000
GREGORIAN_START_DAY = -141427                 # 1582-10-15
GREGORIAN_START_US = -12219292800000000       # 1582-10-15T00:00:00Z

# formats (the families of the reference's truncation_format); TIMESTAMP_DAYS accepts YEAR .. WEEK
YEAR, QUARTER, MONTH, WEEK, DAY, HOUR, MINUTE, SECOND, MILLISECOND, MICROSECOND, INVALID = range(11)
NAMES = {"YEAR": YEAR, "YYYY": YEAR, "YY": YEAR, "QUARTER": QUARTER, "MONTH": MONTH, "MM": MONTH, "MON": MONTH, "WEEK": WEEK,
         "DAY": DAY, "DD": DAY, "HOUR": HOUR, "MINUTE": MINUTE, "SECOND": SECOND, "MILLISECOND": MILLISECOND,
         "MICROSECOND": MICROSECOND}
UNIT_US = {DAY: US_PER_DAY, HOUR: 3_600_000_000, MINUTE: 60_000_000, SECOND: 1_000_000, MILLISECOND: 1000}


def _s16(y):
    return ((y + 32768) & 0xFFFF) - 32768


def civil_from_days(d):
    """(y (int16-reduced), m, d) of proleptic Gregorian day counts (int64 arrays)"""
    z = np.asarray(d, np.int64) + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    dd = doy - (153 * mp + 2) // 5 + 1
    m = np.where(mp < 10, mp + 3, mp - 9)
    return _s16(yoe + era * 400 + (m <= 2)), m, dd


def _doy(m, d):
    return (153 * (m + np.where(m > 2, -3, 9)) + 2) // 5 + d - 1


def days_from_civil(y, m, d):
    y = np.asarray(y, np.int64) - (np.asarray(m) <= 2)
    era = y // 400
    yoe = y - era * 400
    return era * 146097 + yoe * 365 + yoe // 4 - yoe // 100 + _doy(m, d) - 719468


def days_from_julian(y, m, d):
    y = np.asarray(y, np.int64) - (np.asarray(m) <= 2)
    era = y // 4
    yoe = y - era * 4
    return era * 1461 + yoe * 365 + _doy(m, d) - 719470


def julian_from_days(d):
    z = np.asarray(d, np.int64) + 719470
    era = z // 1461
    doe = z - era * 1461
    yoe = (doe - doe // 1460) // 365
    doy = doe - 365 * yoe
    mp = (5 * doy + 2) // 153
    dd = doy - (153 * mp + 2) // 5 + 1
    m = np.where(mp < 10, mp + 3, mp - 9)
    return _s16(yoe + era * 4 + (m <= 2)), m, dd


def _key(y, m, d):
    return y * 512 + m * 32 + d


def _g2j_day(days, keep_late):
    y, m, d = civil_from_days(days)
    k = _key(y, m, d)
    out = days_from_julian(y, m, d)
    if keep_late:
        out = np.where(k >= _key(1582, 10, 15), days, out)
    return np.where((k > _key(1582, 10, 4)) & (k < _key(1582, 10, 15)), GREGORIAN_START_DAY, out)


def _j2g_day(days):
    return days_from_civil(*julian_from_days(days))


def rebase(direction, type_id, values):
    """the rebased values, in the input's dtype (int32 days / int64 micros); every row, null or not"""
    if type_id == TIMESTAMP_DAYS:
        v = np.asarray(values).view(np.int32).astype(np.int64)
        if direction == GREGORIAN_TO_JULIAN:
            out = _g2j_day(v, True)
        else:
            out = np.where(v >= GREGORIAN_START_DAY, v, _j2g_day(np.minimum(v, GREGORIAN_START_DAY - 1)))
        return out.astype(np.int32)
    t = np.asarray(values).view(np.int64)
    days = t // US_PER_DAY
    tod = t - days * US_PER_DAY
    nd = _g2j_day(days, False) if direction == GREGORIAN_TO_JULIAN else _j2g_day(np.minimum(days, GREGORIAN_START_DAY - 1))
    with np.errstate(over="ignore"):
        out = nd.astype(np.int64) * np.int64(US_PER_DAY) + tod         # wraps, as the reference's int64 arithmetic does
    return np.where(t >= GREGORIAN_START_US, t, out)


def parse_format(fmt):
    """the format of a str / bytes name (only a-z upper-cased), INVALID when none"""
    b = fmt.encode("utf-8") if isinstance(fmt, str) else bytes(fmt)
    up = bytes(c ^ 0x20 if 0x61 <= c <= 0x7A else c for c in b)
    try:
        return NAMES.get(up.decode("ascii"), INVALID)
    except UnicodeDecodeError:
        return INVALID


def fits(fmt, type_id):
    return fmt != INVALID and (type_id == TIMESTAMP_MICROSECONDS or fmt <= WEEK)


def _trunc_days(days, fmt):
    if fmt == WEEK:
        return days - (days + 3) % 7
    y, m, _ = civil_from_days(days)
    if fmt == YEAR:
        m = np.ones_like(m)
    elif fmt == QUARTER:
        m = (m - 1) // 3 * 3 + 1
    return days_from_civil(y, m, np.ones_like(m))


def trunc_values(type_id, values, fmt):
    """values truncated to one format that fits the type, every row"""
    if type_id == TIMESTAMP_DAYS:
        return _trunc_days(np.asarray(values).view(np.int32).astype(np.int64), fmt).astype(np.int32)
    t = np.asarray(values).view(np.int64)
    if fmt == MICROSECOND:
        return t.copy()
    days = t // US_PER_DAY
    with np.errstate(over="ignore"):
        if fmt <= WEEK:
            return _trunc_days(days, fmt).astype(np.int64) * np.int64(US_PER_DAY)
        tod = t - days * US_PER_DAY
        base = days_from_civil(*civil_from_days(days)).astype(np.int64)
        return base * np.int64(US_PER_DAY) + tod // UNIT_US[fmt] * UNIT_US[fmt]


def _zero_nulls(out, valid):
    return np.where(valid, out, 0).astype(out.dtype)


def truncate_scalar(type_id, values, valid, fmt):
    """(values, valid) of truncate(datetime, fmt); valid None means no nulls.  Null rows hold 0."""
    n = len(np.asarray(values).view(np.int32 if type_id == TIMESTAMP_DAYS else np.int64))
    v = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    f = parse_format(fmt if fmt is not None else "")
    dtype = np.int32 if type_id == TIMESTAMP_DAYS else np.int64
    if not fits(f, type_id):
        return np.zeros(n, dtype), np.zeros(n, bool)
    return _zero_nulls(trunc_values(type_id, values, f), v), v


def truncate_column(type_id, values, valid, formats):
    """(values, valid) of truncate(datetime, format column): formats is a list of str / bytes, None for a null row; the
    datetime has one row (broadcast) or len(formats)."""
    dtype = np.int32 if type_id == TIMESTAMP_DAYS else np.int64
    vals = np.asarray(values).view(dtype)
    n = len(formats)
    if len(vals) == 1:
        vals = np.repeat(vals, n)
        valid = None if valid is None else np.repeat(np.asarray(valid, bool)[:1], n)
    v = np.ones(n, bool) if valid is None else np.asarray(valid, bool).copy()
    codes = np.array([INVALID if f is None else parse_format(f) for f in formats], np.int64)
    ok = v & np.array([fits(c, type_id) for c in codes], bool) if n else v
    out = np.zeros(n, dtype)
    for c in np.unique(codes[ok]):
        sel = ok & (codes == c)
        out[sel] = trunc_values(type_id, vals[sel], int(c))
    return out, ok
