"""An independent per-value model of DateTimeUtils' rebase and truncation for years 1 .. 9999: Python's datetime.date
gives the proleptic Gregorian calendar, and the Julian calendar comes from the Julian day number (JDN) formulas of the
Explanatory Supplement to the Astronomical Almanac, not from Hinnant's algorithms.  No int16 year reduction: the model
holds only where the year stays in range."""
import datetime as dt

EPOCH = dt.date(1970, 1, 1)
JDN_EPOCH = 2440588                     # JDN of 1970-01-01
US = 86_400_000_000
UNITS = {"DAY": US, "DD": US, "HOUR": 3_600_000_000, "MINUTE": 60_000_000, "SECOND": 1_000_000, "MILLISECOND": 1000}


def greg(days):
    d = EPOCH + dt.timedelta(days=days)
    return d.year, d.month, d.day


def greg_days(y, m, d):
    """a Gregorian y/m/d to days; an out-of-month day (Feb 29 of a common year) runs on into the next month"""
    return (dt.date(y, m, 1) - EPOCH).days + d - 1


def julian_jdn(y, m, d):
    a = (14 - m) // 12
    yy, mm = y + 4800 - a, m + 12 * a - 3
    return d + (153 * mm + 2) // 5 + 365 * yy + yy // 4 - 32083


def julian_from_jdn(j):
    c = j + 32082
    d = (4 * c + 3) // 1461
    e = c - 1461 * d // 4
    m = (5 * e + 2) // 153
    return d - 4800 + m // 10, m + 3 - 12 * (m // 10), e - (153 * m + 2) // 5 + 1


def g2j_day(days, keep_late=True):
    ymd = greg(days)
    if (1582, 10, 4) < ymd < (1582, 10, 15):
        return -141427
    if keep_late and ymd >= (1582, 10, 15):
        return days
    return julian_jdn(*ymd) - JDN_EPOCH


def j2g_day(days):
    if days >= -141427:
        return days
    return greg_days(*julian_from_jdn(days + JDN_EPOCH))


def g2j_us(t):
    if t >= -12219292800000000:
        return t
    days, tod = divmod(t, US)
    return g2j_day(days, keep_late=False) * US + tod


def j2g_us(t):
    if t >= -12219292800000000:
        return t
    days, tod = divmod(t, US)
    return j2g_day(days) * US + tod


def trunc_day(days, fmt):
    y, m, _ = greg(days)
    f = fmt.upper()
    if f in ("YEAR", "YYYY", "YY"):
        return greg_days(y, 1, 1)
    if f == "QUARTER":
        return greg_days(y, (m - 1) // 3 * 3 + 1, 1)
    if f in ("MONTH", "MM", "MON"):
        return greg_days(y, m, 1)
    if f == "WEEK":
        return days - (EPOCH + dt.timedelta(days=days)).weekday()      # Monday = 0
    return None


def trunc_us(t, fmt):
    f = fmt.upper()
    if f == "MICROSECOND":
        return t
    days, tod = divmod(t, US)
    r = trunc_day(days, f)
    if r is not None:
        return r * US
    unit = UNITS.get(f)
    return None if unit is None else days * US + tod // unit * unit
