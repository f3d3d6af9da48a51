"""Independent model of CAST(string AS TIMESTAMP) and CAST(string AS DATE), written from Spark's grammar
(SparkDateTimeUtils.stringToTimestamp / stringToDate, Spark 3.5) as regular expressions, with integer civil-day
arithmetic (Python's datetime stops at year 9999).  Zones named in a time-alone string are resolved through
timezone_model (java.time semantics over the system's tzdata).

timestamp(s, ...) -> (valid, row) where row is the six intermediate columns for a valid string, and for an invalid one
(1, seconds, micros, 2, 0, -1) when the only fault is a zone name the map lacks, else None (only the result is defined).
date(s) -> epoch day or None.
"""
import re

import timezone_model as TZM

_WS = bytes(list(range(0, 33)) + [127])
_TIME = rb"(\d{1,2})(?::(\d{1,2})(?::(\d{1,2})(?:\.(\d*))?)?)?"
_TAIL = rb"((?:[^0-9].*)?)"                      # a zone starts at the first non-digit after the seconds
_DATE_TIME = re.compile(rb"([+-]?)(\d{4,6})(?:-(\d{1,2})(?:-(\d{1,2})(?:[ T]" + _TIME + rb")?)?)?" + _TAIL, re.S)
_T_TIME = re.compile(rb"T" + _TIME + _TAIL, re.S)
_H_M_TIME = re.compile(rb"(\d{1,2}):(\d{1,2})(?::(\d{1,2})(?:\.(\d*))?)?" + _TAIL, re.S)
_OFFSET = re.compile(rb"(\d{1,2})|(\d\d)(\d\d)?(\d\d)?|(\d{1,2}):(\d{1,2})(?::(\d\d))?")
_SPARK320_SIGN = re.compile(rb"([+-])(\d{0,2})(?:[: ](\d{1,2})(?:[: ](\d{1,2}))?)?")


def days_from_civil(y, m, d):
    """Days from 1970-01-01 of a proleptic Gregorian date: whole years, then the months of the year."""
    def leaps_before(year):                       # leap years in [1, year) counted from year 1 (negative years too)
        n = year - 1
        return n // 4 - n // 100 + n // 400
    days = 365 * (y - 1970) + leaps_before(y) - leaps_before(1970)
    cum = (0, 31, 59, 90, 120, 151, 181, 212, 243, 273, 304, 334)
    leap = y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)
    return days + cum[m - 1] + (1 if leap and m > 2 else 0) + d - 1


def _month_days(y, m):
    if m == 2:
        return 29 if (y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)) else 28
    return 30 if m in (4, 6, 9, 11) else 31


def _valid_date(y, m, d):
    return 1 <= m <= 12 and 1 <= d <= _month_days(y, m)


def _offset(text, spark_320):
    """Seconds of an offset after its sign, or None."""
    m = _OFFSET.fullmatch(text)
    if not m:
        return None
    if m.group(1) is not None:
        h, mi, s = int(m.group(1)), 0, 0
    elif m.group(2) is not None:
        h, mi, s = int(m.group(2)), int(m.group(3) or 0), int(m.group(4) or 0)
    else:
        if spark_320 and len(m.group(6)) == 1:
            return None
        if m.group(7) is not None and len(m.group(6)) != 2:
            return None
        h, mi, s = int(m.group(5)), int(m.group(6)), int(m.group(7) or 0)
    if h > 18 or mi > 59 or s > 59 or h * 3600 + mi * 60 + s > 18 * 3600:
        return None
    return h * 3600 + mi * 60 + s


def zone(text, spark_320):
    """('fixed', seconds) | ('name', bytes) | None (an invalid zone) for the text after the time, its spaces dropped."""
    text = text.lstrip(_WS)
    if text == b"Z":
        return ("fixed", 0)
    for prefix in (b"UTC", b"GMT", b"UT", b""):
        if text.startswith(prefix) and (prefix or text[:1] in (b"+", b"-")):
            rest = text[len(prefix):]
            if prefix and rest == b"":
                return ("fixed", 0)
            if prefix == b"GMT" and rest == b"0":
                return ("fixed", 0)
            if rest[:1] in (b"+", b"-"):
                o = _offset(rest[1:], spark_320)
                return None if o is None else ("fixed", o if rest[:1] == b"+" else -o)
            if prefix:
                return ("name", text)
    if text == b"U":
        return None
    return ("name", text)


def _micros(frac):
    frac = (frac or b"")[:6]
    return int(frac.ljust(6, b"0")) if frac else 0


def timestamp(s, default_tz, default_epoch_day, names, zones, now, spark_320, spark_400):
    """names: dict bytes -> index; zones: index -> IANA zone name; now: UTC seconds; returns (valid, row) as the module
    doc says."""
    if s is None:
        return False, (1, 0, 0, 0, 0, -1)
    t = s.strip(_WS)
    just_time = False
    m = _DATE_TIME.fullmatch(t)
    if m and (m.group(2) is not None):
        sign, y, mo, d = m.group(1), int(m.group(2)), int(m.group(3) or 1), int(m.group(4) or 1)
        h, mi, sec, frac, tail = m.group(5), m.group(6), m.group(7), m.group(8), m.group(9)
        year = -y if sign == b"-" else y
        time_given = h is not None
    else:
        leading_space = len(s.lstrip(_WS)) < len(s)
        m = None if (spark_400 and leading_space) else _T_TIME.fullmatch(t)   # SPARK-52351
        m = m or _H_M_TIME.fullmatch(t)
        if not m:
            return False, None
        just_time = True
        year, mo, d = 1970, 1, 1
        h, mi, sec, frac, tail = m.group(1), m.group(2), m.group(3), m.group(4), m.group(5)
        time_given = True
    fields = [int(v) if v is not None else 0 for v in (h, mi, sec)]
    tz = ("none",)
    if tail:
        # a zone may follow the seconds or the fraction only
        if sec is None or not time_given:
            return False, None
        if spark_320 and tail[:1] in (b"+", b"-"):
            z = _SPARK320_SIGN.fullmatch(tail)
            if not z:
                return False, None
            hh, mm = int(z.group(2) or 0), int(z.group(3) or 0)
            if hh > 18 or mm > 59 or hh * 3600 + mm * 60 > 18 * 3600:
                return False, None
            tz = ("fixed", (1 if z.group(1) == b"+" else 0) * (hh * 3600 + mm * 60))
        else:
            tz = zone(tail, spark_320)
            if tz is None:
                return False, None
    if not (-300000 <= year <= 300000) or not _valid_date(year, mo, d):
        return False, None
    if not (fields[0] < 24 and fields[1] < 60 and fields[2] < 60):
        return False, None
    seconds = days_from_civil(year, mo, d) * 86400 + fields[0] * 3600 + fields[1] * 60 + fields[2]
    us = _micros(frac)

    def day_of(local):                            # the day of a local second, truncated toward zero as the cast takes it
        return (abs(local) // 86400) * (1 if local >= 0 else -1)
    if tz[0] == "none":
        return True, (0, seconds + (default_epoch_day * 86400 if just_time else 0), us, 2, 0, default_tz)
    if tz[0] == "fixed":
        return True, (0, seconds + (day_of(now + tz[1]) * 86400 if just_time else 0), us, 1, tz[1], -1)
    idx = names.get(tz[1], -1)
    if idx < 0:
        return False, (1, seconds, us, 2, 0, -1)
    if just_time:
        seconds += day_of(TZM.from_utc(zones[idx], now)) * 86400
    return True, (0, seconds, us, 2, 0, idx)


_DATE = re.compile(rb"([+-]?)(\d{4,7})(?:-(\d{1,2})(?:-(\d{1,2})(?:[ T].*)?)?)?", re.S)


def date(s):
    if s is None:
        return None
    m = _DATE.fullmatch(s.strip(_WS))
    if not m:
        return None
    y = int(m.group(2)) * (-1 if m.group(1) == b"-" else 1)
    mo, d = int(m.group(3) or 1), int(m.group(4) or 1)
    if not _valid_date(y, mo, d):
        return None
    days = days_from_civil(y, mo, d)
    return days if -2**31 <= days < 2**31 else None
