"""numpy restatement of GpuTimeZoneDB's conversions (reference timezones.cu, datetime_utils.cuh:278-588), quirks included.

A time zone table is held as the flat arrays of its two LIST columns:
    list      int32[zones + 1]  offsets of each zone's entries
    utc       int64[entries]    utcInstant, seconds (entry 0 of a zone is INT64_MIN)
    local     int64[entries]    localInstant: utc + offsetAfter for a gap, utc + offsetBefore for an overlap
    off       int32[entries]    offsetAfter, seconds
    rule_list int32[zones + 1]  offsets of each zone's DST integers (0 or 12)
    rules     int32[...]        (month, dayOfMonthIndicator, dayOfWeek 0=Mon..6 / -1, secondsFromMidnight, before, after) x 2

Quirks kept: the seconds of a value are truncated toward zero (a negative sub-second value just below an instant takes the
offset at it); rules are evaluated for the year of the compared seconds, which from UTC is the UTC year; the year's day
count is taken as an int32; the micros overflow check tests `micros >= 224192` at the minimum second; ORC tables give the
raw offset from their last transition on.
"""
import numpy as np

TO_UTC, FROM_UTC = 0, 1
TIMESTAMP_SECONDS, TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS, TIMESTAMP_NANOSECONDS = 13, 14, 15, 16
UNITS = {TIMESTAMP_SECONDS: 1, TIMESTAMP_MILLISECONDS: 1000, TIMESTAMP_MICROSECONDS: 10**6, TIMESTAMP_NANOSECONDS: 10**9}
I64 = np.int64
INT32_MIN = -(2**31)


def _w32(x):
    """int64 -> the int32 it wraps to."""
    return np.asarray(x, I64).astype(np.int32).astype(I64)


def _tdiv(a, b):
    """C's truncating division of int64 arrays by a positive constant."""
    a = np.asarray(a, I64)
    q = a // b
    return q + ((a % b != 0) & (a < 0))


def epoch_day(year, month, day):
    """date_time_utils::to_epoch_day with its int32 / uint32 widths."""
    year, month, day = (np.asarray(v, I64) for v in (year, month, day))
    y = _w32(year - (month <= 2))
    era = _tdiv(np.where(y >= 0, y, y - 399), 400)
    yoe = (y - era * 400) & 0xFFFFFFFF
    t = _w32(153 * np.where(month > 2, month - 3, month + 9))
    doy = _w32(_tdiv(_w32(t + 2), 5) + day - 1) & 0xFFFFFFFF
    doe = (yoe * 365 + yoe // 4 - yoe // 100 + doy) & 0xFFFFFFFF
    return era * 146097 + doe - 719468


def days_in_month(year, month):
    year, month = np.asarray(year, I64), np.asarray(month, I64)
    leap = ((np.fmod(year, 4) == 0) & (np.fmod(year, 100) != 0)) | (np.fmod(year, 400) == 0)
    return np.where(month == 2, np.where(leap, 29, 28), np.where(np.isin(month, (4, 6, 9, 11)), 30, 31))


def weekday(days):
    return np.fmod(np.asarray(days, I64) - (INT32_MIN - 8), 7)


def year_of(seconds):
    """date_time_utils::get_year: the proleptic Gregorian year of floor(s / 86400), the day count as an int32."""
    z = _w32(np.asarray(seconds, I64) // 86400) + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    m = np.where(mp < 10, mp + 3, mp - 9)
    return yoe + era * 400 + (m <= 2)


def rule_instant(year, rule):
    """create_transition_info: the UTC second of a rule (month, dom, dow, time, before, after) in year."""
    month, dom, dow, time, before, _ = (int(v) for v in rule)
    year = np.asarray(year, I64)
    if dom > 0:
        days = epoch_day(year, month, dom)
        if dow >= 0:
            days = days + 6 - np.fmod(weekday(days) + (6 - dow), 7)
    else:
        days = epoch_day(year, month, _w32(days_in_month(year, month) + 1 + dom))
        if dow >= 0:
            days = days - np.fmod(weekday(days) + (7 - dow), 7)
    return days * 86400 + time - before


def rule_offset(direction, s, r0, r1):
    """get_offset_for_local_time (to UTC) / get_offset_for_utc_time (from UTC) of seconds s."""
    s = np.asarray(s, I64)
    y = year_of(s)
    u0, u1 = rule_instant(y, r0), rule_instant(y, r1)
    if direction == TO_UTC:
        gap = r0[5] > r0[4]
        t0, t1 = u0 + (r0[5] if gap else r0[4]), u1 + (r1[4] if gap else r1[5])
    else:
        t0, t1 = u0, u1
    return np.where(s < t0, r0[4], np.where(s < t1, r0[5], r1[5])).astype(I64)


class Table:
    """The flat arrays of a time zone table (see the module doc)."""

    def __init__(self, list_, utc, local, off, rule_list, rules):
        self.list = np.asarray(list_, np.int32)
        self.utc = np.asarray(utc, I64)
        self.local = np.asarray(local, I64)
        self.off = np.asarray(off, np.int32)
        self.rule_list = np.asarray(rule_list, np.int32)
        self.rules = np.asarray(rules, np.int32)

    @property
    def zones(self):
        return len(self.list) - 1

    def zone(self, i):
        b, e = int(self.list[i]), int(self.list[i + 1])
        rb, re_ = int(self.rule_list[i]), int(self.rule_list[i + 1])
        r = self.rules[rb:re_]
        return self.utc[b:e], self.local[b:e], self.off[b:e], (None if len(r) == 0 else (tuple(r[:6]), tuple(r[6:12])))


def zone_offset(direction, s, utc, local, off, rules):
    """The offset in seconds of each of the seconds s in one zone."""
    s = np.asarray(s, I64)
    inst = local if direction == TO_UTC else utc
    idx = np.maximum(np.searchsorted(inst, s, side="right") - 1, 0)
    o = off[idx].astype(I64)
    if rules is not None:
        m = s > inst[-1]
        if m.any():
            o[m] = rule_offset(direction, s[m], *rules)
    return o


def convert(direction, type_id, values, table, tz_index):
    """convertTimestampColumnToUTC / convertUTCTimestampColumnToTimeZone of int64 values of a timestamp type."""
    unit = UNITS[type_id]
    v = np.asarray(values, I64)
    o = zone_offset(direction, _tdiv(v, unit), *table.zone(tz_index))
    with np.errstate(over="ignore"):
        d = o * I64(unit)
        return v - d if direction == TO_UTC else v + d


def add_micros(seconds, micros):
    """overflow_checker::get_timestamp_overflow -> (result, overflowed)."""
    s = np.asarray(seconds, I64)
    us = np.asarray(micros, I64)
    max_sec, min_sec = (2**63 - 1) // 10**6, -(2**63 // 10**6) - 1
    with np.errstate(over="ignore"):
        res = s * I64(10**6) + us
        inside = (s <= max_sec) & (s >= min_sec)
        pos_ovf = us > I64(2**63 - 1) - np.where(inside & (s > 0), s, 0) * I64(10**6)
    ovf = ~inside | ((s > 0) & pos_ovf) | ((s == min_sec) & (us >= 224192))
    return res, ovf


def convert_multi(seconds, micros, invalid, tz_type, tz_offset, table, tz_indices):
    """convertTimestampColumnToUTCWithTzCv -> (int64 micros, valid bool).  An index outside the table, or a zone without
    entries or with other than 0 or 12 rule integers, is a null row."""
    s = np.asarray(seconds, I64)
    n = len(s)
    conv = np.zeros(n, I64)
    known = np.ones(n, bool)
    fixed = np.asarray(tz_type) == 1
    with np.errstate(over="ignore"):
        conv[fixed] = s[fixed] - np.asarray(tz_offset, I64)[fixed]
    idx = np.asarray(tz_indices, I64)
    for z in np.unique(idx[~fixed]):
        rows = (~fixed) & (idx == z)
        if z < 0 or z >= table.zones:
            known[rows] = False
            continue
        utc, local, off, rules = table.zone(int(z))
        nr = int(table.rule_list[z + 1] - table.rule_list[z])
        if len(utc) < 1 or nr not in (0, 12):
            known[rows] = False
            continue
        with np.errstate(over="ignore"):
            conv[rows] = s[rows] - zone_offset(TO_UTC, s[rows], utc, local, off, rules)
    res, ovf = add_micros(conv, micros)
    valid = known & ~np.asarray(invalid, bool) & ~ovf
    return np.where(valid, res, 0), valid


def orc_offset(t, o, raw, ms):
    """get_transition_index (timezones.cu:258-289)."""
    ms = np.asarray(ms, I64)
    if t is None or len(t) == 0:
        return np.full(ms.shape, raw, I64)
    t, o = np.asarray(t, I64), np.asarray(o, I64)
    i = np.searchsorted(t, ms, side="right")
    inside = i < len(t)
    ic = np.minimum(i, len(t) - 1)
    exact = inside & (t[ic] == ms)
    prev = o[np.maximum(i - 1, 0)]
    return np.where(~inside, raw, np.where(exact, o[ic], np.where(i == 0, raw, prev)))


def convert_orc(us, wt, wo, wraw, rt, ro, rraw):
    """convertOrcTimezones of TIMESTAMP_MICROSECONDS values; a None table is a fixed offset."""
    us = np.asarray(us, I64)
    ms = _tdiv(us, 1000)
    w = orc_offset(wt, wo, wraw, ms)
    r = orc_offset(rt, ro, rraw, ms)
    r2 = orc_offset(rt, ro, rraw, ms + _w32(w - r))
    with np.errstate(over="ignore"):
        return us + _w32(w - r2) * I64(1000)
