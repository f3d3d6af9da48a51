"""Python restatement of CastStrings' string-to-timestamp (first phase) and string-to-date parses (reference
cast_string_to_datetime.cu), quirks included.  Strings are bytes; one row at a time.

parse_timestamp(s, ...) -> (result, seconds, micros, tz_type, tz_offset, tz_index), the six columns of
parseTimestampStringsToIntermediate.  parse_date(s) -> epoch day or None.

Quirks kept: trimming drops bytes <= 32 and 127; fraction digits past 6 are truncated; Spark 3.2.0 reads "+hh:mm" right
after the time with a sign of 1 for '+' and 0 for '-' (cast_string_to_datetime.cu:615, 679); a time alone with a fixed
zone or a named one takes its day from (now + offset) / 86400 truncated toward zero (:796-802, :845-851); a name the map
lacks makes the row invalid but keeps tz type 2 and its seconds (:853-857).  Where the reference is undefined this follows
the device: a tenth segment is dropped, a time alone whose named zone maps outside the table is invalid.
"""
from oracle import timezone as OTZ

SUCCESS, INVALID = 0, 1
TZ_NONE, TZ_FIXED, TZ_OTHER, TZ_INVALID = 0, 1, 2, 3


def version_gates(platform, major, minor, patch):
    """(is_vanilla_320, is_vanilla_400_or_later or is_databricks_14_3_or_later) (version.hpp:64-68)."""
    ge = lambda a, b, c: (major, minor, patch) >= (a, b, c)      # noqa: E731
    return (platform == 0 and (major, minor, patch) == (3, 2, 0),
            (platform == 0 and ge(4, 0, 0)) or (platform == 1 and ge(14, 3, 0)))


def _ws(c):
    return c <= 32 or c == 127


def _trim(s):
    a, e = 0, len(s)
    while a < e and _ws(s[a]):
        a += 1
    while a < e and _ws(s[e - 1]):
        e -= 1
    return a, e


def _digits(s, pos, end, maxd):
    """parse_digits (:177-195) -> (count, value, pos)."""
    v = n = 0
    while pos < end and 48 <= s[pos] <= 57:
        v = v * 10 + s[pos] - 48
        pos += 1
        n += 1
        if n == maxd:
            break
    return n, v, pos


def _offset(s, pos, end, sign, is_320):
    """parse_tz_from_sign (:206-284) -> (type, offset, name bounds)."""
    bad = (TZ_INVALID, 0, None)
    hd, hour, pos = _digits(s, pos, end, 2)
    md = sd = minute = second = 0
    if hd == 0:
        return bad
    if pos < end:
        if s[pos] == ord(":"):
            pos += 1
            md, minute, pos = _digits(s, pos, end, 2)
            if md == 0 or (is_320 and md == 1):
                return bad
            if pos < end:
                if s[pos] != ord(":"):
                    return bad
                sd, second, pos = _digits(s, pos + 1, end, 2)
                if sd != 2 or pos < end:
                    return bad
        else:
            if hd != 2:
                return bad
            md, minute, pos = _digits(s, pos, end, 2)
            sd, second, pos = _digits(s, pos, end, 2)
            if md not in (0, 2) or sd not in (0, 2) or pos < end:
                return bad
    if hour > 18 or minute > 59 or second > 59 or hour * 3600 + minute * 60 + second > 18 * 3600:
        return bad
    if sd > 0 and md != 2:
        return bad
    return (TZ_FIXED, sign * (hour * 3600 + minute * 60 + second), None)


def _zone(s, pos, end, is_320):
    """parse_from_tz / parse_tz / try_parse_UT_tz / try_parse_GMT_tz (:301-448)."""
    while pos < end and _ws(s[pos]):
        pos += 1
    if pos >= end:
        return (TZ_INVALID, 0, None)
    if end - pos == 1 and s[pos] == ord("Z"):
        return (TZ_FIXED, 0, None)
    start, c = pos, s[pos]
    pos += 1
    other = (TZ_OTHER, 0, (start, end))
    if c in b"+-":
        return _offset(s, pos, end, 1 if c == ord("+") else -1, is_320)
    if c == ord("U"):
        if pos >= end:
            return (TZ_INVALID, 0, None)
        if s[pos] != ord("T"):
            return other
        pos += 1
        if pos >= end:
            return (TZ_FIXED, 0, None)
        if s[pos] == ord("C"):
            pos += 1
            if pos >= end:
                return (TZ_FIXED, 0, None)
        if s[pos] in b"+-":
            return _offset(s, pos + 1, end, 1 if s[pos] == ord("+") else -1, is_320)
        return other
    if c == ord("G"):
        if end - pos >= 2 and s[pos] == ord("M") and s[pos + 1] == ord("T"):
            if end - pos == 2:
                return (TZ_FIXED, 0, None)
            pos += 2
            if s[pos] in b"+-":
                return _offset(s, pos + 1, end, 1 if s[pos] == ord("+") else -1, is_320)
            if s[pos] == ord("0") and pos + 1 == end:
                return (TZ_FIXED, 0, None)
        return other
    return other


def _valid_digits(seg, n):
    """is_valid_digits (:491-500)."""
    return seg == 6 or (seg == 0 and 4 <= n <= 6) or (seg == 7 and n <= 2) or (seg not in (0, 6, 7) and 0 < n <= 2)


def _leap(y):
    return (y % 4 == 0 and y % 100 != 0) or y % 400 == 0


def valid_month_day(y, m, d):
    if m < 1 or m > 12 or d < 1:
        return False
    return d <= (29 if _leap(y) else 28) if m == 2 else d <= (30 if m in (4, 6, 9, 11) else 31)


def _w32(v):
    return (v + 2**31) % 2**32 - 2**31


def _tdiv(a, b):
    q = abs(a) // b
    return q if a >= 0 else -q


def parse_string(s, is_320, is_400):
    """parse_timestamp_string (:507-705) -> (ok, just_time, tz, seconds, micros), tz = (type, offset, name bounds)."""
    tz = (TZ_NONE, 0, None)
    pos, end = _trim(s)
    fail = lambda: (False, False, tz, 0, 0)                       # noqa: E731
    if pos >= end:
        return fail()
    n = end - pos
    seg = [1970, 1, 1, 0, 0, 0, 0, 0, 0]
    i = j = frac = 0
    cur = cur_n = 0
    just_time = False
    sign = None
    sign320 = None
    if s[pos] in b"+-":
        sign = -1 if s[pos] == ord("-") else 1
        j = 1
    issue_52351 = is_400 and pos > 0

    def close(k):
        nonlocal cur, cur_n
        if not _valid_digits(k, cur_n):
            return False
        if k < 9:
            seg[k] = _w32(cur)
        cur = cur_n = 0
        return True

    while j < n:
        b = s[pos + j]
        if 48 <= b <= 57:
            if i == 6:
                frac += 1
            if i != 6 or cur_n < 6:
                cur = (cur * 10 + b - 48) % 2**32
            cur_n += 1
        elif j == 0 and b == ord("T") and not issue_52351:
            just_time = True
            i += 3
        elif i < 2:
            if b == ord("-"):
                if not close(i):
                    return fail()
                i += 1
            elif i == 0 and b == ord(":") and sign is None:
                just_time = True
                if not _valid_digits(3, cur_n):
                    return fail()
                seg[3] = _w32(cur)
                cur = cur_n = 0
                i = 4
            else:
                return fail()
        elif i == 2:
            if b not in b" T" or not close(i):
                return fail()
            i += 1
        elif i in (3, 4):
            if b != ord(":") or not close(i):
                return fail()
            i += 1
        elif i in (5, 6):
            if not close(i):
                return fail()
            was = i
            i += 1
            if is_320 and b in b"+-":
                sign320 = 1 if b == ord("+") else 0
            elif not (b == ord(".") and was == 5):
                tz = _zone(s, pos + j, end, is_320)
                if tz[0] == TZ_INVALID:
                    return fail()
                j = n - 1
            if i == 6 and b != ord("."):
                i += 1
        else:
            if i < 9 and b in b": ":
                if not close(i):
                    return fail()
                i += 1
            else:
                return fail()
        j += 1
    if not close(i):
        return fail()
    while frac < 6:
        seg[6] *= 10
        frac += 1
    if sign320 is not None:
        h, m = seg[7], seg[8]
        if h > 18 or m > 59 or h * 3600 + m * 60 > 18 * 3600:
            return fail()
        tz = (TZ_FIXED, sign320 * (h * 3600 + m * 60), None)
    year = seg[0] * (sign or 1)
    if not (-300000 <= year <= 300000) or not valid_month_day(year, seg[1], seg[2]):
        return fail()
    if not (0 <= seg[3] < 24 and 0 <= seg[4] < 60 and 0 <= seg[5] < 60 and 0 <= seg[6] < 10**6) or tz[0] == TZ_INVALID:
        return fail()
    days = int(OTZ.epoch_day(year, seg[1], seg[2]))
    return True, just_time, tz, days * 86400 + seg[3] * 3600 + seg[4] * 60 + seg[5], seg[6]


def lookup(name_map, name):
    """The index of name in the map's sorted (bytes, index) pairs, or -1 (thrust::lower_bound, :810-828)."""
    import bisect
    keys = [k for k, _ in name_map]
    i = bisect.bisect_left(keys, name)
    return name_map[i][1] if i < len(keys) and keys[i] == name else -1


def parse_timestamp(s, default_tz, default_epoch_day, name_map, table, now, is_320, is_400):
    """parse_timestamp_string_fn (:741-864).  s is bytes or None (a null row); name_map sorted (bytes, index) pairs;
    table an oracle.timezone.Table."""
    if s is None:
        return (INVALID, 0, 0, TZ_NONE, 0, -1)
    ok, just_time, tz, sec, us = parse_string(s, is_320, is_400)
    ttype, off = tz[0], tz[1]
    if not ok:
        return (INVALID, sec, us, ttype, off, -1)
    if ttype == TZ_NONE:
        return (SUCCESS, sec + (default_epoch_day * 86400 if just_time else 0), us, TZ_OTHER, 0, default_tz)
    if ttype == TZ_FIXED:
        return (SUCCESS, sec + (_tdiv(now + off, 86400) * 86400 if just_time else 0), us, TZ_FIXED, off, -1)
    idx = lookup(name_map, bytes(s[tz[2][0]:tz[2][1]]))
    if idx < 0:
        return (INVALID, sec, us, TZ_OTHER, 0, -1)
    if just_time:
        if idx >= table.zones:
            return (INVALID, sec, us, TZ_OTHER, 0, idx)
        utc, local, offs, rules = table.zone(idx)
        if len(utc) < 1 or int(table.rule_list[idx + 1] - table.rule_list[idx]) not in (0, 12):
            return (INVALID, sec, us, TZ_OTHER, 0, idx)
        local_now = now + int(OTZ.zone_offset(OTZ.FROM_UTC, [now], utc, local, offs, rules)[0])
        sec += _tdiv(local_now, 86400) * 86400
    return (SUCCESS, sec, us, TZ_OTHER, 0, idx)


def parse_date(s):
    """parse_date + parse_string_to_date_fn (:955-1069): the epoch day, or None for a null row."""
    if s is None:
        return None
    pos, end = _trim(s)
    if pos >= end:
        return None
    neg = s[pos] == ord("-")
    if s[pos] in b"+-":
        pos += 1

    def num(pos, lo, hi):
        v = n = 0
        while pos < end and 48 <= s[pos] <= 57:
            n += 1
            if n > hi:
                return None, pos
            v = v * 10 + s[pos] - 48
            pos += 1
        return (v if n >= lo else None), pos

    year, pos = num(pos, 4, 7)
    if year is None:
        return None
    year = -year if neg else year
    month = day = 1
    if pos < end:
        if s[pos] != ord("-"):
            return None
        month, pos = num(pos + 1, 1, 2)
        if month is None:
            return None
        if pos < end:
            if s[pos] != ord("-"):
                return None
            day, pos = num(pos + 1, 1, 2)
            if day is None:
                return None
            if pos < end and s[pos] not in b" T":
                return None
    if not (-10**7 <= year <= 10**7) or not valid_month_day(year, month, day):
        return None
    days = int(OTZ.epoch_day(year, month, day))
    return days if -2**31 <= days < 2**31 else None
