"""An independent calendar for the day-count kernels (datetime.cu, iceberg.cu, cast_datetime.cu), built from the
definition of the two calendars and sharing no formula with civil_date.cuh or the oracles.

- Year-start tables: GSTART[y - Y_LO] is the first day (from 1970-01-01) of proleptic Gregorian year y, JSTART the same
  for the Julian calendar.  Each is a cumulative sum of year lengths from the leap rule (floor remainder, astronomical
  year numbering: year 0 exists and is leap in both), anchored at Gregorian 1970-01-01 = day 0 and at Julian
  1582-10-05 = day -141427 (the day after Julian 1582-10-04 is Gregorian 1582-10-15).  The tables reach past every int32
  day count in both directions, so every int32 day, every wrapped (int16) year and every year whose days can be int32
  has an entry.
- Month tables: MSTART[leap * 14 + m] days of the year before month m (m = 1 .. 12; index 13 is the year's length), and
  MONTH_OF_DOY[leap * 366 + doy] the month of a 0-based day of the year.
- A day is located in its year by searchsorted in the year table; a y/m/d becomes a day as year start + month start +
  d - 1, so a day past the end of its month runs on into the next month (Julian 1500-02-29 is 1500-03-01's day).

On top of those, the contracts of DESIGN 3.6j (rebase, truncation, with the int16 year applied explicitly to the
computed year), 3.6h (Iceberg years / months / days / hours, no wrap) and 3.6m (string to date).  Every function takes
numpy int64 arrays (Calendar()) or torch int64 tensors on the calendar's device (Calendar("cuda")).
"""
import numpy as np

US_PER_DAY = 86_400_000_000
US_PER_HOUR = 3_600_000_000
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
US_DAY_LO, US_DAY_HI = INT64_MIN // US_PER_DAY, INT64_MAX // US_PER_DAY      # the days int64 microseconds reach

# A year has at least 365 days, so this many years either side of 1970 spans every int32 day count; _tables() asserts it
Y_SPAN = 2**31 // 365 + 1
Y_LO, Y_HI = 1970 - Y_SPAN, 1970 + Y_SPAN

GREGORIAN_START = -141427                       # 1582-10-15, the first Gregorian day
GREGORIAN_START_US = GREGORIAN_START * US_PER_DAY

# truncation formats, in the order of the kernels' and oracle/datetime.py's codes
YEAR, QUARTER, MONTH, WEEK, DAY, HOUR, MINUTE, SECOND, MILLISECOND, MICROSECOND = range(10)
UNIT_US = {DAY: US_PER_DAY, HOUR: US_PER_HOUR, MINUTE: 60_000_000, SECOND: 1_000_000, MILLISECOND: 1000}

_MONTH_LEN = [31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]


def leap_gregorian(y):
    return ((y % 4 == 0) & (y % 100 != 0)) | (y % 400 == 0)


def leap_julian(y):
    return y % 4 == 0


def _month_tables():
    mstart = np.zeros((2, 14), np.int64)
    month_of_doy = np.zeros((2, 366), np.int64)
    for leap in (0, 1):
        lens = list(_MONTH_LEN)
        lens[1] += leap
        mstart[leap, 1:] = np.cumsum([0] + lens)
        for m in range(1, 13):
            month_of_doy[leap, mstart[leap, m]: mstart[leap, m + 1]] = m
        if not leap:
            month_of_doy[0, 365] = 13          # no such day: a lookup there is a bug of the caller
    return mstart.reshape(-1), month_of_doy.reshape(-1)


MSTART, MONTH_OF_DOY = _month_tables()


def _year_starts(leap, anchor_year, anchor_day):
    years = np.arange(Y_LO, Y_HI + 2, dtype=np.int64)            # one past Y_HI: every year has its end
    starts = np.concatenate([[0], np.cumsum(365 + leap(years[:-1]).astype(np.int64))])
    return starts - starts[anchor_year - Y_LO] + anchor_day


def _tables():
    g = _year_starts(leap_gregorian, 1970, 0)
    j = _year_starts(leap_julian, 1582, GREGORIAN_START - (MSTART[10] + 5 - 1))   # Julian 1582 is common
    for t in (g, j):
        assert t[0] <= INT32_MIN and t[-1] > INT32_MAX + 1, "the year tables must reach past every int32 day"
    return g, j


GSTART, JSTART = _tables()


def wrap16(y):
    """y reduced to int16 (two's complement), as cuda::std::chrono::year stores it"""
    return (y + 2**15) % 2**16 - 2**15


def wrap32(x):
    return (x + 2**31) % 2**32 - 2**31


def _key(y, m, d):
    """a lexicographic order of (y, m, d) for months 1 .. 12 and days 1 .. 31"""
    return (y * 13 + m) * 32 + d


_GAP_LO, _GAP_HI = _key(1582, 10, 4), _key(1582, 10, 15)


class Calendar:
    def __init__(self, device=None):
        self.torch = device is not None
        if self.torch:
            import torch
            self._t = torch
            conv = lambda a: torch.from_numpy(a).to(device)
        else:
            conv = lambda a: a
        self.gstart, self.jstart = conv(GSTART), conv(JSTART)
        self.mstart, self.month_of_doy = conv(MSTART), conv(MONTH_OF_DOY)

    # ---- backend -----------------------------------------------------------------------------------------------------
    def where(self, c, a, b):
        return self._t.where(c, a, b) if self.torch else np.where(c, a, b)

    def clip(self, x, lo, hi):
        return self._t.clamp(x, lo, hi) if self.torch else np.clip(x, lo, hi)

    def _year_index(self, table, days):
        if self.torch:
            return self._t.searchsorted(table, days, right=True) - 1
        return np.searchsorted(table, days, side="right") - 1

    def micros_of_days(self, days, h):
        """Three int64 microseconds per day of days (inside [US_DAY_LO, US_DAY_HI]), interleaved: the day's first, its
        last, and first + h mod the day's length for h >= 0 (int64 cuts the first day at INT64_MIN, the last at
        INT64_MAX)"""
        first = self.where(days == US_DAY_LO, INT64_MIN, days * US_PER_DAY)       # that product wraps; it is not used
        last = self.where(days == US_DAY_HI, INT64_MAX, days * US_PER_DAY + (US_PER_DAY - 1))
        rows = [first, last, first + h % (last - first + 1)]
        return (self._t.stack(rows, 1) if self.torch else np.stack(rows, 1)).reshape(-1)

    # ---- the calendars -----------------------------------------------------------------------------------------------
    def _ymd(self, table, leap, days):
        i = self._year_index(table, days)
        y = i + Y_LO
        doy = days - table[i]
        row = leap(y) * 1
        m = self.month_of_doy[row * 366 + doy]
        return y, m, doy - self.mstart[row * 14 + m] + 1

    def gregorian_ymd(self, days):
        return self._ymd(self.gstart, leap_gregorian, days)

    def julian_ymd(self, days):
        return self._ymd(self.jstart, leap_julian, days)

    def gregorian_day(self, y, m, d):
        """the day of a Gregorian y/m/d (months 1 .. 12, any day >= 1: past the month's end it runs on)"""
        return self.gstart[y - Y_LO] + self.mstart[leap_gregorian(y) * 14 + m] + d - 1

    def julian_day(self, y, m, d):
        return self.jstart[y - Y_LO] + self.mstart[leap_julian(y) * 14 + m] + d - 1

    # ---- DateTimeUtils (DESIGN 3.6j) ---------------------------------------------------------------------------------
    def rebase_g2j_days(self, days, keep_late=True, ymd=None):
        y, m, d = ymd if ymd is not None else self.gregorian_ymd(days)
        wy = wrap16(y)
        k = _key(wy, m, d)
        out = self.julian_day(wy, m, d)
        if keep_late:
            out = self.where(k >= _GAP_HI, days, out)
        return self.where((k > _GAP_LO) & (k < _GAP_HI), GREGORIAN_START, out)

    def rebase_j2g_days(self, days):
        y, m, d = self.julian_ymd(days)
        return self.where(days >= GREGORIAN_START, days, self.gregorian_day(wrap16(y), m, d))

    def rebase_us(self, t, g2j, ymd=None):
        """ymd: the Gregorian y/m/d of t's floored day, when the caller has it"""
        days = t // US_PER_DAY
        tod = t - days * US_PER_DAY
        nd = self.rebase_g2j_days(days, False, ymd) if g2j else self.rebase_j2g_days(days)
        # |nd| < 2^24 (a wrapped year), so nd * US_PER_DAY + tod stays inside int64: no wrap to model
        return self.where(t >= GREGORIAN_START_US, t, nd * US_PER_DAY + tod)

    def trunc_days(self, days, fmt, ymd=None):
        if fmt == WEEK:
            return wrap32(days - (days + 3) % 7)          # 1970-01-01 was a Thursday; no int16 year on this path
        y, m, _ = ymd if ymd is not None else self.gregorian_ymd(days)
        first = {YEAR: 1, QUARTER: (m - 1) // 3 * 3 + 1, MONTH: m}[fmt]
        return self.gregorian_day(wrap16(y), first, 1)

    def trunc_us(self, t, fmt, ymd=None):
        if fmt == MICROSECOND:
            return t
        days = t // US_PER_DAY
        if fmt <= WEEK:
            return self.trunc_days(days, fmt, ymd) * US_PER_DAY
        y, m, d = ymd if ymd is not None else self.gregorian_ymd(days)
        unit = UNIT_US[fmt]
        return self.gregorian_day(wrap16(y), m, d) * US_PER_DAY + (t - days * US_PER_DAY) // unit * unit

    # ---- IcebergDateTimeUtil (DESIGN 3.6h): the true year, no wrap ----------------------------------------------------
    def iceberg_years(self, days, ymd=None):
        y, _, _ = ymd if ymd is not None else self.gregorian_ymd(days)
        return y - 1970

    def iceberg_months(self, days, ymd=None):
        y, m, _ = ymd if ymd is not None else self.gregorian_ymd(days)
        return (y - 1970) * 12 + m - 1

    @staticmethod
    def iceberg_hours(t):
        return wrap32(t // US_PER_HOUR)

    # ---- CastStrings.toDate (DESIGN 3.6m) ----------------------------------------------------------------------------
    def date_of(self, y, m, d):
        """(day, valid) of a y/m/d the grammar accepted: valid when the date exists, |y| <= 10^7 and its day is an int32;
        day 0 where not valid"""
        ok = (m >= 1) & (m <= 12) & (d >= 1) & (y >= -10**7) & (y <= 10**7) & (y >= Y_LO) & (y <= Y_HI)
        yc, mc = self.clip(y, Y_LO, Y_HI), self.clip(m, 1, 12)
        row = leap_gregorian(yc) * 14 + mc
        ok = ok & (d <= self.mstart[row + 1] - self.mstart[row])
        day = self.gregorian_day(yc, mc, self.clip(d, 1, 31))
        ok = ok & (day >= INT32_MIN) & (day <= INT32_MAX)
        return self.where(ok, day, 0), ok


# the string to date cast's grammar branches (unsigned 4 .. 7 digit years, 1-digit month and day, a trailing ' ' or 'T...')
DATE_VARIANTS = [dict(year_digits=4, plus=False), dict(year_digits=5, month_digits=1, day_digits=1),
                 dict(year_digits=6, plus=False, tail=b" "), dict(year_digits=7, day_digits=1, tail=b"T12:34"),
                 dict(year_digits=4, plus=False, month_digits=1, tail=b"T")]


def render(y, m, d, year_digits=7, month_digits=2, day_digits=2, plus=True, tail=b""):
    """Dates as strings, numpy or torch int64 y / m / d in, (chars, lengths) out: chars a (rows, width) uint8 matrix whose
    row r holds lengths[r] bytes.  The year is zero-padded to year_digits (more digits when |y| needs them) after '-' when
    negative and '+' when not and plus; month and day are zero-padded to month_digits / day_digits; tail follows."""
    torch = None if isinstance(y, np.ndarray) else __import__("torch")
    dev = None if torch is None else y.device

    def full(n, v):
        return np.full(n, v, np.int64) if torch is None else torch.full((n,), v, dtype=torch.int64, device=dev)

    rows = y.shape[0]
    a = abs(y)
    ndig = full(rows, 1)
    for k in range(1, 10):
        ndig = ndig + (a >= 10**k) * 1
    ydig = (ndig < year_digits) * (year_digits - ndig) + ndig
    mdig = (m >= 10) * 1 + 1
    mdig = (mdig < month_digits) * (month_digits - mdig) + mdig
    ddig = (d >= 10) * 1 + 1
    ddig = (ddig < day_digits) * (day_digits - ddig) + ddig
    sign = (y < 0) * 1 if not plus else full(rows, 1)
    lengths = sign + ydig + 1 + mdig + 1 + ddig + len(tail)
    width = int(lengths.max())
    if torch is None:
        out = np.full((rows, width), ord(" "), np.uint8)
        r = np.arange(rows, dtype=np.int64)
    else:
        out = torch.full((rows, width), ord(" "), dtype=torch.uint8, device=dev)
        r = torch.arange(rows, dtype=torch.int64, device=dev)
    flat = out.reshape(-1)

    def put(pos, vals, keep=None):
        idx = r * width + pos
        if keep is not None:
            idx, vals = idx[keep], vals[keep]
        flat[idx] = vals.astype(np.uint8) if torch is None else vals.to(torch.uint8)

    def digits(at, v, n, nmax):
        for k in range(nmax):                                    # digit k from the right
            put(at + n - 1 - k, (v // 10**k) % 10 + 48, k < n)

    put(full(rows, 0), (y < 0) * (ord("-") - ord("+")) + ord("+"), sign == 1)
    at = sign
    digits(at, a, ydig, 10)
    at = at + ydig
    put(at, full(rows, ord("-")))
    digits(at + 1, m, mdig, 2)
    at = at + 1 + mdig
    put(at, full(rows, ord("-")))
    digits(at + 1, d, ddig, 2)
    at = at + 1 + ddig
    for i, c in enumerate(tail):
        put(at + i, full(rows, c))
    return out, lengths


def pack(chars, lengths):
    """A STRING column's (chars, int32 offsets) from render()'s matrix: each row's first lengths[r] bytes"""
    if isinstance(chars, np.ndarray):
        keep = np.arange(chars.shape[1])[None, :] < lengths[:, None]
        return chars[keep], np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    import torch
    keep = torch.arange(chars.shape[1], device=chars.device)[None, :] < lengths[:, None]
    offs = torch.zeros(lengths.shape[0] + 1, dtype=torch.int64, device=chars.device)
    offs[1:] = torch.cumsum(lengths, 0)
    return chars[keep], offs.to(torch.int32)
