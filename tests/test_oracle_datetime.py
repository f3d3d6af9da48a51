"""CPU checks of oracle/datetime.py: the reference's DateTimeUtilsTest values, agreement with the independent model
(tests/datetime_model.py) on every day of 1582, the century leap days, random days and timestamps of years 1 .. 9999
and negative timestamps with a time of day, and hand-derived rows that pin the int16 year reduction."""
import numpy as np
import pytest

import datetime_model as M
from golden import datetime_golden as G
from oracle import datetime as O

D, U = O.TIMESTAMP_DAYS, O.TIMESTAMP_MICROSECONDS
FORMATS = ["YEAR", "YYYY", "YY", "QUARTER", "MONTH", "MM", "MON", "WEEK", "DAY", "DD", "HOUR", "MINUTE", "SECOND", "MILLISECOND",
           "MICROSECOND"]


def _arr(vals, dtype):
    return np.array([0 if v is None else v for v in vals], dtype), np.array([v is not None for v in vals])


@pytest.mark.parametrize("case,direction,t", [(G.REBASE_DAYS_G2J, 0, D), (G.REBASE_DAYS_J2G, 1, D), (G.REBASE_MICROS_G2J, 0, U),
                                              (G.REBASE_MICROS_J2G, 1, U)])
def test_rebase_goldens(case, direction, t):
    vals, valid = _arr(case[0], np.int32 if t == D else np.int64)
    want, _ = _arr(case[1], vals.dtype)
    assert np.array_equal(O.rebase(direction, t, vals)[valid], want[valid])


@pytest.mark.parametrize("case,t", [(G.TRUNC_DAYS, D), (G.TRUNC_MICROS, U)])
def test_truncate_goldens(case, t):
    vals, valid = _arr(case[0], np.int32 if t == D else np.int64)
    want, wvalid = _arr(case[2], vals.dtype)
    out, ok = O.truncate_column(t, vals, valid, case[1])
    assert np.array_equal(ok, wvalid) and np.array_equal(out, want)


def _check_days(days):
    days = np.asarray(days, np.int64)
    g2j, j2g = O.rebase(0, D, days.astype(np.int32)), O.rebase(1, D, days.astype(np.int32))
    for i, d in enumerate(days.tolist()):
        assert g2j[i] == M.g2j_day(d), d
        assert j2g[i] == M.j2g_day(d), d
    for f in FORMATS[:8]:
        got = O.trunc_values(D, days.astype(np.int32), O.parse_format(f))
        assert got.tolist() == [M.trunc_day(d, f) for d in days.tolist()], f


def test_every_day_of_1582():
    start = (M.dt.date(1582, 1, 1) - M.EPOCH).days
    _check_days(np.arange(start, start + 365))


def test_century_leap_days():
    days = []
    for y in range(100, 2001, 100):
        for m, d in ((2, 28), (3, 1)):
            days.append((M.dt.date(y, m, d) - M.EPOCH).days)
        days.append(days[-1] - 1)            # Feb 29 if Gregorian-leap, else Feb 28 again
    # the Julian Feb 29 of each century year, as a Julian day count
    days += [M.julian_jdn(y, 2, 29) - M.JDN_EPOCH for y in range(100, 2001, 100)]
    _check_days(days)


LO, HI = (M.dt.date(1, 1, 1) - M.EPOCH).days, (M.dt.date(9999, 12, 31) - M.EPOCH).days


def test_random_days_and_micros_years_1_to_9999():
    rng = np.random.default_rng(7)
    # the Julian -> Gregorian direction can move a day by up to 2 days: keep clear of year 1's first days
    _check_days(rng.integers(LO + 3, HI, 100_000))
    t = rng.integers((LO + 3) * M.US, HI * M.US, 100_000)
    g2j, j2g = O.rebase(0, U, t), O.rebase(1, U, t)
    assert g2j.tolist() == [M.g2j_us(v) for v in t.tolist()]
    assert j2g.tolist() == [M.j2g_us(v) for v in t.tolist()]
    for f in FORMATS:
        assert O.trunc_values(U, t[:5000], O.parse_format(f)).tolist() == [M.trunc_us(v, f) for v in t[:5000].tolist()], f


def test_negative_micros_with_time_of_day():
    t = np.array([-1, -86_399_999_999, -86_400_000_001, -12219292800000001, -62135596800000000 + 1, -31_556_889_864_403_199],
                 np.int64)
    assert O.rebase(0, U, t).tolist() == [M.g2j_us(v) for v in t.tolist()]
    assert O.rebase(1, U, t).tolist() == [M.j2g_us(v) for v in t.tolist()]
    for f in FORMATS:
        assert O.trunc_values(U, t, O.parse_format(f)).tolist() == [M.trunc_us(v, f) for v in t.tolist()], f


# ---- the int16 year: hand-derived rows ---------------------------------------------------------------------------------
def _civil(y, m, d):
    """days of a proleptic Gregorian y/m/d, any year (exact)"""
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    return era * 146097 + yoe * 365 + yoe // 4 - yoe // 100 + (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1 - 719468


def _julian(y, m, d):
    return M.julian_jdn(y, m, d) - M.JDN_EPOCH


def test_year_40000_example():
    d = _civil(40000, 6, 1)
    assert d == 13_890_324
    # 40000 - 65536 = -25536: the same month and day in year -25536
    assert O.rebase(0, D, np.array([d], np.int32))[0] == _julian(-25536, 6, 1) == -10_046_402
    assert O.trunc_values(D, np.array([d], np.int32), O.YEAR)[0] == _civil(-25536, 1, 1) == -10_046_360


@pytest.mark.parametrize("y,wy", [(32767, 32767), (32768, -32768), (-32768, -32768), (-32769, 32767), (40000, -25536),
                                  (-40000, 25536)])
def test_int16_year_every_op_and_format(y, wy):
    """A date in year y behaves as the same month and day in year wy = int16(y), for every op and every format."""
    for m, dd in ((1, 1), (3, 15), (6, 1), (12, 31)):
        d, wd = _civil(y, m, dd), _civil(wy, m, dd)
        dv = np.array([d], np.int32)
        # Gregorian -> Julian: reinterpreted in the wrapped year (or unchanged when the wrapped date is late)
        want = d if (wy, m, dd) >= (1582, 10, 15) else _julian(wy, m, dd)
        assert O.rebase(0, D, dv)[0] == want
        # Julian -> Gregorian of a Julian day count in year y: the Gregorian days of the wrapped Julian date
        jd = _julian(y, m, dd)
        if jd < -141427:
            assert O.rebase(1, D, np.array([jd], np.int32))[0] == _civil(wy, m, dd)
        wk = int(O.trunc_values(D, dv, O.WEEK)[0])
        assert wk == d - (d + 3) % 7                                     # WEEK keeps the true day
        assert O.trunc_values(D, dv, O.YEAR)[0] == _civil(wy, 1, 1)
        assert O.trunc_values(D, dv, O.QUARTER)[0] == _civil(wy, (m - 1) // 3 * 3 + 1, 1)
        assert O.trunc_values(D, dv, O.MONTH)[0] == _civil(wy, m, 1)
        tod = 12 * 3_600_000_000 + 34 * 60_000_000 + 56_789_012
        t = np.array([d * M.US + tod], np.int64)
        wbase = wd * M.US
        for f, want in ((O.YEAR, _civil(wy, 1, 1) * M.US), (O.MONTH, _civil(wy, m, 1) * M.US), (O.WEEK, wk * M.US),
                        (O.DAY, wbase), (O.HOUR, wbase + 12 * 3_600_000_000), (O.MINUTE, wbase + tod // 60_000_000 * 60_000_000),
                        (O.SECOND, wbase + tod // 1_000_000 * 1_000_000), (O.MILLISECOND, wbase + tod // 1000 * 1000),
                        (O.MICROSECOND, t[0])):
            assert O.trunc_values(U, t, f)[0] == want, (y, m, dd, f)
        # micros rebase: early-out above 1582-10-15, else through the wrapped date
        if t[0] < O.GREGORIAN_START_US:
            assert O.rebase(0, U, t)[0] == _julian(wy, m, dd) * M.US + tod
            jt = np.array([jd * M.US + tod], np.int64)
            assert O.rebase(1, U, jt)[0] == _civil(wy, m, dd) * M.US + tod


def test_parse_format():
    for f in FORMATS:
        assert O.parse_format(f) != O.INVALID and O.parse_format(f.lower()) == O.parse_format(f)
        assert O.parse_format(f.title()) == O.parse_format(f)
    for bad in ["", "Y", "YEARS", "MICROSECONDS", " YEAR", "YEAR ", "ÿear", "MONTH\x00", "QUARTERQUART", b"\xe9t\xe9", "yéar"]:
        assert O.parse_format(bad) == O.INVALID, bad
    assert not O.fits(O.HOUR, D) and O.fits(O.WEEK, D) and O.fits(O.MICROSECOND, U)
