"""CPU checks of tests/calendar_model.py, the independent calendar behind tests/test_gpu_calendar_every_day.py.

Day sets: every year start -1, 0 and +1 across the int32 day range; every day of years -1000 .. 3000; every day of the
two years either side of each int16 wrap (year 32768 * (2k + 1)) inside the int32 range; the first and last 10^6 int32
days.  On them:
- the Gregorian calendar against numpy datetime64 (a third implementation): year from [Y], month from [M], day of month;
- the Julian calendar against datetime_model.py's Julian day number formulas, vectorised;
- the composed contracts against datetime_model.py in years 1 .. 9999, the hand-derived int16 rows of
  test_oracle_datetime.py and the goldens of golden/datetime_golden.py and golden/iceberg_golden.py;
- oracle/datetime.py and oracle/iceberg.py against the model on every row, and oracle/cast_datetime.parse_date on rendered
  strings (the renderings test_gpu_calendar_every_day.py sends to the kernel among them).
"""
import functools

import numpy as np
import pytest

import calendar_model as K
import cast_datetime_model as CM
import datetime_model as M
from golden import datetime_golden as DG
from golden import iceberg_golden as IG
from oracle import cast_datetime as OC
from oracle import datetime as O
from oracle import iceberg as OI

C = K.Calendar()
STEP = 2**20                     # rows per step: numpy's temporaries stay in cache
D, U = O.TIMESTAMP_DAYS, O.TIMESTAMP_MICROSECONDS
US_DAY_LO, US_DAY_HI = K.US_DAY_LO, K.US_DAY_HI


def _gyear(y):
    return K.GSTART[y - K.Y_LO]


def _every_day(y0, y1):
    """every day of Gregorian years y0 .. y1"""
    return np.arange(_gyear(y0), _gyear(y1 + 1), dtype=np.int64)


def _int32(days):
    return days[(days >= K.INT32_MIN) & (days <= K.INT32_MAX)]


def wrap_years():
    """the years where the int16 year jumps (32768 * (2k + 1) and the year before) whose days are int32"""
    y = 32768 * (2 * np.arange(-200, 200) + 1)
    y = y[(y > K.Y_LO) & (y < K.Y_HI)]
    return y[(_gyear(y - 1) >= K.INT32_MIN) & (_gyear(y + 1) - 1 <= K.INT32_MAX)]


@functools.cache
def day_set(name):
    if name == "year_starts":
        st = K.GSTART[1:-1]
        return _int32(np.stack([st - 1, st, st + 1], 1).reshape(-1))     # sorted: years are longer than 2 days
    if name == "years_-1000_3000":
        return _every_day(-1000, 3000)
    if name == "wrap_years":
        return np.concatenate([_every_day(w - 1, w) for w in wrap_years()])
    assert name == "int32_ends"
    return np.concatenate([np.arange(K.INT32_MIN, K.INT32_MIN + 10**6), np.arange(K.INT32_MAX - 10**6 + 1, K.INT32_MAX + 1)])


SETS = ["year_starts", "years_-1000_3000", "wrap_years", "int32_ends"]


def _steps(days):
    for s in range(0, len(days), STEP):
        yield days[s: s + STEP]


def _differ(what, got, want, inputs):
    bad = np.asarray(got) != np.asarray(want)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        pytest.fail(f"{what}: {int(bad.sum())} rows differ, first input {inputs[i]}: got {got[i]}, want {want[i]}")


def test_set_sizes():
    assert len(day_set("year_starts")) > 3 * 11_700_000
    assert day_set("year_starts").min() < K.INT32_MIN + 366 and day_set("year_starts").max() > K.INT32_MAX - 366
    assert len(wrap_years()) == 180 and 32768 in wrap_years() and -32768 in wrap_years()


def test_year_tables():
    years = np.arange(K.Y_LO, K.Y_HI + 2)
    # numpy's own calendar: datetime64[Y] -> [D] is the Gregorian year start
    _differ("GSTART vs datetime64", K.GSTART, (years - 1970).astype("datetime64[Y]").astype("datetime64[D]").astype(np.int64), years)
    _differ("JSTART vs JDN", K.JSTART, M.julian_jdn(years, 1, 1) - M.JDN_EPOCH, years)
    assert K.leap_gregorian(0) and K.leap_julian(0) and not K.leap_gregorian(-100) and K.leap_julian(-100)
    assert K.leap_gregorian(-400) and not K.leap_gregorian(1900) and K.leap_gregorian(-4) and not K.leap_gregorian(-1)
    assert C.gregorian_day(1582, 10, 15) == C.julian_day(1582, 10, 5) == K.GREGORIAN_START
    assert C.julian_day(1500, 2, 29) == C.julian_day(1500, 3, 1) - 1 and C.gregorian_day(1500, 2, 29) == C.gregorian_day(1500, 3, 1)


@pytest.mark.parametrize("name", SETS)
def test_gregorian_against_datetime64(name):
    for days in _steps(day_set(name)):
        y, m, d = C.gregorian_ymd(days)
        dd = days.astype("datetime64[D]")
        mm = dd.astype("datetime64[M]")
        _differ(f"{name} year", y, dd.astype("datetime64[Y]").astype(np.int64) + 1970, days)
        _differ(f"{name} month", (y - 1970) * 12 + m - 1, mm.astype(np.int64), days)
        _differ(f"{name} day", d, (dd - mm.astype("datetime64[D]")).astype(np.int64) + 1, days)
        _differ(f"{name} day of y/m/d", C.gregorian_day(y, m, d), days, days)


@pytest.mark.parametrize("name", SETS)
def test_julian_against_jdn(name):
    for days in _steps(day_set(name)):
        y, m, d = C.julian_ymd(days)
        wy, wm, wd = M.julian_from_jdn(days + M.JDN_EPOCH)
        _differ(f"{name} julian year", y, wy, days)
        _differ(f"{name} julian month", m, wm, days)
        _differ(f"{name} julian day", d, wd, days)
        _differ(f"{name} julian day of y/m/d", C.julian_day(y, m, d), M.julian_jdn(y, m, d) - M.JDN_EPOCH, days)


# ---- the contracts against datetime_model.py (years 1 .. 9999) ---------------------------------------------------------
FORMATS = ["YEAR", "QUARTER", "MONTH", "WEEK", "DAY", "HOUR", "MINUTE", "SECOND", "MILLISECOND", "MICROSECOND"]
LO, HI = (M.dt.date(1, 1, 1) - M.EPOCH).days + 3, (M.dt.date(9999, 12, 31) - M.EPOCH).days   # j2g moves a day by <= 2


def _days_1_9999():
    rng = np.random.default_rng(11)
    starts = day_set("year_starts")
    return np.concatenate([starts[(starts >= LO) & (starts <= HI)], _every_day(1550, 1650), rng.integers(LO, HI, 30_000)])


def test_contracts_against_datetime_model():
    days = _days_1_9999()
    ymd = C.gregorian_ymd(days)
    checks = {"g2j": (C.rebase_g2j_days(days, True, ymd), M.g2j_day), "j2g": (C.rebase_j2g_days(days), M.j2g_day)}
    for f in range(K.WEEK + 1):
        checks[FORMATS[f]] = (C.trunc_days(days, f, ymd), lambda v, f=f: M.trunc_day(v, FORMATS[f]))
    checks["iceberg years"] = (C.iceberg_years(days, ymd), lambda v: M.greg(v)[0] - 1970)
    checks["iceberg months"] = (C.iceberg_months(days, ymd), lambda v: (M.greg(v)[0] - 1970) * 12 + M.greg(v)[1] - 1)
    for what, (got, fn) in checks.items():
        _differ(what, got, [fn(v) for v in days.tolist()], days)
    rng = np.random.default_rng(12)
    t = np.concatenate([days[:20_000] * M.US + rng.integers(0, M.US, 20_000), days[20_000:30_000] * M.US,
                        days[30_000:40_000] * M.US + M.US - 1])
    _differ("g2j us", C.rebase_us(t, True), [M.g2j_us(v) for v in t.tolist()], t)
    _differ("j2g us", C.rebase_us(t, False), [M.j2g_us(v) for v in t.tolist()], t)
    for f, name in enumerate(FORMATS):
        _differ(name, C.trunc_us(t, f), [M.trunc_us(v, name) for v in t.tolist()], t)
    _differ("iceberg hours", C.iceberg_hours(t), [v // 3_600_000_000 for v in t.tolist()], t)


def _civil(y, m, d):
    return int(C.gregorian_day(np.int64(y), m, d))


@pytest.mark.parametrize("y,wy", [(32767, 32767), (32768, -32768), (-32768, -32768), (-32769, 32767), (40000, -25536),
                                  (-40000, 25536)])
def test_int16_year_rows(y, wy):
    """test_oracle_datetime.py's hand-derived rows: a date in year y behaves as the same month and day in int16(y)."""
    assert K.wrap16(y) == wy
    for m, dd in ((1, 1), (3, 15), (6, 1), (12, 31)):
        d = _civil(y, m, dd)
        v = np.array([d], np.int64)
        want = d if (wy, m, dd) >= (1582, 10, 15) else M.julian_jdn(wy, m, dd) - M.JDN_EPOCH
        assert C.rebase_g2j_days(v)[0] == want
        jd = M.julian_jdn(y, m, dd) - M.JDN_EPOCH
        if jd < K.GREGORIAN_START:
            assert C.rebase_j2g_days(np.array([jd]))[0] == _civil(wy, m, dd)
        assert C.trunc_days(v, K.YEAR)[0] == _civil(wy, 1, 1)
        assert C.trunc_days(v, K.QUARTER)[0] == _civil(wy, (m - 1) // 3 * 3 + 1, 1)
        assert C.trunc_days(v, K.MONTH)[0] == _civil(wy, m, 1)
        assert C.trunc_days(v, K.WEEK)[0] == d - (d + 3) % 7
        assert C.iceberg_years(v)[0] == y - 1970
    assert _civil(40000, 6, 1) == 13_890_324
    assert C.rebase_g2j_days(np.array([13_890_324]))[0] == -10_046_402
    assert C.trunc_days(np.array([13_890_324]), K.YEAR)[0] == -10_046_360


def _golden(vals):
    return np.array([0 if v is None else v for v in vals], np.int64), np.array([v is not None for v in vals])


@pytest.mark.parametrize("case,g2j,micros", [(DG.REBASE_DAYS_G2J, True, False), (DG.REBASE_DAYS_J2G, False, False),
                                             (DG.REBASE_MICROS_G2J, True, True), (DG.REBASE_MICROS_J2G, False, True)])
def test_rebase_goldens(case, g2j, micros):
    v, ok = _golden(case[0])
    want, _ = _golden(case[1])
    got = C.rebase_us(v, g2j) if micros else (C.rebase_g2j_days(v) if g2j else C.rebase_j2g_days(v))
    assert np.array_equal(got[ok], want[ok])


@pytest.mark.parametrize("case,micros", [(DG.TRUNC_DAYS, False), (DG.TRUNC_MICROS, True)])
def test_truncate_goldens(case, micros):
    v, ok = _golden(case[0])
    want, wok = _golden(case[2])
    for i in np.flatnonzero(ok & wok):
        f = O.parse_format(case[1][i])
        got = C.trunc_us(v[i: i + 1], f) if micros else C.trunc_days(v[i: i + 1], f)
        assert got[0] == want[i], (case[0][i], case[1][i])


def test_iceberg_goldens():
    for transform, kind, value, want in IG.DATETIME:
        v = np.array([value], np.int64)
        days = v if kind == "date" else v // K.US_PER_DAY
        got = {"years": lambda: C.iceberg_years(days), "months": lambda: C.iceberg_months(days), "days": lambda: days,
               "hours": lambda: C.iceberg_hours(v)}[transform]()
        assert got[0] == want, (transform, kind, value)


# ---- the oracles against the model, every row ----------------------------------------------------------------------
@pytest.mark.parametrize("name", SETS)
def test_oracles_on_days(name):
    for days in _steps(day_set(name)):
        d32 = days.astype(np.int32)
        ymd = C.gregorian_ymd(days)
        _differ(f"{name} g2j", O.rebase(0, D, d32), C.rebase_g2j_days(days, True, ymd), days)
        _differ(f"{name} j2g", O.rebase(1, D, d32), C.rebase_j2g_days(days), days)
        for f in range(K.WEEK + 1):
            _differ(f"{name} {FORMATS[f]}", O.trunc_values(D, d32, f), C.trunc_days(days, f, ymd), days)
        for tr, want in (("years", C.iceberg_years(days, ymd)), ("months", C.iceberg_months(days, ymd)), ("days", days)):
            _differ(f"{name} iceberg {tr}", OI.datetime_transform(tr, OI.TIMESTAMP_DAYS, d32, len(d32)), want, days)


@pytest.mark.parametrize("name", SETS)
def test_oracles_on_micros(name):
    """Each day of the set that int64 microseconds reach, at its first, last and a pseudo-random microsecond."""
    days = day_set(name)
    days = days[(days >= US_DAY_LO) & (days <= US_DAY_HI)]
    t = C.micros_of_days(days, np.random.default_rng(len(days)).integers(0, 2**62, len(days)))
    for ts in _steps(t):
        ymd = C.gregorian_ymd(ts // K.US_PER_DAY)
        _differ(f"{name} g2j us", O.rebase(0, U, ts), C.rebase_us(ts, True, ymd), ts)
        _differ(f"{name} j2g us", O.rebase(1, U, ts), C.rebase_us(ts, False), ts)
        for f, fname in enumerate(FORMATS):
            _differ(f"{name} {fname} us", O.trunc_values(U, ts, f), C.trunc_us(ts, f, ymd), ts)
        for tr, want in (("years", C.iceberg_years(None, ymd)), ("months", C.iceberg_months(None, ymd)),
                         ("days", ts // K.US_PER_DAY), ("hours", C.iceberg_hours(ts))):
            _differ(f"{name} iceberg {tr} us", OI.datetime_transform(tr, OI.TIMESTAMP_MICROSECONDS, ts, len(ts)), want, ts)


# ---- string to date ------------------------------------------------------------------------------------------------
def _strings(chars, lengths):
    return [bytes(r[:n]) for r, n in zip(chars, lengths)]


def _check_dates(y, m, d, **kw):
    """Rendered y/m/d: the oracle's and the regex model's parse against the model's date_of (the grammar accepts every
    rendering with at most 7 year digits)"""
    day, ok = C.date_of(y, m, d)
    ydig = kw.get("year_digits", 7)
    ok = ok & ((abs(y) < 10**7) & (ydig <= 7))
    want = [int(v) if k else None for v, k in zip(day, ok)]
    strs = _strings(*K.render(y, m, d, **kw))
    for fn in (OC.parse_date, CM.date):
        got = [fn(s) for s in strs]
        bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
        assert not bad, f"{fn.__module__}: {len(bad)} rows differ, first {strs[bad[0]]!r}: got {got[bad[0]]}, want {want[bad[0]]}"
    return ok


def _sample_days(n, seed):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.integers(K.INT32_MIN, K.INT32_MAX, n, endpoint=True), day_set("int32_ends")[::40_000],
                           [K.INT32_MIN, K.INT32_MAX, 0, -1, K.GREGORIAN_START]]).astype(np.int64)


def test_date_strings_fixed_width():
    """The rendering the every-day string sweep sends: +-YYYYYYY-MM-DD, 14 bytes, every row a valid date."""
    y, m, d = C.gregorian_ymd(_sample_days(20_000, 1))
    chars, lengths = K.render(y, m, d)
    assert (lengths == 14).all() and chars.shape[1] == 14
    assert _check_dates(y, m, d).all()


@pytest.mark.parametrize("kw", K.DATE_VARIANTS)
def test_date_string_variants(kw):
    y, m, d = C.gregorian_ymd(_sample_days(5_000, 2))
    assert _check_dates(y, m, d, **kw).all()


def test_impossible_and_boundary_dates():
    """Feb 29 of common years, day 31 of 30-day months, months 00 and 13, day 00: null.  Every y/m/d (day 1 .. 31) of the
    boundary years -5877641 and 5881580: null just past int32.  8-digit years and +-10^7: null."""
    rng = np.random.default_rng(3)
    y = rng.integers(-5_877_641, 5_881_581, 4000)
    common = y[~K.leap_gregorian(y)]
    cases = [(common, 2, 29), (y, 4, 31), (y, 6, 31), (y, 9, 31), (y, 11, 31), (y, 0, 1), (y, 13, 1), (y, 1 + y % 12, 0)]
    for yy, mm, dd in cases:
        mm, dd = np.broadcast_to(mm, yy.shape).astype(np.int64), np.broadcast_to(dd, yy.shape).astype(np.int64)
        assert not _check_dates(yy, mm, dd).any()
    for by, first_ok, last_ok in ((-5_877_641, (6, 23), (12, 31)), (5_881_580, (1, 1), (7, 11))):
        mm, dd = [a.reshape(-1) for a in np.meshgrid(np.arange(1, 13), np.arange(1, 32), indexing="ij")]
        ok = _check_dates(np.full(mm.shape, by), mm, dd)
        inside = [(a, b) for a, b, k in zip(mm, dd, ok) if k]
        assert inside[0] == first_ok and inside[-1] == last_ok
    big = np.array([10**7, -10**7, 12_345_678, 2024, 1970, 9_999_999, -9_999_999])
    ones = np.ones(len(big), np.int64)
    assert not _check_dates(big, ones, ones, year_digits=8).any()
    assert not _check_dates(big[-2:], ones[-2:], ones[-2:]).any()                 # 7 digits, outside int32
