"""The calendar kernels over their whole domain, against tests/calendar_model.py's independent calendar on the device.

- every day: all 2^32 int32 days through the rebase in both directions, truncate to YEAR / QUARTER / MONTH / WEEK (a
  scalar format, then a format column that also holds an invalid name and a time format), and Iceberg years / months /
  days of TIMESTAMP_DAYS.
- every day boundary in microseconds: each of the 2.1e8 days int64 microseconds reach, at its first, its last and one
  pseudo-random microsecond (INT64_MIN and INT64_MAX among them), through the rebase, truncate to each of the 10 formats
  (scalar, then a format column) and Iceberg years / months / days / hours.
- every hour boundary: k * 3.6e9 - 1 and k * 3.6e9 for every k that keeps both in int64, through Iceberg hours, every
  int32 wrap of the hour count included.
- every day as a string: all 2^32 int32 days rendered as +-YYYYYYY-MM-DD through CastStrings.toDate; then dates that do
  not exist in every year of the int32 range, every y/m/d of the two boundary years, 8-digit years, and the grammar's
  other branches on sampled days.
- layout: a chunk of each fixed-width sweep from a buffer off 16-byte alignment (map_rows.cuh's element path) with a
  random mask, and a chunk of strings at an unaligned chars buffer with a random mask.

Values, masks and null counts are compared on the device.  A failing comparison reports its row count and the first
failing input with the kernel's and the model's value.  Each sweep prints its row count, time and peak device memory.
"""
import time

import pytest

import calendar_model as K

pytestmark = pytest.mark.gpu

STEP = 2**24                  # rows per kernel call of the day and hour sweeps
DAY_STEP = 2**22              # days per step of the microsecond sweep (3 rows a day)
STRING_STEP = 2**24           # rows per call of the string sweeps
H = K.US_PER_HOUR
DAY_FORMATS = ["YEAR", "quarter", "Month", "WEEK", "Years", "HOUR"]      # YEAR .. WEEK, then an invalid and a time format
US_FORMATS = ["year", "QUARTER", "mon", "Week", "dd", "Hour", "minute", "SECOND", "MilliSecond", "microsecond", "yyyyy"]
NAMES = ["YEAR", "QUARTER", "MONTH", "WEEK", "DAY", "HOUR", "MINUTE", "SECOND", "MILLISECOND", "MICROSECOND"]


@pytest.fixture(scope="module")
def env():
    import gpu_util
    gpu_util.require_cuda()
    import torch

    import srj_b200 as S
    from srj_b200.cast import CastStrings
    from srj_b200.datetime import DateTimeUtils
    from srj_b200.iceberg import IcebergDateTimeUtil

    class Env:
        pass
    e = Env()
    e.torch, e.S, e.DT, e.ICE, e.CAST = torch, S, DateTimeUtils, IcebergDateTimeUtil, CastStrings
    e.cal = K.Calendar("cuda")
    return e


class Tally:
    """Mismatches of one sweep: per comparison, the rows that differ and the first failing input with got and want."""

    def __init__(self, torch, name):
        self.torch, self.name, self.fails = torch, name, {}
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.time()

    def check(self, what, got, want, inputs):
        """got / want: device tensors of one row each per input; inputs: a tensor or a function of a row index"""
        bad = got.to(self.torch.int64) != want.to(self.torch.int64)
        n = int(bad.sum())
        if n:
            i = int(self.torch.nonzero(bad)[0])
            f = self.fails.setdefault(what, [0, None])
            f[0] += n
            if f[1] is None:
                x = inputs(i) if callable(inputs) else inputs[i].item()
                f[1] = f"first input {x!r}: got {got[i].item()!r}, want {want[i].item()!r}"

    def equal(self, what, got, want):
        if got != want:
            self.fails.setdefault(what, [1, f"got {got!r}, want {want!r}"])

    def done(self, rows):
        self.torch.cuda.synchronize()
        print(f"\n{self.name}: {rows} rows in {time.time() - self.t0:.1f} s, "
              f"peak {self.torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
        if self.fails:
            pytest.fail(f"{self.name}: " + "; ".join(f"{w}: {n} rows differ, {first}" for w, (n, first) in self.fails.items()))


# ---- columns ------------------------------------------------------------------------------------------------------
def _col(e, type_id, data, mask=None, nulls=0):
    return e.S.ColumnVector(e.S.DType(type_id), data.numel(), data.view(e.torch.uint8), mask, null_count=nulls)


def _bits(e, mask, n):
    """the first n bits of int32 mask words as a device bool tensor; all true when mask is None"""
    torch = e.torch
    if mask is None:
        return torch.ones(n, dtype=torch.bool, device="cuda")
    sh = torch.arange(32, dtype=torch.int32, device="cuda")
    return ((mask.view(torch.int32).view(-1, 1) >> sh) & 1).view(-1)[:n].bool()


def _random_mask(e, n, seed):
    torch = e.torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    words = torch.randint(-2**31, 2**31, ((n + 31) // 32,), dtype=torch.int64, device="cuda", generator=g).to(torch.int32)
    return words, n - int(_bits(e, words, n).sum())


def _format_column(e, names, n):
    """A STRING column of n rows cycling through names, and each row's format code (-1: not a format)"""
    torch = e.torch
    bs = [s.encode() for s in names]
    reps = -(-n // len(bs))
    lens = torch.tensor([len(b) for b in bs], dtype=torch.int64, device="cuda").repeat(reps)[:n]
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    chars = torch.frombuffer(bytearray(b"".join(bs)), dtype=torch.uint8).cuda().repeat(reps)
    codes = []
    for s in names:
        u = s.upper()
        u = {"YYYY": "YEAR", "YY": "YEAR", "MM": "MONTH", "MON": "MONTH", "DD": "DAY"}.get(u, u)
        codes.append(NAMES.index(u) if u in NAMES else -1)
    code = torch.tensor(codes, dtype=torch.int64, device="cuda").repeat(reps)[:n]
    col = e.S.ColumnVector(e.S.DType(e.S.DType.STRING), n, chars, None, offs.to(torch.int32), null_count=0)
    return col, code


def _check_truncation(e, tally, what, out, want, valid, inputs, width):
    """a truncation's values (0 under nulls), mask and null count"""
    torch = e.torch
    n = want.numel()
    tally.check(f"{what} value", out.data.view(torch.int64 if width == 8 else torch.int32)[:n], torch.where(valid, want, 0), inputs)
    nulls = int((~valid).sum())
    tally.equal(f"{what} null count", out.getNullCount(), nulls)
    if nulls:
        tally.check(f"{what} mask", _bits(e, out.mask, n), valid, inputs)
    else:
        tally.equal(f"{what} has no mask", out.mask is None, True)


def _check_kept(e, tally, what, out, want, col, inputs, width):
    """a rebase's or an Iceberg transform's values (computed under nulls too) and the input's mask and null count"""
    torch = e.torch
    tally.check(f"{what} value", out.data.view(torch.int64 if width == 8 else torch.int32), want, inputs)
    tally.equal(f"{what} null count", out.getNullCount(), col.getNullCount())
    if col.mask is not None:
        tally.equal(f"{what} mask", torch.equal(out.mask.view(torch.int32)[: col.mask.numel()], col.mask.view(torch.int32)), True)


# ---- every int32 day ----------------------------------------------------------------------------------------------
def _days_calls(e, tally, x64, col, tag=""):
    """every days call on the days x64 (int64) held by col, against the model"""
    cal, torch = e.cal, e.torch
    valid = _bits(e, col.mask, x64.numel())
    ymd = cal.gregorian_ymd(x64)
    _check_kept(e, tally, f"g2j days{tag}", e.DT.rebaseGregorianToJulian(col), cal.rebase_g2j_days(x64, True, ymd), col, x64, 4)
    _check_kept(e, tally, f"j2g days{tag}", e.DT.rebaseJulianToGregorian(col), cal.rebase_j2g_days(x64), col, x64, 4)
    want = {}
    for f in range(K.WEEK + 1):
        want[f] = cal.trunc_days(x64, f, ymd)
        _check_truncation(e, tally, f"trunc {NAMES[f]} days{tag}", e.DT.truncate(col, NAMES[f]), want[f], valid, x64, 4)
    fcol, code = _format_column(e, DAY_FORMATS, x64.numel())
    wf = torch.zeros_like(x64)
    for f, w in want.items():
        wf = torch.where(code == f, w, wf)
    _check_truncation(e, tally, f"trunc format column days{tag}", e.DT.truncate(col, fcol), wf, valid & (code >= 0) & (code <= K.WEEK), x64,
                      4)
    del fcol, code, wf, want
    for what, fn, w in (("years", e.ICE.yearsFromEpoch, cal.iceberg_years(x64, ymd)),
                        ("months", e.ICE.monthsFromEpoch, cal.iceberg_months(x64, ymd)), ("days", e.ICE.daysFromEpoch, x64)):
        _check_kept(e, tally, f"iceberg {what} days{tag}", fn(col), w, col, x64, 4)


def _day_chunk(e, c):
    torch = e.torch
    return torch.arange(STEP, dtype=torch.int64, device="cuda") + (K.INT32_MIN + c * STEP)


def test_every_day(env):
    e = env
    tally = Tally(e.torch, "every int32 day")
    rows = 0
    for c in range(2**32 // STEP):
        x64 = _day_chunk(e, c)
        _days_calls(e, tally, x64, _col(e, e.S.DType.TIMESTAMP_DAYS, x64.to(e.torch.int32)))
        rows += x64.numel()
    assert rows == 2**32
    tally.done(f"2^32 = {rows}")


# ---- every day boundary in microseconds ---------------------------------------------------------------------------
def _micros_chunk(e, d0, n):
    torch = e.torch
    days = torch.arange(n, dtype=torch.int64, device="cuda") + d0
    h = (days * -7046029254386353131) & (2**62 - 1)                  # a per-day pseudo-random offset (the product wraps)
    return e.cal.micros_of_days(days, h)


def _micros_calls(e, tally, t, col, tag=""):
    cal, torch = e.cal, e.torch
    valid = _bits(e, col.mask, t.numel())
    days = t // K.US_PER_DAY
    ymd = cal.gregorian_ymd(days)
    _check_kept(e, tally, f"g2j us{tag}", e.DT.rebaseGregorianToJulian(col), cal.rebase_us(t, True, ymd), col, t, 8)
    _check_kept(e, tally, f"j2g us{tag}", e.DT.rebaseJulianToGregorian(col), cal.rebase_us(t, False), col, t, 8)
    want = {}
    for f in range(K.MICROSECOND + 1):
        want[f] = cal.trunc_us(t, f, ymd)
        _check_truncation(e, tally, f"trunc {NAMES[f]} us{tag}", e.DT.truncate(col, NAMES[f]), want[f], valid, t, 8)
    fcol, code = _format_column(e, US_FORMATS, t.numel())
    wf = torch.zeros_like(t)
    for f, w in want.items():
        wf = torch.where(code == f, w, wf)
    _check_truncation(e, tally, f"trunc format column us{tag}", e.DT.truncate(col, fcol), wf, valid & (code >= 0), t, 8)
    del fcol, code, wf, want
    for what, fn, w in (("years", e.ICE.yearsFromEpoch, cal.iceberg_years(None, ymd)),
                        ("months", e.ICE.monthsFromEpoch, cal.iceberg_months(None, ymd)), ("days", e.ICE.daysFromEpoch, days),
                        ("hours", e.ICE.hoursFromEpoch, cal.iceberg_hours(t))):
        _check_kept(e, tally, f"iceberg {what} us{tag}", fn(col), w, col, t, 4)


def test_every_day_boundary_in_micros(env):
    e = env
    tally = Tally(e.torch, "every day boundary in microseconds")
    rows = 0
    ends = set()
    for d0 in range(K.US_DAY_LO, K.US_DAY_HI + 1, DAY_STEP):
        t = _micros_chunk(e, d0, min(DAY_STEP, K.US_DAY_HI + 1 - d0))
        ends |= {K.INT64_MIN, K.INT64_MAX} & {int(t.min()), int(t.max())}
        _micros_calls(e, tally, t, _col(e, e.S.DType.TIMESTAMP_MICROSECONDS, t))
        rows += t.numel()
    assert rows == 3 * (K.US_DAY_HI - K.US_DAY_LO + 1) and ends == {K.INT64_MIN, K.INT64_MAX}
    tally.done(f"3 x {K.US_DAY_HI - K.US_DAY_LO + 1} days = {rows}")


# ---- every hour boundary --------------------------------------------------------------------------------------------
def test_every_hour_boundary(env):
    e = env
    torch = e.torch
    tally = Tally(torch, "every hour boundary")
    k_lo, k_hi = -((-(K.INT64_MIN + 1)) // H), K.INT64_MAX // H          # k * H - 1 and k * H both inside int64
    rows = 0
    for k0 in range(k_lo, k_hi + 1, STEP // 2):
        k = torch.arange(min(STEP // 2, k_hi + 1 - k0), dtype=torch.int64, device="cuda") + k0
        t = torch.stack([k * H - 1, k * H], 1).view(-1)
        want = K.wrap32(torch.stack([k - 1, k], 1).view(-1))          # by construction, not by division
        out = e.ICE.hoursFromEpoch(_col(e, e.S.DType.TIMESTAMP_MICROSECONDS, t))
        tally.check("iceberg hours", out.data.view(torch.int32), want, t)
        rows += t.numel()
        del k, t, want, out
    assert rows == 2 * (k_hi - k_lo + 1)
    tally.done(f"2 x {k_hi - k_lo + 1} hours = {rows}")


# ---- strings ------------------------------------------------------------------------------------------------------
def _string_col(e, y, m, d, mask=None, nulls=0, shift=0, **kw):
    """(column, rendered matrix, row lengths) of the dates y/m/d; shift places the chars that many bytes into their buffer"""
    torch = e.torch
    chars, lengths = K.render(y, m, d, **kw)
    flat, offs = K.pack(chars, lengths)
    if shift:
        buf = torch.empty(flat.numel() + shift, dtype=torch.uint8, device="cuda")
        buf[shift:] = flat
        flat = buf[shift:]
    col = e.S.ColumnVector(e.S.DType(e.S.DType.STRING), y.numel(), flat, mask, offs, null_count=nulls)
    return col, chars, lengths


def _check_dates(e, tally, what, col, want, valid, chars, lengths):
    torch = e.torch
    n = want.numel()

    def show(i):
        return bytes(chars[i, : int(lengths[i])].cpu().tolist())
    out = e.CAST.toDate(col, False)
    tally.check(f"{what} value", out.data.view(torch.int32)[:n], torch.where(valid, want, 0), show)
    tally.equal(f"{what} null count", out.getNullCount(), int((~valid).sum()))
    tally.check(f"{what} mask", _bits(e, out.mask, n), valid, show)


def test_every_day_as_string(env):
    e = env
    torch = e.torch
    tally = Tally(torch, "every int32 day as +-YYYYYYY-MM-DD")
    rows = 0
    for c in range(2**32 // STRING_STEP):
        x = torch.arange(STRING_STEP, dtype=torch.int64, device="cuda") + (K.INT32_MIN + c * STRING_STEP)
        y, m, d = e.cal.gregorian_ymd(x)
        col, chars, lengths = _string_col(e, y, m, d)
        tally.equal("width", int(lengths.min()) == int(lengths.max()) == 14, True)
        _check_dates(e, tally, "toDate", col, x, torch.ones_like(x, dtype=torch.bool), chars, lengths)
        rows += x.numel()
        del x, y, m, d, col, chars, lengths
    assert rows == 2**32
    tally.done(f"2^32 = {rows}")


def test_impossible_dates(env):
    """Every year of the int32 range: Feb 29 of each common year, Apr / Jun / Sep / Nov 31, months 00 and 13, day 00, all
    null.  Every y/m/d of the boundary years (null just past int32), 8-digit years, +-10^7 and 7-digit years outside
    int32."""
    e = env
    torch = e.torch
    tally = Tally(torch, "impossible dates")
    years = torch.arange(-5_877_641, 5_881_581, dtype=torch.int64, device="cuda")
    common = years[~K.leap_gregorian(years)]
    rows = 0
    for yy, m, d in [(common, 2, 29), (years, 4, 31), (years, 6, 31), (years, 9, 31), (years, 11, 31), (years, 0, 1),
                     (years, 13, 1), (years, None, 0)]:
        for s in range(0, yy.numel(), STRING_STEP):
            y = yy[s: s + STRING_STEP]
            mm = y % 12 + 1 if m is None else torch.full_like(y, m)
            dd = torch.full_like(y, d)
            col, chars, lengths = _string_col(e, y, mm, dd)
            _check_dates(e, tally, f"month {m} day {d}", col, torch.zeros_like(y), torch.zeros_like(y, dtype=torch.bool), chars, lengths)
            rows += y.numel()
    mm, dd = torch.meshgrid(torch.arange(1, 13, device="cuda"), torch.arange(1, 32, device="cuda"), indexing="ij")
    mm, dd = mm.reshape(-1).repeat(2), dd.reshape(-1).repeat(2)
    y = torch.tensor([-5_877_641, 5_881_580], device="cuda").repeat_interleave(12 * 31)
    want, valid = e.cal.date_of(y, mm, dd)
    col, chars, lengths = _string_col(e, y, mm, dd)
    _check_dates(e, tally, "boundary years", col, want, valid, chars, lengths)
    tally.equal("boundary years valid rows", int(valid.sum()), 192 + 193)             # Jun 23 .. Dec 31, Jan 1 .. Jul 11
    big = torch.tensor([10**7, -10**7, 12_345_678, -12_345_678, 2024, 1970, 0, 9_999_999, -9_999_999], device="cuda")
    ones = torch.ones_like(big)
    col, chars, lengths = _string_col(e, big, ones, ones, year_digits=8)
    no = torch.zeros_like(big, dtype=torch.bool)
    _check_dates(e, tally, "8-digit years", col, torch.zeros_like(big), no, chars, lengths)
    col, chars, lengths = _string_col(e, big[-2:], ones[-2:], ones[-2:])
    _check_dates(e, tally, "7-digit years outside int32", col, torch.zeros_like(big[-2:]), no[-2:], chars, lengths)
    rows += y.numel() + big.numel() + 2
    tally.done(rows)


def _sample_days(e, n, seed):
    torch = e.torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randint(K.INT32_MIN, K.INT32_MAX + 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    ends = torch.arange(2**16, dtype=torch.int64, device="cuda")
    return torch.cat([x, ends + K.INT32_MIN, K.INT32_MAX - ends])


@pytest.mark.parametrize("kw", K.DATE_VARIANTS)
def test_date_string_variants(env, kw):
    e = env
    torch = e.torch
    tally = Tally(torch, f"date strings {kw}")
    x = _sample_days(e, 2**22, len(str(kw)))
    y, m, d = e.cal.gregorian_ymd(x)
    col, chars, lengths = _string_col(e, y, m, d, **kw)
    _check_dates(e, tally, "toDate", col, x, torch.ones_like(x, dtype=torch.bool), chars, lengths)
    tally.done(x.numel())


# ---- layout ---------------------------------------------------------------------------------------------------------
def test_layout_unaligned_and_masked(env):
    """The last day chunk (past INT32_MAX - 719468) 4 bytes off 16-byte alignment, the first microsecond chunk (INT64_MIN)
    8 bytes off, and a chunk of strings 4 bytes off, each with a random mask."""
    e = env
    torch = e.torch
    tally = Tally(torch, "unaligned, masked")
    x64 = _day_chunk(e, 2**32 // STEP - 1)
    buf = torch.empty(STEP + 4, dtype=torch.int32, device="cuda")
    buf[1: STEP + 1] = x64.to(torch.int32)
    x = buf[1: STEP + 1]
    assert x.data_ptr() % 16 == 4
    mask, nulls = _random_mask(e, STEP, 1)
    assert 0 < nulls < STEP
    _days_calls(e, tally, x64, _col(e, e.S.DType.TIMESTAMP_DAYS, x, mask, nulls), " (unaligned, masked)")
    t = _micros_chunk(e, K.US_DAY_LO, DAY_STEP)
    buf = torch.empty(t.numel() + 2, dtype=torch.int64, device="cuda")
    buf[1: t.numel() + 1] = t
    tb = buf[1: t.numel() + 1]
    assert tb.data_ptr() % 16 == 8
    mask, nulls = _random_mask(e, t.numel(), 2)
    _micros_calls(e, tally, t, _col(e, e.S.DType.TIMESTAMP_MICROSECONDS, tb, mask, nulls), " (unaligned, masked)")
    s = torch.arange(STEP, dtype=torch.int64, device="cuda") + (K.INT32_MAX - STEP + 1)
    y, m, d = e.cal.gregorian_ymd(s)
    mask, nulls = _random_mask(e, STEP, 3)
    col, chars, lengths = _string_col(e, y, m, d, mask, nulls, shift=4)
    assert col.data.data_ptr() % 16 == 4
    _check_dates(e, tally, "toDate (unaligned, masked)", col, s, _bits(e, mask, STEP), chars, lengths)
    tally.done(x.numel() + t.numel() + s.numel())
