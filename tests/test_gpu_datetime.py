"""GPU checks of DateTimeUtils through the Python mirror against oracle/datetime.py: values, masks and null counts of the
rebase in both directions and of the truncation with a scalar or a per-row format, over the full int32 day and int64
microsecond ranges and realistic ones, at row counts that end inside a 4-row group and a mask word, with buffers that are
element-aligned but not 16-byte aligned, with no mask, some nulls and all null, a broadcast datetime row, bad formats,
20M rows per kernel, and four host threads on their own streams."""
import threading

import numpy as np
import pytest

from oracle import datetime as O

pytestmark = pytest.mark.gpu

D, U = O.TIMESTAMP_DAYS, O.TIMESTAMP_MICROSECONDS
ROWS = [0, 1, 3, 4, 31, 33, 1_000_003]
FORMATS = ["YEAR", "YYYY", "YY", "QUARTER", "MONTH", "MM", "MON", "WEEK", "DAY", "DD", "HOUR", "MINUTE", "SECOND", "MILLISECOND",
           "MICROSECOND"]


@pytest.fixture(scope="module")
def S():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200
    return srj_b200


def _dtype(t):
    return np.int32 if t == D else np.int64


def _values(t, n, rng, full):
    if t == D:
        return rng.integers(-2**31, 2**31, n, dtype=np.int64).astype(np.int32) if full else \
            rng.integers(-354285, 47482, n).astype(np.int32)                          # years 1000 .. 2100
    if full:
        return rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64, endpoint=True)
    return rng.integers(-354285 * O.US_PER_DAY, 47482 * O.US_PER_DAY, n, dtype=np.int64)


def _valid(n, rng, kind):
    if kind == "none":
        return None
    if kind == "all":
        return np.zeros(n, bool)
    return rng.random(n) >= 0.2


def _pack(valid):
    if valid is None:
        return None
    bits = np.zeros(((len(valid) + 31) // 32) * 32, np.uint8)
    bits[:len(valid)] = valid
    return np.packbits(bits, bitorder="little").view(np.uint32)


def _col(S, t, vals, valid, misalign=False):
    import torch
    c = S.ColumnVector.from_numpy(t, vals, _pack(valid), size=len(vals))
    if misalign and len(vals):
        w = vals.itemsize
        buf = torch.empty(len(vals) * w + w, dtype=torch.uint8, device="cuda")
        buf[w:] = c.data
        c = S.ColumnVector(S.DType(t), len(vals), buf[w:], c.mask)
        assert c.data.data_ptr() % 16 != 0
    return c


def _host(c, t):
    n = c.size
    vals = c.data.cpu().numpy().view(_dtype(t))[:n] if n else np.zeros(0, _dtype(t))
    if c.mask is None:
        return vals, None
    bits = np.unpackbits(c.mask.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
    return vals, bits


def _check_rebase(S, direction, t, vals, valid, misalign=False):
    from srj_b200.datetime import DateTimeUtils
    fn = DateTimeUtils.rebaseGregorianToJulian if direction == 0 else DateTimeUtils.rebaseJulianToGregorian
    out = fn(_col(S, t, vals, valid, misalign))
    got, gmask = _host(out, t)
    assert out.dtype.type_id == t and out.size == len(vals)
    assert np.array_equal(got, O.rebase(direction, t, vals))                      # every row, null or not
    if valid is None:
        assert gmask is None and out.getNullCount() == 0
    else:
        assert np.array_equal(gmask, valid) and out.getNullCount() == int((~valid).sum())


def _check_trunc(out, t, want, wvalid):
    got, gmask = _host(out, t)
    assert np.array_equal(got, want)
    nulls = int((~wvalid).sum())
    assert out.getNullCount() == nulls
    if nulls == 0:
        assert gmask is None
    else:
        assert np.array_equal(gmask, wvalid)


@pytest.mark.parametrize("t", [D, U])
@pytest.mark.parametrize("direction", [0, 1])
@pytest.mark.parametrize("n", ROWS)
def test_rebase_rows_and_masks(S, t, direction, n):
    rng = np.random.default_rng(n * 4 + direction * 2 + (t == U))
    for full in (True, False):
        for kind in ("none", "some", "all"):
            _check_rebase(S, direction, t, _values(t, n, rng, full), _valid(n, rng, kind), misalign=(kind == "some"))


@pytest.mark.parametrize("t", [D, U])
def test_rebase_edges(S, t):
    if t == D:
        v = np.array([-2**31, -2**31 + 1, 2**31 - 1, 2**31 - 719469, 2**31 - 719468, -141428, -141427, -141426, 13_890_324, -719162,
                      -354285, 0, -1], np.int32)
    else:
        v = np.array([-2**63, -2**63 + 1, 2**63 - 1, O.GREGORIAN_START_US - 1, O.GREGORIAN_START_US, -1, 0, 1,
                      -62135593076345679, -12219292799000001], np.int64)
    for direction in (0, 1):
        _check_rebase(S, direction, t, v, None)


@pytest.mark.parametrize("t", [D, U])
@pytest.mark.parametrize("n", ROWS)
def test_truncate_scalar_every_format(S, t, n):
    from srj_b200.datetime import DateTimeUtils
    rng = np.random.default_rng(100 + n)
    for full in (True, False):
        vals = _values(t, n, rng, full)
        valid = _valid(n, rng, "some")
        for i, f in enumerate(FORMATS + ["bogus", "", "hour"]):
            fmt = f.lower() if i % 2 else f
            col = _col(S, t, vals, valid if i % 3 else None, misalign=(i % 4 == 1))
            want, wvalid = O.truncate_scalar(t, vals, valid if i % 3 else None, fmt)
            _check_trunc(DateTimeUtils.truncate(col, fmt), t, want, wvalid)


def test_truncate_scalar_all_null_and_none_format(S):
    from srj_b200.datetime import DateTimeUtils
    rng = np.random.default_rng(3)
    for t in (D, U):
        vals = _values(t, 33, rng, True)
        for valid, fmt in ((np.zeros(33, bool), "MONTH"), (None, None), (None, "HOUR" if t == D else "WEEKS")):
            want, wvalid = O.truncate_scalar(t, vals, valid, fmt)
            _check_trunc(DateTimeUtils.truncate(_col(S, t, vals, valid), fmt), t, want, wvalid)


def _fmt_col(S, formats):
    bs = [b"" if f is None else (f.encode() if isinstance(f, str) else f) for f in formats]
    offs = np.zeros(len(bs) + 1, np.int32)
    offs[1:] = np.cumsum([len(b) for b in bs])
    chars = np.frombuffer(b"".join(bs), np.uint8) if offs[-1] else np.zeros(0, np.uint8)
    valid = np.array([f is not None for f in formats], bool)
    return S.ColumnVector.from_numpy(S.DType.STRING, chars, _pack(valid) if not valid.all() else None, offs)


def _mixed_formats(n, rng):
    pool = []
    for f in FORMATS:
        pool += [f, f.lower(), f.title(), "".join(c.lower() if j % 2 else c for j, c in enumerate(f))]
    pool += ["", "Y", "YEARS", "MICROSECONDS", "QUARTERQUART", "ÿear", "yéar", b"\xff\xfe", "MONTH\x00", " DAY", None]
    idx = rng.integers(0, len(pool), n)
    return [pool[i] for i in idx]


@pytest.mark.parametrize("t", [D, U])
@pytest.mark.parametrize("n", ROWS)
def test_truncate_column(S, t, n):
    from srj_b200.datetime import DateTimeUtils
    rng = np.random.default_rng(200 + n)
    formats = _mixed_formats(n, rng)
    for full, kind in ((True, "none"), (False, "some"), (True, "all")):
        vals = _values(t, n, rng, full)
        valid = _valid(n, rng, kind)
        want, wvalid = O.truncate_column(t, vals, valid, formats)
        _check_trunc(DateTimeUtils.truncate(_col(S, t, vals, valid, misalign=(kind == "some")), _fmt_col(S, formats)), t, want, wvalid)


@pytest.mark.parametrize("t", [D, U])
def test_truncate_column_broadcast(S, t):
    from srj_b200.datetime import DateTimeUtils
    rng = np.random.default_rng(9)
    formats = _mixed_formats(1000, rng)
    for valid in (None, np.array([True]), np.array([False])):
        vals = _values(t, 1, rng, False)
        want, wvalid = O.truncate_column(t, vals, valid, formats)
        _check_trunc(DateTimeUtils.truncate(_col(S, t, vals, valid), _fmt_col(S, formats)), t, want, wvalid)


def test_truncate_column_errors(S):
    import srj_b200 as SS
    from srj_b200.datetime import DateTimeUtils
    rng = np.random.default_rng(4)
    with pytest.raises(SS.CudfException):
        DateTimeUtils.truncate(_col(S, U, _values(U, 5, rng, False), None), _fmt_col(S, ["YEAR"] * 4))
    with pytest.raises(SS.CudfException):
        DateTimeUtils.truncate(_col(S, U, _values(U, 4, rng, False), None), _col(S, U, _values(U, 4, rng, False), None))
    with pytest.raises(SS.CudfException):
        DateTimeUtils.rebaseGregorianToJulian(S.ColumnVector.from_numpy(S.DType.INT64, np.zeros(4, np.int64)))


def test_time_format_on_days_is_null(S):
    from srj_b200.datetime import DateTimeUtils
    vals = np.arange(-50, 50, dtype=np.int32) * 1000
    for f in ("HOUR", "day", "MicroSecond"):
        out = DateTimeUtils.truncate(_col(S, D, vals, None), f)
        _check_trunc(out, D, np.zeros(100, np.int32), np.zeros(100, bool))
        out = DateTimeUtils.truncate(_col(S, D, vals, None), _fmt_col(S, [f] * 100))
        _check_trunc(out, D, np.zeros(100, np.int32), np.zeros(100, bool))


@pytest.mark.parametrize("kernel", ["rebase_days", "rebase_micros", "trunc_scalar", "trunc_column"])
def test_twenty_million_rows(S, kernel):
    from srj_b200.datetime import DateTimeUtils
    n = 20_000_000
    rng = np.random.default_rng(20)
    t = D if kernel == "rebase_days" else U
    vals = _values(t, n, rng, kernel != "trunc_column")
    valid = _valid(n, rng, "some")
    col = _col(S, t, vals, valid)
    if kernel.startswith("rebase"):
        got, gmask = _host(DateTimeUtils.rebaseJulianToGregorian(col), t)
        assert np.array_equal(got, O.rebase(1, t, vals)) and np.array_equal(gmask, valid)
    elif kernel == "trunc_scalar":
        want, wvalid = O.truncate_scalar(t, vals, valid, "month")
        _check_trunc(DateTimeUtils.truncate(col, "month"), t, want, wvalid)
    else:
        # formats drawn from a pool, built and checked with numpy (a Python list of 20M strings would dominate the test)
        pool = [f.lower() if k else f for f in FORMATS for k in (0, 1)] + ["", "YEARS", "yéar"]
        idx = rng.integers(0, len(pool), n)
        bs = [p.encode() for p in pool]
        mat = np.zeros((len(pool), 12), np.uint8)
        for i, b in enumerate(bs):
            mat[i, :len(b)] = np.frombuffer(b, np.uint8)
        lens = np.array([len(b) for b in bs], np.int64)[idx]
        offs = np.zeros(n + 1, np.int32)
        offs[1:] = np.cumsum(lens)
        chars = mat[idx][np.arange(12)[None, :] < lens[:, None]]
        fcol = S.ColumnVector.from_numpy(S.DType.STRING, chars, None, offs)
        codes = np.array([O.parse_format(p) for p in pool])[idx]
        wvalid = valid & np.isin(codes, [c for c in range(O.INVALID) if O.fits(c, t)])
        want = np.zeros(n, np.int64)
        for c in np.unique(codes[wvalid]):
            sel = wvalid & (codes == c)
            want[sel] = O.trunc_values(t, vals[sel], int(c))
        _check_trunc(DateTimeUtils.truncate(col, fcol), t, want, wvalid)


def test_four_threads_own_streams(S):
    import torch
    from srj_b200.datetime import DateTimeUtils
    errors = []

    def work(k):
        try:
            rng = np.random.default_rng(300 + k)
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                for i in range(5):
                    vals = _values(U, 100_003, rng, True)
                    valid = _valid(100_003, rng, "some")
                    got, _ = _host(DateTimeUtils.rebaseGregorianToJulian(_col(S, U, vals, valid)), U)
                    assert np.array_equal(got, O.rebase(0, U, vals))
                    formats = _mixed_formats(100_003, rng)
                    out = DateTimeUtils.truncate(_col(S, U, vals, valid), _fmt_col(S, formats))
                    stream.synchronize()
                    want, wvalid = O.truncate_column(U, vals, valid, formats)
                    _check_trunc(out, U, want, wvalid)
        except Exception as e:            # noqa: BLE001 - reported below
            errors.append(e)

    th = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
