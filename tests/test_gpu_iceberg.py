"""GPU checks of the Iceberg transforms (srj_b200.iceberg over libsrj_b200.so) against oracle/iceberg.py, which
tests/test_oracle_iceberg.py pins to the Iceberg spec's vectors and an independent per-row model.  Every result is compared
in full: values (offsets and bytes where present), null mask and null count."""
import threading

import numpy as np
import pytest

from oracle import iceberg as O

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
NS = [1, 2, 3, 16, 1024, 2**16, 2**30, 2**30 + 1, INT32_MAX]
FIXED = {O.INT32: "<i4", O.TIMESTAMP_DAYS: "<i4", O.DECIMAL32: "<i4", O.INT64: "<i8", O.TIMESTAMP_MICROSECONDS: "<i8", O.DECIMAL64: "<i8"}


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200 import iceberg as I
    return S, I


def _mask(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _valid(rng, rows, frac):
    return None if frac is None else rng.random(rows) >= frac


def _strings(rows):
    data = b"".join(rows)
    offs = np.concatenate([[0], np.cumsum([len(r) for r in rows], dtype=np.int64)]).astype(np.int32)
    return np.frombuffer(data, np.uint8).copy(), offs


def _dec128(vals):
    return np.array([[v % 2**64, (v >> 64) % 2**64] for v in vals], dtype=np.uint64).view(np.uint8).reshape(-1)


def _dev(S, type_id, data, valid, rows, offsets=None, scale=0):
    mask = _mask(valid) if valid is not None else None
    if type_id == O.LIST:
        import torch
        child = S.ColumnVector.from_numpy(S.DType.UINT8, data, size=len(data))
        return S.ColumnVector(S.DType.LIST, rows, None, None if mask is None else torch.from_numpy(mask.view(np.int32).copy()).cuda(),
                              torch.from_numpy(offsets.copy()).cuda(), child)
    return S.ColumnVector.from_numpy(type_id, data, mask, offsets=offsets, scale=scale, size=rows)


def _check_meta(S, out, inp, rows, type_id):
    assert out.size == rows and out.dtype.type_id == type_id
    if inp.mask is None:
        assert out.mask is None
    else:
        want = np.unpackbits(inp.mask.cpu().numpy().view(np.uint8), bitorder="little")[:rows]
        got = np.unpackbits(out.mask.cpu().numpy().view(np.uint8), bitorder="little")[:rows]
        assert np.array_equal(got, want)
    assert out.getNullCount() == inp.getNullCount()


def _fixed_values(rng, dt, rows):
    info = np.iinfo(np.dtype(dt))
    edge = np.array([0, 1, -1, info.min, info.max, info.min + 1, info.max - 1], dtype=dt)
    v = rng.integers(info.min, info.max, rows, dtype=np.dtype(dt).type, endpoint=True).astype(dt)
    v[: min(rows, len(edge))] = edge[: min(rows, len(edge))]
    return v


# ---- bucket -------------------------------------------------------------------------------------------------------------
def _check_bucket(S, I, type_id, data, valid, rows, n, offsets=None):
    col = _dev(S, type_id, data, valid, rows, offsets)
    out = I.IcebergBucket.computeBucket(col, n)
    _check_meta(S, out, col, rows, S.DType.INT32)
    got = out.data.cpu().numpy().view(np.int32) if rows else np.zeros(0, np.int32)
    want = O.bucket(type_id, data, _mask(valid) if valid is not None else None, rows, n, offsets)
    assert np.array_equal(got, want), (type_id, n, rows)


@pytest.mark.parametrize("type_id", sorted(FIXED))
@pytest.mark.parametrize("rows", [0, 1, 31, 32, 33, 1000, 4099])
def test_bucket_fixed_width(type_id, rows):
    S, I = _s()
    rng = np.random.default_rng(rows * 31 + type_id)
    data = _fixed_values(rng, FIXED[type_id], rows)
    for n in NS:
        _check_bucket(S, I, type_id, data, _valid(rng, rows, [None, 0.3][n % 2]), rows, n)


def test_bucket_ten_million_longs():
    S, I = _s()
    rng = np.random.default_rng(10)
    rows = 10_000_000
    data = rng.integers(INT64_MIN, INT64_MAX, rows, dtype=np.int64)
    _check_bucket(S, I, O.INT64, data, rng.random(rows) >= 0.1, rows, 16)


def test_bucket_decimals_at_the_byte_boundaries():
    S, I = _s()
    v128 = [0, 1, -1, 2**127 - 1, -2**127, -2**127 + 1]
    for k in range(1, 17):
        v128 += [2**(8 * k - 1) - 1, -2**(8 * k - 1), 2**(8 * k - 1) % 2**127, -(2**(8 * k - 1) + 1) if k < 16 else 0]
    v128 = [((v + 2**127) % 2**128) - 2**127 for v in v128]
    rows = len(v128)
    valid = np.arange(rows) % 5 != 3
    for n in NS:
        _check_bucket(S, I, O.DECIMAL128, _dec128(v128), valid, rows, n)
    v64 = np.array([max(min(v, INT64_MAX), INT64_MIN) for v in v128], dtype=np.int64)
    v32 = np.array([max(min(v, INT32_MAX), INT32_MIN) for v in v128], dtype=np.int32)
    for n in (1, 7, INT32_MAX):
        _check_bucket(S, I, O.DECIMAL64, v64, valid, rows, n)
        _check_bucket(S, I, O.DECIMAL32, v32, valid, rows, n)


def test_bucket_decimal128_at_8_byte_alignment():
    import torch
    S, I = _s()
    rng = np.random.default_rng(3)
    rows = 1001
    raw = rng.integers(0, 256, rows * 16, dtype=np.uint8)
    buf = torch.zeros(rows * 16 + 8, dtype=torch.uint8, device="cuda")
    buf[8:] = torch.from_numpy(raw).cuda()
    col = S.ColumnVector(S.DType.DECIMAL128, rows, buf[8:], None)
    out = I.IcebergBucket.computeBucket(col, 1000)
    assert np.array_equal(out.data.cpu().numpy().view(np.int32), O.bucket(O.DECIMAL128, raw, None, rows, 1000))


@pytest.mark.parametrize("type_id", [O.STRING, O.LIST])
def test_bucket_bytes_every_length_and_alignment(type_id):
    """rows of 0..300 bytes starting at every byte alignment (the pad rows shift the next row's start)"""
    S, I = _s()
    rng = np.random.default_rng(type_id)
    rows = []
    for L in range(301):
        for pad in range(4):
            rows.append(bytes(rng.integers(0, 256, pad, dtype=np.uint8)))
            rows.append(bytes(rng.integers(0, 256, L, dtype=np.uint8)))
    chars, offs = _strings(rows)
    valid = rng.random(len(rows)) >= 0.1
    for n in (1, 16, 1024, INT32_MAX):
        _check_bucket(S, I, type_id, chars, valid, len(rows), n, offs)
    _check_bucket(S, I, type_id, chars, None, len(rows), 2**30 + 1, offs)


@pytest.mark.parametrize("type_id", [O.STRING, O.LIST])
def test_bucket_bytes_one_mebibyte_row_and_empty_rows(type_id):
    S, I = _s()
    rng = np.random.default_rng(5)
    rows = [b"", bytes(rng.integers(0, 256, 2**20 + 3, dtype=np.uint8)), b"", b"x"]
    chars, offs = _strings(rows)
    _check_bucket(S, I, type_id, chars, np.array([True, True, False, True]), len(rows), 97, offs)
    chars, offs = _strings([b""] * 40)                          # no bytes at all
    _check_bucket(S, I, type_id, chars, None, 40, 5, offs)


# ---- truncate -----------------------------------------------------------------------------------------------------------
WIDTHS = [1, -1, 2, -2, 10, -10, 1000, INT32_MAX, INT32_MIN]


@pytest.mark.parametrize("type_id", [O.INT32, O.INT64, O.DECIMAL32, O.DECIMAL64, O.DECIMAL128])
@pytest.mark.parametrize("width", WIDTHS)
def test_truncate_integral(type_id, width):
    S, I = _s()
    rng = np.random.default_rng(abs(width) % 1009 + type_id)
    rows = 3001
    if type_id == O.DECIMAL128:
        vals = [0, 1, -1, 2**127 - 1, -2**127, -2**127 + 1, 5, -5] + \
               [int(rng.integers(-2**62, 2**62)) << int(rng.integers(0, 66)) for _ in range(rows - 8)]
        data = _dec128([((v + 2**127) % 2**128) - 2**127 for v in vals])
    else:
        data = _fixed_values(rng, FIXED[type_id], rows)
    valid = rng.random(rows) >= 0.2
    col = _dev(S, type_id, data, valid, rows, scale=-2)
    out = I.IcebergTruncate.truncate(col, width)
    _check_meta(S, out, col, rows, type_id)
    assert out.dtype.scale == -2
    assert np.array_equal(out.data.cpu().numpy(), O.truncate_integral(type_id, data, _mask(valid), rows, width))


@pytest.mark.parametrize("rows", [0, 1, 3, 33])
def test_truncate_integral_small_and_empty(rows):
    S, I = _s()
    rng = np.random.default_rng(rows)
    for type_id in (O.INT32, O.INT64, O.DECIMAL128):
        data = rng.integers(0, 256, rows * (16 if type_id == O.DECIMAL128 else 4 if type_id == O.INT32 else 8), dtype=np.uint8)
        col = _dev(S, type_id, data, None, rows)
        out = I.IcebergTruncate.truncate(col, 7)
        assert out.size == rows
        got = out.data.cpu().numpy() if rows else np.zeros(0, np.uint8)
        assert np.array_equal(got, O.truncate_integral(type_id, data, None, rows, 7))


CHARS = ["a", "Z", "é", "ж", "€", "中", "😀", "𝄞"]
MALFORMED = [b"\x80\x80abc", b"\xc3", b"ab\xe2\x82", b"\xff\xfe\xfd\xfc\xfb", b"\xbf" * 9, b"a\x80b\x80c\x80d\x80",
             b"\xf0\x9f\x98", b"\xe2\x82\xac\x80\x80\x80z"]


def _utf8_rows(rng, count, max_chars):
    rows = [("".join(rng.choice(CHARS, int(rng.integers(0, max_chars))))).encode() for _ in range(count)]
    return rows + MALFORMED + [b"", "€".encode() * 5, "😀".encode() * 5, b"abcd", b"abcde"]


def _check_truncate_bytes(S, I, type_id, chars, offs, valid, width):
    rows = len(offs) - 1
    col = _dev(S, type_id, chars, valid, rows, offs)
    out = I.IcebergTruncate.truncate(col, width)
    _check_meta(S, out, col, rows, type_id)
    want_off, want = O.truncate_bytes(type_id, chars, offs, _mask(valid) if valid is not None else None, rows, width)
    assert np.array_equal(out.offsets.cpu().numpy(), want_off)
    got = (out.data if type_id == O.STRING else out.child.data).cpu().numpy()
    assert np.array_equal(got, want)
    if type_id == O.LIST:
        assert out.child.mask is None and out.child.size == len(want)


@pytest.mark.parametrize("type_id", [O.STRING, O.LIST])
@pytest.mark.parametrize("width", [1, 2, 3, 4, 5, 16, 1000, INT32_MAX])
def test_truncate_bytes(type_id, width):
    S, I = _s()
    rng = np.random.default_rng(width % 1013 + type_id)
    rows = _utf8_rows(rng, 3000, 24)
    rows += [bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)) for _ in range(300)]
    rows += [("".join(rng.choice(CHARS, 700))).encode()]          # long rows: the warp copies them
    chars, offs = _strings(rows)
    valid = rng.random(len(rows)) >= 0.15                         # null rows over non-empty bytes
    _check_truncate_bytes(S, I, type_id, chars, offs, valid, width)
    _check_truncate_bytes(S, I, type_id, chars, offs, None, width)


def test_truncate_string_cuts_at_and_inside_characters():
    S, I = _s()
    rows = [s.encode() for s in ["ab€cd", "€€€", "😀a😀", "aé", "éa", "𝄞𝄞𝄞𝄞", "a" * 17, "€" * 17]]
    chars, offs = _strings(rows)
    for width in range(1, 7):
        _check_truncate_bytes(S, I, O.STRING, chars, offs, None, width)


@pytest.mark.parametrize("type_id", [O.STRING, O.LIST])
def test_truncate_bytes_empty_and_one_mebibyte(type_id):
    S, I = _s()
    chars, offs = _strings([])
    col = _dev(S, type_id, chars, None, 0, offs)
    out = I.IcebergTruncate.truncate(col, 3)
    assert out.size == 0 and out.offsets.cpu().numpy().tolist() == [0]
    rng = np.random.default_rng(11)
    big = ("".join(rng.choice(CHARS, 300_000))).encode()
    chars, offs = _strings([b"", big, b"x", big[:1000]])
    for width in (1, 4, 100_000, INT32_MAX):
        _check_truncate_bytes(S, I, type_id, chars, offs, np.array([True, True, False, True]), width)


def test_truncate_twenty_million_strings():
    S, I = _s()
    rng = np.random.default_rng(20)
    rows = 20_000_000
    lens = rng.integers(0, 12, rows)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pool = np.frombuffer("".join(rng.choice(CHARS, 50_000)).encode(), np.uint8)
    chars = np.resize(pool, int(offs[-1]))
    valid = rng.random(rows) >= 0.1
    _check_truncate_bytes(S, I, O.STRING, chars, offs, valid, 4)


# ---- year / month / day / hour --------------------------------------------------------------------------------------------
def _check_datetime(S, I, transform, type_id, data, valid):
    rows = len(data)
    col = _dev(S, type_id, data, valid, rows)
    fn = {"years": I.IcebergDateTimeUtil.yearsFromEpoch, "months": I.IcebergDateTimeUtil.monthsFromEpoch,
          "days": I.IcebergDateTimeUtil.daysFromEpoch, "hours": I.IcebergDateTimeUtil.hoursFromEpoch}[transform]
    out = fn(col)
    _check_meta(S, out, col, rows, S.DType.TIMESTAMP_DAYS if transform == "days" else S.DType.INT32)
    got = out.data.cpu().numpy().view(np.int32) if rows else np.zeros(0, np.int32)
    assert np.array_equal(got, O.datetime_transform(transform, type_id, data, rows)), transform


@pytest.mark.parametrize("transform", ["years", "months", "days", "hours"])
def test_datetime(transform):
    S, I = _s()
    rng = np.random.default_rng(len(transform))
    D, H = 86_400_000_000, 3_600_000_000
    k = rng.integers(-10**6, 10**6, 500)
    micros = np.concatenate([[0, -1, 1, INT64_MIN, INT64_MAX, INT64_MIN + 1, INT64_MAX - 1],
                             k * D, k * D - 1, k * D + 1, k * H, k * H - 1, k * H + 1,
                             rng.integers(INT64_MIN, INT64_MAX, 5000, dtype=np.int64)]).astype(np.int64)
    valid = rng.random(len(micros)) >= 0.2                        # rows under nulls are computed too
    _check_datetime(S, I, transform, O.TIMESTAMP_MICROSECONDS, micros, valid)
    if transform != "hours":
        days = np.concatenate([[0, -1, 1, INT32_MIN, INT32_MAX, INT32_MIN + 1, INT32_MAX - 1, -719162, -719163, 2932896, 2932897],
                               rng.integers(INT32_MIN, INT32_MAX, 5000)]).astype(np.int32)
        _check_datetime(S, I, transform, O.TIMESTAMP_DAYS, days, rng.random(len(days)) >= 0.2)
        _check_datetime(S, I, transform, O.TIMESTAMP_DAYS, days, None)
    for rows in (0, 1, 5, 33):
        _check_datetime(S, I, transform, O.TIMESTAMP_MICROSECONDS, micros[:rows], None)


# ---- errors, streams ----------------------------------------------------------------------------------------------------
def test_errors():
    S, I = _s()
    from srj_b200 import _native as N
    i64 = _dev(S, O.INT64, np.arange(8, dtype=np.int64), None, 8)
    with pytest.raises(ValueError):
        I.IcebergBucket.computeBucket(i64, 0)
    import torch
    int8_list = S.ColumnVector(S.DType.LIST, 1, None, None, torch.tensor([0, 4], dtype=torch.int32, device="cuda"),
                               S.ColumnVector.from_numpy(1, np.zeros(4, np.int8)))   # LIST<INT8>: not binary
    with pytest.raises(N.CudfException):
        I.IcebergBucket.computeBucket(int8_list, 4)
    with pytest.raises(N.CudfException):
        I.IcebergTruncate.truncate(int8_list, 4)
    with pytest.raises(N.CudfException):
        I.IcebergBucket.computeBucket(_dev(S, 10, np.zeros(8, np.float64), None, 8), 4)        # FLOAT64
    with pytest.raises(N.CudfException):
        I.IcebergTruncate.truncate(i64, 0)
    strs = _dev(S, O.STRING, np.frombuffer(b"abc", np.uint8), None, 1, np.array([0, 3], np.int32))
    for w in (0, -1, INT32_MIN):
        with pytest.raises(N.CudfException):
            I.IcebergTruncate.truncate(strs, w)
    with pytest.raises(ValueError):
        I.IcebergTruncate.truncate(_dev(S, 10, np.zeros(8, np.float64), None, 8), 3)
    with pytest.raises(ValueError):
        I.IcebergDateTimeUtil.hoursFromEpoch(_dev(S, O.TIMESTAMP_DAYS, np.zeros(4, np.int32), None, 4))
    with pytest.raises(ValueError):
        I.IcebergDateTimeUtil.yearsFromEpoch(i64)


def test_threads_each_on_its_own_stream():
    import torch
    S, I = _s()
    rng = np.random.default_rng(8)
    rows = 200_003
    data = rng.integers(INT64_MIN, INT64_MAX, rows, dtype=np.int64)
    strs = _utf8_rows(rng, 20000, 20)
    chars, offs = _strings(strs)
    want_b = O.bucket(O.INT64, data, None, rows, 1000)
    want_o, want_c = O.truncate_bytes(O.STRING, chars, offs, None, len(strs), 3)
    want_h = O.datetime_transform("hours", O.TIMESTAMP_MICROSECONDS, data, rows)
    errors = []

    def work(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(3):
                    b = I.IcebergBucket.computeBucket(_dev(S, O.INT64, data, None, rows), 1000)
                    t = I.IcebergTruncate.truncate(_dev(S, O.STRING, chars, None, len(strs), offs), 3)
                    h = I.IcebergDateTimeUtil.hoursFromEpoch(_dev(S, O.TIMESTAMP_MICROSECONDS, data, None, rows))
                    torch.cuda.current_stream().synchronize()
                    assert np.array_equal(b.data.cpu().numpy().view(np.int32), want_b)
                    assert np.array_equal(t.offsets.cpu().numpy(), want_o) and np.array_equal(t.data.cpu().numpy(), want_c)
                    assert np.array_equal(h.data.cpu().numpy().view(np.int32), want_h)
        except Exception as e:   # noqa: BLE001 - reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
