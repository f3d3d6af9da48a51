"""GPU checks of Arithmetic (srj_b200.arithmetic over libsrj_b200.so) against oracle/arithmetic.py, which
tests/test_oracle_arithmetic.py pins to the reference's tests and an independent integer / fraction model.  Values are
compared bit for bit (a NaN matches any NaN), masks bit for bit over the rows, null counts and the ANSI error row exactly.
Values under null output rows: 0 for multiply, computed from the input's bits for round."""
import zlib

import numpy as np
import pytest

from golden import arithmetic_golden as G
from oracle import arithmetic as A

pytestmark = pytest.mark.gpu

TYPES = {"INT8": (1, np.int8), "INT16": (2, np.int16), "INT32": (3, np.int32), "INT64": (4, np.int64), "FLOAT32": (9, np.float32),
         "FLOAT64": (10, np.float64), "BOOL8": (11, np.uint8), "DECIMAL32": (25, np.int32), "DECIMAL64": (26, np.int64),
         "DECIMAL128": (27, np.uint64)}


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200 import arithmetic as AR
    from srj_b200.bloom import Scalar
    return S, AR, Scalar


def _mask(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _dev(type_id, data, valid=None, scale=0, shift=0):
    """A device column; shift > 0 places the data `shift` elements into its buffer (a sliced, unaligned view)."""
    import torch
    S, _, _ = _s()
    raw = np.ascontiguousarray(data).view(np.uint8).reshape(-1)   # DECIMAL128: (rows, 2) uint64
    rows = len(data)
    width = raw.size // max(rows, 1) if rows else 0
    off = shift * min(width, 8)                                   # DECIMAL128 shifts by 8 bytes, its alignment
    buf = torch.zeros(raw.size + off + 16, dtype=torch.uint8, device="cuda")
    buf[off: off + raw.size] = torch.from_numpy(raw.copy()).cuda()
    view = buf[off: off + raw.size]
    mask = torch.from_numpy(_mask(valid).view(np.int32).copy()).cuda() if valid is not None else None
    nulls = int(len(valid) - np.count_nonzero(valid)) if valid is not None else 0
    return S.ColumnVector(S.DType(type_id, scale), rows, view, mask, null_count=nulls)


def _host(col, t):
    d = col.data.cpu().numpy().view(np.uint8)
    vals = d.view(t) if d.size else np.zeros(0, t)
    if col.mask is None:
        return vals, np.ones(col.size, bool)
    bits = np.unpackbits(col.mask.cpu().numpy().view(np.uint8), bitorder="little")[:col.size].astype(bool)
    return vals, bits


def _same_bits(got, want):
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype.kind == "f":
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        got, want = got[~nan], want[~nan]
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


# ---- multiply ----------------------------------------------------------------------------------------------------------
def _random(t, n, rng):
    if np.dtype(t).kind == "f":
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 30, n)
        return x.astype(t)
    info = np.iinfo(t)
    x = rng.integers(info.min, info.max, n, dtype=np.int64, endpoint=True)
    return (x >> rng.integers(0, 8 * np.dtype(t).itemsize - 1, n)).astype(t)      # magnitudes of every size


def _check_mul(S, AR, Scalar, name, t, a, va, b, vb, ansi, try_mode, ls=False, rs=False, shift=0):
    type_id = TYPES[name][0]
    want, wvalid, werr = A.multiply(a, va, b, vb, ansi, try_mode, ls, rs)

    def operand(x, v, scalar):
        if scalar:
            return Scalar._fixed(type_id, x[0].item() if v else None)
        return _dev(type_id, x, v, shift=shift)
    left, right = operand(a, va, ls), operand(b, vb, rs)
    if werr >= 0:
        with pytest.raises(AR.ExceptionWithRowIndex) as e:
            AR.Arithmetic.multiply(left, right, ansi, try_mode)
        assert e.value.getRowIndex() == werr
        return
    out = AR.Arithmetic.multiply(left, right, ansi, try_mode)
    vals, valid = _host(out, t)
    assert np.array_equal(valid, wvalid)
    assert out.getNullCount() == int(len(wvalid) - wvalid.sum())
    _same_bits(vals, want)


@pytest.mark.parametrize("case", G.MULTIPLY, ids=lambda c: c[0])
def test_multiply_goldens(case):
    S, AR, Scalar = _s()
    name, typ, left, right, ansi, try_mode, want = case
    lt, rt = typ if isinstance(typ, tuple) else (typ, typ)

    def operand(x, tn):
        type_id, t = TYPES[tn]
        if isinstance(x, tuple):
            return Scalar._fixed(type_id, x[1])
        return _dev(type_id, np.array([0 if v is None else v for v in x], t), np.array([v is not None for v in x]))
    if want == "error":
        with pytest.raises(S.CudfException):
            AR.Arithmetic.multiply(operand(left, lt), operand(right, rt), ansi, try_mode)
        return
    if isinstance(want, tuple):
        with pytest.raises(AR.ExceptionWithRowIndex) as e:
            AR.Arithmetic.multiply(operand(left, lt), operand(right, rt), ansi, try_mode)
        assert e.value.getRowIndex() == want[1]
        return
    t = TYPES[lt][1]
    vals, valid = _host(AR.Arithmetic.multiply(operand(left, lt), operand(right, rt), ansi, try_mode), t)
    assert [v.item() if ok else None for v, ok in zip(vals, valid)] == [None if w is None else t(w).item() for w in want]


@pytest.mark.parametrize("name", ["INT8", "INT16", "INT32", "INT64", "FLOAT32", "FLOAT64"])
@pytest.mark.parametrize("mode", ["wrap", "try", "ansi"])
@pytest.mark.parametrize("shape", ["cc", "cs", "sc"])
@pytest.mark.parametrize("null_frac", [0.0, 0.1, 1.0])
def test_multiply_types_modes_shapes(name, mode, shape, null_frac):
    S, AR, Scalar = _s()
    t = TYPES[name][1]
    rng = np.random.default_rng(zlib.crc32(f"{name}{mode}{shape}{null_frac}".encode()))
    n = 5000
    a, b = _random(t, n, rng), _random(t, n, rng)
    va = rng.random(n) >= null_frac if null_frac else None
    vb = rng.random(n) >= null_frac if null_frac else None
    ansi, try_mode = mode == "ansi", mode == "try"
    if shape == "cc":
        _check_mul(S, AR, Scalar, name, t, a, va, b, vb, ansi, try_mode)
        return
    for scalar_valid in (True, False):
        s = _random(t, 1, rng)
        if shape == "cs":
            _check_mul(S, AR, Scalar, name, t, a, va, s, scalar_valid, ansi, try_mode, rs=True)
        else:
            _check_mul(S, AR, Scalar, name, t, s, scalar_valid, b, vb, ansi, try_mode, ls=True)


@pytest.mark.parametrize("n", [1, 31, 33, 2**20 + 7])
@pytest.mark.parametrize("name", ["INT32", "INT64", "INT8"])
def test_multiply_overflow_positions(n, name):
    S, AR, Scalar = _s()
    t = TYPES[name][1]
    hi = np.iinfo(t).max
    rng = np.random.default_rng(n)
    a = rng.integers(-3, 4, n).astype(t)
    b = rng.integers(-3, 4, n).astype(t)
    for pos in sorted({0, n - 1, n // 2}):
        a2 = a.copy()
        a2[pos] = hi
        va = np.ones(n, bool)
        b2 = b.copy()
        b2[pos] = 2
        _check_mul(S, AR, Scalar, name, t, a2, None, b2, None, True, False)             # the error row
        _check_mul(S, AR, Scalar, name, t, a2, None, b2, None, False, True)             # a null row
        if pos + 1 < n:                                                                 # the row after a null
            a3, b3 = a2.copy(), b2.copy()
            a3[pos + 1], b3[pos + 1] = hi, 3
            va[pos] = False
            _check_mul(S, AR, Scalar, name, t, a3, va, b3, None, True, False)
        vb = np.ones(n, bool)                                                           # overflow only under nulls
        vb[pos] = False
        _check_mul(S, AR, Scalar, name, t, a2, None, b2, vb, True, False)


@pytest.mark.parametrize("n", [0, 1, 31, 33, 2**20 + 7])
@pytest.mark.parametrize("shift", [0, 1, 3])
@pytest.mark.parametrize("name", ["INT8", "INT16", "INT64", "FLOAT32"])
def test_multiply_row_counts_and_unaligned(n, shift, name):
    S, AR, Scalar = _s()
    t = TYPES[name][1]
    rng = np.random.default_rng(n + shift)
    a, b = _random(t, n, rng), _random(t, n, rng)
    va = rng.random(n) > 0.1
    _check_mul(S, AR, Scalar, name, t, a, va, b, None, False, True, shift=shift)
    _check_mul(S, AR, Scalar, name, t, a, None, b, None, False, False, shift=shift)


def test_multiply_output_past_2_31_bytes():
    import torch
    S, AR, Scalar = _s()
    n = 2**28 + 5                                              # 8 bytes a row: the output passes 2^31 bytes
    a = torch.arange(n, dtype=torch.int64, device="cuda") - n // 2
    b = (torch.arange(n, dtype=torch.int64, device="cuda") % 7) - 3
    ca = S.ColumnVector(S.DType(4), n, a.view(torch.uint8), None, null_count=0)
    cb = S.ColumnVector(S.DType(4), n, b.view(torch.uint8), None, null_count=0)
    out = AR.Arithmetic.multiply(ca, cb, True, False)
    got = out.data.view(torch.int64)
    assert out.mask is None and out.getNullCount() == 0
    assert torch.equal(got, a * b)
    tail = slice(n - 1000, n)
    want, _, _ = A.multiply(a[tail].cpu().numpy(), None, b[tail].cpu().numpy(), None, True, False)
    assert np.array_equal(got[tail].cpu().numpy(), want)
    a[n - 3] = 2**62                                            # the last rows overflow: the error names the first
    b[n - 3] = 4
    with pytest.raises(AR.ExceptionWithRowIndex) as e:
        AR.Arithmetic.multiply(ca, cb, True, False)
    assert e.value.getRowIndex() == n - 3


# ---- round -------------------------------------------------------------------------------------------------------------
def _float_values(t, n, rng):
    tiny = np.finfo(t).smallest_subnormal
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, tiny, -tiny, tiny * 3, np.finfo(t).tiny, np.finfo(t).max, -np.finfo(t).max,
                         0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 1.25, 0.125, 12345.675, -12345.675, 1.234, 25.66, 154.9, 2346.0], t)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 25, n)
    halves = (rng.integers(-10**6, 10**6, n) + 0.5) / 10.0 ** rng.integers(0, 4, n)
    raw = rng.integers(0, 2**32 if t == np.float32 else 2**63, n, dtype=np.uint64)
    rand = raw.astype(np.uint32).view(np.float32) if t == np.float32 else raw.view(np.float64)
    return np.concatenate([specials, x.astype(t), halves.astype(t), rand.astype(t)])


def _int_values(t, n, rng):
    info = np.iinfo(t)
    edges = [info.min, info.min + 1, info.max, info.max - 1, 0, 1, -1, 5, -5, 15, -15, 25, -25, 125, -125, 126, -126]
    x = _random(t, n, rng)
    return np.concatenate([np.array(edges, np.int64).astype(t), x])


DPS = [-20, -19, -10, -3, -1, 0, 1, 2, 10, 40]


def _check_round(S, AR, name, vals, valid, dp, mode, ansi, scale=0, shift=0):
    type_id, t = TYPES[name]
    if type_id == 27:
        want, werr = A.round_decimal128(vals, scale, dp, mode), -1
    else:
        want, werr = A.round_(vals, valid, dp, mode, ansi, type_id=type_id if type_id in (25, 26) else None, scale=scale)
    col = _dev(type_id, vals, valid, scale=scale, shift=shift)
    if werr >= 0:
        with pytest.raises(AR.ExceptionWithRowIndex) as e:
            AR.Arithmetic.round(col, dp, AR.RoundMode(mode), ansi)
        assert e.value.getRowIndex() == werr
        return
    out = AR.Arithmetic.round(col, dp, AR.RoundMode(mode), ansi)
    got, gvalid = _host(out, t)
    n = len(valid) if valid is not None else (len(vals))
    assert np.array_equal(gvalid, valid if valid is not None else np.ones(n, bool))
    if type_id in (25, 26, 27) and n:
        assert out.dtype.scale == -dp
    _same_bits(got.reshape(-1), np.asarray(want).reshape(-1))


@pytest.mark.parametrize("name", ["INT8", "INT16", "INT32", "INT64", "FLOAT32", "FLOAT64"])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("dp", DPS)
def test_round_numbers(name, mode, dp):
    S, AR, _ = _s()
    t = TYPES[name][1]
    rng = np.random.default_rng(abs(dp) * 7 + mode)
    vals = _float_values(t, 3000, rng) if np.dtype(t).kind == "f" else _int_values(t, 3000, rng)
    valid = rng.random(len(vals)) > 0.1
    for ansi in (False, True):
        _check_round(S, AR, name, vals, valid, dp, mode, ansi)
        if np.dtype(t).kind == "i" and dp < 0:                       # only safe values: the ANSI pass returns a column
            mn, mx = np.iinfo(t).min // 2, np.iinfo(t).max // 2
            _check_round(S, AR, name, np.clip(vals, mn, mx).astype(t), valid, dp, mode, ansi)


@pytest.mark.parametrize("name", ["DECIMAL32", "DECIMAL64", "DECIMAL128"])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("scale", [-4, 0, 3])
def test_round_decimals(name, mode, scale):
    S, AR, _ = _s()
    type_id, t = TYPES[name]
    rng = np.random.default_rng(type_id * 10 + mode + scale)
    n = 2000
    if type_id == 27:
        vals = [int(x) for x in rng.integers(-2**62, 2**62, n)] + [(-1) ** i * (10 ** 37 + 5 * 10 ** (i % 30)) for i in range(200)]
        vals += [-(1 << 127), (1 << 127) - 1, 0, 5, -5, 15, -15, 25, -25]
        data = A.ints_to_dec128(vals)
    else:
        info = np.iinfo(t)
        edges = np.array([info.min, info.max, 0, 5, -5, 15, -15, 25, -25, 10 ** (9 if t == np.int32 else 18) - 1], np.int64).astype(t)
        data = np.concatenate([edges, _random(t, n, rng)])
    rows = len(data)
    valid = rng.random(rows) > 0.1
    for dp in DPS + [4, -4]:                                      # scale up, down, the same (dp = -scale) and zero-fill
        _check_round(S, AR, name, data, valid, dp, mode, False, scale=scale)


@pytest.mark.parametrize("n", [0, 1, 31, 33, 2**20 + 7])
@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("name,dp", [("INT16", -2), ("INT64", -3), ("FLOAT64", 2), ("FLOAT32", -1), ("DECIMAL128", -2), ("DECIMAL64", 1)])
def test_round_row_counts_and_unaligned(n, shift, name, dp):
    S, AR, _ = _s()
    type_id, t = TYPES[name]
    rng = np.random.default_rng(n + shift)
    if type_id == 27:
        vals = A.ints_to_dec128([int(x) for x in rng.integers(-2**62, 2**62, n)])
    elif np.dtype(t).kind == "f":
        vals = (rng.standard_normal(n) * 1000).astype(t)
    else:
        vals = (rng.integers(-10**4, 10**4, n)).astype(t)
    valid = rng.random(n) > 0.1
    _check_round(S, AR, name, vals, valid, dp, 1, True, scale=-2 if type_id in (26, 27) else 0, shift=shift)
    _check_round(S, AR, name, vals, None, dp, 0, False, scale=-2 if type_id in (26, 27) else 0, shift=shift)


@pytest.mark.parametrize("case", G.ROUND, ids=lambda c: c[0])
def test_round_goldens(case):
    S, AR, _ = _s()
    name, typ, scale, vals, dp, mode, ansi, want = case
    type_id, t = TYPES[typ]
    col = _dev(type_id, np.array([0 if v is None else v for v in vals], t), np.array([v is not None for v in vals]), scale=scale)
    if isinstance(want, tuple):
        with pytest.raises(AR.ExceptionWithRowIndex) as e:
            AR.Arithmetic.round(col, dp, AR.RoundMode(mode), ansi)
        assert e.value.getRowIndex() == want[1]
        return
    got, valid = _host(AR.Arithmetic.round(col, dp, AR.RoundMode(mode), ansi), t)
    assert [v.item() if ok else None for v, ok in zip(got, valid)] == [None if w is None else t(w).item() for w in want]


def test_round_rejects_other_types_and_methods():
    S, AR, _ = _s()
    col = _dev(11, np.array([1, 0], np.uint8))
    with pytest.raises(S.CudfException):
        AR.Arithmetic.round(col, 0, AR.RoundMode.HALF_UP)
    with pytest.raises(S.CudfException):
        AR.Arithmetic.round(_dev(3, np.array([1, 2], np.int32)), 0, 7)
    empty = AR.Arithmetic.round(_dev(3, np.zeros(0, np.int32)), 0, 7)   # an empty input returns before any check
    assert empty.size == 0
