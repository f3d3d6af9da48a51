"""GPU checks of DecimalUtils.floatingPointToDecimal (srj_b200.decimal over libsrj_b200.so, csrc/float_to_decimal.cu)
against the C restatement of the reference in oracle/float_to_decimal.c, which tests/test_oracle_float_to_decimal.py pins to
the Python restatement, the reference's test and a model of Spark's intent.  Values, masks, null counts and the failure
row are compared bit for bit; the value under a null row is 0."""
import os
import subprocess
import sys
import tempfile
import threading

import numpy as np
import pytest

from golden import float_to_decimal_golden as G
from oracle import float_to_decimal as D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEC32, DEC64, DEC128 = D.F2D_DECIMAL32, D.F2D_DECIMAL64, D.F2D_DECIMAL128
MAXP = D.F2D_MAX_PRECISION


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200.decimal import DecimalUtils
    return S, DecimalUtils


def _words(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _dev(values, valid=None, shift=0):
    """A device column of values; shift > 0 places it `shift` elements into its buffer (not 16-byte aligned)."""
    import torch
    S, _ = _s()
    raw = np.ascontiguousarray(values).view(np.uint8)
    w = values.dtype.itemsize
    buf = torch.zeros(raw.size + shift * w + 16, dtype=torch.uint8, device="cuda")
    if raw.size:
        buf[shift * w: shift * w + raw.size] = torch.from_numpy(raw.copy()).cuda()
    mask = torch.from_numpy(_words(valid).view(np.int32).copy()).cuda() if valid is not None else None
    t = S.DType.FLOAT32 if values.dtype == np.float32 else S.DType.FLOAT64
    nulls = int(len(valid) - np.count_nonzero(valid)) if valid is not None else 0
    return S.ColumnVector(S.DType(t), len(values), buf[shift * w: shift * w + raw.size], mask, null_count=nulls)


def _cast(col, out_type, precision, scale):
    S, DU = _s()
    return DU.floatingPointToDecimal(col, S.DType(out_type, scale), precision)


def _host(res, out_type):
    col = res.result
    d = col.data.cpu().numpy().view(np.uint8)
    vals = d.view(np.int32) if out_type == DEC32 else d.view(np.int64) if out_type == DEC64 else d.reshape(-1, 16)
    valid = np.ones(col.size, bool) if col.mask is None else \
        np.unpackbits(col.mask.cpu().numpy().view(np.uint8), bitorder="little")[:col.size].astype(bool)
    return vals, valid


def _check(values, out_type, precision, scale, valid=None, shift=0, res=None):
    """Cast on the device and compare everything with the C oracle; returns the oracle's (values, validity, failure)."""
    values = np.ascontiguousarray(values)
    if res is None:
        res = _cast(_dev(values, valid, shift), out_type, precision, scale)
    want, wok, wfirst = D.floating_point_to_decimal_c(values, None if valid is None else _words(valid), out_type, precision, scale)
    got, ok = _host(res, out_type)
    bad = np.flatnonzero(ok != wok)
    assert not bad.size, f"validity differs at rows {bad[:5]}: x = {values[bad[:5]]}"
    same = np.all(got == want, axis=1) if out_type == DEC128 else got == want
    bad = np.flatnonzero(~same)
    assert not bad.size, f"values differ at rows {bad[:5]}: x = {values[bad[:5]]}"
    assert res.failureRowId == wfirst
    nulls = int(len(values) - wok.sum())
    assert res.result.getNullCount() == nulls
    assert (res.result.mask is None) == (nulls == 0)
    return want, wok, wfirst


def _ints(vals, out_type):
    return D.to_ints(vals.reshape(-1)) if out_type == DEC128 else [int(v) for v in vals]


# ---- the reference's test and the hand-derived goldens --------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(G.CASES)), ids=[c[0] for c in G.CASES])
def test_goldens(case):
    name, values, out_type, precision, scale, want, failed = G.CASES[case]
    x = np.array(values, np.float32 if name.startswith("f32") else np.float64)
    res = _cast(_dev(x), out_type, precision, scale)
    got, ok = _host(res, out_type)
    assert [v if o else None for v, o in zip(_ints(got, out_type), ok)] == want
    assert (res.failureRowId >= 0) == failed
    _check(x, out_type, precision, scale, res=res)


# ---- every FLOAT32 bit pattern ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_type,precision,scale", [(DEC32, 9, -2), (DEC32, 9, -9), (DEC64, 18, -6), (DEC128, 38, 0), (DEC128, 38, -10)])
def test_every_float32_pattern(out_type, precision, scale):
    """All 2^32 FLOAT32 patterns in chunks of 2^27, against the C oracle.  With one H100 80GB HBM3 (700 W) the five cases
    took 72 s (each DECIMAL32), 83 s (DECIMAL64) and 190 s (each DECIMAL128), about 10 minutes in all, nearly all of it in
    the CPU oracle and the host copies."""
    chunk = 1 << 27
    for start in range(0, 1 << 32, chunk):
        x = (np.arange(chunk, dtype=np.uint64) + start).astype(np.uint32).view(np.float32)
        _check(x, out_type, precision, scale)


# ---- FLOAT64 ---------------------------------------------------------------------------------------------------------
def _configs():
    for t in (DEC32, DEC64, DEC128):
        p = MAXP[t]
        for s in sorted({-p, -p + 1, -(p // 2), -2, -1, 0, 1, 2, 10, 19, 20, 37, 38}):
            yield t, p, s


@pytest.mark.parametrize("out_type,precision,scale", list(_configs()))
def test_float64_random_bits_and_magnitudes(out_type, precision, scale):
    rng = np.random.default_rng(out_type * 1000 + scale + 100)
    n = 1 << 16
    bits = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False).view(np.float64)
    mags = (10.0 ** rng.uniform(-45, 45, n)) * rng.choice([-1.0, 1.0], n)
    near = (np.round(rng.uniform(-1, 1, n) * 10.0 ** rng.integers(0, 20, n)) / 10.0 ** rng.integers(0, 20, n))
    _check(np.concatenate([bits, mags, near]), out_type, precision, scale)


@pytest.mark.parametrize("out_type", [DEC32, DEC64, DEC128])
def test_float64_k_over_10_to_the_d_at_every_scale(out_type):
    """k / 10^d at every Spark scale d = 0 .. the type's maximum precision, and the legacy scales -1 .. -38."""
    p = MAXP[out_type]
    rng = np.random.default_rng(out_type)
    for d in list(range(0, p + 1)) + list(range(-1, -39, -1)):
        k = rng.integers(-(10 ** min(p, 17)), 10 ** min(p, 17), 4096).astype(np.float64)
        x = k / 10.0 ** d if d >= 0 else k * 10.0 ** -d
        x = np.concatenate([x, np.nextafter(x, np.inf), np.nextafter(x, -np.inf)])
        _check(x, out_type, p, -d)


@pytest.mark.parametrize("out_type", [DEC32, DEC64, DEC128])
def test_ties_bounds_whole_numbers_and_specials(out_type):
    p = MAXP[out_type]
    ties = [1.005, 9.95, 0.125, 2.675, 1.115, 0.5, 1.5, 2.5, 0.05, 0.045, 1e-7 * 5, 123456.785]
    whole = [float(2 ** 53 + i) for i in range(-3, 4)] + [2.0 ** 63 * f for f in (1 - 2 ** -53, 1.0, 1 + 2 ** -52)] + [2.0 ** 64, 2.0 ** 127]
    specials = [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072009e-308, 2.2250738585072014e-308, 1.4e-45, np.nan, np.inf, -np.inf,
                1.7976931348623157e308]
    base = np.array(ties + whole + specials, np.float64)
    base = np.concatenate([base, -base])
    for s in range(-p, 39, 3):
        sp = -s
        edge = [10.0 ** (p - sp)] if p - sp < 309 else []
        e = np.array(edge, np.float64)
        x = np.concatenate([base, e, -e, np.nextafter(e, np.inf), np.nextafter(e, 0), -np.nextafter(e, 0)])
        _check(x, out_type, p, s)


def test_decimal128_can_round_edge():
    """10 * |x| * 10^s against 2^127 in double: rows either side of it round or truncate."""
    for s in (0, 5, 10, 20, 30):
        edge = 2.0 ** 127 / 10.0 / 10.0 ** s
        x = np.nextafter(np.full(64, edge), np.inf)
        for i in range(1, 64):
            x[i] = np.nextafter(x[i - 1], 0 if i < 32 else np.inf) if i != 32 else np.nextafter(edge, np.inf)
        x = np.concatenate([x, x * 0.999999, x * 1.000001, -x])
        _check(x, DEC128, 38, -s)


def test_decimal32_int64_intermediate_wraps_inside_the_bound():
    """DECIMAL32 rows where 10 * |x| * 10^s reaches INT32_MAX take the int64 intermediate; some of their wrapped
    results land inside the bound and are valid, as in the reference."""
    rng = np.random.default_rng(32)
    x = np.concatenate([rng.uniform(2.0 ** 31, 2.0 ** 70, 1 << 16), np.ldexp(1.0, np.arange(31, 90)).astype(np.float64)])
    x = np.concatenate([x, -x])
    _, ok, _ = _check(x, DEC32, 9, 0)
    assert ok.sum() > 0 and (~ok).sum() > 0


# ---- the failure row --------------------------------------------------------------------------------------------------
def test_failure_row_is_the_smallest():
    n = 1 << 20
    x = np.full(n, 1.25)
    assert _check(x, DEC64, 10, -2)[2] == -1
    special = np.arange(0, n, 997)
    x[special] = np.array([np.nan, np.inf, -np.inf])[special % 3]
    valid = np.ones(n, bool)
    valid[5::101] = False
    x[5::101] = 1e30                                                          # null rows are not failures
    assert _check(x, DEC64, 10, -2, valid=valid)[2] == -1
    for rows in ([n - 1], [700_000, 300_001, 999_999], [123_457, 1_000_000]):
        y = x.copy()
        y[rows] = 1e9
        assert _check(y, DEC64, 10, -2, valid=valid)[2] == min(rows)


# ---- sizes, alignment, streams ---------------------------------------------------------------------------------------
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_sizes_and_grid_stride_edges():
    S, DU = _s()
    res = _cast(_dev(np.zeros(0, np.float64)), DEC64, 18, -2)
    assert res.result.size == 0 and res.failureRowId == -1 and res.result.getNullCount() == 0
    wave = 8 * 256 * _sm_count()
    rng = np.random.default_rng(7)
    for n in (1, 31, 33, wave - 1, wave, wave + 1, 2 * wave + 5, (1 << 20) + 7):
        x = rng.uniform(-2e7, 2e7, n)
        valid = rng.random(n) > 0.1
        _check(x, DEC64, 9, -2, valid=valid)
        _check(x.astype(np.float32), DEC32, 9, -2, valid=valid, shift=1)


def test_decimal128_output_past_2gib():
    n = (1 << 27) + 5                                                         # 2^31 + 80 output bytes
    x = np.linspace(-1e20, 1e20, n)
    x[-3:] = [1e30, np.nan, 3.25]
    _check(x, DEC128, 38, -10)


def test_unaligned_slice_side_stream_and_threads():
    import torch
    rng = np.random.default_rng(11)
    x = rng.uniform(-1e6, 1e6, 100_003)
    _check(x, DEC128, 38, -10, shift=1)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        res = _cast(_dev(x), DEC64, 18, -3)
        side.synchronize()
    _check(x, DEC64, 18, -3, res=res)
    errors = []

    def work(seed):
        try:
            y = np.random.default_rng(seed).uniform(-1e9, 1e9, 200_000)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(3):
                    r = _cast(_dev(y), DEC64, 10, -2)
                s.synchronize()
            _check(y, DEC64, 10, -2, res=r)
        except Exception as e:                                               # noqa: BLE001 -- reported below
            errors.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


# ---- the benchmark's outputs ------------------------------------------------------------------------------------------
def test_bench_outputs_match_the_oracle():
    with tempfile.TemporaryDirectory() as td:
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_float_to_decimal.py"), "--rows", "100003", "--steps", "1",
                            "--warmup", "0", "--dump-outputs", td], capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stderr
        names = sorted(f[:-4] for f in os.listdir(td) if f.endswith(".npz"))
        assert len(names) == 5
        for name in names:
            z = np.load(os.path.join(td, name + ".npz"))
            t, p, s = (int(v) for v in z["config"])
            want, wok, wfirst = D.floating_point_to_decimal_c(z["input"], None if z["in_mask"].size == 0 else z["in_mask"], t, p, s)
            assert np.array_equal(z["valid"], wok), name
            assert np.array_equal(z["values"].reshape(want.shape), want), name
            assert int(z["failure_row"]) == wfirst, name
