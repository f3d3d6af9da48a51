"""Arithmetic.round at every decimal place, on the inputs where a division or a tie decides the result
(tests/round_cases.py; its CPU checks are tests/test_round_cases.py).

- FLOAT32: all 2^32 bit patterns at every dp in -39 .. 39, +-40, +-45 and +-300, both modes, against round_cases'
  float64 restatement of the recipe on the device.  One chunk again from a buffer 4 bytes off (the scalar path) with a mask.
- FLOAT64: quotients m / n and e / n near midpoints between doubles, e / n near h + 0.5, subnormal quotients, against
  oracle/arithmetic.py.
- INT8 / INT16: every value at every k up to one past the zero fill, ANSI error rows with nulls over overflowing rows.
  INT32: every value at k = 1 .. 10 against a torch int64 model on the device.  INT64: ties at every k = 1 .. 20.
- DECIMAL32: every value at kd = -9 .. 10.  DECIMAL64 / DECIMAL128: ties at every kd, through several input scales.

Values are compared bit for bit (a NaN matches any NaN; -0.0 is not 0.0), and masks, null counts and ANSI rows exactly.
"""
import time

import numpy as np
import pytest

import round_cases as R
from oracle import arithmetic as A

pytestmark = pytest.mark.gpu

CHUNK = 2 ** 28            # rows per kernel call in the 2^32 sweeps
SUB = 2 ** 23              # rows per step of the device reference (keeps the sweeps within ~4 GiB)
MODES = (R.HALF_UP, R.HALF_EVEN)
INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DECIMAL32, DECIMAL64, DECIMAL128 = 1, 2, 3, 4, 9, 10, 25, 26, 27


@pytest.fixture(scope="module")
def env():
    import gpu_util
    gpu_util.require_cuda()
    import torch

    import srj_b200 as S
    from srj_b200 import arithmetic as AR
    return S, AR, torch


def _round(AR, col, dp, mode, ansi=False):
    return AR.Arithmetic.round(col, dp, AR.RoundMode(mode), ansi)


def _bits_differ(torch, got, want):
    """Rows whose bits differ, a NaN matching any NaN."""
    it = torch.int32 if got.element_size() == 4 else torch.int64
    bad = got.view(it) != want.view(it)
    if got.is_floating_point():
        bad &= ~(torch.isnan(got) & torch.isnan(want))
    return bad


def _report(torch, what, got, want, base=0):
    bad = _bits_differ(torch, got, want)
    i = int(torch.nonzero(bad)[0])
    return f"{what}: {int(bad.sum())} rows differ, first row {base + i}: got {got[i].item()!r}, want {want[i].item()!r}"


def _chunk32(torch, c):
    """Bit patterns [c * CHUNK, (c + 1) * CHUNK) as int32, on the device (no sum leaves int32: CHUNK divides 2^31)."""
    base = (c * CHUNK + 2 ** 31) % 2 ** 32 - 2 ** 31
    return torch.arange(CHUNK, dtype=torch.int32, device="cuda") + base


def _col(S, type_id, data, rows, mask=None, nulls=0, scale=0):
    import torch
    return S.ColumnVector(S.DType(type_id, scale), rows, data.view(torch.uint8), mask, null_count=nulls)


def _random_mask(torch, rows, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    words = torch.randint(-2 ** 31, 2 ** 31, ((rows + 31) // 32,), dtype=torch.int64, device="cuda", generator=g).to(torch.int32)
    w = words.to(torch.int64) & 0xffffffff
    ones = sum(((w >> b) & 1).sum() for b in range(32))
    return words, rows - int(ones)


# ---- FLOAT32: every value ---------------------------------------------------------------------------------------------
def _sweep_float32(S, AR, torch, x, col, label):
    """Every dp and mode on one chunk: the kernel on the whole chunk, the reference in SUB-row steps."""
    counts = torch.zeros(len(R.F32_DPS), 2, dtype=torch.int64, device="cuda")
    for i, dp in enumerate(R.F32_DPS):
        outs = {m: _round(AR, col, dp, m) for m in MODES}
        for out in outs.values():
            assert out.size == x.numel()
            if col.mask is not None:
                assert torch.equal(out.mask, col.mask) and out.getNullCount() == col.getNullCount()
        got = {m: o.data.view(torch.float32) for m, o in outs.items()}
        for s in range(0, x.numel(), SUB):
            want = R.round_float32(x[s: s + SUB], dp)
            for m in MODES:
                counts[i, m] += _bits_differ(torch, got[m][s: s + SUB], want[m]).sum()
        del outs, got                                   # before the next dp allocates its two outputs
    if int(counts.sum()):
        i, m = [int(v) for v in torch.nonzero(counts)[0]]
        dp = R.F32_DPS[i]
        got = _round(AR, col, dp, m).data.view(torch.float32)
        for s in range(0, x.numel(), SUB):
            want = R.round_float32(x[s: s + SUB], dp)[m]
            if _bits_differ(torch, got[s: s + SUB], want).any():
                pytest.fail(_report(torch, f"{label} dp={dp} mode={m} (input bits {x[s:s + SUB].view(torch.int32)[0].item():#x}..)",
                                    got[s: s + SUB], want, s))


def test_float32_every_value(env):
    S, AR, torch = env
    t0 = time.time()
    for c in range(2 ** 32 // CHUNK):
        x = _chunk32(torch, c).view(torch.float32)
        _sweep_float32(S, AR, torch, x, _col(S, FLOAT32, x, CHUNK), f"FLOAT32 chunk {c}")
        del x
    torch.cuda.synchronize()
    print(f"\nFLOAT32 sweep: 2^32 rows x {len(R.F32_DPS)} dp x 2 modes in {time.time() - t0:.1f} s, "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def test_float32_chunk_unaligned_with_mask(env):
    """Chunk 11 (0xb0000000 .. 0xbfffffff: -4.7e-10 .. -2) from a buffer 4 bytes off 16-byte alignment, with nulls."""
    S, AR, torch = env
    buf = torch.empty(CHUNK + 4, dtype=torch.float32, device="cuda")
    buf[1: CHUNK + 1] = _chunk32(torch, 11).view(torch.float32)
    x = buf[1: CHUNK + 1]
    assert x.data_ptr() % 16 == 4
    mask, nulls = _random_mask(torch, CHUNK, 11)
    assert 0 < nulls < CHUNK
    _sweep_float32(S, AR, torch, x, _col(S, FLOAT32, x, CHUNK, mask, nulls), "FLOAT32 unaligned, masked")


# ---- FLOAT64: constructed hard cases ----------------------------------------------------------------------------------
def _dev(S, torch, type_id, data, valid=None, scale=0, shift=0):
    """A device column from host data; shift > 0 places it `shift` elements (8 bytes at most) into its buffer."""
    raw = np.ascontiguousarray(data).view(np.uint8).reshape(-1)
    rows = len(data)
    off = shift * min(raw.size // max(rows, 1), 8)
    buf = torch.zeros(raw.size + off + 16, dtype=torch.uint8, device="cuda")
    buf[off: off + raw.size] = torch.from_numpy(raw.copy()).cuda()
    mask, nulls = None, 0
    if valid is not None:
        b = np.packbits(np.asarray(valid, bool), bitorder="little")
        mask = torch.from_numpy(np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.int32).copy()).cuda()
        nulls = int(len(valid) - np.count_nonzero(valid))
    return S.ColumnVector(S.DType(type_id, scale), rows, buf[off: off + raw.size], mask, null_count=nulls)


def _host(torch, out, t):
    return out.data.cpu().numpy().view(t)


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype.kind == "f":
        nan = np.isnan(want)
        bad = (got.view(np.uint8).reshape(len(got), -1) != want.view(np.uint8).reshape(len(want), -1)).any(1) & ~(nan & np.isnan(got))
    else:
        bad = (got.reshape(len(got), -1) != want.reshape(len(want), -1)).any(1)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        pytest.fail(f"{what}: {int(bad.sum())} rows differ, first row {i}: got {got[i]!r}, want {want[i]!r}")


@pytest.mark.parametrize("dp", R.F64_DPS)
def test_float64_hard_cases(env, dp):
    S, AR, torch = env
    rng = np.random.default_rng(abs(dp) * 2 + (dp > 0))
    cases = R.f64_positive_dp(dp) if dp > 0 else R.f64_negative_dp(-dp)
    rand = rng.integers(0, 2 ** 64, 2 ** 18, dtype=np.uint64).view(np.float64)
    vals = np.concatenate(list(cases.values()) + [R.F64_SPECIALS, rand])
    col = _dev(S, torch, FLOAT64, vals)
    for m in MODES:
        _same(_host(torch, _round(AR, col, dp, m), np.float64), A.round_float(vals, dp, m), f"FLOAT64 dp={dp} mode={m}")


# ---- integers ---------------------------------------------------------------------------------------------------------
def _check_int(S, AR, torch, type_id, t, vals, valid, dp, mode, ansi, shift=0):
    want, werr = A.round_int(vals, valid, dp, mode, ansi)
    col = _dev(S, torch, type_id, vals, valid, shift=shift)
    what = f"type {type_id} dp={dp} mode={mode} ansi={ansi}"
    if werr >= 0:
        with pytest.raises(AR.ExceptionWithRowIndex) as e:
            _round(AR, col, dp, mode, ansi)
        assert e.value.getRowIndex() == werr, what
        return
    out = _round(AR, col, dp, mode, ansi)
    _same(_host(torch, out, t), want, what)
    if valid is not None:
        assert torch.equal(out.mask, col.mask) and out.getNullCount() == col.getNullCount()


@pytest.mark.parametrize("type_id,t,zero_at", [(INT8, np.int8, 3), (INT16, np.int16, 5)])
def test_small_ints_every_value(env, type_id, t, zero_at):
    S, AR, torch = env
    info = np.iinfo(t)
    rng = np.random.default_rng(type_id)
    vals = rng.permutation(np.arange(info.min, info.max + 1)).astype(t)
    for k in range(1, zero_at + 2):
        for m in MODES:
            _check_int(S, AR, torch, type_id, t, vals, None, -k, m, False)
            over = _overflow_rows(vals, k, m)
            assert over.any() == (k == 1 or (t == np.int16 and k <= 3))
            _check_int(S, AR, torch, type_id, t, vals, None, -k, m, True)
            valid = rng.random(len(vals)) > 0.1              # nulls over the first three overflowing rows move the error on
            valid[np.flatnonzero(over)[:3]] = False
            _check_int(S, AR, torch, type_id, t, vals, valid, -k, m, True, shift=k % 2)
            valid[over] = False                              # every overflowing row null: the ANSI call returns
            _check_int(S, AR, torch, type_id, t, vals, valid, -k, m, True)


def _overflow_rows(vals, k, mode):
    """Rows whose exact rounded value leaves the type, from Python integers."""
    info = np.iinfo(vals.dtype)
    d = 10 ** k
    out = np.zeros(len(vals), bool)
    for i, v in enumerate(vals.tolist()):
        q, r = divmod(abs(v), d)
        if r > d - r or (r == d - r and (mode == R.HALF_UP or q & 1)):
            q += 1
        x = -q * d if v < 0 else q * d
        out[i] = not info.min <= x <= info.max
    return out


def _round_int_ref(torch, v, k, mode, bits, decimal):
    """round of int64 values v by 10^k, exact: (q * 10^k wrapped to `bits`, outside the type) or, for a decimal, the
    rounded quotient."""
    d = 10 ** k
    mag = v.abs()
    q = mag // d
    r = mag - q * d
    h = d - r
    q = q + ((r > h) | ((r == h) & ((q & 1) == 1 if mode == R.HALF_EVEN else True))).to(torch.int64)
    x = q if decimal else q * d
    x = torch.where(v < 0, -x, x)
    return x, (x > 2 ** (bits - 1) - 1) | (x < -2 ** (bits - 1))


def test_int32_every_value(env):
    S, AR, torch = env
    t0 = time.time()
    big = 2 ** 62
    for c in range(2 ** 32 // CHUNK):
        x = _chunk32(torch, c)
        col = _col(S, INT32, x, CHUNK)
        for k in range(1, 11):
            for m in MODES:
                got = _round(AR, col, -k, m).data.view(torch.int32)
                bad = torch.zeros((), dtype=torch.int64, device="cuda")
                first = torch.full((), big, dtype=torch.int64, device="cuda")
                for s in range(0, CHUNK, SUB):
                    want, ovf = _round_int_ref(torch, x[s: s + SUB].to(torch.int64), k, m, 32, False)
                    bad += (got[s: s + SUB] != want.to(torch.int32)).sum()
                    rows = torch.arange(s, s + SUB, device="cuda")
                    first = torch.minimum(first, torch.where(ovf, rows, big).min())
                if int(bad):
                    pytest.fail(f"INT32 chunk {c} k={k} mode={m}: {int(bad)} rows differ")
                first = int(first)
                if first == big:
                    assert torch.equal(_round(AR, col, -k, m, True).data.view(torch.int32), got)
                else:
                    with pytest.raises(AR.ExceptionWithRowIndex) as e:
                        _round(AR, col, -k, m, True)
                    assert e.value.getRowIndex() == first, f"INT32 chunk {c} k={k} mode={m}"
        del x, col
    torch.cuda.synchronize()
    print(f"\nINT32 sweep: 2^32 rows x 10 k x 2 modes (and the ANSI pass) in {time.time() - t0:.1f} s")


@pytest.mark.parametrize("k", range(1, 21))
def test_int64_ties(env, k):
    S, AR, torch = env
    vals = np.array(R.int_ties(k, -2 ** 63, 2 ** 63 - 1, seed=k), np.int64)
    rng = np.random.default_rng(k)
    vals = rng.permutation(vals)
    for m in MODES:
        safe = vals[~_overflow_rows(vals, k, m)]
        _check_int(S, AR, torch, INT64, np.int64, vals, None, -k, m, False)
        _check_int(S, AR, torch, INT64, np.int64, vals, None, -k, m, True)
        valid = rng.random(len(vals)) > 0.2
        _check_int(S, AR, torch, INT64, np.int64, vals, valid, -k, m, True, shift=1)
        _check_int(S, AR, torch, INT64, np.int64, safe, None, -k, m, True)


def test_int64_at_19_digits(env):
    """k = 19: 10^19 > 2^63, so |v| >= 5 * 10^18 rounds to +-10^19 wrapped, and only +-4999999999999999999 stay in range."""
    S, AR, torch = env
    h = 5 * 10 ** 18
    edge = [h - 1, h, h + 1, 2 ** 63 - 1, -(h - 1), -h, -(h + 1), -2 ** 63, 0, 1, -1]
    vals = np.array(edge, np.int64)
    wrap = (10 ** 19) % 2 ** 64 - 2 ** 64
    for m in MODES:
        tie = wrap if m == R.HALF_UP else 0                 # 5 * 10^18 is a tie below the even quotient 0
        out = _host(torch, _round(AR, _dev(S, torch, INT64, vals), -19, m), np.int64)
        assert out.tolist() == [0, tie, wrap, wrap, 0, -tie, -wrap, -wrap, 0, 0, 0]
        out = _round(AR, _dev(S, torch, INT64, vals[[0, 4, 8]]), -19, m, True)
        assert _host(torch, out, np.int64).tolist() == [0, 0, 0]
        for i in (2, 3, 6, 7):
            with pytest.raises(AR.ExceptionWithRowIndex) as e:
                _round(AR, _dev(S, torch, INT64, np.array([h - 1, -(h - 1), edge[i], 7], np.int64)), -19, m, True)
            assert e.value.getRowIndex() == 2


# ---- decimals ---------------------------------------------------------------------------------------------------------
def test_decimal32_every_value(env):
    S, AR, torch = env
    for c in range(2 ** 32 // CHUNK):
        x = _chunk32(torch, c)
        for kd in range(-9, 11):
            scale = kd % 3 - 1
            dp = -kd - scale
            col = _col(S, DECIMAL32, x, CHUNK, scale=scale)
            for m in MODES:
                out = _round(AR, col, dp, m)
                assert out.dtype.scale == -dp
                got = out.data.view(torch.int32)
                bad = torch.zeros((), dtype=torch.int64, device="cuda")
                for s in range(0, CHUNK, SUB):
                    v = x[s: s + SUB].to(torch.int64)
                    if kd <= 0:
                        want = v * 10 ** -kd
                    elif kd > 9:
                        want = torch.zeros_like(v)
                    else:
                        want = _round_int_ref(torch, v, kd, m, 32, True)[0]
                    bad += (got[s: s + SUB] != want.to(torch.int32)).sum()
                if int(bad):
                    pytest.fail(f"DECIMAL32 chunk {c} kd={kd} mode={m}: {int(bad)} rows differ")
        del x


def _dec128_extremes():
    m = 10 ** 38 - 1
    return [-2 ** 127, 2 ** 127 - 1, -2 ** 127 + 1, 2 ** 127 - 2, m, -m, m - 1, -(m - 1), 2 ** 64 - 1, -(2 ** 64), 2 ** 64, 2 ** 63]


@pytest.mark.parametrize("kd", range(-18, 20))
def test_decimal64_ties(env, kd):
    S, AR, torch = env
    lo, hi = -2 ** 63, 2 ** 63 - 1
    vals = np.array(R.int_ties(max(kd, 1), lo, hi, seed=kd + 100), np.int64)
    for scale in (-3, 0, 4):
        dp = -kd - scale
        col = _dev(S, torch, DECIMAL64, vals, scale=scale, shift=kd % 2)
        for m in MODES:
            out = _round(AR, col, dp, m)
            assert out.dtype.scale == -dp
            _same(_host(torch, out, np.int64), A.round_decimal(vals, scale, dp, m), f"DECIMAL64 kd={kd} scale={scale} mode={m}")


@pytest.mark.parametrize("kd", range(-38, 40))
def test_decimal128_ties(env, kd):
    S, AR, torch = env
    ints = R.int_ties(max(kd, 1), -2 ** 127, 2 ** 127 - 1, seed=kd + 200) + _dec128_extremes()
    if 19 <= kd <= 20:                                  # either side of the division's one-limb divisor
        ints += [q * 10 ** kd + r for q in (1, 2, 2 ** 64 - 1, 2 ** 64, 10 ** (38 - kd) - 1) for r in (10 ** kd // 2 - 1, 10 ** kd // 2)]
        ints = [v for v in ints if v < 2 ** 127]
        ints += [-v for v in ints]
    data = A.ints_to_dec128(ints)
    for scale in (-2, 0, 5):
        dp = -kd - scale
        col = _dev(S, torch, DECIMAL128, data, scale=scale, shift=kd % 2)
        for m in MODES:
            out = _round(AR, col, dp, m)
            assert out.dtype.scale == -dp
            got = out.data.cpu().numpy().view(np.uint64).reshape(-1, 2)
            _same(got, A.round_decimal128(data, scale, dp, m), f"DECIMAL128 kd={kd} scale={scale} mode={m}")
