"""CPU checks of tests/round_cases.py, the inputs and the float32 reference of tests/test_gpu_round_exhaustive.py: the torch
restatement of the float32 recipe agrees bit for bit with oracle/arithmetic.py's round_float at every decimal place the
GPU sweep uses, and the constructed FLOAT64 and integer cases have the properties they are built for."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import round_cases as R
from oracle import arithmetic as A


def _f32_sample(n: int) -> np.ndarray:
    rng = np.random.default_rng(2024)
    raw = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    exps = rng.integers(0, 9, n // 2)
    halves = ((rng.integers(-2 ** 22, 2 ** 22, n // 2) + 0.5) / 10.0 ** exps).astype(np.float32)
    ints = rng.integers(-2 ** 31, 2 ** 31, n // 4).astype(np.float32)
    edges = np.arange(-2 ** 16, 2 ** 16, dtype=np.int64).astype(np.uint32)       # +-0, subnormals, NaNs, infinities
    edges = np.concatenate([edges, edges ^ 0x7f800000, edges ^ 0x00800000]).view(np.float32)
    return np.concatenate([raw[: n - len(halves) - len(ints) - len(edges)], halves, ints, edges])


F32 = _f32_sample(2 ** 22)


def _same_bits(got: np.ndarray, want: np.ndarray):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    u = np.uint32 if want.dtype == np.float32 else np.uint64
    bad = np.flatnonzero((got.view(u) != want.view(u)) & ~nan)
    assert bad.size == 0, f"{bad.size} differ, first at {bad[0]}: {got[bad[0]]!r} != {want[bad[0]]!r}"


@pytest.mark.parametrize("dp", R.F32_DPS)
def test_float32_reference_matches_oracle(dp):
    x = torch.from_numpy(F32)
    got = R.round_float32(x, dp)
    for mode in (R.HALF_UP, R.HALF_EVEN):
        _same_bits(got[mode].numpy(), A.round_float(F32, dp, mode))


def test_oracle_divides_by_the_c_library_pow():
    """n is pow(10, |dp|) as the host's C library computes it (glibc's 10^23 is one ulp above the nearest double), so
    rounding pow(10, k) to -k places gives it back at every k."""
    n = np.array([math.pow(10.0, k) for k in range(1, 309)])
    for mode in (R.HALF_UP, R.HALF_EVEN):
        got = np.array([A.round_float(n[k - 1: k], -k, mode)[0] for k in range(1, 309)])
        assert np.array_equal(got, n)


def test_float32_reference_keeps_negative_zero():
    x = torch.tensor([-0.0, -0.25, -1e-30, -0.0], dtype=torch.float32)
    for dp in (3, -3, 0):
        for mode in (R.HALF_UP, R.HALF_EVEN):
            assert torch.signbit(R.round_float32(x, dp)[mode]).all()


@pytest.mark.parametrize("k", [k for k in range(1, 24)] + [100, 300, 305, 308])
def test_float64_positive_dp_cases(k):
    """round(e * n) reproduces m, so the recipe divides m by n; and for k >= 9 the quotients sit close to midpoints."""
    n = R.f64_pow10(k)
    c = R.f64_positive_dp(k)
    e = c["mid"][: len(c["mid"]) // 2]
    assert len(e) >= min(16, 10 ** k - 1) and np.all(e > 0)
    m = np.round(e * n)
    assert np.all(m >= 1) and np.all(m < min(n, 2.0 ** 53 + 1))
    dist = [R.midpoint_distance(Fraction(int(v)) / Fraction(n)) for v in m]
    bound = Fraction(1, 2) if k < 9 else Fraction(1, 2 ** 7) if k < 16 else Fraction(1, 2 ** 20)
    assert max(dist) <= bound
    assert min(dist) <= Fraction(1, 2 * 5 ** min(k, 13))    # 10^k = 2^k 5^k: no closer with this divisor
    if k == 308:                                            # the quotient 1 / n and 2 / n are subnormal
        sub = c["sub"][c["sub"] > 0]
        q = np.round(sub * n) / n
        assert np.count_nonzero(np.abs(q) < np.finfo(np.float64).tiny) == 2


@pytest.mark.parametrize("k", [1, 2, 5, 15, 22, 23, 100, 300, 307, 308])
def test_float64_negative_dp_cases(k):
    """e / n is within 4 of e's ulps (over n) of h + 0.5; the "mid" quotients sit close to midpoints."""
    n = R.f64_pow10(k)
    c = R.f64_negative_dp(k)
    half = c["half"][c["half"] > 0]
    assert len(half) >= 6
    for e in half[:: max(1, len(half) // 200)]:
        q = Fraction(float(e)) / Fraction(n)
        assert abs(q - (math.floor(q) + Fraction(1, 2))) <= 4 * Fraction(float(np.spacing(e))) / Fraction(n)
    mid = c["mid"][c["mid"] > 0]
    assert len(mid) >= 16
    dist = [R.midpoint_distance(Fraction(float(e)) / Fraction(n)) for e in mid]
    assert min(dist) <= Fraction(1, 2 * 5 ** min(k, 13))


@pytest.mark.parametrize("k", range(1, 21))
def test_int64_ties(k):
    lo, hi = -2 ** 63, 2 ** 63 - 1
    v = R.int_ties(k, lo, hi)
    assert all(lo <= x <= hi for x in v) and {lo, hi, lo + 1, hi - 1} <= set(v)
    d, h = 10 ** k, 10 ** k // 2
    ties = [x for x in v if abs(x) % d == h]
    if k <= 18:
        for s in (1, -1):
            par = {(abs(x) // d) & 1 for x in ties if x * s > 0}
            assert par == {0, 1}                            # ties below an even and an odd quotient, on both signs
        assert max(abs(x) for x in ties) > hi - d           # the largest tie below 2^63
        assert {abs(x) % d for x in v} >= {h - 1, h, h + 1}
    if k == 19:                                             # 0 or +-10^19 wrapped, around the ANSI bounds
        assert {h - 1, h, h + 1, -(h - 1), -h, -(h + 1)} <= set(v)


def test_int_ties_decimal128_range():
    lo, hi = -2 ** 127, 2 ** 127 - 1
    for k in (1, 19, 20, 37, 38):
        v = R.int_ties(k, lo, hi, seed=k)
        d, h = 10 ** k, 10 ** k // 2
        ties = [x for x in v if abs(x) % d == h]
        assert ties and all(lo <= x <= hi for x in v)
        assert {(abs(x) // d) & 1 for x in ties} == {0, 1} or k == 38
