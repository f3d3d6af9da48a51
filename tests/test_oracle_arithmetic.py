"""CPU checks of oracle/arithmetic.py: it reproduces every golden of tests/golden/arithmetic_golden.py; it agrees with an
independent model in Python integers and fractions for every integer and decimal case (random values and the edges: MIN *
-1, -1 * MIN, MIN * 0, the type bounds, decimal_places -20 .. 20, ties on both sides of zero, storage-edge decimals); and
its float recipe agrees bit for bit with a math.modf / math.floor restatement."""
import math
import random
import struct
from fractions import Fraction

import numpy as np
import pytest

from golden import arithmetic_golden as G
from oracle import arithmetic as A

NP = {"INT8": np.int8, "INT16": np.int16, "INT32": np.int32, "INT64": np.int64, "FLOAT32": np.float32, "FLOAT64": np.float64,
      "DECIMAL32": np.int32}
INTS = (np.int8, np.int16, np.int32, np.int64)


def _col(vals, t):
    valid = np.array([v is not None for v in vals], bool)
    return np.array([0 if v is None else v for v in vals], dtype=t), valid


# ---- goldens -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in G.MULTIPLY if c[6] != "error"], ids=lambda c: c[0])
def test_multiply_goldens(case):
    name, typ, left, right, ansi, try_mode, want = case
    t = NP[typ]
    ls, rs = isinstance(left, tuple), isinstance(right, tuple)
    a, va = (np.array([left[1]], t), True) if ls else _col(left, t)
    b, vb = (np.array([right[1]], t), True) if rs else _col(right, t)
    out, valid, err = A.multiply(a, va, b, vb, ansi, try_mode, ls, rs)
    if isinstance(want, tuple):
        assert err == want[1]
        return
    assert err == -1
    assert [o.item() if ok else None for o, ok in zip(out, valid)] == [None if w is None else t(w).item() for w in want]


@pytest.mark.parametrize("case", G.ROUND, ids=lambda c: c[0])
def test_round_goldens(case):
    name, typ, scale, vals, dp, mode, ansi, want = case
    t = NP[typ]
    v, valid = _col(vals, t)
    out, err = A.round_(v, valid, dp, mode, ansi, type_id=25 if typ == "DECIMAL32" else None, scale=scale)
    if isinstance(want, tuple):
        assert err == want[1]
        return
    assert err == -1
    assert [o.item() if ok else None for o, ok in zip(out, valid)] == [None if w is None else t(w).item() for w in want]


# ---- the integer model -------------------------------------------------------------------------------------------------
def _wrap(x, bits):
    x %= 1 << bits
    return x - (1 << bits) if x >> (bits - 1) else x


def _bounds(t):
    i = np.iinfo(t)
    return int(i.min), int(i.max)


def _edges(t):
    lo, hi = _bounds(t)
    return [lo, lo + 1, -1, 0, 1, hi - 1, hi, lo // 2, hi // 2, 2, -2, 10, -10]


def _samples(t, rng, n=300):
    lo, hi = _bounds(t)
    vals = _edges(t) + [rng.randint(lo, hi) for _ in range(n)]
    vals += [rng.choice([-1, 1]) * rng.randint(0, 1 << rng.randint(0, 8 * np.dtype(t).itemsize - 1)) for _ in range(n)]
    return [min(max(v, lo), hi) for v in vals]


@pytest.mark.parametrize("t", INTS)
@pytest.mark.parametrize("mode", ["wrap", "try", "ansi"])
def test_multiply_agrees_with_python_integers(t, mode):
    rng = random.Random(7)
    lo, hi = _bounds(t)
    bits = 8 * np.dtype(t).itemsize
    xs = _samples(t, rng)
    ys = _samples(t, rng)
    pairs = [(x, y) for x in _edges(t) for y in _edges(t)] + list(zip(xs, ys)) + [(lo, -1), (-1, lo), (lo, 0), (0, lo)]
    rng.shuffle(pairs)
    a = np.array([p[0] for p in pairs], t)
    b = np.array([p[1] for p in pairs], t)
    va = np.array([rng.random() > 0.1 for _ in pairs])
    out, valid, err = A.multiply(a, va, b, None, mode == "ansi", mode == "try")
    want_err = -1
    for i, (x, y) in enumerate(pairs):
        exact = x * y
        ovf = not lo <= exact <= hi
        if mode == "ansi" and ovf and va[i] and want_err < 0:
            want_err = i
        ok = bool(va[i]) and not (ovf and mode != "wrap")
        assert bool(valid[i]) == ok, (x, y)
        assert int(out[i]) == (_wrap(exact, bits) if ok else 0), (x, y)
    assert err == want_err


def _round_model(v, k, mode):
    """v rounded to a multiple of 10^k (k > 0), exactly, with Fraction."""
    d = 10 ** k
    q = Fraction(v, d)
    f = math.floor(q)
    rem = q - f
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and (f % 2 == 1 if mode == A.HALF_EVEN else v > 0)):
        f += 1
    return f * d


@pytest.mark.parametrize("t", INTS)
@pytest.mark.parametrize("mode", [A.HALF_UP, A.HALF_EVEN])
def test_round_int_agrees_with_python_integers(t, mode):
    rng = random.Random(11)
    lo, hi = _bounds(t)
    bits = 8 * np.dtype(t).itemsize
    base = _samples(t, rng, 200)
    for dp in range(-20, 21):
        k = -dp
        ties = []
        if 0 < k <= 19:
            h = 5 * 10 ** (k - 1)
            ties = [s * (m * 10 ** k + h) for m in range(0, 3) for s in (1, -1)] + [s * (m * 10 ** k + h + e) for m in (0, 1) for s in (1, -1) for e in (-1, 1)]
            ties = [x for x in ties if lo <= x <= hi]
        vals = base + ties
        v = np.array(vals, t)
        valid = np.array([rng.random() > 0.05 for _ in vals])
        out, err = A.round_int(v, valid, dp, mode, True)
        want_err = -1
        for i, x in enumerate(vals):
            exact = x if dp >= 0 else _round_model(x, k, mode)
            if dp < 0 and not lo <= exact <= hi and valid[i] and want_err < 0:
                want_err = i
            assert int(out[i]) == _wrap(exact, bits), (x, dp, mode)
        assert err == want_err, dp


def _dec_model(v, scale, dp, mode, bits):
    k = -dp - scale
    if k == 0:
        return v
    if k < 0:
        return _wrap(v * 10 ** (-k), bits)
    if k > {32: 9, 64: 18, 128: 38}[bits]:
        return 0
    r = _round_model(abs(v), k, mode) // 10 ** k
    return -r if v < 0 else r


@pytest.mark.parametrize("bits", [32, 64, 128])
@pytest.mark.parametrize("mode", [A.HALF_UP, A.HALF_EVEN])
def test_round_decimal_agrees_with_fractions(bits, mode):
    rng = random.Random(13 + bits)
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    digits = {32: 9, 64: 18, 128: 38}[bits]
    vals = [lo, lo + 1, hi, hi - 1, 0, 1, -1, 10 ** digits - 1, -(10 ** digits - 1), 10 ** digits, 5, -5, 15, -15, 25, -25]
    vals += [rng.randint(lo, hi) for _ in range(60)] + [rng.randint(-10 ** 6, 10 ** 6) for _ in range(40)]
    for k in range(1, digits + 1):
        h = 5 * 10 ** (k - 1)
        vals += [s * (m * 10 ** k + h + e) for m in (0, 1, 2) for s in (1, -1) for e in (-1, 0, 1)]
    vals = [min(max(v, lo), hi) for v in vals]
    for scale in (-4, 0, 3):
        for dp in range(-20, 21):
            want = [_dec_model(v, scale, dp, mode, bits) for v in vals]
            if bits == 128:
                got = A.dec128_to_ints(A.round_decimal128(A.ints_to_dec128(vals), scale, dp, mode))
            else:
                t = np.int32 if bits == 32 else np.int64
                got = [int(x) for x in A.round_decimal(np.array(vals, t), scale, dp, mode)]
            assert got == want, (scale, dp)
    # scale movements past the type's digits: zeros; a far scale-up wraps
    t = np.int64
    assert not A.round_decimal(np.array([hi if bits == 64 else 1], t), -40, 0, mode).any()


# ---- the float recipe --------------------------------------------------------------------------------------------------
def _f32(x):
    return float(np.float32(x))


def _round_model_float(x, even):
    """round / rint through math.floor: the distance to the floor is exact."""
    if not math.isfinite(x):
        return x
    r = math.floor(x)
    d = x - r
    if d > 0.5 or (d == 0.5 and ((r % 2 == 1) if even else x > 0)):
        r += 1
    return math.copysign(float(r), x) if r == 0 else float(r)


def _recipe_model(x, dp, even, single):
    rnd = _f32 if single else float
    with np.errstate(all="ignore"):
        n = rnd(np.power(np.float64(10.0), abs(dp)))
    if dp == 0:
        return _round_model_float(x, even)
    if dp > 0:
        frac, ip = math.modf(x) if math.isfinite(x) else (math.copysign(0.0, x) if math.isinf(x) else x, x)
        t = _round_model_float(rnd(frac * n) if not (math.isinf(n) and frac == 0) else math.nan, even)
        q = rnd(t / n) if not (math.isinf(t) and math.isinf(n)) else math.nan
        return rnd(ip + q)
    q = rnd(x / n) if not (math.isinf(x) and math.isinf(n)) else math.nan
    t = _round_model_float(q, even)
    return rnd(t * n) if not (t == 0 and math.isinf(n)) else math.nan


def _bits(x, single):
    if math.isnan(x):
        return "nan"
    return struct.pack("<f" if single else "<d", x)


@pytest.mark.parametrize("single", [True, False])
@pytest.mark.parametrize("even", [False, True])
def test_float_recipe_matches_a_math_restatement(single, even):
    rng = np.random.default_rng(5)
    t = np.float32 if single else np.float64
    specials = [0.0, -0.0, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 0.49999997, 1.234, 25.66, 154.9, 2346.0, -1454.0, 125.0, 1e-45 if single else 5e-324,
                -1e-45 if single else -5e-324, 1e-40 if single else 1e-310, 3.4e38 if single else 1.7e308, math.inf, -math.inf, math.nan,
                12345.675, -12345.675, 0.125, 0.375, 1e7, 1e15, 4503599627370497.0]
    raw = rng.integers(0, 2**32 if single else 2**63, 400, dtype=np.uint64)
    rand = (raw.astype(np.uint32).view(np.float32) if single else raw.view(np.float64)).astype(t)
    scaled = (rng.standard_normal(400) * 10.0 ** rng.integers(-6, 12, 400)).astype(t)
    halves = ((rng.integers(-10**6, 10**6, 200) + 0.5) / 10.0 ** rng.integers(0, 4, 200)).astype(t)
    vals = np.concatenate([np.array(specials, t), rand, scaled, halves])
    mode = A.HALF_EVEN if even else A.HALF_UP
    for dp in list(range(-20, 21)) + [40, -40]:
        got = A.round_float(vals, dp, mode)
        for x, g in zip(vals.tolist(), got.tolist()):
            assert _bits(g, single) == _bits(_recipe_model(float(x), dp, even, single), single), (x, dp)


def _non_overflow_range(t, dp, mode):
    """The reference's compute_non_overflow_range (round_float.cu:195-247), restated."""
    lo, hi = _bounds(t)
    safe = {1: -2, 2: -4, 4: -8, 8: -20}[np.dtype(t).itemsize]
    if dp <= safe:
        return lo, hi
    up = mode == A.HALF_UP
    if dp == -19 and np.dtype(t).itemsize == 8:
        return (-4999999999999999999, 4999999999999999999) if up else (-5000000000000000000, 5000000000000000000)
    div = 10 ** -dp
    half, max_q, min_q = div // 2, hi // div, -(-lo // div)            # C's truncating division
    base_pos, base_neg = max_q * div, min_q * div
    even_pos = 1 if not up and max_q % 2 == 0 else 0
    even_neg = 1 if not up and (-min_q) % 2 == 0 else 0
    max_safe = base_pos + half - 1 + even_pos if base_pos <= hi - half - even_pos else hi
    min_safe = base_neg - half + 1 - even_neg if base_neg >= lo + half - 1 + even_neg else lo
    return min_safe, max_safe


@pytest.mark.parametrize("t", INTS)
def test_ansi_round_matches_the_reference_safe_range(t):
    lo, hi = _bounds(t)
    for mode in (A.HALF_UP, A.HALF_EVEN):
        for dp in range(-20, 0):
            mn, mx = _non_overflow_range(t, dp, mode)
            vals = sorted({min(max(v, lo), hi) for c in (lo, hi, mn, mx) for v in range(c - 3, c + 4)})
            for x in vals:
                _, err = A.round_int(np.array([x], t), None, dp, mode, True)
                assert (err == 0) == (not mn <= x <= mx), (t, dp, mode, x)
