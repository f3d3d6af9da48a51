"""CPU checks of oracle/histogram.py: it reproduces every golden of tests/golden/histogram_golden.py and agrees with an
independent pure-Python model (Python's sorted and bisect, exact integers) on random histograms with zero counts, several
nulls, every value kind and positions above 2^53."""
import bisect
import math
import struct

import numpy as np
import pytest

from golden import histogram_golden as G
from oracle import histogram as H


def _f64(x):
    return struct.unpack("<d", struct.pack("<d", x))[0]


def _model_row(values, counts, percentages, is_float):
    """Sort (nulls removed by the caller) by Spark's order with Python's sorted, bisect into the running sums."""
    if not values:
        return None

    def order(v):
        if is_float:
            if math.isnan(v):
                return (2, 0.0)
            return (1, v, math.copysign(1.0, v))          # -0.0 before 0.0
        return (1, int(v))
    pairs = sorted(zip(values, counts), key=lambda vc: order(vc[0]))
    acc, run = [], 0
    for _, c in pairs:
        run += int(c)
        acc.append(run)
    out = []
    for p in percentages:
        position = float(acc[-1] - 1) * p                 # Python floats are IEEE doubles, one rounding per operation
        lower, higher = math.floor(position), math.ceil(position)
        lo = pairs[min(bisect.bisect_left(acc, lower + 1), len(pairs) - 1)][0]
        hi = pairs[min(bisect.bisect_left(acc, higher + 1), len(pairs) - 1)][0]
        tofloat = (lambda x: float(x)) if is_float else (lambda x: float(int(x)))
        if higher == lower or (tofloat(lo) == tofloat(hi) if is_float else int(lo) == int(hi)):
            out.append(tofloat(lo))
        else:
            a = _f64((float(higher) - position) * tofloat(lo))
            b = _f64((position - float(lower)) * tofloat(hi))
            out.append(a + b)
    return out


def _same(a, b):
    return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))


@pytest.mark.parametrize("case", G.PERCENTILES, ids=[c[0] for c in G.PERCENTILES])
def test_percentile_goldens(case):
    _, pairs, pct, want = case
    vals = np.array([v for v, _ in pairs], np.int32)
    cnts = np.array([c for _, c in pairs], np.int64)
    out, ok = H.percentile_from_histogram([0, len(pairs)], vals, None, cnts, pct)
    assert ok.tolist() == [True]
    assert out[0].tolist() == want


@pytest.mark.parametrize("case", G.ROUND_TRIPS, ids=[c[0] for c in G.ROUND_TRIPS])
def test_round_trip_goldens(case):
    _, values, freqs, pct, want = case
    valid = np.array([v is not None for v in values])
    vals = np.array([0 if v is None else v for v in values], np.int32)
    offsets, cv, cvalid, cf = H.create_histogram_if_valid(vals, valid, np.array(freqs, np.int64), True)
    out, ok = H.percentile_from_histogram(offsets, cv, cvalid, cf, pct)
    got = [float(out[r, 0]) if ok[r] else None for r in range(len(values))]
    assert got == want


def test_create_struct_quirk_and_negative():
    vals = np.array([1, 2, 3, 4], np.int64)
    valid = np.array([True, False, True, True])
    v, ok, f = H.create_histogram_if_valid(vals, valid, np.array([2, 5, 0, 1]), False)
    assert ok.tolist() == [True, False, False, True] and f.tolist() == [2, 1, 1, 1]   # nulls get frequency 1
    v, ok, f = H.create_histogram_if_valid(vals, valid, np.array([2, 5, 3, 1]), False)
    assert ok.tolist() == valid.tolist() and f.tolist() == [2, 5, 3, 1]                # no zero: unchanged
    with pytest.raises(ValueError, match="negative"):
        H.create_histogram_if_valid(vals, valid, np.array([2, -1, 3, 1]), True)


def test_all_null_and_empty_rows():
    out, ok = H.percentile_from_histogram([0, 0, 2, 3], np.array([1, 2, 3], np.int32), np.array([False, False, True]),
                                          np.ones(3, np.int64), [0.5])
    assert ok.tolist() == [False, False, True] and out[2, 0] == 3.0
    assert not H.percentile_from_histogram([0, 2], np.array([1, 2]), None, np.ones(2, np.int64), [])[1].any()


KINDS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64, np.bool_]


def _random_values(rng, dt, n):
    if dt == np.bool_:
        return rng.integers(0, 2, n).astype(bool)
    if np.dtype(dt).kind == "f":
        pool = np.array([0.0, -0.0, 1.5, -2.25, np.inf, -np.inf, np.nan, 3.0, 1e300 if dt == np.float64 else 1e30], dt)
        return np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.normal(0, 100, n).astype(dt)).astype(dt)
    info = np.iinfo(dt)
    pool = np.array([info.min, info.max, 0, 1], dt)
    return np.where(rng.random(n) < 0.3, rng.choice(pool, n), rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)).astype(dt)


@pytest.mark.parametrize("dt", KINDS, ids=[np.dtype(k).name for k in KINDS])
def test_oracle_matches_the_independent_model(dt):
    rng = np.random.default_rng(7 + KINDS.index(dt))
    pct = [0.0, 0.25, 0.5, 1.0, 0.3, 0.999] + list(rng.random(4))
    rows = 60
    lens = rng.integers(0, 12, rows)
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = _random_values(rng, dt, n)
    valid = rng.random(n) > 0.25
    big = rng.random(rows) < 0.3                              # totals above 2^53
    counts = rng.integers(0, 4, n).astype(np.int64)          # zero counts included
    for r in np.nonzero(big)[0]:
        counts[offsets[r]:offsets[r + 1]] = rng.integers(2**50, 2**60, lens[r])
    out, ok = H.percentile_from_histogram(offsets, vals, valid, counts, pct)
    is_float = np.dtype(dt).kind == "f"
    for r in range(rows):
        s, e = offsets[r], offsets[r + 1]
        keep = [i for i in range(s, e) if valid[i]]
        want = _model_row([vals[i].item() for i in keep], [int(counts[i]) for i in keep], pct, is_float)
        assert ok[r] == (want is not None)
        if want is not None:
            assert all(_same(float(a), b) for a, b in zip(out[r], want)), (r, out[r], want)
