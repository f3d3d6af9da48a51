"""CPU checks of tests/histogram_scale_model.py, the vectorised percentile model the GPU scale tests compare against: its
key order, hand-derived answers at the clamps, and agreement with oracle/histogram.py on random columns of every value
type with nulls, empty and all-null rows, zero counts, total-0 rows, NaN payloads, signed zeros, infinities, each type's
extremes, totals above 2^53, P = 0 and sliced offsets."""
import numpy as np
import pytest

import histogram_scale_model as M
from oracle import histogram as H

# name -> (numpy dtype, BOOL8)
KINDS = {"int8": (np.int8, False), "int16": (np.int16, False), "int32": (np.int32, False), "int64": (np.int64, False),
         "uint8": (np.uint8, False), "uint16": (np.uint16, False), "uint32": (np.uint32, False), "uint64": (np.uint64, False),
         "float32": (np.float32, False), "float64": (np.float64, False), "bool8": (np.uint8, True)}


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((np.isnan(a) & np.isnan(b)) | (a.view(np.uint64) == b.view(np.uint64))))


def _values(rng, dt, bool8, n):
    if bool8:
        return rng.choice(np.array([0, 1, 2, 127, 255], np.uint8), n)
    if np.dtype(dt).kind == "f":
        nans = (np.array([0x7ff0000000000123, 0xfff8000000000001, 0x7ff8000000000000], np.uint64).view(np.float64) if dt == np.float64
                else np.array([0x7f800123, 0xffc00001, 0x7fc00000], np.uint32).view(np.float32))
        fi = np.finfo(dt)
        pool = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, fi.max, -fi.max, fi.tiny, -fi.smallest_subnormal, 1.5, -1.5], dt), nans])
        return np.where(rng.random(n) < 0.6, rng.choice(pool, n), rng.normal(0, 50, n).astype(dt)).astype(dt)
    info = np.iinfo(dt)
    pool = np.array([info.min, info.min + 1, info.max - 1, info.max, 0, 1], dt)
    return np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)).astype(dt)


def test_key_order():
    f64 = np.array([-np.inf, -1e300, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, 1e300, np.inf], np.float64)
    f32 = f64.astype(np.float32)[[0, 2, 4, 5, 7, 9]]
    for v in (f64, f32):
        k = M.sort_keys(v)
        assert (k[1:] > k[:-1]).all()
        nan = np.array([np.nan, -np.nan], v.dtype)
        nk = M.sort_keys(np.concatenate([nan, np.array([0x7f800001], np.uint32).view(np.float32).astype(v.dtype)]))
        assert (nk == k[-1] + np.uint64(1)).all()                  # every NaN: one key, right above +inf
    for dt in (np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64):
        info = np.iinfo(dt)
        v = np.unique(np.array([info.min, info.min + 1, 0, 1, info.max // 2, info.max // 2 + 1, info.max - 1, info.max], dt))
        k = M.sort_keys(v)
        assert (k[1:] > k[:-1]).all()
    assert M.sort_keys(np.array([0, 1, 2, 255], np.uint8), bool8=True).tolist() == [0, 1, 1, 1]
    assert M.sort_keys(np.array([np.iinfo(np.uint64).max], np.uint64))[0] == ~np.uint64(0)
    assert M.sort_keys(np.array([np.iinfo(np.int64).max], np.int64))[0] == ~np.uint64(0)


def test_clamps_keep_each_rank_in_its_row():
    # row 1 has total 0: rank 0 is the running sum before it, which the search alone places in row 0; row 2's overshoot
    # (total 0, rank 1) would run into row 3 without the clamp to the row's last element
    offsets = [0, 2, 4, 6, 7]
    vals = np.array([1, 2, 5, 9, 4, 3, 8], np.int64)
    counts = np.array([1, 0, 0, 0, 0, 0, 2], np.int64)
    out, ok = M.percentile(offsets, vals, None, counts, [0.0, 0.5, 1.0])
    assert ok.tolist() == [True] * 4
    assert out.tolist() == [[1.0, 1.0, 1.0], [9.0, 7.0, 5.0], [4.0, 3.5, 3.0], [8.0, 8.0, 8.0]]


@pytest.mark.parametrize("name", sorted(KINDS))
def test_model_matches_the_oracle(name):
    dt, bool8 = KINDS[name]
    rng = np.random.default_rng(sorted(KINDS).index(name) + 1)
    rows = 90
    lens = rng.integers(0, 14, rows)
    lens[rng.random(rows) < 0.1] = 0                              # empty rows
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = _values(rng, dt, bool8, n)
    valid = rng.random(n) > 0.25
    counts = rng.integers(0, 4, n).astype(np.int64)              # zero counts
    for r in range(rows):
        s, e = offsets[r], offsets[r + 1]
        if r % 9 == 3:
            valid[s:e] = False                                   # all-null rows
        elif r % 7 == 5:
            counts[s:e] = 0                                      # total-0 rows
        elif r % 11 == 8:
            counts[s:e] = rng.integers(2**50, 2**53, e - s)      # totals above 2^53
    ovals = vals != 0 if bool8 else vals
    pct = [0.0, 0.25, 0.5, 1.0, 1 / 3, 0.999] + list(rng.random(3))
    for slice_from in (0, 1, 37):
        offs = offsets[slice_from:]
        for v in (valid, None):
            want, wok = H.percentile_from_histogram(offs, ovals, v, counts, pct)
            got, ok = M.percentile(offs, vals, v, counts, pct, bool8)
            assert np.array_equal(ok, wok), (slice_from, v is None)
            assert _same(got, want), (slice_from, v is None)
    got, ok = M.percentile(offsets, vals, valid, counts, [], bool8)             # P = 0: every row null
    assert got.shape == (rows, 0) and not ok.any()
    got, ok = M.percentile([5, 5, 5], vals, valid, counts, [0.5], bool8)        # no element: every row null
    assert not ok.any() and (got == 0).all()
