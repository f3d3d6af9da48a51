"""oracle/join.py against the independent model in join_model.py, on random tables of every key type in both null modes,
and both against the goldens of join_golden.py."""
import numpy as np
import pytest

import join_model as M
from golden import join_golden as G
from oracle import join as OJ

TYPES = {"INT8": (1, np.int8), "INT16": (2, np.int16), "INT32": (3, np.int32), "INT64": (4, np.int64), "UINT8": (5, np.uint8),
         "UINT16": (6, np.uint16), "UINT32": (7, np.uint32), "UINT64": (8, np.uint64), "FLOAT32": (9, np.float32),
         "FLOAT64": (10, np.float64), "BOOL8": (11, np.uint8), "TIMESTAMP_DAYS": (12, np.int32), "TIMESTAMP_MICROSECONDS": (15, np.int64),
         "DURATION_NANOSECONDS": (21, np.int64), "DECIMAL32": (25, np.int32), "DECIMAL64": (26, np.int64)}


def _key(name, n, pool, null_frac, rng):
    valid = None if null_frac == 0 else rng.random(n) >= null_frac
    pick = rng.integers(0, pool, n)
    if name == "STRING":
        words = [b"", b"a", b"\x00", b"ab" * 40] + [rng.bytes(int(rng.integers(0, 9))) for _ in range(pool)]
        return OJ.Key(23, [words[i] for i in pick], valid)
    if name == "DECIMAL128":
        return OJ.Key(27, np.stack([(pick * 7 - 3).astype(np.int64), (pick % 2 - 1).astype(np.int64)], axis=1), valid)
    t, dt = TYPES[name]
    if t in (9, 10):
        v = np.array([np.nan, -0.0, 0.0, np.inf, -1.5, 2.25, 7.0], dt)[pick % 7]
        bits = v.view(np.uint32 if t == 9 else np.uint64).copy()
        bits[(pick % 7 == 0) & (np.arange(n) % 2 == 1)] |= 5         # another NaN payload
        return OJ.Key(t, bits.view(dt), valid)
    if t == 11:
        return OJ.Key(t, (pick % 2 * (1 + np.arange(n) % 3)).astype(np.uint8), valid)
    return OJ.Key(t, (pick * 37 - pool).astype(dt), valid)


@pytest.mark.parametrize("name", list(TYPES) + ["STRING", "DECIMAL128"])
@pytest.mark.parametrize("eq", [False, True])
def test_oracle_agrees_with_the_model(name, eq):
    rng = np.random.default_rng(len(name) * 7 + eq)
    for nl, nr, pool, nf in ((60, 50, 8, 0.0), (80, 70, 5, 0.2), (40, 30, 4, 1.0), (0, 10, 3, 0.0), (10, 1, 3, 0.5)):
        left, right = [_key(name, nl, pool, nf, rng)], [_key(name, nr, pool, nf, rng)]
        L, R = OJ.inner_join(left, right, eq)
        assert list(zip(L.tolist(), R.tolist())) == M.inner_join(left, right, eq)


@pytest.mark.parametrize("eq", [False, True])
def test_multi_column_keys(eq):
    rng = np.random.default_rng(3 + eq)
    names = ["INT32", "STRING", "FLOAT64", "DECIMAL128", "BOOL8", "INT64", "UINT16", "DECIMAL32"]
    for ncols in (1, 2, 4, 8):
        left = [_key(n, 200, 3, 0.1, rng) for n in names[:ncols]]
        right = [_key(n, 150, 3, 0.1, rng) for n in names[:ncols]]
        L, R = OJ.inner_join(left, right, eq)
        assert list(zip(L.tolist(), R.tolist())) == M.inner_join(left, right, eq)


def _golden_key(spec):
    name, vals = spec
    valid = np.array([v is not None for v in vals]) if any(v is None for v in vals) else None
    if name == "STRING":
        return OJ.Key(23, [v if v is not None else b"" for v in vals], valid)
    if name == "FLOAT64_BITS":
        return OJ.Key(10, np.array([v or 0 for v in vals], np.uint64).view(np.float64), valid)
    return OJ.Key(3, np.array([v if v is not None else 0 for v in vals], np.int32), valid)


@pytest.mark.parametrize("case", G.INNER, ids=[c[0] for c in G.INNER])
def test_inner_goldens(case):
    _, l, r, eq, want = case
    left, right = [_golden_key(l)], [_golden_key(r)]
    L, R = OJ.inner_join(left, right, eq)
    assert list(zip(L.tolist(), R.tolist())) == want == M.inner_join(left, right, eq)


@pytest.mark.parametrize("case", G.HELPERS, ids=[c[0] for c in G.HELPERS])
def test_helper_goldens(case):
    _, L, R, nl, nr, lo, fo, semi, anti, mr = case
    L, R = np.array(L, np.int32), np.array(R, np.int32)
    for got, model, want in ((OJ.make_left_outer(L, R, nl, nr), M.left_outer(L.tolist(), R.tolist(), nl, nr), lo),
                             (OJ.make_full_outer(L, R, nl, nr), M.full_outer(L.tolist(), R.tolist(), nl, nr), fo)):
        assert (got[0].tolist(), got[1].tolist()) == tuple(model) == tuple(want)
    assert OJ.make_semi(L, nl).tolist() == M.semi(L.tolist(), nl) == semi
    assert OJ.make_anti(L, nl).tolist() == M.anti(L.tolist(), nl) == anti
    assert OJ.get_matched_rows(R, nr).tolist() == M.matched_rows(R.tolist(), nr) == mr


def test_random_helpers_agree():
    rng = np.random.default_rng(17)
    for nl, nr, n in ((0, 0, 0), (1, 3, 5), (100, 90, 300), (33, 65, 64)):
        L = rng.integers(-2, nl + 2, n).astype(np.int32)
        R = rng.integers(-2, nr + 2, n).astype(np.int32)
        L[::5] = OJ.INT32_MIN
        assert [a.tolist() for a in OJ.make_full_outer(L, R, nl, nr)] == list(M.full_outer(L.tolist(), R.tolist(), nl, nr))
        assert OJ.make_semi(R, nr).tolist() == M.semi(R.tolist(), nr) and OJ.make_anti(R, nr).tolist() == M.anti(R.tolist(), nr)
