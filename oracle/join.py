"""JoinPrimitives restated in numpy (reference join_primitives.cu: hash_inner_join over cudf::hash_join, make_left_outer,
make_full_outer, make_semi, make_anti, get_matched_rows).

A key column is Key(type_id, values, valid): values is a numpy array of the raw elements (shape (n, 2) of int64 for
DECIMAL128: low, high), or a sequence of bytes for STRING; valid is a bool array or None (all valid).

inner_join sorts instead of hashing: each column's canonical values (every NaN one NaN, -0.0 as 0.0, BOOL8 as 0 / 1) get
dense codes shared by both sides, rows get the code of their code tuple, and equal codes pair up.  It returns the pairs
sorted by (left, right).  The helpers are exact, in order.
"""
from collections import namedtuple

import numpy as np

Key = namedtuple("Key", "type_id values valid")

INT32_MIN = np.int32(-2 ** 31)
BOOL8, FLOAT32, FLOAT64, STRING, DECIMAL128 = 11, 9, 10, 23, 27


def _canonical(k: Key):
    """the values as a 2-D int64 matrix (or an object array of bytes for STRING) that compares equal exactly when cudf's
    nan_equal_physical_equality_comparator does"""
    if k.type_id == STRING:
        return np.array([bytes(v) for v in k.values] + [b""], dtype=object)[:-1]
    v = np.asarray(k.values)
    if k.type_id == DECIMAL128:
        return v.reshape(-1, 2).astype(np.int64)
    if k.type_id == BOOL8:
        return (v.view(np.uint8) != 0).astype(np.int64).reshape(-1, 1)
    if k.type_id in (FLOAT32, FLOAT64):
        f = v.astype(np.float64)
        f = np.where(f == 0.0, 0.0, f)
        bits = f.view(np.int64).copy()
        bits[np.isnan(f)] = 0x7ff8000000000000
        return bits.reshape(-1, 1)
    return v.astype(np.int64).reshape(-1, 1) if v.dtype != np.uint64 else v.view(np.int64).reshape(-1, 1)


def _codes(left, right, nulls_equal):
    """row codes of both sides (equal codes: equal keys) and the rows that may match at all"""
    nl, nr = len(left[0].values), len(right[0].values)
    cols, ok_l, ok_r = [], np.ones(nl, bool), np.ones(nr, bool)
    for a, b in zip(left, right):
        ca, cb = _canonical(a), _canonical(b)
        if a.type_id == STRING:
            _, inv = np.unique(np.concatenate([ca, cb]), return_inverse=True)
        else:
            _, inv = np.unique(np.concatenate([ca, cb]), axis=0, return_inverse=True)
        inv = inv.reshape(-1).astype(np.int64)
        va = np.ones(nl, bool) if a.valid is None else np.asarray(a.valid, bool)
        vb = np.ones(nr, bool) if b.valid is None else np.asarray(b.valid, bool)
        inv[np.concatenate([~va, ~vb])] = -1
        if not nulls_equal:
            ok_l &= va
            ok_r &= vb
        cols.append(inv)
    _, rows = np.unique(np.stack(cols, axis=1), axis=0, return_inverse=True)
    rows = rows.reshape(-1)
    return rows[:nl], rows[nl:], ok_l, ok_r


def inner_join(left, right, nulls_equal):
    """(L, R) int32, sorted by (L, R): every pair of rows with equal keys"""
    if len(left) == 0 or len(right) == 0:
        raise ValueError("keys table must have at least one column")
    nl, nr = len(left[0].values), len(right[0].values)
    if nl == 0 or nr == 0:
        return np.zeros(0, np.int32), np.zeros(0, np.int32)
    cl, cr, ok_l, ok_r = _codes(left, right, nulls_equal)
    rr = np.nonzero(ok_r)[0]
    order = rr[np.argsort(cr[rr], kind="stable")]
    sorted_codes = cr[order]
    lo = np.searchsorted(sorted_codes, cl, "left")
    hi = np.searchsorted(sorted_codes, cl, "right")
    cnt = np.where(ok_l, hi - lo, 0)
    L = np.repeat(np.arange(nl, dtype=np.int64), cnt)
    start = np.repeat(lo - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
    R = order[start + np.arange(len(L))] if len(L) else np.zeros(0, np.int64)
    idx = np.lexsort((R, L))
    return L[idx].astype(np.int32), R[idx].astype(np.int32)


def matched(m, size):
    """bool[size]: rows an in-range entry of m names"""
    m = np.asarray(m, np.int64)
    out = np.zeros(max(size, 0), bool)
    out[m[(m >= 0) & (m < size)]] = True
    return out


def make_left_outer(L, R, left_size, right_size):
    un = np.nonzero(~matched(L, left_size))[0].astype(np.int32)
    return (np.concatenate([np.asarray(L, np.int32), un]),
            np.concatenate([np.asarray(R, np.int32), np.full(len(un), INT32_MIN, np.int32)]))


def make_full_outer(L, R, left_size, right_size):
    ol, orr = make_left_outer(L, R, left_size, right_size)
    un = np.nonzero(~matched(R, right_size))[0].astype(np.int32)
    return np.concatenate([ol, np.full(len(un), INT32_MIN, np.int32)]), np.concatenate([orr, un])


def make_semi(m, size):
    return np.nonzero(matched(m, size))[0].astype(np.int32)


def make_anti(m, size):
    return np.nonzero(~matched(m, size))[0].astype(np.int32)


def get_matched_rows(m, size):
    return matched(m, size).astype(np.uint8)
