"""An independent model of JoinPrimitives built from Python dicts, sets and lists (no numpy sorting): the inner join is a
dict from key tuples to right rows; floats are normalised by their IEEE bits (every NaN -> one marker, -0.0 -> 0.0),
BOOL8 to bool, a null to a marker that equals itself only when nulls compare equal."""
import math
import struct

NULL = ("null",)
NAN = ("nan",)


def _norm(type_id, v):
    if type_id == 11:                                   # BOOL8
        return bool(int(v))
    if type_id in (9, 10):                              # FLOAT32 / FLOAT64
        f = float(v)
        return NAN if math.isnan(f) else (0.0 if f == 0.0 else f)
    if type_id == 23:
        return bytes(v)
    if type_id == 27:
        lo, hi = (int(x) for x in v)
        return (hi << 64) + (lo & (2 ** 64 - 1))
    return int(v)


def row_keys(cols, r, nulls_equal):
    """the row's key tuple, or None when it can match nothing"""
    key = []
    for k in cols:
        if k.valid is not None and not k.valid[r]:
            if not nulls_equal:
                return None
            key.append(NULL)
        else:
            key.append(_norm(k.type_id, k.values[r]))
    return tuple(key)


def inner_join(left, right, nulls_equal):
    nl, nr = len(left[0].values), len(right[0].values)
    table = {}
    for r in range(nr):
        key = row_keys(right, r, nulls_equal)
        if key is not None:
            table.setdefault(key, []).append(r)
    return sorted((l, r) for l in range(nl) for r in table.get(row_keys(left, l, nulls_equal) or (), []))


def f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def _in_range(m, size):
    return {i for i in m if 0 <= i < size}


def left_outer(L, R, nl, nr):
    hit = _in_range(L, nl)
    un = [i for i in range(nl) if i not in hit]
    return list(L) + un, list(R) + [-2 ** 31] * len(un)


def full_outer(L, R, nl, nr):
    ol, orr = left_outer(L, R, nl, nr)
    hit = _in_range(R, nr)
    un = [i for i in range(nr) if i not in hit]
    return ol + [-2 ** 31] * len(un), orr + un


def semi(m, size):
    return sorted(_in_range(m, size))


def anti(m, size):
    hit = _in_range(m, size)
    return [i for i in range(size) if i not in hit]


def matched_rows(m, size):
    hit = _in_range(m, size)
    return [1 if i in hit else 0 for i in range(size)]
