"""JoinPrimitives.hashInnerJoin on keys built to collide: unequal keys with the same 32-bit row hash, so that the join's
answer rests on keys_equal alone.  Random keys almost never reach that: the chance that any two of n distinct keys share
a hash is about n^2 / 2^33.  tests/join_collide.py solves one free word of a row for a chosen hash.

Every case compares the join with oracle/join.py (sorts, never hashes) under both null modes, checks that the left map is
non-decreasing, and first proves on the device that its families collide: Hash.murmurHash32(0, ...) of columns that hash
as the key columns do (UINT8 / UINT16 / UINT32 of the canonical bits, INT64, DECIMAL128 as INT64 lo then hi, STRING)
equals the model's hash on every non-null row.

Covered: families in every 8-byte type and in DECIMAL128, rows that differ only in the high halves of 8-byte keys, every
<= 4-byte type against a compensating INT32 column, a difference in every column position of 2, 8 and 32 key columns,
null against a colliding value and nulls in the same columns, strings of every length 0 .. 72 and over 4 KB with one
flipped byte at every position, prefixes, tail-only differences and all 16 start alignments mod 4, and chains of 256 to
1,024 colliding keys that wrap from the last bucket, start at bucket 0 or carry the empty slot's upper word."""
import numpy as np
import pytest

import join_collide as JC
from join_collide import (BOOL8, DECIMAL32, DECIMAL64, DECIMAL128, FLOAT32, FLOAT64, INT8, INT16, INT32, INT64, M32,
                          STRING, TIMESTAMP_DAYS, TIMESTAMP_MICROSECONDS, UINT8, UINT16, UINT32, UINT64)
from oracle import join as OJ
from test_gpu_join import NP, check_join, to_dev

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1
EIGHT = [t for t in JC.FIXED_TYPES if JC.WIDTH[t] == 8]
NARROW = [t for t in JC.FIXED_TYPES if JC.WIDTH[t] <= 4]
UINT_OF = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
UTYPE_OF = {1: UINT8, 2: UINT16, 4: UINT32}


class Null:
    """a null key whose data slot holds `under` (a colliding row's value, so that comparing data alone says equal)"""
    def __init__(self, under):
        self.under = under


def model(row):
    return [(t, None if isinstance(v, Null) else v) for t, v in row]


def _data(v):
    return v.under if isinstance(v, Null) else v


def keys(rows):
    """the rows as oracle/join.py key columns (the layout test_gpu_join.to_dev puts on the device)"""
    out = []
    for c, (t, _) in enumerate(rows[0]):
        vals = [r[c][1] for r in rows]
        valid = np.array([not isinstance(v, Null) for v in vals], bool)
        raw = [_data(v) for v in vals]
        w = JC.WIDTH[t]
        if t == STRING:
            values = [bytes(v) for v in raw]
        elif w == 16:
            values = np.array([[v & M64, v >> 64] for v in raw], np.uint64).view(np.int64)
        else:
            values = np.array(raw, UINT_OF[w]).view(NP.get(t, np.int64))
        out.append(OJ.Key(t, values, None if valid.all() else valid))
    return out


def witness(rows):
    """Hash.murmurHash32(0, ...) on the device equals the model's row hash on every non-null row: the collisions the
    model built exist in the kernel's hash"""
    import srj_b200 as S
    rows = [model(r) for r in rows if not any(isinstance(v, Null) for _, v in r)]
    assert rows
    cols = []
    for c, (t, _) in enumerate(rows[0]):
        bits = [JC.canon(t, r[c][1]) if t != STRING else r[c][1] for r in rows]
        w = JC.WIDTH[t]
        if t == STRING:
            cols.append(OJ.Key(STRING, bits, None))
        elif w == 16:
            cols += [OJ.Key(INT64, np.array([b & M64 for b in bits], np.uint64).view(np.int64), None),
                     OJ.Key(INT64, np.array([b >> 64 for b in bits], np.uint64).view(np.int64), None)]
        elif w == 8:
            cols.append(OJ.Key(INT64, np.array(bits, np.uint64).view(np.int64), None))
        else:
            cols.append(OJ.Key(UTYPE_OF[w], np.array(bits, UINT_OF[w]), None))
    got = S.Hash.murmurHash32(0, [to_dev(k) for k in cols]).data.cpu().numpy().view(np.int32)
    want = np.array([JC.signed(JC.row_hash(r)) for r in rows], np.int32)
    assert np.array_equal(got, want), "the device hash differs from the model: the collisions may not exist"


def family(rows):
    """rows that share one row hash and are pairwise unequal keys"""
    assert len({JC.row_hash(model(r)) for r in rows}) == 1
    canon = {tuple(None if isinstance(v, Null) else v if t == STRING else JC.canon(t, v) for t, v in r) for r in rows}
    assert len(canon) == len(rows)
    return rows


def join_both(left, right, eq, min_pairs=1):
    n = check_join(keys(left), keys(right), eq)
    assert n >= min_pairs
    return n


def _rand(t, rng):
    if t == STRING:
        return rng.bytes(int(rng.integers(8, 25)))
    if t == BOOL8:
        return int(rng.integers(0, 2))
    v = int.from_bytes(rng.bytes(JC.WIDTH[t]), "little")
    return JC.canon(t, v) if t in (FLOAT32, FLOAT64) and JC.canon(t, v) != v else v


def _varied(row, c, rng):
    """row with column c changed to another value of its type"""
    t, v = row[c]
    out = list(row)
    if t == BOOL8:
        out[c] = (t, 1 - v)
    elif t == STRING:
        out[c] = (t, bytes([v[0] ^ (1 + int(rng.integers(0, 255)))]) + v[1:])
    else:
        nv = v
        while JC.canon(t, nv) == JC.canon(t, v):
            nv = _rand(t, rng)
        out[c] = (t, nv)
    return out


def _collide(row, change, free, target, rng, filler=None):
    """row with word `change` set to a random value, then word `free` solved so that the row hashes to target"""
    return JC.solve(JC.set_word(row, change, int(rng.integers(0, 1 << 32))), free, target, filler)


# ---------------------------------------------------------------- fixed width
@pytest.mark.parametrize("eq", [False, True])
def test_eight_byte_families(eq):
    rng = np.random.default_rng(100 + eq)
    for t in EIGHT:
        # one column: distinct values that share a hash (lo random, hi solved)
        fams = []
        for _ in range(16):
            base, target = [(t, _rand(t, rng))], int(rng.integers(0, 1 << 32))
            fams.append(family([_collide(base, (0, 0), (0, 1), target, rng, (0, 0)) for _ in range(8)]))
        rows = [r for f in fams for r in f]
        witness(rows)
        join_both(rows, rows[::-1], eq, len(rows))
        # two columns equal in their low halves, unequal in their high halves
        fams = []
        for _ in range(16):
            base, target = [(t, _rand(t, rng)), (t, _rand(t, rng))], int(rng.integers(0, 1 << 32))
            fams.append(family([_collide(base, (0, 1), (1, 1), target, rng, (0, 0)) for _ in range(8)]))
        rows = [r for f in fams for r in f]
        witness(rows)
        join_both(rows, rows[::-1], eq, len(rows))


@pytest.mark.parametrize("eq", [False, True])
def test_decimal128(eq):
    rng = np.random.default_rng(110 + eq)
    rows = []
    for change, free in (((0, 0), (0, 3)), ((0, 1), (0, 3)), ((0, 2), (0, 3)), ((0, 3), (0, 2)), ((0, 1), (0, 0)), ((0, 0), (0, 1))):
        for _ in range(8):       # one column: families whose members differ in `change` and `free` only
            base, target = [(DECIMAL128, int.from_bytes(rng.bytes(16), "little"))], int(rng.integers(0, 1 << 32))
            rows += family([_collide(base, change, free, target, rng) for _ in range(6)])
    witness(rows)
    join_both(rows, rows[::-1], eq, len(rows))
    # pairs that differ in exactly one of the four words, an INT32 column compensating (it leads in half of them)
    for lead in (False, True):
        rows = []
        for j in range(4):
            for _ in range(32):
                a = [(DECIMAL128, int.from_bytes(rng.bytes(16), "little")), (INT32, int(rng.integers(0, 1 << 32)))]
                a = a[::-1] if lead else a
                d = int(lead)
                b = JC.solve(JC.set_word(a, (d, j), JC.get_word(a, (d, j)) ^ (1 << int(rng.integers(0, 32)))), (1 - d, 0), JC.row_hash(a))
                rows += family([a, b])
        witness(rows)
        join_both(rows, rows[::-1], eq, len(rows))


@pytest.mark.parametrize("eq", [False, True])
def test_narrow_types_against_a_compensating_int32(eq):
    rng = np.random.default_rng(120 + eq)
    for t in NARROW:
        for lead in (False, True):                          # the INT32 column after the narrow one, then before it
            d, f = (1, 0) if not lead else (0, 1)
            rows = []
            for _ in range(48):
                a = [(t, _rand(t, rng)), (INT32, int(rng.integers(0, 1 << 32)))]
                a = a[::-1] if lead else a
                rows += family([a, JC.solve(_varied(a, f, rng), (d, 0), JC.row_hash(a))])
            if t == BOOL8:                                  # true as 1, 2 and 255: equal keys
                rows += [[(BOOL8, x), (INT32, 5)][::-1 if lead else 1] for x in (1, 2, 255)]
            if t == FLOAT32:                                # NaN payloads and -0.0 are equal keys; FLOAT32 as the free word
                rows += [[(FLOAT32, x), (INT32, 5)][::-1 if lead else 1] for x in (0x7FC00000, 0xFFC00001, 0x7F800001, 0, 0x80000000)]
                for _ in range(48):
                    a = [(FLOAT32, _rand(FLOAT32, rng)), (INT32, int(rng.integers(0, 1 << 32)))]
                    a = a[::-1] if lead else a
                    rows += family([a, JC.solve(_varied(a, d, rng), (f, 0), JC.row_hash(a), (d, 0))])
            witness(rows)
            join_both(rows, rows[::-1], eq, len(rows))


# ---------------------------------------------------------------- every column position
POOL = [INT32, STRING, INT64, DECIMAL128, FLOAT64, BOOL8, INT16, TIMESTAMP_MICROSECONDS, FLOAT32, UINT8, DECIMAL32, UINT64,
        INT8, UINT16, TIMESTAMP_DAYS, DECIMAL64]


def _free_in(row, c):
    return [a for a in JC.free_words(row) if a[0] == c]


@pytest.mark.parametrize("ncols", [2, 8, 32])
@pytest.mark.parametrize("eq", [False, True])
def test_a_difference_in_every_column_position(ncols, eq):
    rng = np.random.default_rng(130 + ncols + eq)
    types = [STRING, INT64] if ncols == 2 else [POOL[(3 * i + ncols) % len(POOL)] for i in range(ncols)]
    rows = []
    for c in range(ncols):
        for _ in range(4):
            base = [(t, _rand(t, rng)) for t in types]
            target = JC.row_hash(base)
            others = [a for a in JC.free_words(base) if a[0] != c]
            comp = others[int(rng.integers(0, len(others)))]
            filler = next(a for a in JC.free_words(base) if a[0] not in (c, comp[0])) if ncols > 2 else None
            fam = [base, JC.solve(_varied(base, c, rng), comp, target, filler)]
            own = _free_in(base, c)
            if len(own) >= 2:                               # unequal in column c alone
                fam.append(_collide(base, own[0], own[-1], target, rng, None if types[c] != FLOAT64 else own[0]))
            rows += family(fam)
    witness(rows)
    join_both(rows, rows[::-1], eq, len(rows))


# ---------------------------------------------------------------- nulls
@pytest.mark.parametrize("eq", [False, True])
def test_null_against_a_colliding_value(eq):
    rng = np.random.default_rng(140 + eq)
    for t in [INT32, FLOAT32, DECIMAL32, INT64, FLOAT64, TIMESTAMP_MICROSECONDS, DECIMAL128, STRING, INT16, BOOL8, UINT8]:
        for c in range(3):
            rows = []
            for _ in range(8):
                row = [(INT64, _rand(INT64, rng)), (STRING, _rand(STRING, rng))]
                row.insert(c, (t, _rand(t, rng)))
                null = list(row)
                null[c] = (t, None)
                target = JC.row_hash(null)
                own = _free_in(row, c)
                filler = (1 if c == 0 else 0, 0)            # the INT64 column's low half
                if own:                                     # the value solved in column c: the rows differ in validity alone
                    v = JC.solve(row, own[-1], target, filler)
                else:
                    v = JC.solve(row, (2 if c < 2 else 0, 0), target)
                null[c] = (t, Null(v[c][1]))                # the null's data slot holds the value it collides with
                rows += family([null, v])
            witness(rows)
            n = join_both(rows, rows[::-1], eq, len(rows) // 2)
            assert n == (len(rows) if eq else len(rows) // 2)


@pytest.mark.parametrize("eq", [False, True])
def test_nulls_in_the_same_columns(eq):
    rng = np.random.default_rng(150 + eq)
    for t in (INT64, STRING, DECIMAL128, INT32):
        rows = []
        for _ in range(16):
            a = [(t, Null(_rand(t, rng))), (INT64, _rand(INT64, rng)), (STRING, _rand(STRING, rng)), (t, Null(_rand(t, rng)))]
            m = model(a)
            b = _collide(m, (1, 0), (1, 1), JC.row_hash(m), rng)          # unequal in column 1, null in 0 and 3 alike
            c = _collide(m, (2, 0), (2, 1), JC.row_hash(m), rng)          # unequal in column 2
            rows += family([a, [(t, Null(_rand(t, rng)))] + b[1:3] + [a[3]], [a[0]] + c[1:3] + [(t, Null(_rand(t, rng)))]])
            rows.append([(t, Null(_rand(t, rng)))] + a[1:3] + [(t, Null(_rand(t, rng)))])   # a with other data under its nulls
        n = join_both(rows, rows[::-1], eq, 0)
        # with nulls equal, a row matches itself and a matches its copy with other data under its nulls; else none match
        assert n == (len(rows) + 2 * 16 if eq else 0)


# ---------------------------------------------------------------- strings
def _with_int32(s, x=0):
    return [(STRING, s), (INT32, x)]


def _compensate(row, avoid, target, rng):
    """row solved for target in a block of its string that holds none of the bytes `avoid`, or in its INT32 column when
    the string is shorter than 8 bytes"""
    n = len(row[0][1])
    if n < 8:
        return JC.solve(row, (1, 0), target)
    blocks = [j for j in range(n // 4) if not any(4 * j <= p < 4 * j + 4 for p in avoid)]
    return JC.solve(row, (0, blocks[int(rng.integers(0, len(blocks)))]), target)


def _placed(items, pad_byte):
    """every item at each of the four start offsets mod 4 of the chars buffer, each between pads of pad_byte"""
    out, pos = [], 0
    for it in items:
        for start in range(4):
            k = 4 + (start - pos) % 4
            out.append(_with_int32(bytes([pad_byte]) * k, -pad_byte & M32))
            out.append(it)
            pos += k + len(it[0][1])
    out.append(_with_int32(bytes([pad_byte]) * 5, -pad_byte & M32))
    return out


def _string_join(items, eq):
    witness(items)
    left, right = _placed(items, 0xFE), _placed(items[::-1], 0xFD)
    assert join_both(left, right, eq) == 16 * len(items)      # every item with its own copies, at all 16 alignments


LONG = [4097, 4100, 4102, 4103]


@pytest.mark.parametrize("eq", [False, True])
def test_strings_of_every_length(eq):
    rng = np.random.default_rng(160 + eq)
    items = []
    for n in list(range(73)) + LONG:
        base, target = _with_int32(rng.bytes(n), int(rng.integers(0, 1 << 32))), int(rng.integers(0, 1 << 32))
        fam = []
        for i in range(3 if n else 1):                     # one empty string hashes to the target, with one INT32
            s = rng.bytes(n)
            s = bytes([(s[0] + 85 * i) & 0xFF]) + s[1:] if n else s        # members differ in their first byte
            fam.append(JC.solve(_with_int32(s, base[1][1]), (0, n // 4 - 1) if n >= 8 else (1, 0), target))
        items += family(fam)
    _string_join(items, eq)


@pytest.mark.parametrize("eq", [False, True])
def test_strings_one_flipped_byte_at_every_position(eq):
    rng = np.random.default_rng(170 + eq)
    items = []
    for n in list(range(1, 73)) + LONG:
        for p in (range(n) if n < 100 else [0, 3, 4, 2047, n - 5, n - 4, n - 1]):
            for flip in (0x01, 0x80):
                a = _with_int32(rng.bytes(n), int(rng.integers(0, 1 << 32)))
                b = list(a)
                b[0] = (STRING, a[0][1][:p] + bytes([a[0][1][p] ^ flip]) + a[0][1][p + 1:])
                items += family([a, _compensate(b, [p], JC.row_hash(a), rng)])
    _string_join(items, eq)


@pytest.mark.parametrize("eq", [False, True])
def test_strings_against_their_colliding_extensions(eq):
    rng = np.random.default_rng(180 + eq)
    items = []
    for n in range(0, 73):
        a = _with_int32(rng.bytes(n), int(rng.integers(0, 1 << 32)))
        fam = [a]
        for e in range(1, 5):
            b = _with_int32(a[0][1] + rng.bytes(e), a[1][1])
            m = len(b[0][1])
            # b's last whole block takes the compensation (with n % 4 == 0 and e == 4 that is the new block, and a is an
            # exact prefix of b), or b's INT32 column below 4 bytes
            fam.append(JC.solve(b, (0, m // 4 - 1) if m >= 4 else (1, 0), JC.row_hash(a)))
        items += family(fam)
    _string_join(items, eq)


@pytest.mark.parametrize("eq", [False, True])
def test_strings_that_differ_only_in_their_tails(eq):
    rng = np.random.default_rng(190 + eq)
    items, found = [], 0
    while found < 12:                      # one column: the last two of its 2 or 3 tail bytes (a partial final word)
        n = 4 * int(rng.integers(0, 5)) + 2 + found % 2
        pair = JC.tail_collision(_with_int32(rng.bytes(n), int(rng.integers(0, 1 << 32))), (0, n - 2), (0, n - 1))
        if pair:
            items += family(list(pair))
            found += 1
    _string_join(items, eq)
    rows, found = [], 0
    while found < 12:                      # two columns: the last byte of each (1, 2 or 3 tail bytes)
        na, nb = 4 * int(rng.integers(0, 4)) + 1 + found % 3, 4 * int(rng.integers(0, 4)) + 1 + (found // 3) % 3
        pair = JC.tail_collision([(STRING, rng.bytes(na)), (STRING, rng.bytes(nb))], (0, na - 1), (1, nb - 1))
        if pair:
            rows += family(list(pair))
            found += 1
    witness(rows)
    join_both(rows, rows[::-1], eq, len(rows))


# ---------------------------------------------------------------- chains
def _chain_family(kind, size, target, rng):
    if kind == INT64:
        base = [(INT64, _rand(INT64, rng))]
        return family([_collide(base, (0, 0), (0, 1), target, rng) for _ in range(size)])
    if kind == STRING:
        base = [(STRING, rng.bytes(13))]
        return family([_collide(base, (0, 1), (0, 2), target, rng) for _ in range(size)])
    base = [(INT32, 0), (DECIMAL128, int.from_bytes(rng.bytes(16), "little"))]
    return family([_collide(base, (0, 0), (1, 3), target, rng) for _ in range(size)])


def _chain_case(kind, size, target, eq, rng):
    fam = _chain_family(kind, size, target, rng)
    witness(fam)
    right = [fam[i % size] for i in range(2 * size)]          # every key twice
    left = fam[::-1] + fam[: size // 3]
    assert join_both(left, right, eq) == 2 * len(left)


@pytest.mark.parametrize("kind", [INT64, STRING, DECIMAL128])
@pytest.mark.parametrize("eq", [False, True])
def test_chains_of_colliding_keys(kind, eq):
    rng = np.random.default_rng(200 + kind + eq)
    for size in (256, 1024):
        last = JC.buckets(2 * size) - 1                      # the chain starts in the last bucket and wraps to bucket 0
        for target in ((int(rng.integers(0, 1 << 32)) & ~last) | last, 0, M32):
            _chain_case(kind, size, target, eq, rng)


@pytest.mark.parametrize("nl", [2047, 2048, 2049])
def test_a_chain_in_a_million_row_table(nl):
    rng = np.random.default_rng(210 + nl)
    size, nr = 1024, 1 << 20
    last = JC.buckets(nr) - 1
    fam = _chain_family(INT64, size, (int(rng.integers(0, 1 << 32)) & ~last) | last, rng)
    witness(fam)
    fill = rng.integers(-(1 << 62), 1 << 62, nr - 2 * size, dtype=np.int64)
    fam_v = np.array([r[0][1] for r in fam], np.uint64).view(np.int64)
    right = np.concatenate([fill[: nr // 2], fam_v, fam_v, fill[nr // 2:]])
    probe = np.concatenate([fam_v[::-1], fill[: nl]])[: nl].copy()
    probe[1::7] = rng.integers(-(1 << 62), 1 << 62, len(probe[1::7]), dtype=np.int64)     # misses among the hits
    for eq in (False, True):
        check_join([OJ.Key(INT64, probe, None)], [OJ.Key(INT64, right, None)], eq)
