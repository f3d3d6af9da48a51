"""CPU checks of oracle/iceberg.py: against the Iceberg spec's hash vectors and truncate examples, the standard MurmurHash3
vector, hand-derived date / time answers, and the independent per-row model of tests/iceberg_model.py on random and
edge values.  Also the reciprocal remainder the kernels use (reciprocal.cuh) at the divisor extremes."""
import numpy as np
import pytest

import iceberg_model as M
from golden import iceberg_golden as G
from oracle import iceberg as O

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
DIVISORS = [1, 2, 3, 4, 7, 16, 1000, 1024, 2**16, 2**30, 2**30 + 1, 2**31 - 2, INT32_MAX]


def _mask(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _strings(rows):
    data = b"".join(rows)
    offs = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    return np.frombuffer(data, np.uint8).copy(), offs


def _dec128(vals):
    return np.array([[v % 2**64, (v >> 64) % 2**64] for v in vals], dtype=np.uint64).view(np.uint8).reshape(-1)


def test_model_murmur3_matches_the_standard_vector():
    data, want = G.MURMUR3_FOX
    assert M.murmur3_32(data) % 2**32 == want
    h = O.murmur3_rows(np.frombuffer(data, np.uint8)[None, :])
    assert int(h[0]) == want


@pytest.mark.parametrize("kind,value,want", G.HASH)
def test_spec_hash_vectors(kind, value, want):
    if kind in ("int", "long", "date", "timestamp"):
        got = M.hash_long(value)
        tid = {"int": O.INT32, "date": O.TIMESTAMP_DAYS, "long": O.INT64, "timestamp": O.TIMESTAMP_MICROSECONDS}[kind]
        arr = np.array([value], dtype="<i4" if tid in (O.INT32, O.TIMESTAMP_DAYS) else "<i8")
        n = INT32_MAX
        assert O.bucket(tid, arr, None, 1, n)[0] == (want & INT32_MAX) % n
    elif kind.startswith("decimal"):
        got = M.murmur3_32(M.java_bytes(value))
        for tid, arr in ((O.DECIMAL32, np.array([value], "<i4")), (O.DECIMAL64, np.array([value], "<i8")),
                         (O.DECIMAL128, _dec128([value]))):
            assert O.bucket(tid, arr, None, 1, INT32_MAX)[0] == (want & INT32_MAX) % INT32_MAX
    else:
        b = value.encode() if isinstance(value, str) else value
        got = M.murmur3_32(b)
        chars, offs = _strings([b])
        assert O.bucket(O.STRING if isinstance(value, str) else O.LIST, chars, None, 1, INT32_MAX, offs)[0] == \
            (want & INT32_MAX) % INT32_MAX
    assert got == want


@pytest.mark.parametrize("kind,width,value,want", G.TRUNCATE)
def test_spec_truncate_examples(kind, width, value, want):
    if kind == "string":
        chars, offs = _strings([value.encode()])
        o, b = O.truncate_bytes(O.STRING, chars, offs, None, 1, width)
        assert bytes(b) == want.encode() and list(o) == [0, len(want)]
        assert M.trunc_utf8(value.encode(), width) == want.encode()
        return
    tid, dt = {"int": (O.INT32, "<i4"), "long": (O.INT64, "<i8"), "decimal(9,2)": (O.DECIMAL32, "<i4")}[kind]
    out = O.truncate_integral(tid, np.array([value], dt), None, 1, width)
    assert int(out.view(dt)[0]) == want == M.trunc_int(value, width, 32 if dt == "<i4" else 64)


@pytest.mark.parametrize("transform,kind,value,want", G.DATETIME)
def test_datetime_goldens(transform, kind, value, want):
    tid, dt = (O.TIMESTAMP_DAYS, "<i4") if kind == "date" else (O.TIMESTAMP_MICROSECONDS, "<i8")
    assert O.datetime_transform(transform, tid, np.array([value], dt), 1)[0] == want
    days = value if kind == "date" else M.floor_days(value)
    model = {"years": M.years, "months": M.months, "days": lambda d: d}
    assert (M.hours(value) if transform == "hours" else model[transform](days)) == want


def test_bucket_oracle_matches_the_model():
    rng = np.random.default_rng(1)
    rows = 600
    valid = rng.random(rows) >= 0.2
    mask = _mask(valid)
    i32 = np.concatenate([[0, 1, -1, INT32_MIN, INT32_MAX], rng.integers(INT32_MIN, INT32_MAX, rows - 5)]).astype("<i4")
    i64 = np.concatenate([[0, 1, -1, INT64_MIN, INT64_MAX], rng.integers(INT64_MIN, INT64_MAX, rows - 5, dtype=np.int64)])
    d128 = [0, 1, -1, 2**127 - 1, -2**127] + [int(rng.integers(-2**62, 2**62)) << int(rng.integers(0, 64)) for _ in range(rows - 5)]
    d128 = [((v + 2**127) % 2**128) - 2**127 for v in d128]
    strs = [bytes(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8)) for _ in range(rows)]
    chars, offs = _strings(strs)
    for n in (1, 2, 16, 1000, 2**30 + 1, INT32_MAX):
        for tid, arr, vals, enc in [
            (O.INT32, i32, i32, lambda v: (int(v) % 2**64).to_bytes(8, "little")),
            (O.TIMESTAMP_DAYS, i32, i32, lambda v: (int(v) % 2**64).to_bytes(8, "little")),
            (O.INT64, i64, i64, lambda v: (int(v) % 2**64).to_bytes(8, "little")),
            (O.DECIMAL32, i32, i32, lambda v: M.java_bytes(int(v))),
            (O.DECIMAL64, i64, i64, lambda v: M.java_bytes(int(v))),
            (O.DECIMAL128, _dec128(d128), d128, M.java_bytes),
        ]:
            got = O.bucket(tid, arr, mask, rows, n)
            want = [M.bucket_value(M.murmur3_32(enc(v)), n) if ok else 0 for v, ok in zip(vals, valid)]
            assert got.tolist() == want, (tid, n)
        got = O.bucket(O.STRING, chars, mask, rows, n, offs)
        assert got.tolist() == [M.bucket_value(M.murmur3_32(s), n) if ok else 0 for s, ok in zip(strs, valid)]


@pytest.mark.parametrize("k", range(1, 17))
def test_decimal_byte_counts_at_every_boundary(k):
    """BigInteger.toByteArray is k bytes for -2^(8k-1) <= v < 2^(8k-1) and no fewer"""
    vals = [2**(8 * k - 1) - 1, -2**(8 * k - 1)]
    if k < 16:
        vals += [2**(8 * k - 1), -2**(8 * k - 1) - 1]
    be, n = O.decimal_java_bytes(_dec128(vals).view("<i8").reshape(-1, 2))
    assert n.tolist() == [len(M.java_bytes(v)) for v in vals]
    assert n[0] == n[1] == k and (k == 16 or (n[2] == n[3] == k + 1))
    for i, v in enumerate(vals):
        assert bytes(be[i, 16 - n[i]:]) == M.java_bytes(v)


@pytest.mark.parametrize("d", DIVISORS + [2**31])
def test_reciprocal_remainder_at_the_divisor_extremes(d):
    """reciprocal.cuh: mod_v1 (x <= 2^31) and mod_v2 (x <= 2^63) against Python %"""
    m1, m2 = (2**32 - 1) // d, (2**64 - 1) // d
    xs = {0, 1, d - 1, d, d + 1, 2 * d - 1, 2**31 - 1, 2**31, (2**31 // d) * d, (2**31 // d) * d - 1}
    for x in sorted(v for v in xs if 0 <= v <= 2**31):
        r = (x - ((x * m1) >> 32) * d) % 2**32
        assert (r - d if r >= d else r) == x % d, (x, d)
    for x in (0, 1, d - 1, d, 2**63 - 1, 2**63, (2**63 // d) * d, (2**63 // d) * d - 1, d * 2**32 - 1):
        if 0 <= x <= 2**63:
            r = (x - ((x * m2) >> 64) * d) % 2**64
            assert (r - d if r >= d else r) == x % d, (x, d)


WIDTHS = [1, -1, 2, -2, 10, -10, 1000, INT32_MAX, INT32_MIN, 2**30 + 1, -(2**30 + 1)]


@pytest.mark.parametrize("w", WIDTHS)
def test_truncate_integral_oracle_matches_the_model(w):
    rng = np.random.default_rng(abs(w) % 1000)
    i32 = np.concatenate([[0, 1, -1, INT32_MIN, INT32_MAX, INT32_MIN + 1, INT32_MAX - 1, -5, 5],
                          rng.integers(INT32_MIN, INT32_MAX, 200)]).astype("<i4")
    i64 = np.concatenate([[0, 1, -1, INT64_MIN, INT64_MAX, INT64_MIN + 1, -5, 5], rng.integers(INT64_MIN, INT64_MAX, 200, dtype=np.int64)])
    d128 = [0, 1, -1, 2**127 - 1, -2**127, -2**127 + 1, -5, 5] + [int(rng.integers(-2**62, 2**62)) << 60 for _ in range(50)]
    valid = np.ones(len(i32), bool)
    valid[3] = False
    for tid, arr, vals, bits, dt in [(O.INT32, i32, i32, 32, "<i4"), (O.DECIMAL32, i32, i32, 32, "<i4"),
                                     (O.INT64, i64, i64, 64, "<i8"), (O.DECIMAL64, i64, i64, 64, "<i8")]:
        m = _mask(valid[: len(vals)])
        got = O.truncate_integral(tid, arr, m, len(vals), w).view(dt)
        want = [M.trunc_int(int(v), w, bits) if ok else 0 for v, ok in zip(vals, valid[: len(vals)])]
        assert got.tolist() == want, tid
    got = O.truncate_integral(O.DECIMAL128, _dec128(d128), None, len(d128), w).view("<u8").reshape(-1, 2)
    assert [int(lo) | (int(hi) << 64) for lo, hi in got] == [M.trunc_int(v, w, 128) % 2**128 for v in d128]


def test_truncate_wraps_as_the_reference_does():
    # INT32_MIN % -1 is 0; (-5 % INT32_MIN) + INT32_MIN wraps to 2^31 - 5
    assert M.trunc_int(INT32_MIN, -1, 32) == INT32_MIN
    assert M.trunc_int(-5, INT32_MIN, 32) == ((-5 - (2**31 - 5)) + 2**31) % 2**32 - 2**31
    assert M.trunc_int(INT64_MIN, -1, 64) == INT64_MIN
    assert O.truncate_integral(O.INT32, np.array([-5], "<i4"), None, 1, INT32_MIN).view("<i4")[0] == M.trunc_int(-5, INT32_MIN, 32)


CHARS = ["a", "é", "€", "😀"]


@pytest.mark.parametrize("width", [1, 2, 3, 4, 5, 16, 1000, INT32_MAX])
def test_truncate_string_oracle_matches_the_model(width):
    rng = np.random.default_rng(width % 97)
    rows = [("".join(rng.choice(CHARS, int(rng.integers(0, 12))))).encode() for _ in range(300)]
    rows += [b"\x80\x80abc", b"\xc3", b"ab\xe2\x82", b"\xff\xfe\xfd\xfc\xfb", b"", b"\xf0\x9f\x98\x80" * 3]   # malformed too
    chars, offs = _strings(rows)
    valid = np.ones(len(rows), bool)
    valid[::7] = False
    o, b = O.truncate_bytes(O.STRING, chars, offs, _mask(valid), len(rows), width)
    want = [M.trunc_utf8(r, width) if ok else b"" for r, ok in zip(rows, valid)]
    assert [bytes(b[o[i]:o[i + 1]]) for i in range(len(rows))] == want
    o, b = O.truncate_bytes(O.LIST, chars, offs, _mask(valid), len(rows), width)
    assert [bytes(b[o[i]:o[i + 1]]) for i in range(len(rows))] == [r[:width] if ok else b"" for r, ok in zip(rows, valid)]


def test_datetime_oracle_matches_the_model():
    rng = np.random.default_rng(7)
    days = np.concatenate([[0, -1, 1, INT32_MIN, INT32_MAX, -719162, -719163, 2932896, 2932897, 11016, -141427],
                           rng.integers(INT32_MIN, INT32_MAX, 300)]).astype("<i4")
    for tr, fn in (("years", M.years), ("months", M.months), ("days", lambda d: d)):
        assert O.datetime_transform(tr, O.TIMESTAMP_DAYS, days, len(days)).tolist() == [fn(int(d)) for d in days]
    D, H = 86_400_000_000, 3_600_000_000
    micros = np.concatenate([[0, -1, 1, INT64_MIN, INT64_MAX, D, D - 1, D + 1, -D, -D - 1, -D + 1, H, H - 1, -H, -H - 1],
                             rng.integers(INT64_MIN, INT64_MAX, 300, dtype=np.int64)])
    for tr, fn in (("years", lambda t: M.years(M.floor_days(t))), ("months", lambda t: M.months(M.floor_days(t))),
                   ("days", M.floor_days), ("hours", M.hours)):
        assert O.datetime_transform(tr, O.TIMESTAMP_MICROSECONDS, micros, len(micros)).tolist() == [fn(int(t)) for t in micros]
