"""JoinPrimitives on the device against oracle/join.py: the inner join's pair multiset and its non-decreasing left map, and
the outer / semi / anti / matched-rows helpers byte for byte.  Covers every fixed-width key type, DECIMAL128 and STRING
(empty and > 4 KB strings), one to eight mixed key columns, both null modes at 0 / 10 / 100 % nulls, empty sides, build
sizes either side of each table size, left sizes at tile edges, heavy duplicates, unaligned buffers, four threads on their
own streams, 50 M probe rows and a join of more than 2^31 pairs."""
import threading

import numpy as np
import pytest
import torch

from oracle import join as OJ

pytestmark = pytest.mark.gpu

INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8 = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11
TS_DAYS, TS_S, TS_MS, TS_US, TS_NS, DUR_D, DUR_S, DUR_MS, DUR_US, DUR_NS = range(12, 22)
STRING, DEC32, DEC64, DEC128 = 23, 25, 26, 27
NP = {INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, UINT8: np.uint8, UINT16: np.uint16, UINT32: np.uint32,
      UINT64: np.uint64, FLOAT32: np.float32, FLOAT64: np.float64, BOOL8: np.uint8, TS_DAYS: np.int32, DUR_D: np.int32, DEC32: np.int32,
      DEC64: np.int64}
FIXED = [INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8, TS_DAYS, TS_S, TS_MS, TS_US, TS_NS, DUR_D,
         DUR_S, DUR_MS, DUR_US, DUR_NS, DEC32, DEC64]


def _np_type(t):
    return NP.get(t, np.int64)


def _values(t, n, pool, rng):
    """n values drawn from `pool` distinct keys, so that both sides share keys"""
    pick = rng.integers(0, pool, n)
    if t == STRING:
        words = [b"", b"a", b"ab", b"abc\x00", bytes(range(200, 256)), b"x" * 4100, b"x" * 4099 + b"y"] + \
                [rng.bytes(int(rng.integers(0, 40))) for _ in range(max(0, pool - 7))]
        return [words[i % len(words)] for i in pick]
    if t == DEC128:
        lo = (pick.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)).view(np.int64)
        return np.stack([lo, (pick % 3 - 1).astype(np.int64)], axis=1)
    if t == FLOAT32:
        specials = np.array([np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf], np.float32)
        v = (pick.astype(np.float32) * np.float32(0.5)) - 3
        v[pick < 6] = specials[pick[pick < 6]]
        bits = v.view(np.uint32).copy()
        bits[(pick == 0) & (np.arange(n) % 2 == 1)] = 0x7fc00123          # another NaN payload
        return bits.view(np.float32)
    if t == FLOAT64:
        specials = np.array([np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf])
        v = pick.astype(np.float64) * 0.25 - 3
        v[pick < 6] = specials[pick[pick < 6]]
        bits = v.view(np.uint64).copy()
        bits[(pick == 0) & (np.arange(n) % 2 == 1)] = 0xfff0000000000001  # a signalling NaN
        return bits.view(np.float64)
    if t == BOOL8:
        return (pick % 3 * (np.arange(n) % 2 + 1)).astype(np.uint8)       # 0, and true as 1, 2 or 4
    return (pick * 2654435761 - pool).astype(_np_type(t))


def _key(t, n, pool, null_frac, rng):
    valid = None if null_frac == 0 else rng.random(n) >= null_frac
    return OJ.Key(t, _values(t, n, pool, rng), valid)


def _mask(valid, n):
    if valid is None:
        return None
    b = np.packbits(np.asarray(valid, bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4 + (4 if len(b) == 0 else 0), np.uint8)])


def to_dev(k: OJ.Key, scale=0, shift=0):
    """a device column; shift > 0 places the data `shift` bytes past a 256-byte boundary"""
    import srj_b200 as S
    n = len(k.values)
    mask = _mask(k.valid, n)
    dmask = torch.from_numpy(mask.view(np.int32).copy()).cuda() if mask is not None else None
    if k.type_id == STRING:
        lens = np.array([len(v) for v in k.values], np.int64)
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        raw = np.frombuffer(b"".join(k.values), np.uint8)
        data = torch.zeros(len(raw) + shift + 1, dtype=torch.uint8, device="cuda")[shift:shift + len(raw)]
        data.copy_(torch.from_numpy(raw.copy()))
        return S.ColumnVector(S.DType(STRING), n, data, dmask, torch.from_numpy(offs).cuda())
    raw = np.ascontiguousarray(k.values).view(np.uint8).reshape(-1)
    data = torch.zeros(len(raw) + shift, dtype=torch.uint8, device="cuda")[shift:]
    data.copy_(torch.from_numpy(raw.copy()))
    return S.ColumnVector(S.DType(k.type_id, scale), n, data, dmask)


def run_join(left, right, eq, shift=0):
    import srj_b200 as S
    from srj_b200.join import JoinPrimitives
    gl, gr = JoinPrimitives.hashInnerJoin(S.Table([to_dev(k, shift=shift) for k in left]), S.Table([to_dev(k, shift=shift) for k in right]), eq)
    return gl.data.cpu().numpy(), gr.data.cpu().numpy()


def check_join(left, right, eq, shift=0):
    L, R = run_join(left, right, eq, shift)
    assert len(L) == len(R)
    assert np.all(np.diff(L.astype(np.int64)) >= 0), "the left map is not non-decreasing"
    idx = np.lexsort((R, L))
    wl, wr = OJ.inner_join(left, right, eq)
    assert np.array_equal(L[idx], wl) and np.array_equal(R[idx], wr)
    return len(L)


@pytest.mark.parametrize("t", FIXED + [DEC128, STRING])
@pytest.mark.parametrize("eq", [False, True])
def test_every_key_type(t, eq):
    rng = np.random.default_rng(t * 2 + eq)
    left, right = [_key(t, 3000, 300, 0.1, rng)], [_key(t, 2000, 300, 0.1, rng)]
    assert check_join(left, right, eq) > 0


@pytest.mark.parametrize("ncols", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("null_frac", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("eq", [False, True])
def test_mixed_key_columns_and_nulls(ncols, null_frac, eq):
    rng = np.random.default_rng(ncols * 100 + int(null_frac * 10) + eq)
    types = [[INT32, STRING, INT64, DEC128, FLOAT64, BOOL8, INT16, TS_US][(i * 3 + ncols) % 8] for i in range(ncols)]
    left = [_key(t, 5000, 3, null_frac, rng) for t in types]
    right = [_key(t, 4000, 3, null_frac, rng) for t in types]
    n = check_join(left, right, eq)
    if null_frac == 1.0 and not eq:
        assert n == 0


@pytest.mark.parametrize("nl,nr", [(0, 10), (10, 0), (0, 0)])
def test_either_side_empty(nl, nr):
    rng = np.random.default_rng(5)
    assert check_join([_key(INT32, nl, 4, 0, rng)], [_key(INT32, nr, 4, 0, rng)], True) == 0


@pytest.mark.parametrize("nr", [1, 2, 3, 4, 5, 7, 8, 9, 63, 64, 65, 1023, 1024, 1025, 4095, 4096, 4097, 65535, 65536, 65537])
def test_build_sizes_at_table_size_edges(nr):
    rng = np.random.default_rng(nr)
    check_join([_key(INT64, 3000, nr + 5, 0, rng)], [_key(INT64, nr, nr + 5, 0, rng)], False)


@pytest.mark.parametrize("nl", [1, 255, 256, 257, 2047, 2048, 2049, 4096, 10241])
def test_left_sizes_at_tile_edges(nl):
    rng = np.random.default_rng(nl)
    check_join([_key(STRING, nl, 50, 0.1, rng), _key(INT32, nl, 2, 0, rng)], [_key(STRING, 700, 50, 0.1, rng), _key(INT32, 700, 2, 0, rng)], True)


def test_heavy_duplicates():
    rng = np.random.default_rng(9)
    left = [OJ.Key(INT64, np.full(3000, 42, np.int64), None)]
    right = [OJ.Key(INT64, np.concatenate([np.full(2000, 42, np.int64), np.arange(1000, 1500, dtype=np.int64)]), None)]
    assert check_join(left, right, False) == 3000 * 2000
    check_join([_key(INT32, 20000, 5, 0.05, rng)], [_key(INT32, 5000, 5, 0.05, rng)], True)


def test_float_and_string_edges():
    nan_a = np.array([0x7ff8000000000000, 0x7ff8000000000123, 0xfff0000000000001, 0x8000000000000000, 0], np.uint64).view(np.float64)
    left = [OJ.Key(FLOAT64, nan_a, None)]
    right = [OJ.Key(FLOAT64, nan_a[::-1].copy(), None)]
    L, R = run_join(left, right, False)
    pairs = set(zip(L.tolist(), R.tolist()))
    assert pairs == {(a, b) for a in range(3) for b in (2, 3, 4)} | {(a, b) for a in (3, 4) for b in (0, 1)}   # NaNs; zeros
    # null against the empty string: equal only as two nulls (nulls equal), never as null == ""
    s_left = [OJ.Key(STRING, [b"", b"", b"a"], np.array([True, False, True]))]
    s_right = [OJ.Key(STRING, [b"", b""], np.array([False, True]))]
    assert set(zip(*[m.tolist() for m in run_join(s_left, s_right, True)])) == {(0, 1), (1, 0)}
    assert set(zip(*[m.tolist() for m in run_join(s_left, s_right, False)])) == {(0, 1)}


def test_unaligned_buffers():
    rng = np.random.default_rng(11)
    types = [INT64, DEC128, STRING, INT32, FLOAT64]
    left = [_key(t, 3001, 40, 0.1, rng) for t in types]
    right = [_key(t, 2003, 40, 0.1, rng) for t in types]
    check_join(left, right, True, shift=8)       # 8 bytes off a 16- and 32-byte boundary: element-aligned only


def test_decimal_scale_mismatch_and_schema_errors():
    import srj_b200 as S
    from srj_b200.join import JoinPrimitives
    a = OJ.Key(DEC64, np.arange(4, dtype=np.int64), None)
    with pytest.raises(S.CudfException):
        JoinPrimitives.hashInnerJoin(S.Table([to_dev(a, scale=-2)]), S.Table([to_dev(a, scale=-3)]), True)
    e = OJ.Key(DEC64, np.zeros(0, np.int64), None)
    gl, gr = JoinPrimitives.hashInnerJoin(S.Table([to_dev(e, scale=-2)]), S.Table([to_dev(a, scale=-3), to_dev(a)]), True)
    assert gl.getRowCount() == gr.getRowCount() == 0


def _helpers_check(L, R, nl, nr):
    from srj_b200.join import GatherMap, JoinPrimitives
    dl, dr = GatherMap(torch.from_numpy(L.astype(np.int32)).cuda()), GatherMap(torch.from_numpy(R.astype(np.int32)).cuda())
    for got, want in ((JoinPrimitives.makeLeftOuter(dl, dr, nl, nr), OJ.make_left_outer(L, R, nl, nr)),
                      (JoinPrimitives.makeFullOuter(dl, dr, nl, nr), OJ.make_full_outer(L, R, nl, nr))):
        assert np.array_equal(got[0].data.cpu().numpy(), want[0]) and np.array_equal(got[1].data.cpu().numpy(), want[1])
    assert np.array_equal(JoinPrimitives.makeSemi(dl, nl).data.cpu().numpy(), OJ.make_semi(L, nl))
    assert np.array_equal(JoinPrimitives.makeAnti(dl, nl).data.cpu().numpy(), OJ.make_anti(L, nl))
    mr = JoinPrimitives.getMatchedRows(dr, nr)
    assert mr.mask is None and np.array_equal(mr.data.cpu().numpy(), OJ.get_matched_rows(R, nr))


@pytest.mark.parametrize("nl,nr,n", [(0, 0, 0), (5, 0, 0), (0, 5, 0), (1, 1, 1), (31, 33, 40), (32, 64, 100), (8191, 8193, 20000),
                                     (8192, 16385, 3), (100000, 70000, 250000)])
def test_helpers_byte_for_byte(nl, nr, n):
    rng = np.random.default_rng(nl + nr + n)
    L = rng.integers(-3, nl + 3, n) if nl else rng.integers(-3, 3, n)
    R = rng.integers(-3, nr + 3, n) if nr else rng.integers(-3, 3, n)
    L[:: 7] = OJ.INT32_MIN
    _helpers_check(L.astype(np.int32), R.astype(np.int32), nl, nr)


def test_helpers_from_a_join():
    rng = np.random.default_rng(21)
    left, right = [_key(INT32, 30000, 20000, 0.05, rng)], [_key(INT32, 25000, 20000, 0.05, rng)]
    L, R = OJ.inner_join(left, right, False)
    _helpers_check(L, R, 30000, 25000)


def test_four_threads_on_their_own_streams():
    rng = np.random.default_rng(31)
    cases = [([_key(t, 40000, 5000, 0.1, rng)], [_key(t, 30000, 5000, 0.1, rng)]) for t in (INT64, STRING, DEC128, FLOAT32)]
    results, errors = [None] * 4, []

    def work(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                results[i] = run_join(*cases[i], True)
                torch.cuda.current_stream().synchronize()
        except Exception as e:        # noqa: BLE001  (reported below)
            errors.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for (L, R), (left, right) in zip(results, cases):
        idx = np.lexsort((R, L))
        wl, wr = OJ.inner_join(left, right, True)
        assert np.array_equal(L[idx], wl) and np.array_equal(R[idx], wr)


def test_fifty_million_probe_rows():
    import srj_b200 as S
    from srj_b200.join import JoinPrimitives
    rng = np.random.default_rng(41)
    nr, nl = 1_000_000, 50_000_000
    perm = rng.permutation(nr)
    right = torch.from_numpy((perm.astype(np.int64) * 7)).cuda()
    left = torch.randint(0, 14 * nr, (nl,), dtype=torch.int64, device="cuda", generator=torch.Generator("cuda").manual_seed(7))
    gl, gr = JoinPrimitives.hashInnerJoin(S.Table([S.ColumnVector(S.DType(INT64), nl, left.view(torch.uint8))]),
                                          S.Table([S.ColumnVector(S.DType(INT64), nr, right.view(torch.uint8))]), False)
    hit = (left % 7 == 0) & (left < 7 * nr)
    want_l = torch.nonzero(hit).view(-1).to(torch.int32)
    inv = torch.empty(nr, dtype=torch.int64, device="cuda")
    inv[torch.from_numpy(perm).cuda()] = torch.arange(nr, device="cuda")
    want_r = inv[left[hit] // 7].to(torch.int32)
    assert torch.equal(gl.data, want_l) and torch.equal(gr.data, want_r)


def test_more_than_two_to_the_31_pairs():
    import srj_b200 as S
    from srj_b200.join import JoinPrimitives
    nr, nl = 65_536, 32_769
    if torch.cuda.get_device_properties(0).total_memory < 40 * 2 ** 30:
        pytest.skip("needs a card with 40 GB")
    right = torch.full((nr,), 5, dtype=torch.int32, device="cuda")
    left = torch.full((nl,), 5, dtype=torch.int32, device="cuda")
    gl, gr = JoinPrimitives.hashInnerJoin(S.Table([S.ColumnVector(S.DType(INT32), nl, left.view(torch.uint8))]),
                                          S.Table([S.ColumnVector(S.DType(INT32), nr, right.view(torch.uint8))]), False)
    assert gl.getRowCount() == nl * nr > 2 ** 31
    del left, right
    for b in range(0, nl, 1024):                          # per left row: 65,536 entries, its own index, right rows summing right
        e = min(nl, b + 1024)
        lrows = gl.data[b * nr:e * nr].view(e - b, nr)
        assert bool((lrows == torch.arange(b, e, device="cuda", dtype=torch.int32).view(-1, 1)).all())
        rrows = gr.data[b * nr:e * nr].view(e - b, nr).to(torch.int64)
        assert bool((rrows.sum(1) == nr * (nr - 1) // 2).all()) and bool((rrows.pow(2).sum(1) == (nr - 1) * nr * (2 * nr - 1) // 6).all())
        assert bool((rrows.min(1).values == 0).all()) and bool((rrows.max(1).values == nr - 1).all())
