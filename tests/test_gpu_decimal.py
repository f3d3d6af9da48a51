"""GPU checks of DecimalUtils (srj_b200.decimal over libsrj_b200.so) against oracle/decimal.py, which
tests/test_oracle_decimal.py pins to the reference's DecimalUtilsTest cases, hand-derived edges and an independent model.
Every valid row's overflow flag and value are compared, and both output columns' masks and null counts."""
import threading

import numpy as np
import pytest

from oracle import decimal as O

pytestmark = pytest.mark.gpu

MAX38 = 10**38 - 1
OPS = {O.MULTIPLY: "multiply", O.DIVIDE: "divide", O.INTEGER_DIVIDE: "intdiv", O.REMAINDER: "remainder", O.ADD: "add",
       O.SUBTRACT: "subtract"}
# (a_scale, b_scale, out_scale) per op: Spark's result scales, positive cudf scales, and each divide / remainder path
GRID = {
    O.MULTIPLY: [(-10, -10, -6), (-2, -2, -4), (0, 0, 0), (-38, -38, -38), (-5, -3, -10), (2, 1, 0), (3, 2, 7), (-19, -19, -2),
                 (-1, 0, -30)],
    O.DIVIDE: [(-10, -10, -6), (-2, -5, -10), (0, -38, -38), (-38, 0, -38), (-6, -2, -20), (2, -3, 0), (-1, -1, 10), (5, -30, -40),
               (0, 0, -39), (0, 38, -38), (4, 0, 0)],
    O.REMAINDER: [(-2, -3, -3), (-3, -2, -3), (-10, -10, -10), (-2, -5, -2), (0, 3, 0), (-38, -1, -38), (2, 0, 0), (0, -20, -20)],
    O.ADD: [(-10, -2, -10), (-2, -10, -6), (0, 0, 0), (3, -3, -5), (-38, 38, -38), (-1, -1, 2), (-6, -6, -6), (10, 20, 12)],
}
GRID[O.INTEGER_DIVIDE] = [(a, b, 0) for a, b, _ in GRID[O.DIVIDE]] + [(-2, -3, 1), (0, 0, -2)]
GRID[O.SUBTRACT] = GRID[O.ADD]


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200 import decimal as D
    return S, D


def _mask(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _values(rng, n, edges=True):
    """signed values of 1-38 digits, both signs, with 0, +-(10^38 - 1), powers of ten and +-1 mixed in"""
    digits = rng.integers(1, 39, n)
    vals = [int(rng.integers(1, 10)) * 10 ** (int(d) - 1) + int.from_bytes(rng.bytes(16), "little") % 10 ** (int(d) - 1) if d > 1
            else int(rng.integers(0, 10)) for d in digits]
    vals = [-v if s else v for v, s in zip(vals, rng.random(n) < 0.5)]
    if edges:
        special = [0, 1, -1, MAX38, -MAX38, 10**37, -10**37, 5, -5, 15, -25, 10**19, 2**63, -2**63, 2**64]
        for i, v in zip(rng.choice(n, min(n, 3 * len(special)), replace=False), special * 3):
            vals[int(i)] = v
    return vals


def _col(S, vals, scale, valid=None, offset=0):
    """a DECIMAL128 column; offset bytes (0 or 8) in front of its data, so that 8 gives an 8-byte-aligned input"""
    import torch
    raw = np.concatenate([np.zeros(offset, np.uint8), O.from_ints(vals)])
    t = torch.from_numpy(raw).cuda()[offset:]
    m = None if valid is None else torch.from_numpy(_mask(valid).view(np.int32).copy()).cuda()
    return S.ColumnVector(S.DType(S.DType.DECIMAL128, scale), len(vals), t, m)


def _check(op, tbl, a, b, sa, sb, so, va=None, vb=None, interim=True):
    n = len(a)
    want = [O.row(op, x, y, sa, sb, so, interim) for x, y in zip(a, b)]
    valid = np.ones(n, bool)
    for v in (va, vb):
        if v is not None:
            valid &= np.asarray(v, bool)
    ovf_col, val_col = tbl.getColumn(0), tbl.getColumn(1)
    ovf = ovf_col.data.cpu().numpy()
    w = 8 if op == O.INTEGER_DIVIDE else 16
    got = val_col.data.cpu().numpy()
    gvals = [int.from_bytes(got[w * i:w * i + w].tobytes(), "little", signed=True) for i in range(n)]
    for i in np.nonzero(valid)[0]:
        assert (bool(ovf[i]), gvals[i]) == (bool(want[i][0]), want[i][1]), (OPS[op], sa, sb, so, a[i], b[i], i)
    want_mask, want_nulls = O.mask_and(None if va is None else _mask(va), None if vb is None else _mask(vb), n)
    for c in (ovf_col, val_col):
        assert c.getNullCount() == want_nulls
        if want_mask is None:
            assert c.mask is None
        else:
            bits = np.unpackbits(c.mask.cpu().numpy().view(np.uint8), bitorder="little")[:n]
            assert np.array_equal(bits, np.unpackbits(want_mask.view(np.uint8), bitorder="little")[:n])
    assert val_col.getType().type_id == (S_INT64 if op == O.INTEGER_DIVIDE else S_DEC128)
    if op != O.INTEGER_DIVIDE:
        assert val_col.getType().scale == so


S_INT64, S_DEC128 = 4, 27


def _call(D, op, a, b, so, interim=True):
    if op == O.MULTIPLY:
        return D.DecimalUtils.multiply128(a, b, so, interim)
    if op == O.DIVIDE:
        return D.DecimalUtils.divide128(a, b, so)
    if op == O.INTEGER_DIVIDE:
        return D.DecimalUtils.integerDivide128(a, b) if so == 0 else D._binary(O.INTEGER_DIVIDE, a, b, so, False, "intdiv")
    if op == O.REMAINDER:
        return D.DecimalUtils.remainder128(a, b, so)
    if op == O.ADD:
        return D.DecimalUtils.add128(a, b, so)
    return D.DecimalUtils.subtract128(a, b, so)


@pytest.mark.parametrize("op", sorted(OPS))
def test_scale_grid(op):
    S, D = _s()
    rng = np.random.default_rng(100 + op)
    n = 1500
    for sa, sb, so in GRID[op]:
        O.check_scales(op, sa, sb, so)
        a, b = _values(rng, n), _values(rng, n)
        if op in (O.DIVIDE, O.INTEGER_DIVIDE, O.REMAINDER):
            b[:6] = [0, 1, -1, 10, -10, 3]
        for interim in ((True, False) if op == O.MULTIPLY else (True,)):
            tbl = _call(D, op, _col(S, a, sa), _col(S, b, sb), so, interim)
            _check(op, tbl, a, b, sa, sb, so, interim=interim)


def test_divide_paths_ties_and_small_divisors():
    S, D = _s()
    # ties of both signs at each divide path, divisors +-1 / 0, exact powers of ten
    a = [5, -5, 15, -15, 25, 1, -1, 10**37, -10**37, MAX38, -MAX38, 7, 0, 2, -2, 10**38 - 5]
    b = [10, 10, -10, -10, 2, 2, 2, 1, -1, 1, -1, 0, 3, 4, -4, 10]
    for sa, sb, so in [(0, 0, 0), (0, 0, -1), (0, 0, -39), (0, 0, -60), (-3, 0, -2), (1, 0, 0), (0, 0, 1), (0, -38, -38), (0, 0, -114)]:
        for op in (O.DIVIDE, O.INTEGER_DIVIDE):
            tbl = _call(D, op, _col(S, a, sa), _col(S, b, sb), so)
            _check(op, tbl, a, b, sa, sb, so)


def test_integer_divide_around_int64_limits():
    S, D = _s()
    a, b = [], []
    for q in (2**63 - 1, 2**63, 2**63 + 1, -2**63, -2**63 - 1, 2**64, -2**64 + 1, 2**70 + 3):
        for d in (1, -1, 7, -3):
            a.append(q * d if abs(q * d) <= MAX38 else q)
            b.append(d)
    tbl = D.DecimalUtils.integerDivide128(_col(S, a, 0), _col(S, b, 0))
    _check(O.INTEGER_DIVIDE, tbl, a, b, 0, 0, 0)


def test_multiply_precision10_edges_and_early_exit():
    S, D = _s()
    a, b = [], []
    for k in range(0, 39):
        for x, y in ((10**k, 10**(38 - k)), (10**k, 10**(38 - k) - 1), (10**k + 1, 10**(38 - k)), (-(10**k), 10**(38 - k) + 1)):
            a.append(x if abs(x) <= MAX38 else MAX38)
            b.append(y if abs(y) <= MAX38 else MAX38)
    a += [MAX38, -MAX38, MAX38, 0]
    b += [MAX38, MAX38, 1, MAX38]
    for sa, sb, so in [(0, 0, 0), (0, 0, -1), (-10, -10, -6), (-20, -20, -38), (0, 0, -38), (1, 1, 0)]:
        for interim in (True, False):
            tbl = D.DecimalUtils.multiply128(_col(S, a, sa), _col(S, b, sb), so, interim)
            _check(O.MULTIPLY, tbl, a, b, sa, sb, so, interim=interim)


def test_multiply_far_below_the_product_scale():
    # product scales far below a_scale + b_scale: every row takes the early exit (overflow, 0), including rows whose
    # interim cast rounds first (products of 40+ digits), where e0 - k must not wrap around int32
    S, D = _s()
    a = [10**20, -(10**20), MAX38, 1, 0, 10**19]
    b = [10**20, 10**20, MAX38, 1, 0, 10**19]
    for sa, sb, so in ((0, 0, -(2**31) + 1), (0, 0, -(2**31)), (2**31 - 1, 2**31 - 1, -(2**31)), (5, -(2**31), -(2**31) + 3), (0, 0, -40),
                       (0, 0, -39)):
        for interim in (True, False):
            tbl = D.DecimalUtils.multiply128(_col(S, a, sa), _col(S, b, sb), so, interim)
            _check(O.MULTIPLY, tbl, a, b, sa, sb, so, interim=interim)


def test_remainder_divisor_rounding_to_zero():
    S, D = _s()
    a = [123456, -123456, 7, -7, MAX38, 10**20]
    b = [4, -4, 49, -50, 3, 5]         # at rem_scale = b_scale + 2 these divisors round to 0, 0, 0, 1 (HALF_UP of 0.50), 0, 0
    tbl = D.DecimalUtils.remainder128(_col(S, a, 0), _col(S, b, 0), 2)
    _check(O.REMAINDER, tbl, a, b, 0, 0, 2)


@pytest.mark.parametrize("masks", ["none", "a", "b", "both", "all_null"])
def test_masks_and_null_counts(masks):
    S, D = _s()
    rng = np.random.default_rng(7)
    n = 777
    a, b = _values(rng, n), _values(rng, n)
    va = rng.random(n) > 0.3 if masks in ("a", "both") else None
    vb = rng.random(n) > 0.2 if masks in ("b", "both") else None
    if masks == "all_null":
        va = np.zeros(n, bool)
    for op in sorted(OPS):
        sa, sb, so = GRID[op][0]
        tbl = _call(D, op, _col(S, a, sa, va), _col(S, b, sb, vb), so)
        _check(op, tbl, a, b, sa, sb, so, va, vb)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1023, 1024, 1025, 4 * 256 + 3])
def test_row_counts_and_tile_edges(n):
    S, D = _s()
    rng = np.random.default_rng(n)
    a, b = _values(rng, n, edges=n > 50), _values(rng, n, edges=n > 50)
    va = rng.random(n) > 0.1
    for op in sorted(OPS):
        sa, sb, so = GRID[op][0]
        tbl = _call(D, op, _col(S, a, sa, va), _col(S, b, sb), so)
        assert tbl.getRowCount() == n
        _check(op, tbl, a, b, sa, sb, so, va)


def test_eight_byte_aligned_inputs_and_unaligned_flags():
    import ctypes as C
    import torch
    S, D = _s()
    from srj_b200 import _native as N
    rng = np.random.default_rng(3)
    n = 1001
    a, b = _values(rng, n), _values(rng, n)
    for op in sorted(OPS):
        sa, sb, so = GRID[op][0]
        for off_a, off_b in ((8, 0), (0, 8), (8, 8)):
            tbl = _call(D, op, _col(S, a, sa, offset=off_a), _col(S, b, sb, offset=off_b), so)
            _check(op, tbl, a, b, sa, sb, so)
        ca, cb = _col(S, a, sa), _col(S, b, sb)
        want = [O.row(op, x, y, sa, sb, so) for x, y in zip(a, b)]
        w = 8 if op == O.INTEGER_DIVIDE else 16
        for k in range(4):                     # the overflow output at byte offsets 0-3; the values 8-byte aligned
            ovf = torch.zeros(n + 8, dtype=torch.uint8, device="cuda")
            out = torch.zeros(n * w + 16, dtype=torch.uint8, device="cuda")
            nulls = C.c_int64(-1)
            N.check(N.lib().srj_decimal128_binary(op, C.byref(ca._c()), C.byref(cb._c()), so, 1, ovf.data_ptr() + k, out.data_ptr() + 8,
                                                  None, C.byref(nulls), int(torch.cuda.current_stream().cuda_stream)))
            g = ovf.cpu().numpy()
            assert nulls.value == 0 and not g[:k].any() and not g[k + n:].any()
            assert np.array_equal(g[k:k + n], np.array([r[0] for r in want], np.uint8))
            vals = out.cpu().numpy()[8:8 + n * w]
            assert np.array_equal(vals, O.from_ints([r[1] for r in want], w))


def test_one_million_rows_in_full():
    # every row of every op compared with the oracle, 10 % nulls on a
    S, D = _s()
    n = 1_000_000
    rng = np.random.default_rng(1_000_000)
    a, b = _values(rng, n), _values(rng, n)
    va = rng.random(n) > 0.1
    for op in sorted(OPS):
        sa, sb, so = GRID[op][0]
        tbl = _call(D, op, _col(S, a, sa, va), _col(S, b, sb), so)
        _check(op, tbl, a, b, sa, sb, so, va)


def test_ten_million_rows_sampled():
    import torch
    S, D = _s()
    n = 10_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    raw = torch.randint(-2**63, 2**63 - 1, (n, 2), dtype=torch.int64, device="cuda", generator=g)
    raw[:, 1] >>= 24                      # |v| < 2^103 < 10^38 - 1
    rb = torch.randint(-2**63, 2**63 - 1, (n, 2), dtype=torch.int64, device="cuda", generator=g)
    rb[:, 1] >>= 40
    ca = S.ColumnVector(S.DType(S.DType.DECIMAL128, -10), n, raw.view(torch.uint8).view(-1))
    cb = S.ColumnVector(S.DType(S.DType.DECIMAL128, -10), n, rb.view(torch.uint8).view(-1))
    rng = np.random.default_rng(11)
    idx = np.unique(np.concatenate([np.arange(2048), n - 1 - np.arange(2048), rng.integers(0, n, 8000)]))
    ha = O.to_ints(raw.cpu().numpy().view(np.uint8).reshape(-1)[np.repeat(idx * 16, 16) + np.tile(np.arange(16), len(idx))])
    hb = O.to_ints(rb.cpu().numpy().view(np.uint8).reshape(-1)[np.repeat(idx * 16, 16) + np.tile(np.arange(16), len(idx))])
    for op, so in ((O.MULTIPLY, -6), (O.DIVIDE, -6), (O.INTEGER_DIVIDE, 0), (O.REMAINDER, -10), (O.ADD, -10), (O.SUBTRACT, -10)):
        tbl = _call(D, op, ca, cb, so)
        ovf = tbl.getColumn(0).data.cpu().numpy()
        w = 8 if op == O.INTEGER_DIVIDE else 16
        vals = tbl.getColumn(1).data.cpu().numpy().reshape(-1, w)
        for j, i in enumerate(idx):
            f, v = O.row(op, ha[j], hb[j], -10, -10, so)
            assert bool(ovf[i]) == f and int.from_bytes(vals[i].tobytes(), "little", signed=True) == v, (op, int(i))
        # whole-output checksum against a second run on an 8-byte-aligned copy of the inputs (the non-vector path)
        a8 = torch.zeros(n * 16 + 8, dtype=torch.uint8, device="cuda")
        a8[8:] = ca.data
        tbl2 = _call(D, op, S.ColumnVector(ca.dtype, n, a8[8:]), cb, so)
        assert torch.equal(tbl2.getColumn(0).data, tbl.getColumn(0).data)
        assert torch.equal(tbl2.getColumn(1).data, tbl.getColumn(1).data)


def test_non_default_stream_and_threads():
    import torch
    S, D = _s()
    rng = np.random.default_rng(9)
    n = 3000
    a, b = _values(rng, n), _values(rng, n)
    va = rng.random(n) > 0.25
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        tbl = D.DecimalUtils.multiply128(_col(S, a, -10, va), _col(S, b, -10), -6)
    s.synchronize()
    _check(O.MULTIPLY, tbl, a, b, -10, -10, -6, va)

    errors = []

    def work(t):
        try:
            op = sorted(OPS)[t % len(OPS)]
            sa, sb, so = GRID[op][t % len(GRID[op])]
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(3):
                    tb = _call(D, op, _col(S, a, sa, va), _col(S, b, sb), so)
                st.synchronize()
            _check(op, tb, a, b, sa, sb, so, va)
        except Exception as e:   # noqa: BLE001
            errors.append(repr(e))

    ths = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errors, errors
