"""GPU checks of ZOrder (srj_b200.zorder over libsrj_b200.so) against oracle/zorder.py, which tests/test_oracle_zorder.py pins
to the reference's test inputs, hand-derived answers, the curve's properties and an independent model.  interleaveBits is
compared byte for byte (offsets and bytes); hilbertIndex value for value."""
import ctypes as C
import threading

import numpy as np
import pytest

from golden import zorder_golden as G
from oracle import zorder as Z

pytestmark = pytest.mark.gpu

SIZES = {1: (1, 5, 11), 2: (2, 6), 4: (3, 7, 9, 12, 17, 25), 8: (4, 8, 10, 13, 14, 15, 16, 18, 19, 20, 21, 26), 16: (27,)}
WIDTH = {t: w for w, ts in SIZES.items() for t in ts}
INT32 = 3


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200.zorder import ZOrder
    return S, ZOrder


def _mask(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _host_col(rng, width, rows, nulls, special=False):
    """(raw bytes uint8[rows * W], mask or None); nulls: None (no mask), a fraction, or 1.0 (all null)"""
    raw = rng.integers(0, 256, rows * width, dtype=np.uint8)
    if special and rows:
        words = raw.reshape(rows, width)
        words[: rows // 4] = 0xFF                                   # -1 / NaN bit patterns (all ones)
        words[rows // 4: rows // 2, -1] |= 0x80                     # negative
        if width in (4, 8):                                         # quiet / signalling NaNs and -0.0
            nan = {4: [0x7FC00001, 0x7F800001, 0x80000000], 8: [0x7FF8000000000001, 0x7FF0000000000001, 1 << 63]}[width]
            dt = np.uint32 if width == 4 else np.uint64
            words.reshape(-1).view(dt)[: len(nan)] = np.array(nan, dtype=dt)
    mask = None
    if nulls is not None:
        mask = _mask(rng.random(rows) >= nulls)
    return raw, mask


def _dev(S, type_id, raw, mask, rows):
    return S.ColumnVector.from_numpy(type_id, raw, mask, size=rows)


def _check_interleave(S, ZOrder, type_id, hosts, rows):
    width = WIDTH[type_id]
    out = ZOrder.interleaveBits(rows, *[_dev(S, type_id, r, m, rows) for r, m in hosts])
    want_offs, want = Z.interleave_bits(hosts, width, rows)
    assert out.dtype.type_id == S.DType.LIST and out.mask is None and out.getNullCount() == 0 and out.size == rows
    assert np.array_equal(out.offsets.cpu().numpy(), want_offs)
    assert np.array_equal(out.child.data.cpu().numpy(), want)


@pytest.mark.parametrize("type_id", sorted(WIDTH))
def test_interleave_every_fixed_width_type(type_id):
    S, ZOrder = _s()
    rng = np.random.default_rng(type_id)
    rows = 1000
    for n in (1, 3, 4):
        _check_interleave(S, ZOrder, type_id, [_host_col(rng, WIDTH[type_id], rows, 0.1 if c % 2 else None, special=True)
                                               for c in range(n)], rows)


@pytest.mark.parametrize("ncols", [1, 2, 3, 4, 5, 7, 8, 9, 16, 17, 33, 64, 224, 225, 300])
@pytest.mark.parametrize("type_id", [1, 2, 3, 4, 27])
def test_interleave_column_counts(ncols, type_id):
    S, ZOrder = _s()
    width = WIDTH[type_id]
    rows = 1037 if ncols * width <= 1024 else 261
    rng = np.random.default_rng(ncols * 31 + type_id)
    hosts = [_host_col(rng, width, rows, [None, 0.3, 1.0][c % 3], special=c % 5 == 0) for c in range(ncols)]
    _check_interleave(S, ZOrder, type_id, hosts, rows)


@pytest.mark.parametrize("type_id,ncols", [(3, 32), (3, 33), (4, 16), (4, 17), (1, 128), (1, 129), (27, 8), (27, 9),
                                           (2, 63), (2, 65)])
def test_interleave_both_sides_of_the_staging_threshold(type_id, ncols):
    """rows of up to 128 bytes are staged per warp in shared memory, wider ones are written directly"""
    S, ZOrder = _s()
    rng = np.random.default_rng(ncols)
    rows = 3 * 256 + 17
    _check_interleave(S, ZOrder, type_id, [_host_col(rng, WIDTH[type_id], rows, 0.5 if c == 1 else None) for c in range(ncols)], rows)


@pytest.mark.parametrize("rows", [0, 1, 31, 32, 33, 63, 255, 256, 257, 8 * 256 + 1, 100_003])
@pytest.mark.parametrize("type_id,ncols", [(3, 4), (1, 3), (2, 5), (4, 16), (27, 2), (1, 200)])
def test_interleave_row_counts(rows, type_id, ncols):
    S, ZOrder = _s()
    rng = np.random.default_rng(rows + ncols)
    _check_interleave(S, ZOrder, type_id, [_host_col(rng, WIDTH[type_id], rows, 0.1 if c == 0 else None) for c in range(ncols)], rows)


def test_interleave_10m_rows_delta_shape():
    S, ZOrder = _s()
    rng = np.random.default_rng(10)
    rows = 10_000_000
    _check_interleave(S, ZOrder, INT32, [_host_col(rng, 4, rows, 0.1) for _ in range(4)], rows)


@pytest.mark.parametrize("case", G.INTERLEAVE, ids=[c[0] for c in G.INTERLEAVE])
def test_interleave_reference_cases(case):
    S, ZOrder = _s()
    _, width, rows, columns = case
    tid = {1: 1, 2: 2, 4: 3}[width]
    if not columns:
        out = ZOrder.interleaveBits(rows)
        assert out.size == rows and out.offsets.cpu().numpy().tolist() == [0] * (rows + 1) and out.child.size == 0
        return
    hosts = []
    for c in columns:
        raw = b"".join(((v or 0) & ((1 << (8 * width)) - 1)).to_bytes(width, "little") for v in c)
        hosts.append((np.frombuffer(raw, np.uint8).copy(), _mask([v is not None for v in c]) if None in c else None))
    _check_interleave(S, ZOrder, tid, hosts, rows)


def test_interleave_known_answers():
    S, ZOrder = _s()
    for width, values, want in G.INTERLEAVE_KNOWN:
        tid = {1: 1, 2: 2, 4: 3}[width]
        cols = [_dev(S, tid, np.frombuffer((v & ((1 << 8 * width) - 1)).to_bytes(width, "little"), np.uint8).copy(), None, 1)
                for v in values]
        assert ZOrder.interleaveBits(1, *cols).child.data.cpu().numpy().tobytes() == want
    dec = _dev(S, 27, np.frombuffer(G.DECIMAL128_BYTES, np.uint8).copy(), None, 1)
    assert ZOrder.interleaveBits(1, dec).child.data.cpu().numpy().tobytes() == G.DECIMAL128_BYTES[::-1]


def test_interleave_errors_raise_cudf_exception():
    S, ZOrder = _s()
    from srj_b200 import _native as N
    a = _dev(S, INT32, np.zeros(16, np.uint8), None, 4)
    b = _dev(S, 4, np.zeros(32, np.uint8), None, 4)
    with pytest.raises(N.CudfException):
        ZOrder.interleaveBits(4, a, b)
    s = S.ColumnVector.from_numpy(S.DType.STRING, np.zeros(4, np.uint8), offsets=np.array([0, 1, 2, 3, 4], np.int32))
    with pytest.raises(N.CudfException):
        ZOrder.interleaveBits(4, s)


def _c_abi_interleave(S, cols, rows, width, shift_in, shift_out, stream):
    """srj_interleave_bits with inputs `shift_in` bytes into their tensors and outputs `shift_out` bytes off alignment"""
    import torch
    from srj_b200 import _native as N
    n = len(cols)
    views = []
    for raw, mask in cols:
        t = torch.from_numpy(np.concatenate([np.zeros(shift_in, np.uint8), raw])).cuda()
        views.append(S.ColumnVector(S.DType(WIDTH_TYPE[width]), rows, t[shift_in:],
                                    torch.from_numpy(mask.view(np.int32)).cuda() if mask is not None else None))
    offs = torch.zeros(4 * (rows + 1) + shift_out, dtype=torch.uint8, device="cuda")
    data = torch.zeros(rows * n * width + shift_out, dtype=torch.uint8, device="cuda")
    arr = S._carray(views)
    N.check(N.lib().srj_interleave_bits(arr, n, rows, offs.data_ptr() + shift_out, data.data_ptr() + shift_out, stream))
    return offs, data, views


WIDTH_TYPE = {1: 1, 2: 2, 4: 3, 8: 4, 16: 27}


@pytest.mark.parametrize("width,ncols,shift_in", [(1, 3, 1), (2, 4, 2), (4, 4, 4), (8, 16, 8), (16, 3, 16), (4, 40, 4),
                                                  (16, 3, 8), (16, 9, 8)])
def test_interleave_element_aligned_inputs_and_unaligned_outputs(width, ncols, shift_in):
    """inputs one element into their tensors (DECIMAL128 also 8 bytes in: it needs 8-byte alignment only), outputs at
    every byte offset"""
    import torch
    S, _ = _s()
    rng = np.random.default_rng(width)
    rows = 1000
    hosts = [_host_col(rng, width, rows, 0.2 if c == 0 else None) for c in range(ncols)]
    want_offs, want = Z.interleave_bits(hosts, width, rows)
    for shift_out in (1, 2, 3, 5):
        offs, data, _ = _c_abi_interleave(S, hosts, rows, width, shift_in, shift_out, int(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert np.array_equal(offs.cpu().numpy()[shift_out:].view(np.int32), want_offs)
        assert np.array_equal(data.cpu().numpy()[shift_out:], want)


def test_interleave_at_exactly_int32_max_output_bytes():
    """one INT8 column of INT32_MAX rows: the output is the input (nulls as 0) and the offsets are 0 .. INT32_MAX"""
    import torch
    S, ZOrder = _s()
    rows = 2**31 - 1
    g = torch.Generator(device="cuda").manual_seed(3)
    raw = torch.randint(0, 256, (rows,), dtype=torch.uint8, device="cuda", generator=g)
    mask = torch.randint(-2**31, 2**31 - 1, ((rows + 31) // 32,), dtype=torch.int32, device="cuda", generator=g)
    out = ZOrder.interleaveBits(rows, S.ColumnVector(S.DType(1), rows, raw, mask))
    assert out.child.size == rows
    step = 1 << 28
    for s in range(0, rows + 1, step):
        e = min(rows + 1, s + step)
        assert torch.equal(out.offsets[s:e].to(torch.int64), torch.arange(s, e, dtype=torch.int64, device="cuda"))
    bits = mask.view(torch.uint8)
    for s in range(0, rows, step):
        e = min(rows, s + step)
        r = torch.arange(s, e, device="cuda")
        valid = (bits[r >> 3] >> (r & 7).to(torch.uint8)) & 1
        assert torch.equal(out.child.data[s:e], raw[s:e] * valid)
        del r, valid
    rng = np.random.default_rng(1)
    idx = np.concatenate([rng.integers(0, rows, 4096), [0, 31, 32, rows - 33, rows - 32, rows - 1]])
    hv = raw[torch.from_numpy(idx).cuda()].cpu().numpy()
    hm = np.unpackbits(bits.cpu().numpy(), bitorder="little")[idx]
    assert np.array_equal(out.child.data[torch.from_numpy(idx).cuda()].cpu().numpy(), hv * hm)


def test_interleave_non_default_stream_and_threads():
    import torch
    S, ZOrder = _s()
    rng = np.random.default_rng(5)
    rows = 50_000
    hosts = [_host_col(rng, 8, rows, 0.1) for _ in range(6)]
    want_offs, want = Z.interleave_bits(hosts, 8, rows)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = ZOrder.interleaveBits(rows, *[_dev(S, 4, r, m, rows) for r, m in hosts])
    s.synchronize()
    assert np.array_equal(out.child.data.cpu().numpy(), want)

    errors = []

    def work(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                cols = [_dev(S, 4, r, m, rows) for r, m in hosts[i % 3:]]
                o = ZOrder.interleaveBits(rows, *cols)
                h = ZOrder.hilbertIndex(16, rows, *[_dev(S, 3, r[: 4 * rows], m, rows) for r, m in hosts[:3]])
            st.synchronize()
            sub = hosts[i % 3:]
            assert np.array_equal(o.child.data.cpu().numpy(), Z.interleave_bits(sub, 8, rows)[1])
            assert np.array_equal(h.data.cpu().numpy().view(np.int64),
                                  Z.hilbert_index(16, [(r[: 4 * rows], m) for r, m in hosts[:3]], rows))
        except Exception as e:  # noqa: BLE001
            errors.append(e)
    ts = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


# ---- hilbertIndex
def _check_hilbert(S, ZOrder, bits, hosts, rows):
    out = ZOrder.hilbertIndex(bits, rows, *[_dev(S, INT32, r, m, rows) for r, m in hosts])
    assert out.dtype.type_id == S.DType.INT64 and out.mask is None and out.size == rows
    assert np.array_equal(out.data.cpu().numpy().view(np.int64), Z.hilbert_index(bits, hosts, rows))


def _int32_col(rng, rows, nulls):
    v = rng.integers(-2**31, 2**31, rows, dtype=np.int64).astype(np.int32)
    v[: rows // 8] = rng.integers(0, 64, rows // 8)                         # small values, inside every num_bits range
    return v.view(np.uint8), (_mask(rng.random(rows) >= nulls) if nulls else None)


@pytest.mark.parametrize("ncols", [1, 2, 3, 4])
def test_hilbert_every_num_bits(ncols):
    S, ZOrder = _s()
    rng = np.random.default_rng(ncols)
    rows = 2000
    for bits in range(1, 33):
        if bits * ncols > 64:
            continue
        _check_hilbert(S, ZOrder, bits, [_int32_col(rng, rows, 0.2 if c == 0 else None) for c in range(ncols)], rows)


@pytest.mark.parametrize("ncols", [2, 4, 8, 16, 32, 64])
def test_hilbert_64_bit_shapes(ncols):
    S, ZOrder = _s()
    rng = np.random.default_rng(ncols + 100)
    rows = 3000
    _check_hilbert(S, ZOrder, 64 // ncols, [_int32_col(rng, rows, 0.1 if c % 3 == 0 else None) for c in range(ncols)], rows)


def test_hilbert_reference_and_known_cases():
    S, ZOrder = _s()
    for _, bits, rows, columns in G.HILBERT:
        if not columns:
            out = ZOrder.hilbertIndex(bits, rows)
            assert out.size == rows and not out.data.cpu().numpy().any()
            continue
        hosts = [(np.array([v or 0 for v in c], np.int32).view(np.uint8), _mask([v is not None for v in c]) if None in c else None)
                 for c in columns]
        _check_hilbert(S, ZOrder, bits, hosts, rows)
    for bits, values, want in G.HILBERT_KNOWN:
        cols = [_dev(S, INT32, np.array([v or 0], np.int32).view(np.uint8), _mask([v is not None]) if v is None else None, 1)
                for v in values]
        assert ZOrder.hilbertIndex(bits, 1, *cols).data.cpu().numpy().view(np.int64).tolist() == [want]


def test_hilbert_10m_rows_and_unaligned_output():
    import torch
    S, ZOrder = _s()
    from srj_b200 import _native as N
    rng = np.random.default_rng(11)
    rows = 10_000_000
    hosts = [_int32_col(rng, rows, 0.1) for _ in range(3)]
    _check_hilbert(S, ZOrder, 21, hosts, rows)
    small = [(r[: 4 * 999], m) for r, m in hosts]
    views = [_dev(S, INT32, r, m, 999) for r, m in small]
    out = torch.zeros(8 * 999 + 3, dtype=torch.uint8, device="cuda")
    N.check(N.lib().srj_hilbert_index(21, S._carray(views), 3, 999, out.data_ptr() + 3, int(torch.cuda.current_stream().cuda_stream)))
    assert np.array_equal(out.cpu().numpy()[3:].view(np.int64), Z.hilbert_index(21, small, 999))


def test_hilbert_errors_raise_cudf_exception():
    S, ZOrder = _s()
    from srj_b200 import _native as N
    a = _dev(S, INT32, np.zeros(16, np.uint8), None, 4)
    for bits, cols in [(0, [a]), (33, [a]), (22, [a, a, a])]:
        with pytest.raises(N.CudfException):
            ZOrder.hilbertIndex(bits, 4, *cols)
    with pytest.raises(N.CudfException):
        ZOrder.hilbertIndex(4, 4, _dev(S, 4, np.zeros(32, np.uint8), None, 4))
