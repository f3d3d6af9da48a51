"""GPU checks of Histogram (srj_b200.histogram over libsrj_b200.so) against oracle/histogram.py, which
tests/test_oracle_histogram.py pins to the reference's tests, hand-derived answers and an independent model.  Results are
compared bit for bit (a NaN matches any NaN), masks bit for bit."""
import threading

import numpy as np
import pytest

from golden import histogram_golden as G
from oracle import histogram as H

pytestmark = pytest.mark.gpu

K = 8192                                      # SRJ_HISTOGRAM_CTA_ELEMENTS
NP = {1: np.int8, 2: np.int16, 3: np.int32, 4: np.int64, 5: np.uint8, 6: np.uint16, 7: np.uint32, 8: np.uint64, 9: np.float32,
      10: np.float64, 11: np.uint8}
BOOL8, INT32, INT64, FLOAT64, STRING = 11, 3, 4, 10, 23


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200.histogram import Histogram
    return S, Histogram


def _mask(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _bits(col, n):
    if col.mask is None:
        return np.ones(n, bool)
    return np.unpackbits(col.mask.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)


def _values(rng, t, n):
    dt = NP[t]
    if t == BOOL8:
        return rng.choice(np.array([0, 1, 2, 255], np.uint8), n)
    if np.dtype(dt).kind == "f":
        nan_payload = np.array([0x7ff0000000000123, 0xfff8000000000001], np.uint64).view(np.float64) if dt == np.float64 else \
            np.array([0x7f800123, 0xffc00001], np.uint32).view(np.float32)
        pool = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -1.5, 7.0], dt), nan_payload.astype(dt, copy=False)])
        return np.where(rng.random(n) < 0.6, rng.choice(pool, n), rng.normal(0, 50, n).astype(dt)).astype(dt)
    info = np.iinfo(dt)
    pool = np.array([info.min, info.max, info.min + 1, info.max - 1, 0, 1], dt)
    return np.where(rng.random(n) < 0.4, rng.choice(pool, n), rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)).astype(dt)


def _oracle_vals(t, vals):
    return vals != 0 if t == BOOL8 else vals


def _hist_view(S, t, offsets, vals, valid, counts, slice_from=0):
    """LIST<STRUCT<T, INT64>>; slice_from > 0 views the offsets from that row on (offsets[0] != 0)."""
    import torch
    vcol = S.ColumnView.from_numpy(t, np.ascontiguousarray(vals), _mask(valid) if valid is not None else None, size=len(vals))
    ccol = S.ColumnView.from_numpy(INT64, np.ascontiguousarray(counts, np.int64), size=len(counts))
    st = S.ColumnView.makeStructView(vcol, ccol)
    off = torch.from_numpy(np.asarray(offsets, np.int32).copy()).cuda()
    return S.ColumnView.makeListView(off[slice_from:], st)


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(nan | (a.view(np.uint64) == b.view(np.uint64))))


def _check(S, Hs, t, offsets, vals, valid, counts, pct, slice_from=0):
    view = _hist_view(S, t, offsets, vals, valid, counts, slice_from)
    offs = np.asarray(offsets, np.int64)[slice_from:]
    want, ok = H.percentile_from_histogram(offs, _oracle_vals(t, vals), valid, counts, pct)
    rows, P = len(offs) - 1, len(pct)
    flat = Hs.percentileFromHistogram(view, pct, False)
    got = flat.data.cpu().numpy().view(np.float64)
    early = P == 0 or offs[-1] == offs[0]
    if early:
        assert flat.size == rows and not _bits(flat, rows).any()
    else:
        assert flat.size == rows * P
        assert np.array_equal(_bits(flat, rows * P), np.repeat(ok, P))
        assert _same(got.reshape(rows, P)[ok], want[ok])
        assert np.all(got.reshape(rows, P)[~ok] == 0.0)
    lists = Hs.percentileFromHistogram(view, pct, True)
    lo = lists.offsets.cpu().numpy()
    assert np.array_equal(_bits(lists, rows), ok)
    assert np.array_equal(lo, np.concatenate([[0], np.cumsum(ok)]) * P)
    assert _same(lists.child.data.cpu().numpy().view(np.float64), want[ok].reshape(-1))


PCTS = {"p0": [0.0], "p25": [0.25], "p50": [0.5], "p100": [1.0], "four": [0.0, 0.25, 0.5, 1.0],
        "p101": [i / 100 for i in range(101)]}


@pytest.mark.parametrize("t", sorted(NP), ids=[str(t) for t in sorted(NP)])
@pytest.mark.parametrize("pname", sorted(PCTS))
def test_every_type_and_percentage_set(t, pname):
    S, Hs = _s()
    rng = np.random.default_rng(t * 31 + len(pname))
    lens = rng.integers(0, 40, 300)
    lens[:5] = [0, 1, 2, 3, 300]
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = _values(rng, t, n)
    valid = rng.random(n) > 0.2
    valid[offsets[3]:offsets[4]] = False                       # an all-null row
    counts = rng.integers(0, 5, n).astype(np.int64)
    counts[valid & (counts == 0) & (rng.random(n) < 0.5)] = 1
    _check(S, Hs, t, offsets, vals, valid, counts, PCTS[pname])


@pytest.mark.parametrize("t", [INT64, FLOAT64, 9, 8, BOOL8])
def test_lengths_at_every_tier_edge_in_one_column(t):
    S, Hs = _s()
    rng = np.random.default_rng(5 + t)
    lens = np.array([0, 1, 2, 31, 32, 33, 255, 256, 257, K - 1, K, K + 1, 5_000_000, 3, 2 * K + 7, 0], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = _values(rng, t, n)
    valid = rng.random(n) > 0.1
    counts = rng.integers(1, 4, n).astype(np.int64)
    _check(S, Hs, t, offsets, vals, valid, counts, [0.0, 0.25, 0.5, 1.0, 0.37, 0.999])
    _check(S, Hs, t, offsets, vals, None, counts, [i / 100 for i in range(101)])


@pytest.mark.parametrize("big", [False, True], ids=["ones", "above_2_53"])
def test_counts_of_one_and_totals_above_2_53(big):
    S, Hs = _s()
    rng = np.random.default_rng(11 + big)
    lens = np.array([1, 2, 5, 100, 1000, K, K + 1, 70000], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = rng.integers(-10**6, 10**6, n).astype(np.int64)
    # totals pass 2^53 from the 1,000-element row on and stay below 2^63 on the 70,000-element one
    counts = rng.integers(2**44, 2**46, n).astype(np.int64) if big else np.ones(n, np.int64)
    _check(S, Hs, INT64, offsets, vals, None, counts, [0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 1.0, 1 / 3])


def test_zero_counts_nulls_and_degenerate_rows():
    S, Hs = _s()
    vals = np.array([3, 1, 2, 9, 5, 5, 7, 4, 4, 8, 6], np.int32)
    valid = np.array([1, 0, 1, 1, 0, 0, 1, 1, 1, 0, 1], bool)
    counts = np.array([0, 3, 2, 0, 1, 1, 0, 0, 0, 2, 0], np.int64)
    offsets = [0, 4, 6, 9, 9, 11]                                # zero counts, several nulls, all-null, empty, all-zero counts
    _check(S, Hs, INT32, offsets, vals, valid, counts, [0.0, 0.5, 0.75, 1.0])


def test_p0_sliced_and_no_elements():
    S, Hs = _s()
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 600, 200)
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = _values(rng, FLOAT64, n)
    counts = rng.integers(1, 9, n).astype(np.int64)
    _check(S, Hs, FLOAT64, offsets, vals, None, counts, [])                      # P = 0: every row null
    _check(S, Hs, FLOAT64, offsets, vals, None, counts, [0.5, 0.9], slice_from=17)  # offsets[0] != 0
    _check(S, Hs, INT32, [0, 0, 0], np.zeros(0, np.int32), None, np.zeros(0, np.int64), [0.5, 0.2])   # no element at all
    view = _hist_view(S, INT32, [0], np.zeros(0, np.int32), None, np.zeros(0, np.int64))
    assert Hs.percentileFromHistogram(view, [0.5], False).size == 0                  # no rows
    assert Hs.percentileFromHistogram(view, [0.5], True).size == 0


def test_errors_raise_the_java_exceptions():
    S, Hs = _s()
    view = _hist_view(S, INT32, [0, 2], np.array([1, 2], np.int32), None, np.ones(2, np.int64))
    with pytest.raises(S.CudfException, match="LIST"):
        Hs.percentileFromHistogram(view.child.children[0], [0.5], False)
    bad = _hist_view(S, STRING, [0, 0], np.zeros(0, np.uint8), None, np.zeros(0, np.int64))
    with pytest.raises(S.CudfException, match="Unsupported type"):
        Hs.percentileFromHistogram(bad, [0.5], False)
    rows = 2**16
    big = _hist_view(S, INT32, np.zeros(rows + 1, np.int32), np.zeros(0, np.int32), None, np.zeros(0, np.int64))
    with pytest.raises(S.CudfColumnSizeOverflowException):
        Hs.percentileFromHistogram(big, np.full(2**15, 0.5), False)


@pytest.mark.parametrize("lists", [False, True], ids=["struct", "lists"])
@pytest.mark.parametrize("t", [INT32, FLOAT64, 27, BOOL8, 1])
def test_create_histogram_if_valid(lists, t):
    S, Hs = _s()
    rng = np.random.default_rng(t + 100 * lists)
    n = 5000
    width = 16 if t == 27 else np.dtype(NP[t]).itemsize
    raw = rng.integers(0, 256, n * width, dtype=np.uint8)
    for valid, freqs in ((rng.random(n) > 0.3, rng.integers(0, 4, n)), (None, rng.integers(1, 4, n)), (rng.random(n) > 0.3, rng.integers(1, 4, n)),
                         (None, np.where(rng.random(n) < 0.01, 0, rng.integers(1, 1 << 40, n)))):
        v = S.ColumnView.from_numpy(t, raw, _mask(valid) if valid is not None else None, size=n)
        f = S.ColumnView.from_numpy(INT64, freqs.astype(np.int64), size=n)
        out = Hs.createHistogramIfValid(v, f, lists)
        rowsv = raw.reshape(n, width)
        want = H.create_histogram_if_valid(np.arange(n), valid, freqs, lists)
        st = out.child if lists else out
        if lists:
            assert np.array_equal(out.offsets.cpu().numpy(), want[0])
            want = want[1:]
        idx, wvalid, wfreq = want
        m = len(idx)
        assert st.size == m
        vcol, fcol = st.children
        assert np.array_equal(vcol.data.cpu().numpy().reshape(m, width), rowsv[idx])
        assert np.array_equal(_bits(vcol, m), wvalid) and vcol.getNullCount() == int((~wvalid).sum())
        assert np.array_equal(fcol.data.cpu().numpy().view(np.int64), wfreq)
    neg = S.ColumnView.from_numpy(INT64, np.array([1, -1, 2] + [1] * (n - 3), np.int64), size=n)
    with pytest.raises(S.CudfException, match="negative"):
        Hs.createHistogramIfValid(S.ColumnView.from_numpy(t, raw, size=n), neg, lists)
    empty = Hs.createHistogramIfValid(S.ColumnView.from_numpy(t, raw[:0], size=0), S.ColumnView.from_numpy(INT64, np.zeros(0, np.int64), size=0),
                                      lists)
    assert empty.size == 0 and (not lists or empty.offsets.cpu().tolist() == [0])


@pytest.mark.parametrize("case", G.ROUND_TRIPS, ids=[c[0] for c in G.ROUND_TRIPS])
def test_reference_round_trips_through_the_mirror(case):
    S, Hs = _s()
    _, values, freqs, pct, want = case
    valid = np.array([v is not None for v in values])
    vals = np.array([0 if v is None else v for v in values], np.int32)
    v = S.ColumnView.from_numpy(INT32, vals, None if valid.all() else _mask(valid), size=len(vals))
    f = S.ColumnView.from_numpy(INT64, np.array(freqs, np.int64), size=len(freqs))
    hist = Hs.createHistogramIfValid(v, f, True)
    out = Hs.percentileFromHistogram(hist, pct, False)
    got = out.data.cpu().numpy().view(np.float64)
    ok = _bits(out, len(values))
    assert [float(got[i]) if ok[i] else None for i in range(len(values))] == want


def test_goldens_on_the_device():
    S, Hs = _s()
    for _, pairs, pct, want in G.PERCENTILES:
        view = _hist_view(S, INT32, [0, len(pairs)], np.array([p[0] for p in pairs], np.int32), None, np.array([p[1] for p in pairs], np.int64))
        got = Hs.percentileFromHistogram(view, pct, True).child.data.cpu().numpy().view(np.float64)
        assert got.tolist() == want


def test_four_threads_on_their_own_streams():
    import torch
    S, Hs = _s()
    rng = np.random.default_rng(42)
    cases = []
    for i in range(4):
        lens = rng.integers(0, 3000, 400)
        lens[0] = 20000 + i
        offsets = np.concatenate([[0], np.cumsum(lens)])
        n = int(offsets[-1])
        vals = _values(rng, FLOAT64, n)
        counts = rng.integers(1, 5, n).astype(np.int64)
        want, ok = H.percentile_from_histogram(offsets, vals, None, counts, [0.1, 0.5, 0.9])
        cases.append((offsets, vals, counts, want, ok))
    errors = []

    def run(i):
        try:
            offsets, vals, counts, want, ok = cases[i]
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(3):
                    view = _hist_view(S, FLOAT64, offsets, vals, None, counts)
                    out = Hs.percentileFromHistogram(view, [0.1, 0.5, 0.9], False)
                    got = out.data.cpu().numpy().view(np.float64).reshape(-1, 3)
                    torch.cuda.current_stream().synchronize()
                    assert _same(got[ok], want[ok])
        except Exception as e:   # noqa: BLE001
            errors.append(e)
    ts = [threading.Thread(target=run, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


GUARD = 64                                    # sentinel words right after each output buffer
SENTINEL = 0x5A5A5A5A


def _guarded(torch, words):
    return torch.full((words + GUARD,), SENTINEL, dtype=torch.int32, device="cuda")


def _guard_intact(t, words):
    return bool((t[words:].cpu().numpy().view(np.uint32) == SENTINEL).all())


@pytest.mark.parametrize("zeros", [0.0, 0.01, 0.4, 1.0])
def test_create_lists_writes_only_the_kept_rows_mask(zeros):
    """The list child's mask is ceil(kept / 32) words: the call writes no word past it."""
    import ctypes as C
    import torch
    S, _ = _s()
    from srj_b200 import _native as N
    rng = np.random.default_rng(int(zeros * 100))
    n = 100_003
    vals = rng.integers(-1000, 1000, n).astype(np.int32)
    valid = rng.random(n) > 0.3
    freqs = np.where(rng.random(n) < zeros, 0, rng.integers(1, 9, n)).astype(np.int64)
    v = S.ColumnView.from_numpy(INT32, vals, _mask(valid), size=n)
    f = S.ColumnView.from_numpy(INT64, freqs, size=n)
    cv, cf = v._c(), f._c()
    lib = N.lib()
    stream = torch.cuda.current_stream().cuda_stream
    ws = torch.empty(lib.srj_histogram_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    kept, nulls = C.c_int64(0), C.c_int64(0)
    N.check(lib.srj_histogram_create_size(C.byref(cv), C.byref(cf), 1, C.byref(kept), C.byref(nulls), ws.data_ptr(), stream))
    k = kept.value
    words = (k + 31) // 32
    mask = _guarded(torch, words)
    out_v = torch.empty(max(k, 1), dtype=torch.int32, device="cuda")
    out_f = torch.empty(max(k, 1), dtype=torch.int64, device="cuda")
    offs = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    N.check(lib.srj_histogram_create(C.byref(cv), C.byref(cf), 1, out_v.data_ptr(), mask.data_ptr(), out_f.data_ptr(), offs.data_ptr(),
                                     ws.data_ptr(), stream))
    torch.cuda.synchronize()
    _, wv, wvalid, wf = H.create_histogram_if_valid(vals, valid, freqs, True)
    assert k == len(wv) and _guard_intact(mask, words)
    got = np.unpackbits(mask[:words].cpu().numpy().view(np.uint8), bitorder="little")[:k].astype(bool)
    assert np.array_equal(got, wvalid) and nulls.value == int((~wvalid).sum())
    assert np.array_equal(out_v[:k].cpu().numpy(), wv) and np.array_equal(out_f[:k].cpu().numpy(), wf)


@pytest.mark.parametrize("lists", [False, True], ids=["flat", "lists"])
def test_percentile_writes_only_its_outputs(lists):
    """Flat output: a mask bit per double (ceil(rows * P / 32) words); lists: a bit per row.  Nothing past either."""
    import ctypes as C
    import torch
    S, _ = _s()
    from srj_b200 import _native as N
    rng = np.random.default_rng(9 + lists)
    lens = rng.integers(0, 30, 1001)
    lens[7] = K + 5                                             # one row on the select path
    offsets = np.concatenate([[0], np.cumsum(lens)])
    n = int(offsets[-1])
    vals = rng.normal(0, 9, n)
    valid = rng.random(n) > 0.3
    counts = rng.integers(1, 5, n).astype(np.int64)
    pct = np.array([0.1, 0.5, 0.9])
    view = _hist_view(S, FLOAT64, offsets, vals, valid, counts)
    cin = view._c()
    rows, P = len(lens), len(pct)
    lib = N.lib()
    stream = torch.cuda.current_stream().cuda_stream
    ws = torch.empty(lib.srj_percentile_workspace_bytes(rows, n, P), dtype=torch.uint8, device="cuda")
    nv, nvals = C.c_int64(0), C.c_int64(0)
    N.check(lib.srj_percentile_from_histogram_size(C.byref(cin), P, int(lists), C.byref(nv), C.byref(nvals), ws.data_ptr(), stream))
    m = nvals.value
    mwords = ((rows if lists else m) + 31) // 32
    out = torch.full((m + GUARD,), np.nan, dtype=torch.float64, device="cuda")
    mask = _guarded(torch, mwords)
    offs = _guarded(torch, rows + 1)
    N.check(lib.srj_percentile_from_histogram(C.byref(cin), pct.ctypes.data_as(C.c_void_p), P, int(lists), out.data_ptr(), mask.data_ptr(),
                                              offs.data_ptr() if lists else None, ws.data_ptr(), stream))
    torch.cuda.synchronize()
    want, ok = H.percentile_from_histogram(offsets, vals, valid, counts, list(pct))
    assert _guard_intact(mask, mwords) and np.isnan(out[m:].cpu().numpy()).all()
    bits = np.unpackbits(mask[:mwords].cpu().numpy().view(np.uint8), bitorder="little")
    if lists:
        assert _guard_intact(offs, rows + 1) and m == ok.sum() * P
        assert np.array_equal(bits[:rows].astype(bool), ok) and _same(out[:m].cpu().numpy(), want[ok].reshape(-1))
    else:
        assert m == rows * P and np.array_equal(bits[:m].astype(bool), np.repeat(ok, P))
        assert _same(out[:m].cpu().numpy().reshape(rows, P)[ok], want[ok])
