"""GPU parity tests of the wide variable-width from_rows path (from_rows_wide.cu + strings_wide_kernel) against
the CPU oracle: slab planning over different schemas, partial tiles, 32-row group boundaries of the offsets
protocol, unaligned row buffers (SAFE tiles), buffer-edge hand copies, non-canonical rows, sliced outputs."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from util import cols_equal, random_table

pytestmark = pytest.mark.gpu

WIDE_SCHEMAS = {
    # config C3 (3096-byte fixed section, 64 STRING columns, one slab)
    "c3": [O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 64,
    # odd alignments: 1/2-byte fields between strings, validity offset not a multiple of 4
    "odd": [O.INT8, O.STRING, O.INT16, O.DECIMAL128, O.STRING, O.INT64, O.BOOL8, O.INT32, O.STRING, O.FLOAT64, O.INT8] * 20,
    # more STRING columns than the fast gather takes (generic gather finishing the offsets)
    "many_strings": [O.STRING] * 70 + [O.INT64] * 40,
    "strings_first": [O.STRING] * 12 + [O.INT64] * 100,
    "strings_last": [O.INT64] * 100 + [O.STRING] * 12,
    "one_slab": [O.STRING, O.INT32] * 50,
    # 512 columns, 128 STRING columns: more than kWMaxCols, so the whole-row kernel serves it
    "c3x2": [O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 128,
    # 9 STRING columns spread over 2 KB: exercises the "previous pair too far" planning fallback
    "sparse_strings": ([O.STRING] + [O.INT64] * 30) * 9,
}


def _gpu():
    import gpu_util
    gpu_util.require_cuda()
    return gpu_util


def _check_table(G, tbl, data, offs, nrows, types, cols=None):
    ocols, onulls = O.convert_from_rows(data, offs, nrows, types)
    for i, (g, o) in enumerate(zip(tbl.columns, ocols)):
        h = G.to_host(g)
        assert np.array_equal(h.mask, o.mask), f"mask, column {i}"
        if types[i] == O.STRING:
            assert np.array_equal(h.offsets, o.offsets), f"offsets, column {i}: first diff {np.flatnonzero(h.offsets != o.offsets)[:4]}"
            assert np.array_equal(h.data, o.data), f"chars, column {i}: first diff {np.flatnonzero(h.data != o.data)[:4]}"
        else:
            assert cols_equal(h, o, check_null_payload=True), f"column {i}"
        assert g.getNullCount() == int(onulls[i]), f"null count, column {i}"
        if cols is not None:
            assert cols_equal(h, cols[i])


@pytest.mark.parametrize("nrows", [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1000, 4099])
@pytest.mark.parametrize("name", sorted(WIDE_SCHEMAS))
def test_wide_from_rows(name, nrows):
    G = _gpu()
    import srj_b200 as S
    types = WIDE_SCHEMAS[name]
    cols = random_table(types, nrows, seed=nrows * 3 + len(types))
    (offs, data), = O.convert_to_rows(cols)
    tbl = S.RowConversion.convertFromRows(G.rows_to_device(offs, data), [S.DType(t) for t in types])
    _check_table(G, tbl, data, offs, nrows, types, cols)


@pytest.mark.parametrize("shift", [1, 4, 8, 24])
@pytest.mark.parametrize("name", ["c3", "odd", "many_strings"])
def test_wide_unaligned_row_buffer(name, shift):
    """The rows child sliced at +1/+4 (rows not 8-byte aligned: SAFE tiles read global memory byte-wise) and at
    +8/+24 (aligned rows, but the first row's 16-byte TMA window would start before the buffer and the last
    one's would end past it: hand copies at both ends)."""
    G = _gpu()
    import srj_b200 as S
    types = WIDE_SCHEMAS[name]
    nrows = 1500
    cols = random_table(types, nrows, seed=77 + shift)
    (offs, data), = O.convert_to_rows(cols)
    big = torch.zeros(len(data) + 64, dtype=torch.uint8, device="cuda")
    big[shift:shift + len(data)] = torch.from_numpy(data).cuda()
    child = S.ColumnVector(S.DType.INT8, len(data), big[shift:shift + len(data)])
    assert child.data.data_ptr() % 16 == shift % 16
    vec = S.ColumnVector(S.DType.LIST, nrows, None, None, torch.from_numpy(offs).cuda(), child)
    tbl = S.RowConversion.convertFromRows(vec, [S.DType(t) for t in types])
    _check_table(G, tbl, data, offs, nrows, types, cols)


def test_wide_exact_size_buffer_edges():
    """rows buffer whose end is not 16-byte aligned inside an exact-size allocation (tail hand copy)."""
    G = _gpu()
    import srj_b200 as S
    types = WIDE_SCHEMAS["c3"]
    for nrows in (5, 70):
        cols = random_table(types, nrows, seed=5 + nrows)
        (offs, data), = O.convert_to_rows(cols)
        tbl = S.RowConversion.convertFromRows(G.rows_to_device(offs, data), [S.DType(t) for t in types])
        _check_table(G, tbl, data, offs, nrows, types, cols)


@pytest.mark.parametrize("name", ["c3", "many_strings"])
def test_wide_non_canonical_rows(name):
    """Rows whose chars are stored in a different order (pairs updated): phase 1 must flag them and phase 2 must
    follow the stored pair offsets (RC:1143) -- also while it finishes the group-local offsets."""
    G = _gpu()
    import srj_b200 as S
    types = WIDE_SCHEMAS[name]
    n = 700
    cols = random_table(types, n, seed=21)
    (offs, data), = O.convert_to_rows(cols)
    st, sz, voff, spr = O.compute_layout(types)
    sidx = [i for i, t in enumerate(types) if t == O.STRING]
    a_col, b_col = sidx[3], sidx[4]                      # swap the chars of two neighbouring STRING columns
    data = data.copy()
    for r in range(0, n, 7):                             # every 7th row only: canonical and permuted rows mixed
        row = data[offs[r]:offs[r + 1]]
        (oa, la), (ob, lb) = row[st[a_col]:st[a_col] + 8].view(np.uint32), row[st[b_col]:st[b_col] + 8].view(np.uint32)
        A, B = row[oa:oa + la].copy(), row[ob:ob + lb].copy()
        row[oa:oa + lb] = B
        row[oa + lb:oa + lb + la] = A
        row[st[b_col]:st[b_col] + 8].view(np.uint32)[:] = (oa, lb)
        row[st[a_col]:st[a_col] + 8].view(np.uint32)[:] = (oa + lb, la)
    tbl = S.RowConversion.convertFromRows(G.rows_to_device(offs, data), [S.DType(t) for t in types])
    _check_table(G, tbl, data, offs, n, types, cols)


def test_wide_sliced_output_buffers():
    """Output columns that are element-offset slices of larger allocations (odd INT8 pointers, INT32 data at
    4 mod 16, chars at odd addresses) through the C ABI directly."""
    G = _gpu()
    import ctypes as C
    import srj_b200 as S
    from srj_b200 import _native as N
    types = WIDE_SCHEMAS["odd"]
    nrows = 2050
    cols = random_table(types, nrows, seed=99)
    (offs, data), = O.convert_to_rows(cols)
    ocols, onulls = O.convert_from_rows(data, offs, nrows, types)
    dts = [S.DType(t) for t in types]
    plan = S.Plan.get(dts)
    d_rows = torch.from_numpy(data).cuda()
    d_offs = torch.from_numpy(offs).cuda()
    words = (nrows + 31) // 32
    outs = []
    for d, o in zip(dts, ocols):
        mask = torch.empty(words + 1, dtype=torch.int32, device="cuda")[1:]
        if d.type_id == S.DType.STRING:
            outs.append(S.ColumnVector(d, nrows, None, mask, torch.empty(nrows + 2, dtype=torch.int32, device="cuda")[1:]))
        else:
            sz = d.size_in_bytes()
            outs.append(S.ColumnVector(d, nrows, torch.empty((nrows + 1) * sz, dtype=torch.uint8, device="cuda")[sz:], mask))
    nulls = torch.zeros(len(dts), dtype=torch.int64, device="cuda")
    totals = torch.zeros(len(dts) + 1, dtype=torch.int64, device="cuda")
    lib = N.lib()
    st = int(torch.cuda.current_stream().cuda_stream)
    carr = (N.SrjColumn * len(outs))()
    for i, c in enumerate(outs):
        carr[i] = c._c()
    ws = torch.empty(max(8, lib.srj_from_rows_workspace_bytes(plan.handle, nrows)), dtype=torch.uint8, device="cuda")
    N.check(lib.srj_convert_from_rows_fixed(plan.handle, d_rows.data_ptr(), d_offs.data_ptr(), d_rows.numel(), nrows, carr,
                                            nulls.data_ptr(), totals.data_ptr(), None, ws.data_ptr(), st))
    h_tot = totals.cpu().numpy()
    assert h_tot[len(dts)] == 0                                   # canonical rows, no overflow
    for i, d in enumerate(dts):
        if d.type_id == S.DType.STRING:
            assert h_tot[i] == len(ocols[i].data)
            outs[i].data = torch.empty(int(h_tot[i]) + 3, dtype=torch.uint8, device="cuda")[3:]     # odd chars pointer
            carr[i] = outs[i]._c()
    N.check(lib.srj_convert_from_rows_strings(plan.handle, d_rows.data_ptr(), d_offs.data_ptr(), d_rows.numel(), nrows, carr,
                                              totals.data_ptr(), ws.data_ptr(), st))
    torch.cuda.synchronize()
    assert np.array_equal(nulls.cpu().numpy(), onulls)
    for i, (g, o) in enumerate(zip(outs, ocols)):
        h = G.to_host(g)
        assert np.array_equal(h.mask, o.mask), f"mask, column {i}"
        if types[i] == O.STRING:
            assert np.array_equal(h.offsets, o.offsets) and np.array_equal(h.data, o.data), f"string column {i}"
        else:
            assert cols_equal(h, o, check_null_payload=True), f"column {i}"


def test_wide_long_strings_take_the_slow_gather():
    """Strings longer than 32 bytes and tiles whose chars exceed a stage (direct mode) in a wide schema."""
    G = _gpu()
    import srj_b200 as S
    types = [O.INT64, O.STRING] * 40
    nrows = 300
    cols = random_table(types, nrows, seed=8, max_str=32)
    rng = np.random.default_rng(3)
    # make two columns long: ~200-byte strings in one, a few 40 KB strings in another
    for ci, lens in ((1, rng.integers(100, 300, nrows)), (41, np.where(np.arange(nrows) % 37 == 0, 40_000, 3))):
        offs = np.zeros(nrows + 1, np.int32)
        np.cumsum(lens, out=offs[1:])
        cols[ci] = O.HCol(O.STRING, rng.integers(32, 127, int(offs[-1]), dtype=np.uint8), None, offs, 0, nrows)
    (offs, data), = O.convert_to_rows(cols)
    tbl = S.RowConversion.convertFromRows(G.rows_to_device(offs, data), [S.DType(t) for t in types])
    _check_table(G, tbl, data, offs, nrows, types, cols)


# ======================================== to_rows (to_rows_wide.cu) =================================================
def _check_to_rows(cols):
    G = _gpu()
    import srj_b200 as S
    batches = O.convert_to_rows(cols)
    out = S.RowConversion.convertToRows(G.table_to_device(cols))
    assert len(out) == len(batches)
    for o, (offs, data) in zip(out, batches):
        goffs, gdata = G.rows_to_host(o)
        assert np.array_equal(goffs, offs)
        assert np.array_equal(gdata, data), f"first diff at byte {np.flatnonzero(gdata != data)[:5]} of {len(data)}"


WIDE_TO_ROWS = dict(WIDE_SCHEMAS)
WIDE_TO_ROWS.update({
    # 8 KB of 16-byte fields in front of 10 STRING columns
    "dec_slabs": [O.DECIMAL128] * 500 + [O.STRING] * 10,
    # size_per_row not a multiple of 8: the variable section starts inside an 8-byte store unit
    "phase": [O.INT64] * 70 + [O.STRING] * 9 + [O.INT8] * 3,
    # 33 STRING columns: 8 warps x 5 columns, the last warp of a tile has none
    "str33": [O.STRING] * 33 + [O.INT32] * 90,
})


@pytest.mark.parametrize("nrows", [1, 31, 32, 33, 64, 65, 1000, 4099])
@pytest.mark.parametrize("name", sorted(WIDE_TO_ROWS))
def test_wide_to_rows(name, nrows):
    types = WIDE_TO_ROWS[name]
    _check_to_rows(random_table(types, nrows, seed=nrows * 5 + len(types)))


@pytest.mark.parametrize("null_frac", [0.0, 0.5, 1.0])
def test_wide_to_rows_null_masks(null_frac):
    """0.0: no masks at all (NULL mask pointers = all valid); 1.0: every value null (payload still copied)."""
    _check_to_rows(random_table(WIDE_SCHEMAS["odd"], 2500, seed=17, null_frac=null_frac))


@pytest.mark.parametrize("max_str", [0, 1, 31, 32, 33, 100])
def test_wide_to_rows_string_lengths(max_str):
    """0: empty chars buffers; <= 32: word mover; > 32: the byte-wise rounds (and tiles that exceed the images)."""
    _check_to_rows(random_table(WIDE_SCHEMAS["c3"], 777, seed=max_str, max_str=max_str))


def test_wide_to_rows_huge_rows_fall_back():
    """Rows far larger than the tile images raise the flag; the generic kernel behind redoes the batch."""
    rng = np.random.default_rng(4)
    types = WIDE_SCHEMAS["strings_last"]
    n = 200
    cols = random_table(types, n, seed=2)
    lens = np.where(np.arange(n) % 50 == 7, 90_000, 4)
    offs = np.zeros(n + 1, np.int32)
    np.cumsum(lens, out=offs[1:])
    cols[105] = O.HCol(O.STRING, rng.integers(32, 127, int(offs[-1]), dtype=np.uint8), None, offs, 0, n)
    _check_to_rows(cols)


def test_wide_to_rows_unaligned_column_buffers():
    """Chars at odd addresses (cp.async chunks that start below the buffer: head bytes by hand), fixed-width data,
    masks and offsets as element-offset slices of larger allocations (cudf's alignment contract: element-aligned)."""
    G = _gpu()
    import srj_b200 as S
    types = WIDE_SCHEMAS["c3"]
    n = 1300
    cols = random_table(types, n, seed=31)
    batches = O.convert_to_rows(cols)

    def shifted(t, nbytes):
        raw = t.view(torch.uint8).reshape(-1)
        big = torch.empty(raw.numel() + nbytes, dtype=torch.uint8, device="cuda")
        big[nbytes:] = raw
        return big[nbytes:]

    dcols = []
    for c, t in zip(cols, types):
        d = G.to_device(c)
        if t == O.STRING:
            d.data = shifted(d.data, 5)
            d.offsets = shifted(d.offsets, 4).view(torch.int32)
        else:
            d.data = shifted(d.data, S.DType(t).size_in_bytes())
        if d.mask is not None:
            d.mask = shifted(d.mask, 4).view(torch.int32)
        dcols.append(d)
    out = S.RowConversion.convertToRows(S.Table(dcols))
    assert len(out) == 1
    goffs, gdata = G.rows_to_host(out[0])
    assert np.array_equal(goffs, batches[0][0])
    assert np.array_equal(gdata, batches[0][1]), f"first diff at byte {np.flatnonzero(gdata != batches[0][1])[:5]}"


def test_wide_round_trip_is_identity():
    G = _gpu()
    import srj_b200 as S
    types = WIDE_SCHEMAS["c3"]
    cols = random_table(types, 9000, seed=12)
    out = S.RowConversion.convertToRows(G.table_to_device(cols))
    tbl = S.RowConversion.convertFromRows(out[0], [S.DType(t) for t in types])
    for g, c in zip(tbl.columns, cols):
        assert cols_equal(G.to_host(g), c)
