"""The UnsafeRow codec (csrc/unsafe_row.cu) against the independent model (tests/unsafe_row_model.py) at the edges its
launches have: grid-stride sweeps, the per-warp shared-memory stage, the path without row offsets, 256 fields, type
and value edges, row counts of zero and row bytes at INT32_MAX, rows from another writer, and concurrent callers.

to_rows and from_rows run at most 8 CTAs of 256 rows per SM, the chars gather at most 16 CTAs of 8 warps x 32 rows;
a warp assembles its 32 rows in a 12 KB stage when they fit and writes in place otherwise.  Row counts and string
lengths come from unsafe_row_model.plan() and the device's SM count, so the cases stay on those edges on any GPU.

Compared whole: to_rows -- every row byte, padding included, and the row offsets; from_rows -- every column byte
(the payload under a NULL too), the mask words with their zero tail bits, STRING offsets and chars, the null counts.
Output buffers are filled with a sentinel first, so a byte the kernels leave unwritten shows.  Large tables are built
on the device and compared in chunks of rows."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

import unsafe_row_model as M
from oracle import oracle as O
from test_gpu_unsafe_row import SCHEMAS as GPU_SCHEMAS
from test_unsafe_row_model import ALL_TYPES, _dec_cases
from util import TYPE_BY_NAME, col_from_values, random_table

pytestmark = pytest.mark.gpu

S_, I8, I32, I64, D128 = O.STRING, O.INT8, O.INT32, O.INT64, O.DECIMAL128
METRIC = [I32, I64, D128, S_] * 64
CHUNK = 16 * 1024
INT32_MAX = 2**31 - 1


def _gpu():
    import gpu_util
    gpu_util.require_cuda()
    return gpu_util


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rows_sweep() -> int:
    return _sms() * M.ROWS_GRID_PER_SM * M.THREADS


def _chars_sweep() -> int:
    return _sms() * M.CHARS_GRID_PER_SM * M.THREADS


def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- tables
class _HostCol:
    """Rows [lo, hi) of a device column on the host, in the shape the model reads (lo a multiple of 32)."""

    def __init__(self, dc, lo, hi):
        t = dc.dtype.type_id
        self.type_id, self.size = t, hi - lo
        self.mask = None if dc.mask is None else dc.mask[lo // 32:(hi + 31) // 32].cpu().numpy().view(np.uint32)
        self.offsets = None
        if t == S_:
            o = dc.offsets[lo:hi + 1].cpu().numpy().astype(np.int64)
            self.data = dc.data[int(o[0]):int(o[-1])].cpu().numpy()
            self.offsets = o - o[0]
        else:
            w = M.FIXED_WIDTH.get(t, 16)
            self.data = dc.data[lo * w:hi * w].cpu().numpy()


def _random_mask(n, null_frac, g):
    if null_frac == 0:
        return None
    words = (n + 31) // 32
    bits = torch.zeros(words * 32, dtype=torch.int64, device="cuda")
    bits[:n] = (torch.rand(n, device="cuda", generator=g) >= null_frac).to(torch.int64)
    w = (bits.view(words, 32) << torch.arange(32, device="cuda")).sum(1)
    return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)


def _valid_of(mask, n):
    if mask is None:
        return torch.ones(n, dtype=torch.bool, device="cuda")
    r = torch.arange(n, device="cuda")
    return ((mask[r >> 5] >> (r & 31)) & 1).bool()


def _dev_table(types, n, seed, null_frac=0.2, max_str=12):
    """Seeded columns on the device: random bytes (BOOL8 in {0, 1}), DECIMAL128 values of every toByteArray length,
    strings of 0..max_str bytes, NULL strings empty, mask tail bits zero."""
    import srj_b200 as S
    g = torch.Generator(device="cuda").manual_seed(seed)
    cols = []
    for t in types:
        mask = _random_mask(n, null_frac, g)
        if t == S_:
            lens = torch.randint(0, max_str + 1, (n,), device="cuda", generator=g, dtype=torch.int64)
            lens = torch.where(_valid_of(mask, n), lens, 0)
            offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
            torch.cumsum(lens, 0, out=offs[1:])
            chars = torch.randint(0, 256, (max(int(offs[-1]), 1),), device="cuda", generator=g, dtype=torch.uint8)
            cols.append(S.ColumnVector(S.DType(t), n, chars, mask, offs.to(torch.int32)))
        elif t == D128:
            raw = torch.randint(0, 256, (n, 16), device="cuda", generator=g, dtype=torch.uint8)
            k = torch.randint(1, 17, (n, 1), device="cuda", generator=g)
            neg = (raw.gather(1, k - 1) & 0x80) != 0
            fill = torch.where(neg, 255, 0).to(torch.uint8)
            raw = torch.where(torch.arange(16, device="cuda")[None, :] < k, raw, fill)
            cols.append(S.ColumnVector(S.DType(t), n, raw.reshape(-1), mask))
        else:
            w = M.FIXED_WIDTH[t]
            data = torch.randint(0, 256, (n * w,), device="cuda", generator=g, dtype=torch.uint8)
            if t == O.BOOL8:
                data &= 1
            cols.append(S.ColumnVector(S.DType(t), n, data, mask))
    return cols


def _host_table(cols):
    return [_gpu().to_device(c) for c in cols]


# ---------------------------------------------------------------------------------------------- C ABI calls
def _abi():
    from srj_b200 import _native as N
    return N, N.lib(), int(torch.cuda.current_stream().cuda_stream)


def _to_rows(dcols, n, with_offsets=True):
    """srj_unsafe_row_sizes + srj_convert_to_unsafe_rows into a sentinel-filled buffer -> (offsets or None, rows)."""
    N, lib, st = _abi()
    ws = torch.empty(max(8, lib.srj_unsafe_row_workspace_bytes(len(dcols), n)), dtype=torch.uint8, device="cuda")
    carr = (N.SrjColumn * len(dcols))(*[c._c() for c in dcols])
    offs = None
    if with_offsets:
        offs = torch.empty(n + 1, dtype=torch.int32, device="cuda")
        total = C.c_int64(0)
        N.check(lib.srj_unsafe_row_sizes(carr, len(dcols), n, offs.data_ptr(), C.byref(total), ws.data_ptr(), st))
        nbytes = total.value
    else:
        nbytes = n * M.layout([c.dtype.type_id for c in dcols]).row_base
    rows = torch.full((max(nbytes, 8),), 0xA5, dtype=torch.uint8, device="cuda")
    N.check(lib.srj_convert_to_unsafe_rows(carr, len(dcols), n, None if offs is None else offs.data_ptr(), rows.data_ptr(),
                                           ws.data_ptr(), st))
    torch.cuda.synchronize()
    return offs, rows[:nbytes]


def _from_rows(types, rows, offs, n):
    """srj_convert_from_unsafe_rows (+ _strings) into sentinel-filled outputs -> (columns, null counts)."""
    import srj_b200 as S
    N, lib, st = _abi()
    words = max(1, (n + 31) // 32)
    outs = []
    for t in types:
        mask = torch.full((words,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        if t == S_:
            outs.append(S.ColumnVector(S.DType(t), n, None, mask, torch.full((n + 1,), -7, dtype=torch.int32, device="cuda")))
        else:
            outs.append(S.ColumnVector(S.DType(t), n, torch.full((max(1, n * M.FIXED_WIDTH.get(t, 16)),), 0xA5,
                                                                 dtype=torch.uint8, device="cuda"), mask))
    nulls = torch.full((len(types),), -1, dtype=torch.int64, device="cuda")
    ws = torch.empty(max(8, lib.srj_unsafe_row_workspace_bytes(len(types), n)), dtype=torch.uint8, device="cuda")
    carr = (N.SrjColumn * len(outs))(*[c._c() for c in outs])
    optr = None if offs is None else offs.data_ptr()
    N.check(lib.srj_convert_from_unsafe_rows(rows.data_ptr(), optr, n, carr, len(outs), nulls.data_ptr(), ws.data_ptr(), st))
    sidx = [i for i, t in enumerate(types) if t == S_]
    if sidx:
        for i in sidx:
            outs[i].data = torch.full((max(1, int(outs[i].offsets[n])),), 0xA5, dtype=torch.uint8, device="cuda")
        carr = (N.SrjColumn * len(outs))(*[c._c() for c in outs])
        N.check(lib.srj_convert_from_unsafe_rows_strings(rows.data_ptr(), optr, n, carr, len(outs), st))
    torch.cuda.synchronize()
    return outs, nulls.cpu().numpy()


# ---------------------------------------------------------------------------------------------- comparisons
def _chunks(n, chunk=CHUNK):
    return [(lo, min(n, lo + chunk)) for lo in range(0, n, chunk)]


def _row_span(offs, types, lo, hi):
    if offs is None:
        rb = M.layout(types).row_base
        return lo * rb, hi * rb, None
    o = offs[lo:hi + 1].cpu().numpy().astype(np.int64)
    return int(o[0]), int(o[-1]), o - o[0]


def _check_to_rows(host_cols, offs, rows, n, types, spans=None):
    """Device rows against the model's, over `spans` ((lo, hi) row ranges, lo a multiple of 32; default: all)."""
    if offs is not None:
        assert int(offs[0]) == 0 and int(offs[n]) == rows.numel(), "row offsets: first / last"
    elif spans is None:
        assert rows.numel() == n * M.layout(types).row_base
    for lo, hi in spans or _chunks(n):
        want_o, want_d = M.to_rows(host_cols(lo, hi))
        b0, b1, got_o = _row_span(offs, types, lo, hi)
        if got_o is not None:
            assert np.array_equal(got_o, want_o), f"row offsets in rows [{lo}, {hi}): first diff " \
                f"{lo + np.flatnonzero(got_o != want_o)[:4]}"
        got = rows[b0:b1].cpu().numpy()
        assert np.array_equal(got, want_d), f"row bytes of rows [{lo}, {hi}): first diff at byte " \
            f"{b0 + np.flatnonzero(got != want_d)[:5]}"


def _check_from_rows(types, outs, nulls, offs, rows, n, spans=None):
    """Device columns against the model's reading of the device rows (which _check_to_rows or the case pinned)."""
    whole = spans is None
    total = np.zeros(len(types), np.int64)
    for lo, hi in spans or _chunks(n):
        b0, b1, ro = _row_span(offs, types, lo, hi)
        want = M.from_rows(rows[b0:b1].cpu().numpy(), ro, types, n=hi - lo)
        total += want.null_counts
        for f, (t, g) in enumerate(zip(types, outs)):
            if g.mask is None:
                assert want.null_counts[f] == 0, f"field {f}: no mask but NULLs in rows [{lo}, {hi})"
            else:
                m = g.mask[lo // 32:(hi + 31) // 32].cpu().numpy().view(np.uint32)
                assert np.array_equal(m, want.masks[f]), f"mask words of field {f}, rows [{lo}, {hi}): first diff " \
                    f"{lo // 32 + np.flatnonzero(m != want.masks[f])[:4]}"
            if t == S_:
                o = g.offsets[lo:hi + 1].cpu().numpy().astype(np.int64)
                assert np.array_equal(o - o[0], want.offsets[f]), f"offsets of field {f}, rows [{lo}, {hi})"
                got = g.data[int(o[0]):int(o[-1])].cpu().numpy()
            else:
                w = M.FIXED_WIDTH.get(t, 16)
                got = g.data[lo * w:hi * w].cpu().numpy()
            assert np.array_equal(got, want.data[f]), f"bytes of field {f}, rows [{lo}, {hi}): first diff " \
                f"{np.flatnonzero(got != want.data[f])[:4]}"
    if whole:
        assert np.array_equal(np.asarray(nulls), total), f"null counts {np.asarray(nulls)} vs {total}"
        for t, g in zip(types, outs):
            if t == S_:
                assert int(g.offsets[0]) == 0 and g.data.numel() == max(1, int(g.offsets[n]))


def _check_round_trip_on_device(dcols, outs, nulls, n):
    """from(to(x)) against x on the device, whole: values where valid, 0 under a NULL (the slot of a NULL is 0),
    NULL strings empty, the same mask words and null counts."""
    for f, (c, g) in enumerate(zip(dcols, outs)):
        valid = _valid_of(c.mask, n)
        if g.mask is not None and c.mask is not None:
            assert torch.equal(g.mask[:(n + 31) // 32], c.mask[:(n + 31) // 32]), f"mask words, field {f}"
        assert int(nulls[f]) == int((~valid).sum()), f"null count, field {f}"
        if c.dtype.type_id == S_:
            assert torch.equal(g.offsets, c.offsets), f"string offsets, field {f}"
            k = int(c.offsets[n])
            assert torch.equal(g.data[:k], c.data[:k]), f"chars, field {f}"
        else:
            w = M.FIXED_WIDTH.get(c.dtype.type_id, 16)
            want = torch.where(valid.repeat_interleave(w), c.data[:n * w], 0)
            assert torch.equal(g.data[:n * w], want), f"values, field {f}"


def _host_of(dcols):
    return lambda lo, hi: [_HostCol(c, lo, hi) for c in dcols]


def _host_cols_of(cols):
    """Host columns sliced to [lo, hi) by the model itself."""
    class _Range:
        def __init__(self, c, lo, hi):
            self.type_id, self.size, self.mask = c.type_id, hi - lo, None
            w = None if c.type_id == S_ else M.FIXED_WIDTH.get(c.type_id, 16)
            valid = c.valid()[lo:hi]
            self.mask = None if c.mask is None else O.pack_mask(valid)
            if w is None:
                o = c.offsets.astype(np.int64)
                self.offsets = o[lo:hi + 1] - o[lo]
                self.data = c.data[o[lo]:o[hi]]
            else:
                self.offsets = None
                self.data = np.ascontiguousarray(c.data).view(np.uint8)[lo * w:hi * w]
    return lambda lo, hi: [_Range(c, lo, hi) for c in cols]


def _both_ways_whole(types, cols, with_offsets=True):
    """Host columns through the C ABI both ways, compared whole with the model."""
    _gpu()
    n = cols[0].size
    dcols = _host_table(cols)
    offs, rows = _to_rows(dcols, n, with_offsets)
    _check_to_rows(_host_cols_of(cols), offs, rows, n, types)
    outs, nulls = _from_rows(types, rows, offs, n)
    _check_from_rows(types, outs, nulls, offs, rows, n)


# ======================================================================= 1. the metric's shape
def test_metric_shape_256_columns_past_a_chars_sweep():
    """[INT32, INT64, DECIMAL128, STRING] x 64 with 20 % NULLs through UnsafeRowConversion, past three to_rows /
    from_rows sweeps and one chars-gather sweep, ending 17 rows into a warp.  Two chars sweeps would be about 1.08 M
    rows: more than 2^31 bytes of rows of this schema, which one call refuses."""
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    n = _chars_sweep() + 4096 + 17
    dcols = _dev_table(METRIC, n, seed=256)
    rows = UR.convertToRows(S.Table(dcols))
    offs, data = rows.offsets, rows.child.data
    p = M.plan(METRIC, n, _sms(), offs.cpu().numpy())
    assert (p.rows_sweeps, p.chars_sweeps) == (3, 2) and n % 32 == 17 and p.smem == 8 * 12288 + 256 * 44 + 16
    _check_to_rows(_host_of(dcols), offs, data, n, METRIC)
    back = UR.convertFromRows(rows, [S.DType(t) for t in METRIC])
    outs = back.columns
    nulls = [c.getNullCount() for c in outs]
    _check_round_trip_on_device(dcols, outs, nulls, n)
    # the model's own reading of the rows, at both ends and across each sweep boundary
    spans = [(0, 4096), (n // 32 * 32 - 4096, n)] + [(b - 2048, b + 2048) for b in (_rows_sweep(), 2 * _rows_sweep(),
                                                                                   _chars_sweep())]
    _check_from_rows(METRIC, outs, nulls, offs, data, n, spans)
    del rows, back, outs, dcols
    _free()


@pytest.mark.parametrize("fields", [255, 256])
@pytest.mark.parametrize("kind", [I32, I64, D128, S_], ids=["INT32", "INT64", "DECIMAL128", "STRING"])
def test_255_and_256_fields_of_one_kind(kind, fields):
    types = [kind] * fields
    n = 2 * 256 + 37
    cols = random_table(types, n, seed=fields + kind)
    _both_ways_whole(types, cols)


def test_a_257th_field_is_refused_everywhere():
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    types = [I32] * 257
    with pytest.raises(S.CudfException):
        UR.layout([S.DType(t) for t in types])
    with pytest.raises(M.UnsupportedSchema):
        M.layout(types)
    N, lib, st = _abi()
    dcols = _host_table(random_table(types, 5, seed=1))
    carr = (N.SrjColumn * 257)(*[c._c() for c in dcols])
    ws = torch.empty(lib.srj_unsafe_row_workspace_bytes(257, 5), dtype=torch.uint8, device="cuda")
    offs = torch.zeros(6, dtype=torch.int32, device="cuda")
    rows = torch.zeros(5 * 4096, dtype=torch.uint8, device="cuda")
    nulls = torch.zeros(257, dtype=torch.int64, device="cuda")
    total = C.c_int64(0)
    with pytest.raises(S.CudfException):
        N.check(lib.srj_unsafe_row_sizes(carr, 257, 5, offs.data_ptr(), C.byref(total), ws.data_ptr(), st))
    with pytest.raises(S.CudfException):
        N.check(lib.srj_convert_to_unsafe_rows(carr, 257, 5, None, rows.data_ptr(), ws.data_ptr(), st))
    with pytest.raises(S.CudfException):
        N.check(lib.srj_convert_from_unsafe_rows(rows.data_ptr(), None, 5, carr, 257, nulls.data_ptr(), ws.data_ptr(), st))
    with pytest.raises(S.CudfException):
        N.check(lib.srj_convert_from_unsafe_rows_strings(rows.data_ptr(), offs.data_ptr(), 5, carr, 257, st))
    torch.cuda.synchronize()
    assert not rows.any(), "a refused call wrote rows"


# ======================================================================= 2. stage edges with row offsets
STAGE_SCHEMA = [S_, I32, S_]      # the STRING sizes set each warp's bytes; INT32 has NULLs, the last STRING is all NULL
_STAGE_FIXED = M.layout(STAGE_SCHEMA).fixed_bytes        # 32 bytes: bitset + 3 slots


def _padded_sizes(k, total):
    """k padded string sizes (multiples of 8, >= 8) summing to total - k * fixed: a warp of k rows of `total` bytes."""
    words = (total - k * _STAGE_FIXED) // 8
    assert (total - k * _STAGE_FIXED) % 8 == 0 and words >= k
    s = np.full(k, words // k, np.int64)
    s[: words % k] += 1
    return 8 * s


def _stage_table(warp_bytes, seed):
    """Columns whose warp w spans exactly warp_bytes[w] = (bytes, rows) (the last warp may be partial), and the row
    offsets that gives."""
    rng = np.random.default_rng(seed)
    n = 32 * (len(warp_bytes) - 1) + warp_bytes[-1][1]
    padded = np.concatenate([_padded_sizes(k, b) for b, k in warp_bytes])
    lens = padded - rng.integers(0, 8, n)                 # within 7 bytes below the padded size: padding varies
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    chars = rng.integers(0, 256, int(offs[-1]), dtype=np.uint8)
    s0 = O.HCol(S_, chars, None, offs.astype(np.int32), 0, n)
    i32 = O.HCol(I32, rng.integers(0, 256, 4 * n, dtype=np.uint8), O.pack_mask(rng.random(n) >= 0.2), None, 0, n)
    s2 = O.HCol(S_, np.zeros(0, np.uint8), np.zeros((n + 31) // 32, np.uint32), np.zeros(n + 1, np.int32), 0, n)
    ro = np.zeros(n + 1, np.int64)
    np.cumsum(padded + _STAGE_FIXED, out=ro[1:])
    return [s0, i32, s2], ro


STAGED, IN_PLACE = M.STAGE, M.STAGE + 8


def test_stage_edges_alternate_in_a_cta_and_flip_between_sweeps():
    """Warps of exactly 12,288 bytes (staged) and 12,296 bytes (in place), alternating inside every CTA; a CTA's warp
    that is staged in its first grid-stride sweep is in place in its second and the reverse; a third sweep ends on a
    partial warp of 9 rows at the edge, once staged and once in place."""
    _gpu()
    sweep_warps = _rows_sweep() // 32
    for last in (STAGED, IN_PLACE):
        nw = 2 * sweep_warps + 3
        wb = [((STAGED if (w + w // sweep_warps) % 2 == 0 else IN_PLACE), 32) for w in range(nw - 1)] + [(last, 9)]
        cols, ro = _stage_table(wb, seed=last)
        n = cols[0].size
        p = M.plan(STAGE_SCHEMA, n, _sms(), ro)
        assert p.rows_sweeps == 3 and p.staged.tolist() == [b == STAGED for b, _ in wb]
        assert p.staged[0] and not p.staged[1] and not p.staged[sweep_warps] and p.staged[sweep_warps + 1]
        _both_ways_whole(STAGE_SCHEMA, cols)
        _free()


def test_a_row_larger_than_the_stage():
    cols = random_table([S_, I32, S_], 100, seed=4, max_str=40)
    big = np.random.default_rng(1).integers(0, 256, 13001, dtype=np.uint8)
    o = cols[0].offsets.astype(np.int64)
    r = 40
    chars = np.concatenate([cols[0].data[:o[r]], big, cols[0].data[o[r + 1]:]])
    lens = np.diff(o)
    lens[r] = len(big)
    offs = np.zeros(101, np.int64)
    np.cumsum(lens, out=offs[1:])
    valid = cols[0].valid()
    valid[r] = True
    cols[0] = O.HCol(S_, chars, O.pack_mask(valid), offs.astype(np.int32), 0, 100)
    ro, _ = M.to_rows(cols)
    p = M.plan([S_, I32, S_], 100, _sms(), ro)
    assert ro[r + 1] - ro[r] > M.STAGE and p.staged.tolist() == [True, False, True, True]
    _both_ways_whole([S_, I32, S_], cols)


# ======================================================================= 3. no row offsets (C ABI)
OFFSET_LESS = {
    "int64_x47_384B": [I64] * 47,                          # every warp staged
    "int64_x48_392B": [I64] * 48,                          # full warps in place, a partial last warp staged
    "dec_384B": [I64] * 32 + [D128] * 5,                   # the same edge through 16 * ndec
    "dec_392B": [I64] * 30 + [D128] * 6,
    "fixed_256": (ALL_TYPES[:18] * 15)[:256],              # 2080-byte rows: staged only up to 5 rows
}


def _offset_less_n(where, sms):
    if where == "two_sweeps":
        return 2 * sms * M.ROWS_GRID_PER_SM * M.THREADS + 32 * 5 + 5
    return 2 * 256 + 32 * 2 + int(where.split("_")[1])


@pytest.mark.parametrize("where", ["tail_1", "tail_5", "tail_31", "two_sweeps"])
@pytest.mark.parametrize("name", list(OFFSET_LESS))
def test_offset_less_stage_edges(name, where):
    _gpu()
    types = OFFSET_LESS[name]
    n = _offset_less_n(where, _sms())
    row = M.layout(types).row_base
    p = M.plan(types, n, _sms())
    assert p.stage == min(M.STAGE, 32 * row)
    assert bool(p.staged[0]) == (row <= 384) and bool(p.staged[-1]) == ((n % 32 or 32) * row <= p.stage)
    if where == "two_sweeps":
        assert p.rows_sweeps == 3
    dcols = _dev_table(types, n, seed=n % 1000 + len(types))
    offs, rows = _to_rows(dcols, n, with_offsets=False)
    _check_to_rows(_host_of(dcols), None, rows, n, types)
    outs, nulls = _from_rows(types, rows, None, n)
    _check_from_rows(types, outs, nulls, None, rows, n)
    del dcols, rows, outs
    _free()


# ======================================================================= 4. the benchmark's workload
def test_unsafe_c2_at_50m_rows_without_row_offsets():
    """bench.py's unsafe_c2 table: 50 M rows of [INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, BOOL8, TIMESTAMP_US] x 4,
    264-byte rows, 20 % NULLs.  Every column, mask and null count on the device; rows and columns against the model at
    both ends and in random 4 K-row windows."""
    _gpu()
    types = [I8, O.INT16, I32, I64, O.FLOAT32, O.FLOAT64, O.BOOL8, O.TIMESTAMP_MICROSECONDS] * 4
    n = 50_000_000
    assert M.layout(types).row_base == 264
    dcols = _dev_table(types, n, seed=42)
    offs, rows = _to_rows(dcols, n, with_offsets=False)
    outs, nulls = _from_rows(types, rows, None, n)
    _check_round_trip_on_device(dcols, outs, nulls, n)
    rng = np.random.default_rng(50)
    spans = [(0, 65536), (n - 65536, n)] + [(lo, lo + 4096) for lo in (rng.integers(0, (n - 4096) // 32, 6) * 32).tolist()]
    _check_to_rows(_host_of(dcols), None, rows, n, types, spans)
    _check_from_rows(types, outs, nulls, None, rows, n, spans)
    del dcols, rows, outs
    _free()


# ======================================================================= 5. types
def _edge_values(t):
    if t == D128:
        return [v for v, _ in _dec_cases()]
    if t == S_:
        return [b"", None, b"x" * 7, b"y" * 8, b"z" * 9, b"\xc3\xa9" * 20]
    if t in (O.FLOAT32, O.FLOAT64):
        b = "bits32" if t == O.FLOAT32 else "bits64"
        return [(b, 0x7FC00001 if t == O.FLOAT32 else 0xFFF8000000000001), -0.0, (b, 1), float("inf"), 1.5, None]
    w = M.FIXED_WIDTH[t]
    if t in (O.UINT8, O.UINT16, O.UINT32, O.UINT64, O.BOOL8):
        top = 1 if t == O.BOOL8 else 2 ** (8 * w) - 1
        return [0, top, (top + 1) // 2, None, 1]
    lo, hi = -2 ** (8 * w - 1), 2 ** (8 * w - 1) - 1
    return [lo, hi, -1, 0, None, 1, -719162 if w >= 4 else -3]


def test_every_accepted_type_at_its_value_edges():
    """Each type ur_classify accepts, at the known-answer values of the model's tests; the slots of negative
    TIMESTAMP_DAYS / INT32 values and of UINT32 / UINT16 values with the top bit set keep zero upper bytes, a DECIMAL32
    -1 is the long -1, float payloads move bit for bit."""
    vals = {t: _edge_values(t) for t in ALL_TYPES}
    n = max(len(v) for v in vals.values()) * 3
    names = {v: k for k, v in TYPE_BY_NAME.items()}
    cols = [col_from_values(names[t], (vals[t] * n)[:n]) for t in ALL_TYPES]
    _both_ways_whole(ALL_TYPES, cols)
    offs, rows = _to_rows(_host_table(cols), n)
    row0 = rows[: int(offs[1])].cpu().numpy()
    slot = {t: row0[8 + 8 * f:16 + 8 * f].tobytes() for f, t in enumerate(ALL_TYPES)}
    assert slot[O.TIMESTAMP_DAYS] == b"\x00\x00\x00\x80" + bytes(4)          # INT32 min, not sign-extended
    assert slot[O.UINT32] == bytes(8) and slot[O.UINT16] == bytes(8)
    assert slot[O.DECIMAL32] == (-2**31).to_bytes(8, "little", signed=True)
    assert slot[O.FLOAT32] == b"\x01\x00\xc0\x7f" + bytes(4)
    row1 = rows[int(offs[1]): int(offs[2])].cpu().numpy()
    s1 = {t: row1[8 + 8 * f:16 + 8 * f].tobytes() for f, t in enumerate(ALL_TYPES)}
    assert s1[O.UINT32] == b"\xff" * 4 + bytes(4) and s1[O.UINT16] == b"\xff\xff" + bytes(6)
    assert s1[O.TIMESTAMP_DAYS] == b"\xff\xff\xff\x7f" + bytes(4)
    row2 = rows[int(offs[2]): int(offs[3])].cpu().numpy()
    s2 = {t: row2[8 + 8 * f:16 + 8 * f].tobytes() for f, t in enumerate(ALL_TYPES)}
    assert s2[O.TIMESTAMP_DAYS] == b"\xff" * 4 + bytes(4) and s2[O.DECIMAL32] == b"\xff" * 8
    assert s2[O.UINT32] == b"\x00\x00\x00\x80" + bytes(4) and s2[O.UINT16] == b"\x00\x80" + bytes(6)


@pytest.mark.parametrize("t", [O.DURATION_DAYS, O.DURATION_NANOSECONDS, O.LIST, O.STRUCT],
                         ids=["DURATION_DAYS", "DURATION_NANOSECONDS", "LIST", "STRUCT"])
def test_unsupported_types_are_refused(t):
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    with pytest.raises(S.CudfException):
        UR.layout([S.DType(I32), S.DType(t)])
    if t in (O.DURATION_DAYS, O.DURATION_NANOSECONDS):
        w = 4 if t == O.DURATION_DAYS else 8
        c = S.ColumnVector(S.DType(t), 3, torch.zeros(3 * w, dtype=torch.uint8, device="cuda"))
        with pytest.raises(S.CudfException):
            UR.convertToRows(S.Table([c]))


# ======================================================================= 6. sizes
@pytest.mark.parametrize("types", [[I32, D128], [I32, S_, D128, S_]], ids=["no_strings", "strings"])
def test_zero_rows(types):
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    cols = random_table(types, 0, seed=1)
    rows = UR.convertToRows(S.Table(_host_table(cols)))
    assert rows.size == 0 and rows.offsets.cpu().tolist() == [0] and rows.child.size == 0
    back = UR.convertFromRows(rows, [S.DType(t) for t in types])
    for t, c in zip(types, back.columns):
        assert c.size == 0 and c.getNullCount() == 0
        if t == S_:
            assert c.offsets.cpu().tolist() == [0]
    offs, data = _to_rows(_host_table(cols), 0, with_offsets=S_ in types)
    outs, nulls = _from_rows(types, data, offs, 0)
    assert nulls.tolist() == [0] * len(types)
    for t, g in zip(types, outs):
        if t == S_:
            assert g.offsets.cpu().tolist() == [0]


def test_int8_rows_at_int32_max_bytes():
    """One INT8 field: 16-byte rows.  134,217,727 rows are 2,147,483,632 bytes and convert; one more row is refused."""
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    n = 134_217_727
    assert 16 * n <= INT32_MAX < 16 * (n + 1)
    dcols = _dev_table([I8], n + 1, seed=8)
    c = dcols[0]
    mask = c.mask.clone()
    mask[-1] &= 0x7FFFFFFF                               # row n's bit: the mask of n rows has a zero tail
    small = S.ColumnVector(c.dtype, n, c.data[:n], mask)
    rows = UR.convertToRows(S.Table([small]))
    assert rows.child.size == 16 * n
    offs, data = rows.offsets, rows.child.data
    assert torch.equal(offs.view(-1)[-2:].cpu(), torch.tensor([16 * (n - 1), 16 * n], dtype=torch.int32))
    w = data.view(torch.int64).view(n, 2)
    valid = _valid_of(mask, n)
    assert torch.equal(w[:, 0], (~valid).to(torch.int64)), "bitset words"
    assert torch.equal(w[:, 1], torch.where(valid, c.data[:n].to(torch.int64), 0)), "slots"
    del w
    rng = np.random.default_rng(9)
    spans = [(n // 32 * 32 - 65536, n)] + [(lo, lo + 4096) for lo in (rng.integers(0, n // 32 - 200, 4) * 32).tolist()]
    _check_to_rows(_host_of([small]), offs, data, n, [I8], spans)
    back = UR.convertFromRows(rows, [S.DType(I8)])
    _check_round_trip_on_device([small], back.columns, [back.columns[0].getNullCount()], n)
    _check_from_rows([I8], back.columns, None, offs, data, n, spans)
    del rows, back, data, offs
    _free()
    with pytest.raises(S.CudfColumnSizeOverflowException):
        UR.convertToRows(S.Table([c]))
    del dcols, c, small
    _free()


def test_string_rows_at_int32_max_bytes():
    """One STRING field of 8-byte strings: 24-byte rows.  89,478,485 rows are 2,147,483,640 bytes and convert, the
    chars of the last rows sit just under 2^31; one more row is refused."""
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    n = 89_478_485
    assert 24 * n <= INT32_MAX < 24 * (n + 1)
    g = torch.Generator(device="cuda").manual_seed(24)
    chars = torch.randint(0, 256, (8 * (n + 1),), device="cuda", generator=g, dtype=torch.uint8)
    offs_in = torch.arange(0, 8 * (n + 2), 8, dtype=torch.int32, device="cuda")
    col = S.ColumnVector(S.DType(S_), n, chars[:8 * n], None, offs_in[:n + 1])
    rows = UR.convertToRows(S.Table([col]))
    assert rows.child.size == 24 * n
    offs, data = rows.offsets, rows.child.data
    w = data.view(torch.int64).view(n, 3)
    assert not bool(w[:, 0].any()), "bitset words"
    assert bool((w[:, 1] == (16 << 32) | 8).all()), "slots"
    assert torch.equal(w[:, 2], chars[:8 * n].view(torch.int64)), "chars in the rows"
    del w
    spans = [(n // 32 * 32 - 65536, n), (0, 4096)]
    _check_to_rows(_host_of([col]), offs, data, n, [S_], spans)
    back = UR.convertFromRows(rows, [S.DType(S_)])
    out = back.columns[0]
    assert torch.equal(out.offsets, offs_in[:n + 1]) and torch.equal(out.data, chars[:8 * n])
    _check_from_rows([S_], back.columns, None, offs, data, n, spans)
    del rows, back, out, data, offs
    _free()
    with pytest.raises(S.CudfColumnSizeOverflowException):
        UR.convertToRows(S.Table([S.ColumnVector(S.DType(S_), n + 1, chars, None, offs_in)]))
    del chars, offs_in, col
    _free()


# ======================================================================= 7. rows from another writer
@pytest.mark.parametrize("where", ["small", "past_a_chars_sweep"])
def test_rows_from_another_writer(where):
    """Rows whose variable-length entries are in reverse field order behind 8-byte gaps: the readers follow the slots."""
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    types = [S_, D128, I32, S_, I64, D128, S_]
    n = 1000 + 7 if where == "small" else _chars_sweep() + 33
    cols = random_table(types, n, seed=n % 997, max_str=20)
    offs, data = M.to_rows_permuted(cols)
    assert int(offs[-1]) <= INT32_MAX
    rows = _gpu().rows_to_device(offs, data)
    back = UR.convertFromRows(rows, [S.DType(t) for t in types])
    want = M.from_rows(data, offs, types)
    assert want.null_counts.tolist() == [c.null_count() for c in cols]
    outs = back.columns
    for f, (t, g) in enumerate(zip(types, outs)):
        assert g.getNullCount() == want.null_counts[f]
        if g.mask is not None:
            assert np.array_equal(g.mask.cpu().numpy().view(np.uint32)[:(n + 31) // 32], want.masks[f]), f
        if t == S_:
            assert np.array_equal(g.offsets.cpu().numpy(), want.offsets[f]), f
        assert np.array_equal(g.data.cpu().numpy(), want.data[f]), f"field {f}"
    # and the model's reading is the input, NULL payloads zeroed
    ro, rd = M.to_rows(cols)
    regular = M.from_rows(rd, ro, types)
    for f in range(len(types)):
        assert np.array_equal(regular.data[f], want.data[f])
    del rows, back
    _free()


# ======================================================================= 8. threads and streams
def test_four_threads_on_their_own_streams():
    _gpu()
    import srj_b200 as S
    from srj_b200.unsaferow import UnsafeRowConversion as UR
    names = ["mixed", "fixed_only", "strings_only", "decimals"]
    work = {}
    for i, name in enumerate(names):
        types = GPU_SCHEMAS[name]
        cols = random_table(types, 3000 + 517 * i, seed=70 + i)
        work[name] = (types, cols, M.to_rows(cols))
    errors = []
    dev = torch.cuda.current_device()

    def run(name):
        try:
            torch.cuda.set_device(dev)
            types, cols, (want_o, want_d) = work[name]
            want = M.from_rows(want_d, want_o, types)
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                for _ in range(3):
                    dt = S.Table(_host_table(cols))
                    rows = UR.convertToRows(dt)
                    back = UR.convertFromRows(rows, [S.DType(t) for t in types])
                    stream.synchronize()
                    assert np.array_equal(rows.offsets.cpu().numpy(), want_o), name
                    assert np.array_equal(rows.child.data.cpu().numpy(), want_d), name
                    for f, (t, g) in enumerate(zip(types, back.columns)):
                        assert g.getNullCount() == want.null_counts[f], (name, f)
                        if t == S_:
                            assert np.array_equal(g.offsets.cpu().numpy(), want.offsets[f]), (name, f)
                        assert np.array_equal(g.data.cpu().numpy(), want.data[f]), (name, f)
        except BaseException as e:                       # noqa: BLE001  (re-raised in the main thread)
            errors.append((name, e))

    threads = [threading.Thread(target=run, args=(nm,)) for nm in names]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
