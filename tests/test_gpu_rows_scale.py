"""The row-conversion kernels against the independent JCUDF model (tests/jcudf_model.py) at the row counts where their
persistent grids cycle.

Every from_rows / to_rows kernel runs at most one CTA per SM, deals tiles (or super-tiles) round-robin and stages them
through a shared-memory ring.  A CTA's ring is only exercised fully once it has wrapped its stages, and the round-robin
only once a CTA takes a second tile; both need more rows than the oracle-checked tests use.  The row counts here come
from the planning rules restated in tests/row_plans.py and the device's SM count, so they stay on those edges on any
GPU.  Each case names the kernel and template instantiation it was written for, and checks through torch.profiler that
it ran.

Compared whole: from_rows -- every column's bytes including the payload under nulls, the mask words with their zero
tail bits, STRING offsets and chars, the null counts, the chars totals and the status word; to_rows -- every row byte
including the padding, and the LIST offsets."""
import re
import warnings

import numpy as np
import pytest
import torch

import jcudf_model as M
import row_plans as P
from oracle import oracle as O
from util import random_table

pytestmark = pytest.mark.gpu

S_, I8, I16, I32, I64, D128 = O.STRING, O.INT8, O.INT16, O.INT32, O.INT64, O.DECIMAL128


def _gpu():
    import gpu_util
    gpu_util.require_cuda()
    return gpu_util


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------- profiling
def _norm(name: str) -> str:
    return re.sub(r"\s+", "", name)


def _ran(names, kernel):
    k = _norm(kernel)
    if "<" in k:
        return any(k in _norm(n) for n in names)
    return any(re.search(r"\b" + kernel + r"\b", n) for n in names)


def _profiled(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # a first device record, completed before fn() starts, so that the profiler's activity buffer is in place
        # when fn()'s first kernels finish
        torch.zeros(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        out = fn()
        torch.cuda.synchronize()
    return out, {e.name for e in prof.events()}


def _run_checked(fn, check, kernels):
    """fn() on the device, check(result) against the model, and each of `kernels` seen running.

    torch.profiler does not always deliver every kernel record of a short window.  The launchers' choices depend only on
    the schema and the sizes, so every run of the same call launches the same kernels: the call is profiled again, up
    to five times, until each named kernel has been seen, and every run's result is checked.  One unprofiled run goes
    first, so that plan creation, module loading and first-use allocations fall outside the profiled windows."""
    check(fn())
    seen = set()
    for attempt in range(5):
        out, names = _profiled(fn)
        check(out)
        del out
        seen |= names
        missing = [k for k in kernels if not _ran(seen, k)]
        if not missing:
            return
        if attempt < 4:
            warnings.warn(f"profiler run {attempt + 1} recorded no {missing}; profiling the same call again")
    assert not missing, f"{missing} did not run in 5 profiled runs; recorded: {sorted(seen)}"


# ---------------------------------------------------------------------------------------------- device calls
def _from_rows_device(types, d_offs, d_rows, n):
    """srj_convert_from_rows_fixed + _strings through the C ABI: the columns, the null counts and the chars totals with
    the status word behind them (what RowConversion.convertFromRows reads but does not return)."""
    import srj_b200 as S
    from srj_b200 import _native as N
    dts = [S.DType(t) for t in types]
    plan = S.Plan.get(dts)
    lib = N.lib()
    words = (n + 31) // 32
    outs = []
    for d in dts:
        mask = torch.empty(max(words, 1), dtype=torch.int32, device="cuda")
        if d.type_id == S.DType.STRING:
            outs.append(S.ColumnVector(d, n, None, mask, torch.empty(n + 1, dtype=torch.int32, device="cuda")))
        else:
            outs.append(S.ColumnVector(d, n, torch.empty(n * d.size_in_bytes(), dtype=torch.uint8, device="cuda"), mask))
    nc = len(dts)
    nulls = torch.full((nc,), -1, dtype=torch.int64, device="cuda")
    totals = torch.full((nc + 1,), -1, dtype=torch.int64, device="cuda")
    ws = torch.empty(max(8, lib.srj_from_rows_workspace_bytes(plan.handle, n)), dtype=torch.uint8, device="cuda")
    st = int(torch.cuda.current_stream().cuda_stream)
    carr = (N.SrjColumn * nc)()
    for i, c in enumerate(outs):
        carr[i] = c._c()
    N.check(lib.srj_convert_from_rows_fixed(plan.handle, d_rows.data_ptr(), d_offs.data_ptr(), d_rows.numel(), n, carr,
                                            nulls.data_ptr(), totals.data_ptr(), None, ws.data_ptr(), st))
    if any(t == S_ for t in types):
        h_tot = totals.cpu().numpy()
        for i, t in enumerate(types):
            if t == S_:
                outs[i].data = torch.empty(max(int(h_tot[i]), 1), dtype=torch.uint8, device="cuda")
                carr[i] = outs[i]._c()
        N.check(lib.srj_convert_from_rows_strings(plan.handle, d_rows.data_ptr(), d_offs.data_ptr(), d_rows.numel(), n,
                                                  carr, totals.data_ptr(), ws.data_ptr(), st))
    torch.cuda.synchronize()
    return outs, nulls.cpu().numpy(), totals.cpu().numpy()


def _check_from_rows(types, want: M.FromRows, n):
    def check(res):
        outs, nulls, totals = res
        nc = len(types)
        words = (n + 31) // 32
        for i, (t, g) in enumerate(zip(types, outs)):
            mask = g.mask.cpu().numpy().view(np.uint32)[:words]
            assert np.array_equal(mask, want.masks[i]), f"mask words, column {i}: first diff " \
                f"{np.flatnonzero(mask != want.masks[i])[:4]}"
            if t == S_:
                offs = g.offsets.cpu().numpy()
                assert np.array_equal(offs, want.offsets[i]), f"offsets, column {i}: first diff " \
                    f"{np.flatnonzero(offs != want.offsets[i])[:4]}"
                chars = g.data.cpu().numpy()[: int(want.char_totals[i])]
                assert np.array_equal(chars, want.data[i]), f"chars, column {i}: first diff " \
                    f"{np.flatnonzero(chars != want.data[i])[:4]}"
            else:
                got = g.data.cpu().numpy()
                assert np.array_equal(got, want.data[i]), f"column {i}: first diff at byte " \
                    f"{np.flatnonzero(got != want.data[i])[:4]}"
        assert np.array_equal(nulls, want.null_counts), "null counts"
        assert np.array_equal(totals[:nc], want.char_totals), "chars totals"
        assert int(totals[nc]) == want.status, f"status word {int(totals[nc])}, model {want.status}"
    return check


def _from_rows_case(types, cols, kernels, mutate=None):
    """Rows of `cols` by the model (optionally rewritten by `mutate(offs, data)`), converted back on the device and
    compared with the model's columns; `kernels` (None: not profiled) must be seen running.  Returns the model's status
    word."""
    _gpu()
    n = cols[0].size
    (offs, data), = M.to_rows(cols)
    if mutate is not None:
        mutate(offs, data)
    var = any(t == S_ for t in types)
    want = M.from_rows(data, offs if var else None, n, types)
    d_offs = torch.from_numpy(offs).cuda()
    d_rows = torch.from_numpy(data).cuda()
    del data
    fn, check = (lambda: _from_rows_device(types, d_offs, d_rows, n)), _check_from_rows(types, want, n)
    if kernels is None:
        check(fn())
    else:
        _run_checked(fn, check, kernels)
    return want.status


def _strings_kernel(types):
    return "strings_wide_kernel" if P.strings_wide_eligible(types) else "strings_from_rows_kernel"


def _from_rows_kernels(types):
    """What launches for a schema: the phase-1 kernel (instantiation named) and, with STRING columns, the scan and the
    chars gather."""
    if any(t == S_ for t in types):
        if P.wide_refusal(types) is None:
            return [P.wide_kernel_name(types), "wide_group_scan_kernel", _strings_kernel(types)]
        return [P.from_rows_kernel_name(types), _strings_kernel(types)]
    return [P.from_rows_kernel_name(types)]


# ======================================================================= from_rows_kernel, fixed width
FIXED = {
    # one schema per tiling class of srj_plan_create
    "c1_three_stages": [I32, I64, O.FLOAT64, O.BOOL8],                          # S <= 128: 3 x 64 KB, R = 512
    "c4_store_sales": [I32] * 9 + [I64, I32] + [O.DECIMAL32] * 12,             # S = 104: 3 stages, R = 512
    "c2_two_stages": [I8, I16, I32, I64, O.FLOAT32, O.FLOAT64, O.BOOL8, O.TIMESTAMP_MICROSECONDS] * 4,  # R = 512
    "r256": [I64] * 48,                                                         # R = 256
    "pivot_r64": [I64] * 191 + [I32],                                           # R = 64
    "dec200_r16": [D128] * 200,                                                 # R = 16
    "dec520_r8": [D128] * 520,                                                  # R = 8
    "shrunk_i32x3000": [I32] * 3000,                                            # stages shrunk below 100 KB
}


def _fixed_counts(types, sms):
    tl = P.from_rows_tiling(types)
    sup = P.from_rows_super_rows(types)
    # the last count: every CTA wraps its ring and takes a second super-tile, and the table ends on a partial tile
    return {"grid_minus_1": sms * sup - 1, "grid": sms * sup, "grid_plus_1": sms * sup + 1,
            "ring_wrap": (tl.num_stages + 1) * sms * sup + tl.tile_rows + 1}


def _fixed_ids():
    return [f"{name}-{k}-{P.from_rows_kernel_name(t)}" for name, t in FIXED.items() for k in
            ("grid_minus_1", "grid", "grid_plus_1", "ring_wrap")]


@pytest.mark.parametrize("name,where", [(n, k) for n in FIXED for k in ("grid_minus_1", "grid", "grid_plus_1", "ring_wrap")],
                         ids=_fixed_ids())
def test_fixed_from_rows_at_cycle_points(name, where):
    types = FIXED[name]
    n = _fixed_counts(types, _sms())[where]
    assert P.from_rows_tiling(types).num_stages in (2, 3)
    cols = random_table(types, n, seed=n % 1000 + len(types))
    _from_rows_case(types, cols, _from_rows_kernels(types))


@pytest.mark.parametrize("kind", ["murmur3", "xxhash64"])
def test_fused_hash_c4_when_every_cta_wraps(kind):
    """from_rows + partition hash of C4 at the ring-wrap row count: the hash of the columns just written."""
    G = _gpu()
    import srj_b200 as S
    types = FIXED["c4_store_sales"]
    n = _fixed_counts(types, _sms())["ring_wrap"]
    cols = random_table(types, n, seed=44, null_frac=0.04)
    (offs, data), = M.to_rows(cols)
    want = M.from_rows(data, None, n, types)
    keys = [1, 9]
    kc = [O.HCol(types[k], want.data[k], want.masks[k], None, 0, n) for k in keys]
    want_h = O.xxhash64(kc, 42) if kind == "xxhash64" else O.murmur_hash3_32(kc, 42)
    rows = G.rows_to_device(offs, data)

    def check(res):
        tbl, h = res
        assert np.array_equal(h.data.cpu().numpy().view(want_h.dtype), want_h)
        for i, g in enumerate(tbl.columns):
            assert np.array_equal(g.data.cpu().numpy(), want.data[i]), f"column {i}"
    _run_checked(lambda: S.RowConversion.convertFromRowsWithHash(rows, [S.DType(t) for t in types], keys, kind=kind,
                                                                 seed=42),
                 check, [P.from_rows_kernel_name(types)])


# ======================================================================= from_rows_kernel, variable width (VAR = 1)
VAR = {
    "mixed": [I32, S_, I64, D128, S_, O.BOOL8, S_, I16],
    "simple_string": [S_],
    "c3_small": [I32, I64, D128, S_] * 8,
}


@pytest.mark.parametrize("name", sorted(VAR), ids=lambda n: f"{n}-{P.from_rows_kernel_name(VAR[n])}")
def test_var_from_rows_second_super_tile(name):
    """2 super-tiles per CTA + 33 rows: the adaptive tile cut starts again in a CTA's second super-tile."""
    types = VAR[name]
    assert P.wide_refusal(types) is not None
    n = 2 * _sms() * P.from_rows_super_rows(types) + 33
    _from_rows_case(types, random_table(types, n, seed=n % 977), _from_rows_kernels(types))


# ======================================================================= from_rows_wide_kernel
WIDE = {
    "g4_520b": [S_] * 8 + [I64] * 56,                                  # G = 4, one slab, 520-B rows
    "g3_one_slab": [S_, I32] * 50,                                     # G = 3
    "g2_odd": [I8, S_, I16, D128, S_, I64, O.BOOL8, I32, S_, O.FLOAT64, I8] * 20,   # G = 2
    "g1_c3": [I32, I64, D128, S_] * 64,                                # G = 1, one 3096-B slab
    "two_slabs_dec": [D128] * 250 + [S_] * 10,
    "three_slabs_dec": [D128] * 400 + [S_] * 8,
    "two_slabs_448_cols": [S_] * 8 + [I64] * 440,
}


def _wide_id(name):
    w = P.plan_wide(WIDE[name])
    return f"{name}-{w.nslabs}slab-{P.wide_kernel_name(WIDE[name])}"


def test_wide_schemas_cover_every_g_and_slab_count():
    assert {P.plan_wide(t).G for t in WIDE.values()} == {1, 2, 3, 4}
    assert {P.plan_wide(t).nslabs for t in WIDE.values()} == {1, 2, 3}


@pytest.mark.parametrize("name", list(WIDE), ids=[_wide_id(n) for n in WIDE])
def test_wide_from_rows_every_cta_wraps(name):
    """(NS + 1) tiles per CTA + 1 row: every CTA wraps its ring and the last tile holds one row."""
    types = WIDE[name]
    w = P.plan_wide(types)
    n = (w.nstages + 1) * _sms() * w.R + 1
    _from_rows_case(types, random_table(types, n, seed=n % 991), _from_rows_kernels(types))


SLAB_PAIR_128 = [S_] * 8 + [I64] * 180 + [S_] + [I64] * 15 + [S_] + [I64] * 195
SLAB_PAIR_136 = [S_] * 8 + [I64] * 180 + [S_] + [I64] * 16 + [S_] + [I64] * 196
EDGES = {
    # each pair: the wide plan on one side, the whole-row kernel on the other
    "strings_7": [S_] * 7 + [I64] * 56,
    "strings_8": [S_] * 8 + [I64] * 56,
    "spr_511": [S_] * 8 + [I64] * 54 + [I32] + [I8] * 2,
    "spr_512": [S_] * 8 + [I64] * 54 + [I32] + [I8] * 3,
    "cols_448": [S_] * 8 + [I64] * 440,
    "cols_449": [S_] * 8 + [I64] * 441,
    "slab_pair_128_back": SLAB_PAIR_128,
    "slab_pair_136_back": SLAB_PAIR_136,
}


def test_selection_edges_are_where_the_plan_says():
    assert M.layout(EDGES["spr_511"]).size_per_row == 511 and M.layout(EDGES["spr_512"]).size_per_row == 512
    for refused, taken in (("strings_7", "strings_8"), ("spr_511", "spr_512"), ("cols_449", "cols_448"),
                           ("slab_pair_136_back", "slab_pair_128_back")):
        assert P.wide_refusal(EDGES[refused]) is not None, refused
        assert P.wide_refusal(EDGES[taken]) is None, taken
    assert P.plan_wide(SLAB_PAIR_128).nslabs == 2


def _edge_id(name):
    return f"{name}-{_from_rows_kernels(EDGES[name])[0]}"


@pytest.mark.parametrize("name", list(EDGES), ids=[_edge_id(n) for n in EDGES])
def test_wide_selection_edges(name):
    types = EDGES[name]
    n = 2 * _sms() * 32 + 65
    _from_rows_case(types, random_table(types, n, seed=len(types)), _from_rows_kernels(types))


@pytest.mark.parametrize("groups,extra", [(4095, 0), (4096, 0), (4096, 1), (2 * 4096, 1)],
                         ids=["4095_groups", "4096_groups", "4096_groups_plus_1_row", "8192_groups_plus_1_row"])
def test_wide_group_scan_chunks(groups, extra):
    """wide_group_scan_kernel takes kGsThreads x kGsPer 32-row groups per CTA: the chars before a later chunk are the
    sum over every earlier one."""
    assert P.GS_CHUNK_GROUPS == 4096
    types = WIDE["g4_520b"]
    n = groups * 32 + extra
    _from_rows_case(types, random_table(types, n, seed=groups + extra), _from_rows_kernels(types))


# ======================================================================= strings_wide_kernel
def _strings_schema(k):
    # alternate the phase-1 kernel in front of the gather: wide plan (group-local offsets) or the whole-row kernel
    return [S_] * k + [I64] * 60 if k in (8, 16, 33, 64) else [I32, I32] + [S_] * k


@pytest.mark.parametrize("k", [8, 9, 16, 17, 33, 63, 64, 65],
                         ids=lambda k: f"{k}_strings-{_strings_kernel(_strings_schema(k))}")
def test_strings_gather_wraps_its_ring(k):
    """More than 7 x SMs 32-row tiles: every CTA goes round its 2 * kSwNG-stage ring more than once."""
    types = _strings_schema(k)
    assert sum(t == S_ for t in types) == k
    assert P.strings_wide_eligible(types) == (k <= 64)
    n = (P.SW_STAGES + 1) * _sms() * 32 + 33
    _from_rows_case(types, random_table(types, n, seed=k, max_str=24), _from_rows_kernels(types))


@pytest.mark.parametrize("k", [16, 9])
def test_non_canonical_rows_in_the_second_ring_cycle(k):
    """Rows whose chars are stored out of column order (pairs updated to match) only in 32-row groups that the gather's
    CTAs reach on their second pass round the ring, and in the final partial group.  Phase 1 must flag them in its later
    tiles, or the canonical fast path would gather the wrong bytes."""
    types = _strings_schema(k)
    sms = _sms()
    n = (P.SW_STAGES + 1) * sms * 32 + 17
    lay = M.layout(types)
    sidx = [c for c, t in enumerate(types) if t == S_]
    a_col, b_col = sidx[2], sidx[3]
    rows = list(range(P.SW_STAGES * sms * 32, (P.SW_STAGES + 1) * sms * 32, 97)) + [n - 3, n - 1]

    def mutate(offs, data):
        for r in rows:
            row = data[offs[r]:offs[r + 1]]
            pa, pb = row[lay.starts[a_col]:lay.starts[a_col] + 8], row[lay.starts[b_col]:lay.starts[b_col] + 8]
            (oa, la), (ob, lb) = pa.view(np.uint32).copy(), pb.view(np.uint32).copy()
            A, B = row[oa:oa + la].copy(), row[ob:ob + lb].copy()
            row[oa:oa + lb] = B
            row[oa + lb:oa + lb + la] = A
            pb.view(np.uint32)[:] = (oa, lb)
            pa.view(np.uint32)[:] = (oa + lb, la)

    cols = random_table(types, n, seed=k + 100, null_frac=0.0, max_str=24)
    la, lb = (np.diff(cols[c].offsets.astype(np.int64)) for c in (a_col, b_col))
    rows = [r for r in rows if la[r] > 0 and lb[r] > 0]      # a swap of two non-empty strings breaks the column order
    assert len(rows) > 10 and rows[-1] >= n - 3
    status = _from_rows_case(types, cols, _from_rows_kernels(types), mutate=mutate)
    assert status == M.STATUS_NON_CANONICAL


# ======================================================================= to_rows
def _to_rows_case(cols, kernels):
    G = _gpu()
    import srj_b200 as S
    want = M.to_rows(cols)
    dev = G.table_to_device(cols)

    def check(out):
        assert len(out) == len(want)
        for o, (offs, data) in zip(out, want):
            goffs, gdata = G.rows_to_host(o)
            assert np.array_equal(goffs, offs), f"offsets: first diff {np.flatnonzero(goffs != offs)[:4]}"
            assert np.array_equal(gdata, data), f"first diff at byte {np.flatnonzero(gdata != data)[:5]} of {len(data)}"
    _run_checked(lambda: S.RowConversion.convertToRows(dev), check, kernels)


@pytest.mark.parametrize("name", ["c2_two_stages", "c1_three_stages"])
def test_to_rows2_second_pass_and_generic_tail(name):
    """kT2Super tiles on every CTA, one more tile (the round-robin's second pass) and R + 1 rows: the last full tile is
    a second pass, the one row behind it goes to the generic kernel."""
    types = FIXED[name]
    R = P.to_rows2_R(types)
    assert R >= 128
    n = P.T2_SUPER * R * _sms() + R + 1
    _to_rows_case(random_table(types, n, seed=R + 5), ["to_rows2_kernel", "to_rows_kernel"])


def test_to_rows_w_second_pass():
    """More than 2 x kTwWarps x 32 x SMs rows: every to_rows_w_kernel warp takes a third 32-row group."""
    types = VAR["mixed"]
    n = 2 * P.TW_WARPS * 32 * _sms() + 33
    cols = random_table(types, n, seed=8)
    assert P.to_rows_var_kernel(types, int(M.row_sizes(cols).sum()), n) == "to_rows_w_kernel"
    _to_rows_case(cols, ["to_rows_w_kernel"])


def test_to_rows3_three_super_tiles_per_cta():
    types = WIDE["g1_c3"]
    cols = random_table(types, 64, seed=1, max_str=25)
    nbytes = int(M.row_sizes(cols).sum())
    sup = P.to_rows3_super_rows(types, nbytes, 64)
    assert sup >= 16
    n = 3 * _sms() * sup + 7
    cols = random_table(types, n, seed=2, max_str=25)
    assert P.to_rows_var_kernel(types, int(M.row_sizes(cols).sum()), n) == "to_rows3_kernel"
    _to_rows_case(cols, ["to_rows3_kernel"])


@pytest.mark.parametrize("n", [P.RS_CHUNK - 1, P.RS_CHUNK, P.RS_CHUNK + 1, 2 * P.RS_CHUNK + 1, 7 * P.RS_CHUNK - 1])
def test_row_size_scan_across_chunks(n):
    """The row sizes are scanned in chunks of kRsChunk rows: the LIST offsets after a chunk carry every earlier one."""
    types = [I32, S_, I64, S_, I8]
    _to_rows_case(random_table(types, n, seed=n, max_str=40), ["to_rows_w_kernel"])


# ======================================================================= one whole C3 batch
def test_wide_c3_batch_of_500k_rows():
    """One full C3 batch (15,625 groups, 4 scan chunks), compared whole.  Not profiled, and last in this file: the
    kernels of this schema are attested by the g1_c3 case of test_wide_from_rows_every_cta_wraps, and after this
    multi-gigabyte call torch.profiler was seen to miss kernel records of later windows in the same process."""
    types = WIDE["g1_c3"]
    n = 500_000
    assert (n + 31) // 32 > 3 * P.GS_CHUNK_GROUPS
    _from_rows_case(types, random_table(types, n, seed=3), None)
