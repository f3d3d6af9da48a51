"""GPU parity tests of the variable-width to_rows kernels (csrc/to_rows_var.cu) against the CPU oracle, through the
C ABI.  The launcher picks to_rows3_kernel when the average row is between about stage/64 and stage/8 bytes (a few KB:
the C3 shape) and to_rows_w_kernel for narrow rows.  So that every string schema of tests/row_conversion.cpp
(SimpleString, DoubleString, ManyStrings, BigStrings) reaches to_rows3_kernel, those tests append a block of 256
DECIMAL128 columns (4 KB per row) to it.  Each test checks through torch.profiler that the kernel it names ran.
Bit-exact: every row byte incl. the zero padding, and the LIST offsets."""
import re
import warnings

import numpy as np
import pytest

from oracle import oracle as O
from util import random_table

pytestmark = pytest.mark.gpu

WIDE = [O.DECIMAL128] * 256   # 4 KB of fixed-width fields: moves a narrow string schema to to_rows3_kernel


def _gpu():
    import gpu_util
    gpu_util.require_cuda()
    return gpu_util


def _ran(names, kernel):
    return any(re.search(r"\b" + kernel + r"\b", n) for n in names)


def _profiled(fn):
    """fn()'s result and the names of the events torch.profiler recorded with CUDA activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.name for e in prof.events()}


def _check_rows(G, out, batches):
    assert len(out) == len(batches)
    for o, (offs, data) in zip(out, batches):
        goffs, gdata = G.rows_to_host(o)
        assert np.array_equal(goffs, offs)
        assert np.array_equal(gdata, data), f"first diff at byte {np.flatnonzero(gdata != data)[:5]}"


def _check(cols, kernels=()):
    """Rows of `cols` on the device == the oracle's, and each of `kernels` ran during the conversion.

    torch.profiler does not always deliver every kernel record of a short window (a run can come back with the
    runtime calls but without some or all of its kernels).  The launcher's choice depends only on the schema and
    the sizes, so every run of the same call launches the same kernels: the call is profiled again, up to five
    times, until each named kernel has been seen, and every run's rows are compared with the oracle."""
    G = _gpu()
    import srj_b200 as S
    batches = O.convert_to_rows(cols)
    dev = G.table_to_device(cols)
    seen = set()
    for attempt in range(5):
        out, names = _profiled(lambda: S.RowConversion.convertToRows(dev))
        _check_rows(G, out, batches)
        seen |= names
        missing = [k for k in kernels if not _ran(seen, k)]
        if not missing:
            break
        if attempt < 4:
            warnings.warn(f"profiler run {attempt + 1} recorded no {missing}; profiling the same call again")
    assert not missing, f"{missing} did not run in 5 profiled runs; recorded: {sorted(seen)}"


SCHEMAS = {
    "simple_string": [O.STRING],
    "double_string": [O.INT32, O.STRING, O.STRING],
    "mixed": [O.INT32, O.STRING, O.INT64, O.DECIMAL128, O.STRING, O.BOOL8, O.STRING, O.INT16, O.INT8],
    "c3_small": [O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 8,
    "many_strings": [O.STRING] * 50,
    "strings_200": [O.STRING] * 200 + [O.INT16],          # more than 48 blocks of 4 -> wider blocks
    "all_widths": [O.INT8, O.STRING, O.INT16, O.INT32, O.STRING, O.INT64, O.DECIMAL128, O.FLOAT32, O.BOOL8] * 5,
}


@pytest.mark.parametrize("nrows", [1, 7, 8, 33, 1000, 20_011])
@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_forced_var_kernel_matches_oracle(name, nrows):
    types = SCHEMAS[name]
    if len(types) * nrows > 1_500_000:
        nrows = 1_500_000 // len(types)
    _check(random_table(types + WIDE, nrows, seed=nrows + 101), kernels=["to_rows3_kernel"])


@pytest.mark.parametrize("max_str", [0, 3, 33, 40, 200])
def test_string_lengths_around_the_word_path_limit(max_str):
    """<= 32 bytes: register word path; longer: warp-cooperative copy; 0: all-empty strings."""
    types = [O.INT64, O.STRING, O.STRING, O.INT32, O.STRING] + WIDE
    _check(random_table(types, 5000, seed=max_str + 5, max_str=max_str), kernels=["to_rows3_kernel"])


@pytest.mark.parametrize("nrows", [24, 4099, 30_000])
def test_c3_shape_picks_the_var_kernel(nrows):
    """256 columns, ~3.9 KB rows (the C3 config) -> to_rows3_kernel by the launcher's own rule."""
    types = [O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 64
    _check(random_table(types, nrows, seed=nrows, max_str=25), kernels=["to_rows3_kernel"])


def test_no_null_masks_and_unaligned_tail():
    types = [O.INT32, O.STRING, O.INT64, O.STRING] + WIDE
    _check(random_table(types, 3001, seed=9, null_frac=0.0), kernels=["to_rows3_kernel"])


def test_rows_larger_than_the_stage_fall_back():
    """A row that cannot fit the image buffer raises the flag; the generic kernel behind redoes the batch.
    to_rows_kernel is launched behind every to_rows3_kernel and returns at once unless the flag is up, so seeing it
    only shows the launch; the rows matching the oracle, the 300 KB row included, show that it redid the batch."""
    rng = np.random.default_rng(4)
    big = [bytes(rng.integers(32, 127, n, dtype=np.uint8)) for n in (0, 1, 300_000, 5, 0, 70_000, 3)]
    vals = big + [b"", None, b"x"] * 10
    c0 = O.strings_col(vals)
    c1 = O.HCol(O.INT64, rng.integers(0, 2**62, len(vals)).astype(np.int64).view(np.uint8), None, None, 0, len(vals))
    c2 = O.strings_col([b"tail%d" % i for i in range(len(vals))])
    _check([c0, c1, c2], kernels=["to_rows3_kernel", "to_rows_kernel"])


def test_medium_rows_use_partial_tiles():
    """~12 KB rows: 8 rows per tile, super-tiles with remainders."""
    rng = np.random.default_rng(21)
    n = 777
    cols = []
    for c in range(4):
        vals = [bytes(rng.integers(32, 127, int(rng.integers(0, 6000)), dtype=np.uint8)) if rng.random() > 0.1 else None
                for _ in range(n)]
        cols.append(O.strings_col(vals))
    cols.append(O.HCol(O.INT64, rng.integers(0, 2**62, n).astype(np.int64).view(np.uint8), None, None, 0, n))
    _check(cols, kernels=["to_rows3_kernel"])


# ---- narrow rows: the warp-private kernel (to_rows_w_kernel) is picked by the launcher's own rule -------------------
@pytest.mark.parametrize("nrows", [1, 31, 32, 33, 1000, 50_003])
@pytest.mark.parametrize("name", ["simple_string", "double_string", "mixed", "c3_small", "all_widths"])
def test_narrow_rows_pick_the_warp_kernel(name, nrows):
    _check(random_table(SCHEMAS[name], nrows, seed=nrows + 7), kernels=["to_rows_w_kernel"])


def test_narrow_rows_without_masks_and_long_strings():
    types = [O.INT32, O.STRING, O.INT64, O.STRING, O.INT8]
    _check(random_table(types, 4001, seed=3, null_frac=0.0), kernels=["to_rows_w_kernel"])
    _check(random_table(types, 4001, seed=4, max_str=200), kernels=["to_rows_w_kernel"])     # > 32 bytes: warp-cooperative copy


def test_narrow_table_with_one_huge_row_falls_back():
    """Average row is small (warp kernel chosen) but one row exceeds a warp's buffer: flag -> generic kernel.
    As above, to_rows_kernel is launched whether or not the flag is raised; the rows matching the oracle, the
    40 KB row included, show that it redid the batch."""
    rng = np.random.default_rng(8)
    n = 3000
    vals = [bytes(rng.integers(32, 127, int(rng.integers(0, 20)), dtype=np.uint8)) for _ in range(n)]
    vals[1777] = bytes(rng.integers(32, 127, 40_000, dtype=np.uint8))
    c0 = O.strings_col(vals)
    c1 = O.HCol(O.INT64, rng.integers(0, 2**62, n).astype(np.int64).view(np.uint8), None, None, 0, n)
    _check([c1, c0], kernels=["to_rows_w_kernel", "to_rows_kernel"])
