"""Pins the independent UnsafeRow model (unsafe_row_model.py) on the CPU: byte for byte against the per-row restatement
oracle/unsafe_row.py in both directions, on rows in a layout the encoder never writes, against hand-derived known
answers, and guards the launch constants the model restates from csrc/unsafe_row.cu."""
import os
import re
import time

import numpy as np
import pytest

import unsafe_row_model as M
from oracle import oracle as O
from oracle import unsafe_row as U
from test_gpu_unsafe_row import SCHEMAS as GPU_SCHEMAS
from util import col_from_values, random_table

# every type csrc/unsafe_row.cu's ur_classify accepts
ALL_TYPES = [O.INT8, O.UINT8, O.BOOL8, O.INT16, O.UINT16, O.INT32, O.UINT32, O.FLOAT32, O.TIMESTAMP_DAYS, O.DECIMAL32,
             O.INT64, O.UINT64, O.FLOAT64, O.TIMESTAMP_SECONDS, O.TIMESTAMP_MILLISECONDS, O.TIMESTAMP_MICROSECONDS,
             O.TIMESTAMP_NANOSECONDS, O.DECIMAL64, O.DECIMAL128, O.STRING]
SCHEMAS = {**GPU_SCHEMAS, "every_type": ALL_TYPES}


def test_type_ids_and_widths_agree_with_the_oracle():
    assert set(ALL_TYPES) == M.SUPPORTED
    for t in M.FIXED_WIDTH:
        assert M.FIXED_WIDTH[t] == O.size_of(t), t
    assert (M.STRING, M.DECIMAL128, M.LIST, M.STRUCT, M.DURATION_DAYS) == (O.STRING, O.DECIMAL128, O.LIST, O.STRUCT,
                                                                         O.DURATION_DAYS)


def _assert_model_matches_oracle(types, cols):
    offs, data = U.to_unsafe_rows(cols)
    mo, md = M.to_rows(cols)
    assert np.array_equal(mo, offs), f"offsets: first diff {np.flatnonzero(mo != offs)[:4]}"
    assert np.array_equal(md, data), f"row bytes: first diff {np.flatnonzero(md != data)[:4]}"
    want = U.from_unsafe_rows(data, offs, types)
    got = M.from_rows(data, offs, types)
    for f, (t, w) in enumerate(zip(types, want)):
        assert np.array_equal(got.masks[f], O.pack_mask(w.valid())), f"mask, field {f}"
        assert got.null_counts[f] == w.null_count(), f"null count, field {f}"
        assert np.array_equal(got.data[f], np.ascontiguousarray(w.data).view(np.uint8)), f"bytes, field {f}"
        if t == O.STRING:
            assert np.array_equal(got.offsets[f], w.offsets), f"string offsets, field {f}"


@pytest.mark.parametrize("null_frac", [0.0, 0.2, 1.0], ids=["no_nulls", "nulls_20", "all_null"])
@pytest.mark.parametrize("nrows", [0, 1, 31, 32, 33, 1000])
@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_model_matches_oracle(name, nrows, null_frac):
    types = SCHEMAS[name]
    _assert_model_matches_oracle(types, random_table(types, nrows, seed=nrows * 7 + len(types), null_frac=null_frac))


def test_permuted_rows_decode_to_the_columns():
    types = SCHEMAS["every_type"] + [O.STRING, O.DECIMAL128] * 3
    n = 300
    cols = random_table(types, n, seed=5)
    offs, data = M.to_rows(cols)
    poffs, pdata = M.to_rows_permuted(cols)
    lay = M.layout(types)
    nvar = lay.ndec + lay.nstr
    assert np.array_equal(np.diff(poffs), np.diff(offs) + 8 * nvar)
    assert not np.array_equal(pdata[:len(data)], data)
    want = M.from_rows(data, offs, types)
    got = M.from_rows(pdata, poffs, types)
    oracle = U.from_unsafe_rows(pdata, poffs, types)              # the oracle's reader follows the slots too
    for f, t in enumerate(types):
        assert np.array_equal(got.masks[f], want.masks[f]) and np.array_equal(got.data[f], want.data[f]), f
        assert np.array_equal(np.ascontiguousarray(oracle[f].data).view(np.uint8), want.data[f]), f
        if t == O.STRING:
            assert np.array_equal(got.offsets[f], want.offsets[f]) and np.array_equal(oracle[f].offsets, want.offsets[f])


def test_permuted_layout_by_hand():
    """(STRING "ab", DECIMAL128 1): entries in reverse field order, each behind 8 zero bytes."""
    cols = [col_from_values("STRING", [b"ab"]), col_from_values("DECIMAL128", [1])]
    offs, data = M.to_rows_permuted(cols)
    # bitset | slot 0 | slot 1 | gap | decimal (16) | gap | "ab" + 6
    assert offs.tolist() == [0, 24 + 8 + 16 + 8 + 8]
    assert data[8:16].view(np.uint64)[0] == (56 << 32) | 2 and data[16:24].view(np.uint64)[0] == (32 << 32) | 1
    assert not data[24:32].any() and data[32] == 1 and not data[33:56].any() and data[56:58].tobytes() == b"ab"


def test_model_speed_on_the_256_column_schema():
    """The GPU tests check large tables through the model in chunks of rows: 32 K rows of the 256-field mixed schema
    take about a second each way on one CPU core.  A per-row loop would take minutes."""
    types = [O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 64
    cols = random_table(types, 32 * 1024, seed=1)
    t0 = time.perf_counter()
    offs, data = M.to_rows(cols)
    t1 = time.perf_counter()
    M.from_rows(data, offs, types)
    t2 = time.perf_counter()
    assert t1 - t0 < 3.0 and t2 - t1 < 3.0, f"model of 32 K rows x 256 fields: to_rows {t1 - t0:.2f} s, from_rows {t2 - t1:.2f} s"


# ---------------------------------------------------------------------------------------------- known answers
def _dec_col(vals, valid=None):
    raw = b"".join(int(v).to_bytes(16, "little", signed=True) for v in vals)
    mask = None if valid is None else O.pack_mask(np.array(valid, bool))
    return O.HCol(O.DECIMAL128, np.frombuffer(raw, np.uint8).copy(), mask, None, 0, len(vals))


def _dec_cases():
    """(value, toByteArray length) on both sides of each length boundary: a k-byte two's complement holds
    [-2^(8k-1), 2^(8k-1) - 1]."""
    out = [(0, 1)]
    for k in range(1, 17):
        top = 2 ** (8 * k - 1)
        out += [(top - 1, k), (-top, k), (-(top - 1), k)]
        if k < 16:
            out += [(top, k + 1), (-top - 1, k + 1)]
    return out


def test_decimal128_every_byte_array_length():
    cases = _dec_cases()
    assert {L for _, L in cases} == set(range(1, 17))
    col = _dec_col([v for v, _ in cases])
    offs, data = M.to_rows([col])
    assert np.array_equal(offs, np.arange(len(cases) + 1) * 32)      # bitset, slot, 16 reserved bytes
    for r, (v, L) in enumerate(cases):
        row = data[offs[r]:offs[r + 1]]
        assert row[:8].tobytes() == bytes(8)
        assert row[8:16].view(np.uint64)[0] == (16 << 32) | L, (v, L)
        assert row[16:16 + L].tobytes() == v.to_bytes(L, "big", signed=True) and not row[16 + L:].any(), v
    assert [data[offs[r] + 16:offs[r] + 16 + L].tobytes() for r, (v, L) in enumerate(cases[:6])] == \
        [b"\x00", b"\x7f", b"\x80", b"\x81", b"\x00\x80", b"\xff\x7f"]        # 0, 127, -128, -127, 128, -129
    back = M.from_rows(data, offs, [O.DECIMAL128])
    assert back.data[0].tobytes() == col.data.tobytes()
    _assert_model_matches_oracle([O.DECIMAL128], [col])


def _slot(t, v):
    (offs, data) = M.to_rows([col_from_values(t, [v])])
    return data[8:16].tobytes()


def test_fixed_width_slots_keep_zero_upper_bytes():
    assert _slot("TIMESTAMP_DAYS", -1) == b"\xff\xff\xff\xff" + bytes(4)
    assert _slot("TIMESTAMP_DAYS", -719162) == (-719162 & 0xFFFFFFFF).to_bytes(8, "little")
    assert _slot("UINT32", 2**31) == b"\x00\x00\x00\x80" + bytes(4)
    assert _slot("UINT32", 2**32 - 1) == b"\xff" * 4 + bytes(4)
    assert _slot("UINT16", 2**15) == b"\x00\x80" + bytes(6)
    assert _slot("UINT8", 255) == b"\xff" + bytes(7)
    assert _slot("INT32", -4) == b"\xfc\xff\xff\xff" + bytes(4)
    assert _slot("DECIMAL32", -1) == b"\xff" * 8                       # a decimal of precision <= 18 is a long
    assert _slot("DECIMAL32", -2**31) == (-2**31).to_bytes(8, "little", signed=True)
    assert _slot("UINT64", 2**64 - 1) == b"\xff" * 8
    assert _slot("TIMESTAMP_NANOSECONDS", -1) == b"\xff" * 8


def test_float_payloads_are_copied_bit_for_bit():
    assert _slot("FLOAT32", ("bits32", 0x7FC00001)) == b"\x01\x00\xc0\x7f" + bytes(4)
    assert _slot("FLOAT64", ("bits64", 0xFFF8000000000001)) == (0xFFF8000000000001).to_bytes(8, "little")
    assert _slot("FLOAT32", -0.0) == b"\x00\x00\x00\x80" + bytes(4)
    assert _slot("FLOAT64", -0.0) == bytes(7) + b"\x80"
    assert _slot("FLOAT32", ("bits32", 1)) == b"\x01" + bytes(7)           # smallest denormal
    assert _slot("FLOAT64", ("bits64", 1)) == b"\x01" + bytes(7)
    for t, bits in (("FLOAT32", 0x7FC00001), ("FLOAT64", 0xFFF8000000000001), ("FLOAT32", 1)):
        col = col_from_values(t, [("bits32" if t == "FLOAT32" else "bits64", bits)])
        offs, data = M.to_rows([col])
        assert M.from_rows(data, offs, [col.type_id]).data[0].tobytes() == col.data.tobytes()


@pytest.mark.parametrize("fields", [63, 64, 65, 128, 129, 256])
def test_bitset_words(fields):
    nulls = {0, fields - 1} | ({64} if fields > 64 else set())
    cols = [col_from_values("INT8", [None if f in nulls else f % 127 + 1]) for f in range(fields)]
    offs, data = M.to_rows(cols)
    words = (fields + 63) // 64
    assert offs.tolist() == [0, 8 * words + 8 * fields]
    want = [0] * words
    for f in nulls:
        want[f // 64] |= 1 << (f % 64)
    assert data[:8 * words].view(np.uint64).tolist() == want
    slots = data[8 * words:].view(np.uint64)
    assert all(slots[f] == (0 if f in nulls else f % 127 + 1) for f in range(fields))
    back = M.from_rows(data, offs, [O.INT8] * fields)
    assert [int(k) for k in back.null_counts] == [int(f in nulls) for f in range(fields)]
    _assert_model_matches_oracle([O.INT8] * fields, cols)


def test_empty_string_against_null_string():
    cols = [col_from_values("STRING", [b""]), col_from_values("STRING", [None]), col_from_values("STRING", [b"q"])]
    offs, data = M.to_rows(cols)
    w = data.view(np.uint64)
    assert offs.tolist() == [0, 40] and w[0] == 0b010
    assert w[1] == (32 << 32) | 0 and w[2] == 0 and w[3] == (32 << 32) | 1
    assert data[32:40].tobytes() == b"q" + bytes(7)
    back = M.from_rows(data, offs, [O.STRING] * 3)
    assert back.null_counts.tolist() == [0, 1, 0] and [o.tolist() for o in back.offsets] == [[0, 0], [0, 0], [0, 1]]
    _assert_model_matches_oracle([O.STRING] * 3, cols)


def test_layout_refusals():
    assert M.layout([O.INT64] * 256).fixed_bytes == 32 + 2048
    for bad in ([], [O.INT64] * 257, [O.DURATION_DAYS], [O.LIST], [O.STRUCT], [O.INT32, O.DICTIONARY32]):
        with pytest.raises(M.UnsupportedSchema):
            M.layout(bad)


# ---------------------------------------------------------------------------------------------- launch rules
def test_plans_of_the_offset_less_edges():
    """47 INT64 fields: 384-byte rows, a whole warp fits the 12 KB stage.  48: 392 bytes, full warps go in place and
    only a partial last warp of at most 31 rows is staged.  The same edge through 16 * ndec."""
    for types, row, full_staged in (([O.INT64] * 47, 384, True), ([O.INT64] * 48, 392, False),
                                    ([O.INT64] * 32 + [O.DECIMAL128] * 5, 384, True),
                                    ([O.INT64] * 30 + [O.DECIMAL128] * 6, 392, False)):
        assert M.layout(types).row_base == row
        p = M.plan(types, 3 * 256 + 31, 132)
        assert p.stage == min(12288, 32 * row)
        assert len(p.staged) == 25 and p.staged[:-1].tolist() == [full_staged] * 24 and p.staged[-1]
    p = M.plan([O.INT64] * 256, 3 * 256 + 5, 132)
    assert p.stage == 12288 and not p.staged[:-1].any() and p.staged[-1]
    assert not M.plan([O.INT64] * 256, 3 * 256 + 6, 132).staged[-1]


def test_plan_grids():
    p = M.plan([O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 64, 1_081_361, 132, np.zeros(1_081_362, np.int64))
    assert (p.rows_grid, p.rows_per_sweep, p.rows_sweeps) == (1056, 270_336, 5)
    assert (p.chars_grid, p.chars_per_sweep, p.chars_sweeps) == (2112, 540_672, 3)
    assert p.smem == 8 * 12288 + 256 * 44 + 16
    p = M.plan([O.INT8], 1, 132)
    assert (p.rows_grid, p.chars_grid, p.rows_sweeps, p.stage) == (1, 1, 1, 32 * 16)


_SRC = os.path.join(os.path.dirname(__file__), "..", "spark-rapids-jni_b200", "csrc", "unsafe_row.cu")


def _const(src, name):
    m = re.search(r"constexpr\s+int\s+" + name + r"\s*=\s*([^;/]+);", src)
    assert m, f"{name} not found"
    return m.group(1).strip()


def test_launch_constants_match_the_source():
    """The GPU edge tests size their tables from plan().  If the codec is retuned, they would silently stop reaching
    the stage and sweep edges they were written for: fail here instead."""
    src = open(_SRC).read()
    assert _const(src, "kUrStage") == "12 * 1024" and M.STAGE == 12 * 1024
    assert int(_const(src, "kUrBatch")) == M.BATCH and int(_const(src, "kUrMaxCols")) == M.MAX_FIELDS
    assert src.count("__launch_bounds__(256)") == 4 and M.THREADS == 256
    # ur_grid: one CTA per 256 rows, at most 8 per SM; the chars gather: at most 16 per SM
    assert "std::min<int64_t>((n + 255) / 256, int64_t{sm_count()} * 8)" in src and M.ROWS_GRID_PER_SM == 8
    assert "std::min<int64_t>((n + 255) / 256, int64_t{sm_count()} * 16)" in src and M.CHARS_GRID_PER_SM == 16
    # the grid-stride steps of the three kernels
    assert src.count("blk * 256 < n; blk += gridDim.x") == 2
    assert "d0 = (static_cast<int64_t>(blockIdx.x) * 8 + warp_id()) * 32; d0 < n; d0 += static_cast<int64_t>(gridDim.x) * 256" in src
    # the stage: kUrStage with row offsets, else 32 rows rounded to 16 bytes; a warp is staged when its rows fit
    assert "if (d_row_offsets) return kUrStage;" in src
    assert "return std::min(kUrStage, (32 * fixed_row_bytes + 15) & ~15);" in src
    assert src.count("staged   = b1 - b0 <= stage;") == 1 and src.count("staged = b1 - b0 <= stage;") == 1
    assert src.count("ur_stage(d_row_offsets, t.fixed_bytes + 16 * t.ndec)") == 2
    assert src.count("8 * static_cast<size_t>(stage) + static_cast<size_t>(ncols) * (sizeof(UrCol) + 4) + 16") == 2
    assert re.search(r"struct UrCol \{\s*const uint8_t\* data;[^}]*const uint32_t\* mask;[^}]*const int32_t\* offsets;"
                     r"[^}]*int32_t kind;[^}]*int32_t width;[^}]*int32_t sext;[^}]*int32_t pad;\s*\};", src)
    assert M.DESC_BYTES == 3 * 8 + 4 * 4
