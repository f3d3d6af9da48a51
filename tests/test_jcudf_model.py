"""Pins the independent JCUDF model (jcudf_model.py) on the CPU: byte for byte against the C oracle on random tables of
every row-conversion schema the GPU tests use and on the edge-value tables of hash_edges.py, against hand-derived rows,
and guards the planning constants row_plans.py restates from csrc/."""
import os
import re

import numpy as np
import pytest

import hash_edges as E
import jcudf_model as M
import row_plans as P
from oracle import oracle as O
from test_gpu_rows import FIXED_SCHEMAS, STRING_SCHEMAS
from test_gpu_to_rows_var import SCHEMAS as VAR_SCHEMAS
from test_gpu_wide import WIDE_TO_ROWS
from util import col_from_values, random_table

SCHEMAS = {**{f"rows.{k}": v for k, v in {**FIXED_SCHEMAS, **STRING_SCHEMAS}.items()},
           **{f"wide.{k}": v for k, v in WIDE_TO_ROWS.items()},
           **{f"to_rows_var.{k}": v for k, v in VAR_SCHEMAS.items()}}


def _assert_same(types, cols):
    n = cols[0].size
    want = O.convert_to_rows(cols)
    got = M.to_rows(cols)
    assert len(got) == len(want)
    for (go, gd), (wo, wd) in zip(got, want):
        assert np.array_equal(go, wo), f"offsets: first diff {np.flatnonzero(go != wo)[:4]}"
        assert np.array_equal(gd, wd), f"row bytes: first diff {np.flatnonzero(gd != wd)[:4]}"
    offs, data = want[0]
    var = any(t == O.STRING for t in types)
    ocols, onulls = O.convert_from_rows(data, offs if var else None, n, types)
    m = M.from_rows(data, offs if var else None, n, types)
    assert np.array_equal(m.null_counts, onulls)
    assert m.status == 0
    for i, (t, oc) in enumerate(zip(types, ocols)):
        assert np.array_equal(m.masks[i], oc.mask[: (n + 31) // 32]), f"mask, column {i}"
        assert np.array_equal(m.data[i], np.ascontiguousarray(oc.data).view(np.uint8)), f"column {i}"
        if t == O.STRING:
            assert np.array_equal(m.offsets[i], oc.offsets), f"offsets, column {i}"
            assert m.char_totals[i] == len(oc.data)
        else:
            assert m.char_totals[i] == 0


@pytest.mark.parametrize("nrows", [0, 1, 31, 32, 33, 5003])
@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_model_matches_oracle(name, nrows):
    types = SCHEMAS[name]
    _assert_same(types, random_table(types, nrows, seed=nrows * 11 + len(types)))


@pytest.mark.parametrize("t", list(E.EDGES), ids=[str(t) for t in E.EDGES])
def test_model_matches_oracle_on_edge_values(t):
    """Edge values of each type, next to a STRING and a 1-byte field (so the field lands at every alignment), with no
    mask, some nulls and all nulls; null strings keep their edge lengths."""
    types = [t, O.INT8, t, O.STRING, O.INT16, t]
    cols = E.edge_cols(types, 2 * len(E.EDGES[t]) + 37, nulls=[None, 0.3, "all", 0.5, None, 0.2], seed=t)
    _assert_same(types, cols)


def test_model_matches_oracle_on_non_canonical_rows():
    types = [O.INT32, O.STRING, O.INT64, O.STRING]
    n = 300
    (offs, data), = O.convert_to_rows(random_table(types, n, seed=21, null_frac=0.0))
    lay = M.layout(types)
    for r in range(0, n, 3):            # column 3's chars first, then column 1's: pairs updated
        row = data[offs[r]:offs[r + 1]]
        p1, p3 = row[lay.starts[1]:lay.starts[1] + 8].view(np.uint32), row[lay.starts[3]:lay.starts[3] + 8].view(np.uint32)
        (o1, l1), (o3, l3) = p1.copy(), p3.copy()
        a, b = row[o1:o1 + l1].copy(), row[o3:o3 + l3].copy()
        row[o1:o1 + l3] = b
        row[o1 + l3:o1 + l3 + l1] = a
        p3[:] = (o1, l3)
        p1[:] = (o1 + l3, l1)
    m = M.from_rows(data, offs, n, types)
    ocols, _ = O.convert_from_rows(data, offs, n, types)
    assert m.status == M.STATUS_NON_CANONICAL
    for c in (1, 3):
        assert np.array_equal(m.offsets[c], ocols[c].offsets) and np.array_equal(m.data[c], ocols[c].data)


# ---------------------------------------------------------------------------------------------- known answers
def test_javadoc_example_and_config_layouts():
    lay = M.layout([O.BOOL8, O.INT16, O.DURATION_DAYS])                   # RowConversion.java:77-85
    assert lay.starts == [0, 2, 4] and lay.validity_offset == 8 and lay.size_per_row == 9 and lay.fixed_row_size == 16
    lay = M.layout([O.DURATION_DAYS, O.INT16, O.BOOL8])                   # RowConversion.java:99-103
    assert lay.starts == [0, 4, 6] and lay.size_per_row == 8 and lay.fixed_row_size == 8
    cols = [col_from_values("BOOL8", [1, 0]), col_from_values("INT16", [0x1234, None]),
            O.HCol(O.DURATION_DAYS, np.array([0x0A0B0C0D, 7], np.int32).view(np.uint8), None, None, 0, 2)]
    (offs, data), = M.to_rows(cols)
    assert offs.tolist() == [0, 16, 32]
    assert data[:16].tolist() == [1, 0, 0x34, 0x12, 0x0D, 0x0C, 0x0B, 0x0A, 0b111, 0, 0, 0, 0, 0, 0, 0]
    assert data[24] == 0b101
    assert M.layout([O.INT32, O.INT64, O.FLOAT64, O.BOOL8]).size_per_row == 26                              # C1
    lay = M.layout([O.INT32, O.INT64, O.DECIMAL128, O.STRING] * 64)                                          # C3
    assert lay.starts[:8] == [0, 8, 16, 32, 40, 48, 64, 80] and (lay.validity_offset, lay.size_per_row) == (3064, 3096)
    lay = M.layout([O.INT32] * 9 + [O.INT64, O.INT32] + [O.DECIMAL32] * 12)                                  # C4
    assert lay.starts[:12] == [0, 4, 8, 12, 16, 20, 24, 28, 32, 40, 48, 52] and lay.size_per_row == 103


def test_pivot_like_layout():
    """tests/row_conversion.cpp:457-498: 191 x INT64 + INT32; the int at byte 1528, rows 1560 bytes apart."""
    n = 100
    ints = (0x11223344 + np.arange(n)).astype(np.int32)
    cols = [O.HCol(O.INT64, np.zeros(n, np.int64).view(np.uint8), None, None, 0, n) for _ in range(191)]
    cols.append(O.HCol(O.INT32, ints.view(np.uint8), None, None, 0, n))
    (offs, data), = M.to_rows(cols)
    assert np.array_equal(offs, np.arange(n + 1) * 1560)
    assert np.array_equal(data.reshape(n, 1560)[:, 1528:1532].copy().view(np.int32).ravel(), ints)


def _both(cols):
    """The rows by the model, checked equal to the oracle's, and read back by the model."""
    (offs, data), = M.to_rows(cols)
    (o2, d2), = O.convert_to_rows(cols)
    assert np.array_equal(offs, o2) and np.array_equal(data, d2)
    return offs, data


def test_decimal128_after_int8_is_16_byte_aligned():
    cols = [col_from_values("INT8", [0x7F, -1]), col_from_values("DECIMAL128", [1, None])]
    offs, data = _both(cols)
    assert M.layout([O.INT8, O.DECIMAL128]).starts == [0, 16]
    row0 = [0x7F] + [0] * 15 + [1] + [0] * 15 + [0b11] + [0] * 7
    row1 = [0xFF] + [0] * 15 + [0] * 16 + [0b01] + [0] * 7          # null DECIMAL128: payload (zeros) copied
    assert offs.tolist() == [0, 40, 80] and data.tolist() == row0 + row1


def test_string_pairs_after_1_and_2_byte_fields():
    cols = [col_from_values("INT8", [5]), col_from_values("STRING", [b"ab"]), col_from_values("INT16", [0x0102]),
            col_from_values("STRING", [b"xyz"])]
    offs, data = _both(cols)
    # INT8 @0, pair @4 (4-aligned), INT16 @12, pair @16, validity @24, size_per_row 25; chars from 25, row ends at 30
    assert data.tolist() == [5, 0, 0, 0, 25, 0, 0, 0, 2, 0, 0, 0, 2, 1, 0, 0, 27, 0, 0, 0, 3, 0, 0, 0, 0x0F,
                             ord("a"), ord("b"), ord("x"), ord("y"), ord("z"), 0, 0]
    assert offs.tolist() == [0, 32]
    m = M.from_rows(data, offs, 1, [c.type_id for c in cols])
    assert bytes(m.data[1]) == b"ab" and bytes(m.data[3]) == b"xyz" and m.offsets[3].tolist() == [0, 3]


@pytest.mark.parametrize("ncols,null_col,want", [
    (8, 7, [0x7F]), (9, 8, [0xFF, 0x00]), (9, 0, [0xFE, 0x01]),
    (64, 63, [0xFF] * 7 + [0x7F]), (65, 64, [0xFF] * 8 + [0x00]), (65, 9, [0xFF, 0xFD] + [0xFF] * 6 + [0x01])])
def test_validity_bytes(ncols, null_col, want):
    cols = [col_from_values("INT8", [c]) if c != null_col else col_from_values("INT8", [None]) for c in range(ncols)]
    offs, data = _both(cols)
    vbytes = (ncols + 7) // 8
    assert data[ncols:ncols + vbytes].tolist() == want
    assert len(data) == (ncols + vbytes + 7) // 8 * 8 and not data[ncols + vbytes:].any()
    m = M.from_rows(data, None, 1, [O.INT8] * ncols)
    assert m.null_counts.tolist() == [int(c == null_col) for c in range(ncols)]


def test_empty_and_null_strings():
    cols = [col_from_values("STRING", [b""]), col_from_values("STRING", [None]), col_from_values("STRING", [b"q"])]
    offs, data = _both(cols)
    assert data.tolist() == [25, 0, 0, 0, 0, 0, 0, 0, 25, 0, 0, 0, 0, 0, 0, 0, 25, 0, 0, 0, 1, 0, 0, 0, 0b101,
                             ord("q"), 0, 0, 0, 0, 0, 0]
    m = M.from_rows(data, offs, 1, [O.STRING] * 3)
    assert m.null_counts.tolist() == [0, 1, 0] and m.char_totals.tolist() == [0, 0, 1] and m.status == 0


def test_build_batches_rule():
    """RC:1500-1517 with the overflow guard: <= INT32_MAX bytes a batch, cut on 32-row boundaries."""
    sizes = np.full(100_000, 65536, np.int64)
    b = M.build_batches(sizes)
    assert b == O.build_batches(sizes.astype(np.uint64))
    assert b[1] == 32736 and all((hi - lo) * 65536 <= 2**31 - 1 for lo, hi in zip(b[:-1], b[1:]))
    b = M.build_batches(np.full(3_000_000, 816, np.int64))                  # test_batch_split_over_2gib
    assert b[1] == (2**31 - 1 + 815) // 816 // 32 * 32 and b[-1] == 3_000_000
    rng = np.random.default_rng(1)
    sizes = rng.integers(1, 400_000, 30_000) // 8 * 8 + 8
    assert M.build_batches(sizes) == O.build_batches(sizes.astype(np.uint64))


# ---------------------------------------------------------------------------------------------- planning constants
_CSRC = os.path.join(os.path.dirname(__file__), "..", "spark-rapids-jni_b200", "csrc")


def _src(name):
    return open(os.path.join(_CSRC, name)).read()


def _const(src, name):
    m = re.search(r"constexpr\s+int\s+" + name + r"\s*=\s*([^;/]+);", src)
    assert m, f"{name} not found"
    return m.group(1).strip()


def test_planning_constants_and_tile_rule_match_the_sources():
    """The GPU scale tests size their tables from row_plans.py.  If a planner is retuned, they would silently stop
    reaching the cycle points they were written for: fail here instead."""
    capi, fr, frw = _src("capi.cu"), _src("from_rows.cu"), _src("from_rows_wide.cu")
    strs, tr, trv = _src("strings.cu"), _src("to_rows.cu"), _src("to_rows_var.cu")
    for s in (capi, fr, frw, strs, tr, trv):
        assert str(P.SMEM_BUDGET) in s
    # srj_plan_create: 64 KB x 3 stages up to 128-byte rows, 100 KB x 2 above; 512-row cap; shrink by 3/4
    assert re.search(r"if \(S <= 128\) \{ tl\.num_stages = 3; tl\.stage_bytes = 64 \* 1024; \}", capi)
    assert re.search(r"else\s+\{ tl\.num_stages = 2; tl\.stage_bytes = 100 \* 1024; \}", capi)
    # one tile-rounding rule, for the first tile and after every shrink
    assert capi.count("if (R > 512) R = 512;") == 1 and capi.count("set_tile_rows(tl, S);") == 2
    assert "tl.stage_bytes = (tl.stage_bytes * 3 / 4) & ~127;" in capi
    assert (P.FR_NARROW_MAX, P.FR_NARROW_STAGE, P.FR_WIDE_STAGE, P.FR_MAX_TILE) == (128, 64 * 1024, 100 * 1024, 512)
    assert int(_const(fr, "kMaxStages")) == P.FR_MAX_STAGES and int(_const(fr, "kStageSlack")) == P.FR_STAGE_SLACK
    assert re.search(r"p\.super_rows\s*=\s*static_cast<int64_t>\(p\.tile_rows\) \* \(row_offsets \? 8 : 2\);", fr)
    assert (P.FR_SUPER_VAR, P.FR_SUPER_FIXED) == (8, 2)
    assert "launch_variant<11>" in fr
    # plan_wide
    assert int(_const(frw, "kWMaxCols")) == P.W_MAX_COLS
    assert re.search(r"const int slab_cap = (\d+);", frw).group(1) == str(P.W_SLAB_CAP)
    assert int(_const(frw, "kWMaxG")) == P.W_MAX_G and int(_const(frw, "kWMaxStages")) == P.W_MAX_STAGES
    assert int(_const(frw, "kWSlack")) == P.W_SLACK
    assert "if (nstr < 8 || spr < 512 || nc > kWMaxCols) return false;" in frw
    assert "if (nominal - begin > 128) return false;" in frw and "if (tables > 64 * 1024) return false;" in frw
    assert "launch_wide_variant<12>" in frw
    assert (int(_const(frw, "kGsThreads")), int(_const(frw, "kGsPer"))) == (P.GS_THREADS, P.GS_PER)
    # strings_wide_kernel
    assert int(_const(strs, "kSwNG")) == P.SW_NG and _const(strs, "kSwStages") == "2 * kSwNG"
    assert (int(_const(strs, "kSwMaxWpt")), int(_const(strs, "kSwMaxCpw"))) == (P.SW_MAX_WPT, P.SW_MAX_CPW)
    assert "return nstr >= 8 && nstr <= kSwMaxWpt * kSwMaxCpw;" in strs
    assert (_const(strs, "kScanThreads"), _const(strs, "kScanIter"), _const(strs, "kScanChunk")) == \
        ("256", "kScanThreads * 4", "kScanIter * 4") and P.STR_SCAN_CHUNK == 4096
    # to_rows
    assert int(_const(tr, "kT2Super")) == P.T2_SUPER and "const int budget = 225 * 1024 - tables;" in tr
    assert int(_const(tr, "kRsChunk")) == P.RS_CHUNK and "kRsChunkHost = 4096" in capi
    assert int(_const(trv, "kTwWarps")) == P.TW_WARPS
    assert (int(_const(trv, "kT3MaxBlocks")), int(_const(trv, "kT3MaxItems"))) == (P.T3_MAX_BLOCKS, P.T3_MAX_ITEMS)


def test_plans_of_the_scale_schemas():
    """Hand-checked plans the GPU scale tests rely on."""
    S, I64 = O.STRING, O.INT64
    assert P.plan_wide([S] * 8 + [I64] * 56).G == 4 and M.layout([S] * 8 + [I64] * 56).size_per_row == 520
    assert P.plan_wide([O.DECIMAL128] * 250 + [S] * 10).nslabs == 2
    assert P.plan_wide([O.DECIMAL128] * 400 + [S] * 8).nslabs == 3
    assert P.plan_wide([S] * 8 + [I64] * 440).nslabs == 2
    c3 = [O.INT32, I64, O.DECIMAL128, S] * 64
    assert (P.plan_wide(c3).G, P.plan_wide(c3).nslabs) == (1, 1)
    assert P.wide_refusal([O.INT32, I64, O.DECIMAL128, S] * 128) == "more than kWMaxCols columns"
    assert P.wide_refusal([O.DECIMAL128] * 500 + [S] * 10) == "more than kWMaxCols columns"
    tl = P.from_rows_tiling([O.INT8, O.INT16, O.INT32, I64, O.FLOAT32, O.FLOAT64, O.BOOL8, O.TIMESTAMP_MICROSECONDS] * 4)
    assert (tl.tile_rows, tl.num_stages) == (512, 2)
    assert P.from_rows_tiling([O.INT32] * 3000).stage_bytes < P.FR_WIDE_STAGE
    assert P.strings_wide_split(33) == (8, 5) and P.strings_wide_split(8) == (2, 4)
