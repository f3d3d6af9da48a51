"""CPU tests of the shuffle model (tests/shuffle_model.py): the model against the oracle byte for byte on the Kudo goldens
(tests/golden/kudo_golden.py) and on edge tables, golden round trips through both, partition ids and the stable
partition against the oracle on the hash edge keys, and a guard that ties the edge lists of the GPU tests to the dispatch
constants of csrc/partition.cu and csrc/kudo.cu."""
import os
import re
import struct

import numpy as np
import pytest

import hash_edges as E
import shuffle_model as M
from golden import kudo_golden as KG
from oracle import kudo as K
from oracle import oracle as O
from util import random_table

CSRC = os.path.join(os.path.dirname(__file__), "..", "spark-rapids-jni_b200", "csrc")

# the dispatch constants the GPU edge tests are placed on (checked against the sources below)
MOVE_COLS, MOVE_GROUP_B, MOVE_MAX_RPT, PART_MAX_P, KUDO_MAX_COLS = 48, 16, 8, 16384, 256
PADDING_COLUMN_COUNTS, PADDING_ROW_COUNTS = M.PADDING_COLUMN_COUNTS, M.PADDING_ROW_COUNTS


def part_tile_rows(P: int) -> int:
    """partition.cu part_tile_rows: 4096 rows, doubled while below 8 rows per partition."""
    t = 4096
    while t < 8 * P:
        t *= 2
    return t


def assert_mcol_equal(got: M.MCol, want: M.MCol, what: str, nullable=True):
    assert got.type_id == want.type_id and got.size == want.size, what
    assert got.data == want.data, f"{what}: data"
    assert got.offsets == want.offsets, f"{what}: offsets"
    assert got.valid == want.valid, f"{what}: validity"
    if nullable:
        assert got.nullable == want.nullable, f"{what}: nullability"


def oracle_as_mcol(c: O.HCol) -> M.MCol:
    m = M.from_host(c)
    m.valid = m.valid if m.valid is not None else [True] * c.size
    return m


# ---- the model against the oracle and the goldens --------------------------------------------------------------------------
@pytest.mark.parametrize("case", KG.CASES, ids=[c["name"] for c in KG.CASES])
def test_golden_bytes_and_round_trip(case):
    tables, parts, want = M.golden_tables(case)
    buf, offs = M.write_parts(tables, parts)
    for (ti, s, n), a, b in zip(parts, offs, offs[1:]):
        assert buf[a:b] == K.write_partition(tables[ti], s, n), f"partition {(ti, s, n)} differs from the oracle"
    types = [c.type_id for c in tables[0]]
    got = M.assemble(buf, offs, types)
    for i, (g, w) in enumerate(zip(got, want)):
        assert_mcol_equal(g, w, f"model column {i}")
    ob = K.assemble(np.frombuffer(buf, np.uint8), np.array(offs, np.int64), types)
    for i, (g, w) in enumerate(zip(ob, want)):
        assert_mcol_equal(oracle_as_mcol(g), w, f"oracle column {i}", nullable=False)


def test_golden_list_covers_the_reference_cases():
    names = {c["name"].split("[")[0].split("/")[0] for c in KG.CASES}
    assert names == {"Simple", "Strings", "SimpleWithStrings", "Nulls", "ShortNulls", "PurgeNulls", "EmptySplits",
                     "EmptyInputs", "FixedPoint", "MixedValidity", "testMergeTableWithDifferentValidity", "testMergeString",
                     "testSerializeValidity"}
    assert sum(c["name"].startswith("ShortNulls/word") for c in KG.CASES) == 32 + 6
    purge = next(c for c in KG.CASES if c["name"].startswith("PurgeNulls"))
    assert M.golden_tables(purge)[2][0].nullable is False              # 0 rows: no partition carries validity


def test_known_partition_bytes():
    """testSerializeValidity by hand: rows [509, 512) of an INT32 column with a mask: header 28 + 1, validity byte 63
    (rows 504..511, all valid) padded to 3, no offsets, 12 data bytes."""
    case = next(c for c in KG.CASES if c["name"] == "testSerializeValidity")
    tables, parts, _ = M.golden_tables(case)
    b, _ = M.write_parts(tables, parts)
    assert struct.unpack(">7i", b[:28]) == (0x4B554430, 509, 3, 3, 0, 15, 1)
    assert b[28] == 1 and b[29] == 0xFF and b[30:32] == b"\0\0" and b[32:] == struct.pack("<3i", 509, 510, 511)


@pytest.mark.parametrize("name", list(KG.CONCAT_SCHEDULES))
def test_concat_validity_schedules(name):
    """KudoConcatValidityTest: slices (start, n) of seeded validity appended one after another."""
    tables, parts, want_valid = concat_validity_case(name)
    buf, offs = M.write_parts(tables, parts)
    got = M.assemble(buf, offs, [O.INT8])[0]
    assert got.valid == want_valid and got.nullable == any(s is not None and n > 0 for s, n in KG.CONCAT_SCHEDULES[name])
    ob = K.assemble(np.frombuffer(buf, np.uint8), np.array(offs, np.int64), [O.INT8])[0]
    assert ob.valid().tolist() == want_valid


def concat_validity_case(name, seed=0):
    """-> (tables, parts, validity of the assembled column): one INT8 table per slice; a slice with a start carries its
    seeded bits at rows [start, start + n) of a mask, one without a start has no mask."""
    rng = np.random.Generator(np.random.Philox(seed))
    tables, parts, want = [], [], []
    for s, n in KG.CONCAT_SCHEDULES[name]:
        rows = (s or 0) + n
        vals = rng.integers(-128, 128, rows).astype(np.int8).view(np.uint8)
        if s is None:
            tables.append([M.HostCol(O.INT8, vals, None, None, 0, rows)])
            want += [True] * n
        else:
            bits = rng.random(rows) < 0.5
            tables.append([M.HostCol(O.INT8, vals, M.pack_valid(bits.tolist()), None, 0, rows)])
            want += bits[s:].tolist()
        parts.append((len(tables) - 1, s or 0, n))
    return tables, parts, want


# ---- Kudo edge tables ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncols", [1, 7, 8, 9, 255, 256])
def test_kudo_column_counts_against_the_oracle(ncols):
    types = [[O.INT8, O.STRING, O.INT64, O.DECIMAL128, O.INT16, O.FLOAT32][c % 6] for c in range(ncols)]
    cols = random_table(types, 67, seed=ncols, all_valid_cols=range(0, ncols, 3))
    splits = [0, 0, 1, 9, 30, 67]
    mb, mo = M.split(cols, splits)
    ob, oo = K.split(cols, splits)
    assert mb == ob.tobytes() and mo == oo.tolist()
    hs = M.header_size(ncols)
    assert hs == 28 + (ncols + 7) // 8
    for p in range(len(splits) - 1):
        vlen = struct.unpack(">i", mb[mo[p] + 12:mo[p] + 16])[0]
        assert (hs + vlen) % 4 == 0                                        # header + validity padded to 4
    got = M.assemble(mb, mo, types)
    for g, c in zip(got, cols):
        w = M.from_host(c)
        assert g.data == w.data and g.offsets == w.offsets and g.valid == (w.valid or [True] * c.size)


def test_validity_padding_takes_every_value():
    """The validity padding, 3 - (28 + bitset + validity bytes - 1) % 4, over 1, 8, 9 and 17 masked columns and slices of
    1, 9, 17 and 25 rows (1 to 4 validity bytes per column): every padding 0..3 is produced."""
    seen = set()
    for ncols in PADDING_COLUMN_COUNTS:
        for n in PADDING_ROW_COUNTS:
            cols = random_table([O.INT32] * ncols, 40, seed=ncols + n, null_frac=0.3)
            b = M.write_partition(cols, 0, n)
            vlen = struct.unpack(">i", b[12:16])[0]
            assert M.validity_padding(b) == vlen - ncols * ((n + 7) // 8)
            seen.add(M.validity_padding(b))
            assert b == K.write_partition(cols, 0, n)
    assert seen == {0, 1, 2, 3}


def test_every_validity_slice_against_the_oracle():
    tables, parts = M.validity_slice_schedule(lambda rows: random_table([O.INT16], rows, seed=1, null_frac=0.5),
                                              lambda rows: random_table([O.INT16], rows, seed=2, null_frac=0.0))
    for ti, s, n in parts[:2000]:
        assert M.write_partition(tables[ti], s, n) == K.write_partition(tables[ti], s, n)
    buf, offs = M.write_parts(tables, parts)
    got = M.assemble(buf, offs, [O.INT16])[0]
    want = M.concat_slices(tables, parts)[0]
    assert got.valid == want.valid and got.data == want.data
    seen, at = set(), 0
    for ti, s, n in parts:
        if ti == 0:
            seen.add((s % 8, n, at % 32))
        at += n
    assert seen == {(r, n, o) for r in range(8) for n in range(1, 41) for o in range(32)}


# ---- HashPartitioning --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 2, 1024, 1025, 16384])
def test_partition_ids_and_stable_partition_against_the_oracle(P):
    types = [O.INT32, O.INT64, O.STRING, O.DECIMAL128, O.FLOAT64, O.INT8, O.BOOL8, O.DECIMAL32]
    for k, t in enumerate(types):
        cols = E.edge_cols([t, O.INT32], 300, nulls=[0.2, None], seed=k)
        ids = M.partition_ids(cols, P)
        assert ids == O.partition_ids(cols, P).tolist(), f"type {t}"
    keys = E.edge_cols([O.INT32, O.STRING, O.INT64], 2000, nulls=[0.1, 0.3, None], seed=9)
    ids = M.partition_ids(keys, P)
    offs, gather, scatter = M.stable_partition(ids, P)
    want_cols, want_offs, want_g = O.stable_partition(keys, np.array(ids, np.int32), P)
    assert offs == want_offs.tolist() and gather == want_g.tolist()
    assert [scatter[g] for g in gather] == list(range(len(ids)))
    for c, w in zip(keys, want_cols):
        m = M.take(c, gather)
        assert m.data == M._bytes(w.data) and m.mask_words() == M._bytes(w.mask) and m.offsets == (w.offsets.tolist() if w.offsets is not None else None)


# ---- the dispatch constants the edge lists are placed on ------------------------------------------------------------------------
def _const(src, name, file):
    m = re.search(r"constexpr\s+\w+\s+" + name + r"\s*=\s*([^;]+);", src)
    assert m, f"{name} not found in {file}"
    return eval(m.group(1).split("//")[0], {})                       # e.g. 1 << 14


def test_shuffle_dispatch_constants_match_the_edge_tests_in_their_modules():
    part = open(os.path.join(CSRC, "partition.cu")).read()
    kudo = open(os.path.join(CSRC, "kudo.cu")).read()
    assert _const(part, "kMoveCols", "partition.cu") == MOVE_COLS
    assert _const(part, "kMoveGroupB", "partition.cu") == MOVE_GROUP_B
    assert _const(part, "kMoveMaxRpt", "partition.cu") == MOVE_MAX_RPT
    assert _const(part, "kPartMaxP", "partition.cu") == PART_MAX_P
    assert _const(part, "kPartThreads", "partition.cu") == 1024
    assert _const(kudo, "kKudoMaxCols", "kudo.cu") == KUDO_MAX_COLS
    # part_tile_rows: 4096, doubled while below 8 x P
    assert re.search(r"int32_t t = 4096;\s*while \(t < 8 \* P\) t <<= 1;", part)
    # the tile kernel takes plans whose tile is at most kMoveMaxRpt x 1024 rows; larger plans move row by row
    assert re.search(r"if \(tile > kMoveMaxRpt \* kPartThreads\) return SRJ_EUNSUPPORTED;", part)
    assert part_tile_rows(1024) == MOVE_MAX_RPT * 1024 and part_tile_rows(1025) > MOVE_MAX_RPT * 1024
    assert re.search(r"num_partitions > \(1 << 14\)", part) and re.search(r"P > 65535", kudo)
    # the rank kernel's warps: min(32, 51200 / P - 1): 2 warps and 196,608 B of shared memory at P = 16384
    assert re.search(r"\(200 \* 1024\) / \(static_cast<int64_t>\(P\) \* 4\) - 1", part)
    w = max(1, min(32, 51200 // PART_MAX_P - 1))
    assert w == 2 and (w + 1) * PART_MAX_P * 4 == 196_608
    assert [part_tile_rows(P) for P in (1, 512, 513, 1024, 1025, 2048, 16384)] == [4096, 4096, 8192, 8192, 16384, 16384, 131072]
