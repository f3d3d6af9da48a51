"""Pins the independent hash model (spark_hash_model.py) on the CPU: against every golden of the reference's tests, and
against the C oracle on the edge-value tables of hash_edges.py.  Also guards the dispatch constants of csrc/hash.cu that
the GPU edge tests size their tables from."""
import os
import re

import numpy as np
import pytest

import hash_edges as E
import spark_hash_model as M
from golden import hash_golden as GOLD
from golden import hash_nested_golden as NG
from oracle import oracle as O
from util import cols_from_case

KIND = {"murmur": "murmur3", "xxhash64": "xxhash64", "hive": "hive"}


def _oracle(kind, cols, seed):
    if kind == "xxhash64":
        return O.xxhash64(cols, seed)
    if kind == "murmur3":
        return O.murmur_hash3_32(cols, seed & 0xFFFFFFFF)
    return O.hive_hash(cols)


# ---------------------------------------------------------------- the model against the goldens
@pytest.mark.parametrize("case", GOLD.CASES, ids=[c["name"] for c in GOLD.CASES])
def test_model_matches_golden(case):
    got = M.hash_rows(KIND[case["kind"]], cols_from_case(case), case["seed"])
    assert got.tolist() == list(case["expected"]), case["src"]


@pytest.mark.parametrize("name,build,want", NG.XX_CASES, ids=[c[0] for c in NG.XX_CASES])
def test_model_matches_nested_xxhash64_golden(name, build, want):
    assert M.hash_rows("xxhash64", [build()], 42).tolist() == want


@pytest.mark.parametrize("name,build,want", NG.HIVE_CASES, ids=[c[0] for c in NG.HIVE_CASES])
def test_model_matches_nested_hive_golden(name, build, want):
    assert M.hash_rows("hive", [build()]).tolist() == want


def test_model_murmur_lists_and_structs_hash_like_their_elements():
    """HashTest.java:225-270: a list of ints hashes like the columns of its elements; a struct like its fields."""
    il = NG.lists_of([None, [0, -2, 3], [NG.INT_MAX], [5, -6, None], [NG.INT_MIN], None], NG.ints)
    c1, c2, c3 = (NG.ints([None, 0, None, 5, NG.INT_MIN, None]), NG.ints([None, -2, NG.INT_MAX, None, None, None]),
                  NG.ints([None, 3, None, -6, None, None]))
    want = M.hash_rows("murmur3", [c1, c2, c3], 1868)
    assert np.array_equal(M.hash_rows("murmur3", [il], 1868), want)
    assert np.array_equal(M.hash_rows("murmur3", [O.struct_col(c1, c2, c3)], 1868), want)


def test_java_big_integer_bytes():
    """BigInteger.valueOf(v).toByteArray() for values whose minimal length is easy to get wrong."""
    cases = {0: "00", 1: "01", -1: "ff", 127: "7f", 128: "0080", -128: "80", -129: "ff7f", 255: "00ff", -256: "ff00",
             2**63: "008000000000000000", -2**63: "8000000000000000", -2**63 - 1: "ff7fffffffffffffff",
             2**64: "010000000000000000", 2**127 - 1: "7f" + "ff" * 15, -2**127: "80" + "00" * 15}
    for v, hexb in cases.items():
        assert M.java_big_integer_bytes(v).hex() == hexb, v


# ---------------------------------------------------------------- the model against the oracle on the edge tables
@pytest.mark.parametrize("nulls", [None, 0.3, "all"], ids=["no_mask", "nulls", "all_null"])
@pytest.mark.parametrize("t", list(E.EDGES), ids=[str(t) for t in E.EDGES])
def test_model_matches_oracle_per_type(t, nulls):
    n = 2 * len(E.EDGES[t]) + 5
    cols = E.edge_cols([t, t], n, nulls=[nulls, None], seed=t)
    for kind, seed in (("xxhash64", 42), ("xxhash64", -7), ("murmur3", 42), ("murmur3", 0xDEADBEEF), ("hive", 0)):
        kc = E.hive_ok(cols) if kind == "hive" else cols
        if not kc:
            continue
        assert np.array_equal(M.hash_rows(kind, kc, seed), _oracle(kind, kc, seed)), kind


def test_model_matches_oracle_all_types_mixed():
    types = list(E.EDGES) * 2
    cols = E.edge_cols(types, 600, nulls=[None, 0.2, 0.5] * len(types), seed=3)
    for kind in ("xxhash64", "murmur3", "hive"):
        kc = E.hive_ok(cols) if kind == "hive" else cols
        assert np.array_equal(M.hash_rows(kind, kc, 42), _oracle(kind, kc, 42)), kind


@pytest.mark.parametrize("name", list(E.nested_edge_keys(1)))
def test_model_matches_oracle_nested(name):
    col = E.nested_edge_keys(300, seed=11)[name]
    kinds = ["xxhash64"] + (["murmur3"] if name != "list_of_struct" else []) + (["hive"] if E.nested_hive_ok(col) else [])
    for kind in kinds:
        assert np.array_equal(M.hash_rows(kind, [col], 42), O.nested_hash(kind, [col], 42)), kind


def test_oracle_partition_ids_of_nested_keys_use_murmur3():
    """GpuHashPartitioning over LIST / STRUCT keys: pmod of their murmur3 hash (with murmur3's level-null rule)."""
    keys = E.nested_edge_keys(300, seed=4)
    kc = [keys["struct_bool_double_string"], keys["list_list_string"]]
    for P in (7, 200):
        ids = O.partition_ids(kc, P)
        assert np.array_equal(ids, O.spark_pmod(O.nested_hash("murmur3", kc, 42), P))
        assert ids.tolist() == [M.pmod(int(h), P) for h in M.hash_rows("murmur3", kc, 42)]


# ---------------------------------------------------------------- dispatch constants
def test_hash_dispatch_constants_match_the_edge_tests():
    """The GPU edge tests place their row and column counts on the dispatch edges of csrc/hash.cu.  If the dispatch is
    retuned, they would silently stop reaching the paths they were written for: fail here instead."""
    src = open(os.path.join(os.path.dirname(__file__), "..", "spark-rapids-jni_b200", "csrc", "hash.cu")).read()

    def const(name):
        m = re.search(r"constexpr\s+int\s+" + name + r"\s*=\s*(\d+)\s*;", src)
        assert m, f"{name} not found in hash.cu"
        return int(m.group(1))

    assert const("kHsRows") == E.HS_ROWS
    assert const("kHsMaxCols") == E.HS_MAX_COLS
    assert const("kHashColsPerLaunch") == E.HASH_COLS_PER_LAUNCH
    # launch_hash_stream declines tables below 4 chunks and launches with more key columns than kHsMaxCols
    assert re.search(r"hp\.ncols\s*>\s*kHsMaxCols\s*\|\|\s*num_rows\s*<\s*4\s*\*\s*kHsRows", src)
    assert E.STREAM_MIN_ROWS == 4 * E.HS_ROWS
    # ... and any key column that is not 16-byte aligned, or a STRING key
    assert re.search(r"col\.data\)\s*&\s*15", src) and re.search(r"col\.mask\)\s*&\s*15", src)
    assert re.search(r"col\.size\s*==\s*0\)\s*return SRJ_OK", src)
    # ... and keys whose chunk (values + 256-byte mask pieces) does not fit twice in the stage budget
    m = re.search(r"\(([\d\s*]+)\)\s*/\s*p\.stage_bytes", src)
    assert m and np.prod([int(x) for x in m.group(1).split("*")]) == E.STAGE_BUDGET
    assert re.search(r"p\.nstages\s*<\s*2\)\s*return SRJ_OK", src)
    assert re.search(r"off \+= 256", src) and re.search(r"\(off \+ 127\) & ~127", src)
