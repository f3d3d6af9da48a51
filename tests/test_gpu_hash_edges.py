"""The row hashes on the GPU at the edge values of every key type (hash_edges.py), through every dispatch path of
csrc/hash.cu, the fused from_rows hash, nested keys and hash partitioning.

Every result is compared with the C oracle on all rows and with the independent model (spark_hash_model.py) on all rows
of the narrower tables and on a fixed sample of the larger ones.  The test ids name the path a table is sized for:
  perthread   : fewer than STREAM_MIN_ROWS rows, row_hash_kernel (general) or row_hash_plain_kernel (4/8-byte keys)
  stream      : whole HS_ROWS chunks on row_hash_stream_kernel, the tail rows on the per-thread kernels
  declined    : large tables the streaming kernel refuses (too many keys, unaligned data or mask, STRING keys)
  chunked     : more key columns than one launch carries; the later chunks start from the previous chunk's hashes
"""
import numpy as np
import pytest
import torch

import hash_edges as E
import spark_hash_model as M
from hash_edges import HASH_COLS_PER_LAUNCH, HS_MAX_COLS, HS_ROWS, STREAM_MIN_ROWS
from oracle import oracle as O

pytestmark = pytest.mark.gpu

KINDS = ("xxhash64", "murmur3", "hive")
SEEDS = {"xxhash64": 42, "murmur3": 42, "hive": 0}
MODEL_BUDGET = 400_000          # element hashes the model computes per table and hash (beyond it: a fixed row sample)


def _gpu():
    import gpu_util
    gpu_util.require_cuda()
    return gpu_util


def _device_hash(kind, dcols, seed):
    import srj_b200 as S
    if kind == "xxhash64":
        return S.Hash.xxhash64(seed, dcols).data.cpu().numpy().view(np.int64)
    if kind == "murmur3":
        return S.Hash.murmurHash32(seed, dcols).data.cpu().numpy().view(np.int32)
    return S.Hash.hiveHash(dcols).data.cpu().numpy().view(np.int32)


def _oracle_hash(kind, cols, seed):
    if any(c.type_id in (O.LIST, O.STRUCT) for c in cols):
        return O.nested_hash(kind, cols, seed)
    if kind == "xxhash64":
        return O.xxhash64(cols, seed)
    if kind == "murmur3":
        return O.murmur_hash3_32(cols, seed)
    return O.hive_hash(cols)


def model_rows(n, ncols):
    """All rows if the table is small enough, otherwise the rows at the chunk edges plus a seeded sample."""
    if n * max(ncols, 1) <= MODEL_BUDGET:
        return np.arange(n)
    edges = [r for k in range(0, n // HS_ROWS + 1) for r in (k * HS_ROWS - 1, k * HS_ROWS) if 0 <= r < n]
    rng = np.random.Generator(np.random.Philox(n))
    sample = rng.choice(n, size=max(64, MODEL_BUDGET // max(ncols, 1) - len(edges) - 2), replace=False)
    return np.unique(np.concatenate([edges, [0, n - 1], sample]).astype(np.int64))


def check(kind, cols, got, seed, what=""):
    want = _oracle_hash(kind, cols, seed)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{kind} {what}: GPU != oracle at rows {bad[:8].tolist()} of {len(got)}"
    rows = model_rows(len(got), len(cols))
    m = M.hash_rows(kind, cols, seed, rows)
    bad = rows[np.flatnonzero(got[rows] != m)]
    assert bad.size == 0, f"{kind} {what}: GPU != model at rows {bad[:8].tolist()} of {len(got)}"


def run_all(cols, dcols=None, kinds=KINDS, what=""):
    """Hash `cols` with every kind on the GPU (from `dcols` if given: the same columns, placed differently) and check."""
    G = _gpu()
    dcols = dcols if dcols is not None else [G.to_device(c) for c in cols]
    for kind in kinds:
        idx = [i for i, c in enumerate(cols) if kind != "hive" or c.type_id in E.HIVE_TYPES]
        if not idx:
            continue
        kc, kd = [cols[i] for i in idx], [dcols[i] for i in idx]
        check(kind, kc, _device_hash(kind, kd, SEEDS[kind]), SEEDS[kind], what)


def _shifted(t: torch.Tensor, shift: int) -> torch.Tensor:
    """The bytes of t in a new allocation, `shift` bytes past its (256-byte aligned) start."""
    big = torch.zeros(t.numel() * t.element_size() + 64, dtype=torch.uint8, device=t.device)
    v = big[shift: shift + t.numel() * t.element_size()]
    v.copy_(t.contiguous().view(torch.uint8))
    return v


BY_SIZE = {1: [O.BOOL8, O.INT8, O.UINT8], 2: [O.INT16, O.UINT16, O.INT16],
           4: [O.INT32, O.FLOAT32, O.UINT32, O.TIMESTAMP_DAYS, O.DECIMAL32],
           8: [O.INT64, O.FLOAT64, O.UINT64, O.TIMESTAMP_MICROSECONDS, O.DECIMAL64, O.TIMESTAMP_NANOSECONDS],
           16: [O.DECIMAL128, O.DECIMAL128]}
PLAIN = [O.INT32, O.INT64, O.DECIMAL64, O.TIMESTAMP_MILLISECONDS, O.UINT32, O.TIMESTAMP_DAYS]
MIXED = [0.25, None]            # every other key column has a mask


# ---------------------------------------------------------------- per-thread kernels (fewer than STREAM_MIN_ROWS rows)
@pytest.mark.parametrize("nulls", [None, 0.3, "all"], ids=["no_mask", "nulls", "all_null"])
@pytest.mark.parametrize("t", list(E.EDGES), ids=[f"perthread_type{t}" for t in E.EDGES])
def test_perthread_every_type(t, nulls):
    n = 3 * len(E.EDGES[t]) + 11
    run_all(E.edge_cols([t, t], n, nulls=[nulls, None], seed=t), what=f"type {t}")


@pytest.mark.parametrize("path,types", [("perthread_plain", PLAIN), ("perthread_general", list(E.EDGES))])
def test_perthread_tables(path, types):
    cols = E.edge_cols(types, 5003, nulls=MIXED * len(types), seed=1)
    assert not E.streams(cols)
    run_all(cols, what=path)


def test_perthread_8191_rows_does_not_stream():
    """One row short of the streaming threshold: the per-thread kernels take the whole table."""
    types = [BY_SIZE[s][0] for s in sorted(BY_SIZE)]
    cols = E.edge_cols(types, STREAM_MIN_ROWS - 1, nulls=MIXED * len(types), seed=2)
    assert not E.streams(cols) and E.streams(E.edge_cols(types, STREAM_MIN_ROWS))
    run_all(cols, what="8191 rows")


# ---------------------------------------------------------------- streaming kernel
STREAM_ROWS = [STREAM_MIN_ROWS, STREAM_MIN_ROWS + 1, STREAM_MIN_ROWS + HS_ROWS - 1, 3 * HS_ROWS * 2, 3 * HS_ROWS * 5,
               200_003]


@pytest.mark.parametrize("nrows", STREAM_ROWS, ids=[f"rows{n}" for n in STREAM_ROWS])
@pytest.mark.parametrize("size", sorted(BY_SIZE), ids=[f"stream_size{s}" for s in sorted(BY_SIZE)])
def test_stream_element_sizes(size, nrows):
    """Every element width through the streaming kernel's shared-memory loads, with and without masks in one launch;
    row counts at the chunk edges (exactly 4 chunks, one tail row, a 2047-row tail, whole chunks with no tail)."""
    cols = E.edge_cols(BY_SIZE[size], nrows, nulls=MIXED * len(BY_SIZE[size]), seed=size)
    assert E.streams(cols)
    run_all(cols, what=f"size {size}, {nrows} rows")


@pytest.mark.parametrize("nulls", [None, 0.0, 0.5, "all", "mixed"],
                         ids=["stream_no_masks", "stream_masks_no_nulls", "stream_masks", "stream_all_null",
                              "stream_mixed_masks"])
def test_stream_mask_modes(nulls):
    types = [BY_SIZE[s][0] for s in sorted(BY_SIZE)]
    pats = [0.3, None, "all", 0.0, 0.3] if nulls == "mixed" else nulls
    cols = E.edge_cols(types, STREAM_MIN_ROWS + HS_ROWS - 1, nulls=pats, seed=5)
    assert E.streams(cols)
    run_all(cols, what=str(nulls))


# ---------------------------------------------------------------- streaming declined
def test_declined_17_keys():
    types = ([BY_SIZE[s][0] for s in (1, 2, 4)] * 6)[:HS_MAX_COLS + 1]     # narrow keys: only their count declines
    cols = E.edge_cols(types, STREAM_MIN_ROWS + 777, nulls=MIXED * len(types), seed=6)
    assert not E.streams(cols) and E.streams(cols[:HS_MAX_COLS])
    run_all(cols, what="17 keys")


@pytest.mark.parametrize("what", ["declined_data_shifted_one_element", "declined_mask_shifted_4_bytes"])
def test_declined_unaligned(what):
    """Element-aligned but not 16-byte aligned column buffers: the table goes to the per-thread kernels."""
    G = _gpu()
    types = [O.INT8, O.INT16, O.FLOAT32, O.FLOAT64, O.DECIMAL128, O.INT64]
    n = STREAM_MIN_ROWS + HS_ROWS + 5
    cols = E.edge_cols(types, n, nulls=[0.3] * len(types), seed=7)
    assert E.streams(cols)          # at aligned addresses the streaming kernel would take these keys
    dcols = []
    for c in cols:
        dc = G.to_device(c)
        if what.startswith("declined_data") and E.SIZE[c.type_id] < 16:
            dc.data = _shifted(dc.data, E.SIZE[c.type_id])
            assert dc.data.data_ptr() % 16 != 0
        if what.startswith("declined_mask"):
            dc.mask = _shifted(dc.mask, 4).view(torch.int32)
            assert dc.mask.data_ptr() % 16 == 4
        dcols.append(dc)
    run_all(cols, dcols, what=what)


def test_declined_string_key_among_fixed_keys():
    types = [O.STRING, O.INT32, O.DECIMAL128, O.FLOAT64, O.BOOL8, O.STRING]
    run_all(E.edge_cols(types, STREAM_MIN_ROWS + HS_ROWS - 1, nulls=[0.2, None, 0.2, None, 0.2, None], seed=8),
            what="STRING keys")


# ---------------------------------------------------------------- column chunks
CHUNK_POOLS = {   # kinds -> (types of the first 48 keys, narrow types of the later keys)
    "xx_mm": (E.FIXED_TYPES, [O.INT8, O.BOOL8, O.INT16, O.UINT8, O.INT32, O.FLOAT32, O.TIMESTAMP_DAYS]),
    "hive": ([t for t in E.FIXED_TYPES if t in E.HIVE_TYPES], [O.INT8, O.BOOL8, O.INT16, O.INT32, O.FLOAT32,
                                                               O.TIMESTAMP_DAYS]),
}


@pytest.mark.parametrize("nrows", [STREAM_MIN_ROWS + 777, 3001])
@pytest.mark.parametrize("ncols", [HASH_COLS_PER_LAUNCH + 1, 64, 2 * HASH_COLS_PER_LAUNCH + 1])
@pytest.mark.parametrize("kinds", ["xx_mm", "hive"])
def test_chunked_columns(kinds, ncols, nrows):
    """The first 48 keys on the per-thread kernels; from 8192 rows on, a later chunk of at most 16 narrow keys
    streams and must start from the hashes the previous chunk left in the output (xxhash64 / murmur3: the running
    hash; hive: the 31-fold so far)."""
    first, narrow = CHUNK_POOLS[kinds]
    pool = first + ([O.STRING] if nrows < STREAM_MIN_ROWS else [])
    types = [pool[i % len(pool)] if i < HASH_COLS_PER_LAUNCH else narrow[i % len(narrow)] for i in range(ncols)]
    cols = E.edge_cols(types, nrows, nulls=MIXED * ncols, seed=ncols)
    last = cols[(ncols - 1) // HASH_COLS_PER_LAUNCH * HASH_COLS_PER_LAUNCH:]
    assert E.streams(last) == (nrows >= STREAM_MIN_ROWS) and not E.streams(cols[:HASH_COLS_PER_LAUNCH])
    run_all(cols, kinds=("xxhash64", "murmur3") if kinds == "xx_mm" else ("hive",),
            what=f"chunked_{ncols}cols_{nrows}rows")


# ---------------------------------------------------------------- fused from_rows + hash
@pytest.mark.parametrize("schema", ["fixed", "wide_strings"])
@pytest.mark.parametrize("kind", KINDS)
def test_from_rows_with_hash_edge_keys(kind, schema):
    G = _gpu()
    import srj_b200 as S
    # at most 16 keys: DECIMAL128 first (so the 3-key run has it), every decimal and every element rule among them
    keyt = [O.DECIMAL128, O.BOOL8, O.FLOAT64, O.DECIMAL32, O.DECIMAL64, O.INT8, O.INT16, O.INT32, O.INT64, O.UINT8,
            O.UINT16, O.UINT32, O.UINT64, O.FLOAT32, O.TIMESTAMP_DAYS, O.TIMESTAMP_MICROSECONDS]
    keyt = [t for t in keyt if kind != "hive" or t in E.HIVE_TYPES]
    types = keyt + ([O.STRING, O.INT64] * 30 if schema == "wide_strings" else [O.INT16])
    n = STREAM_MIN_ROWS + HS_ROWS - 1
    cols = E.edge_cols(types, n, nulls=[0.2] * len(types), seed=9)
    (offs, data), = O.convert_to_rows(cols)
    vec = G.rows_to_device(offs, data)
    dts = [S.DType(t, c.scale) for t, c in zip(types, cols)]
    for keys in ([0, 1, 2], list(range(len(keyt)))):
        _, h = S.RowConversion.convertFromRowsWithHash(vec, dts, keys, kind=kind, seed=SEEDS[kind])
        kc = [cols[k] for k in keys]
        got = h.data.cpu().numpy().view(np.int64 if kind == "xxhash64" else np.int32)
        check(kind, kc, got, SEEDS[kind], f"{schema} keys {keys}")


# ---------------------------------------------------------------- nested keys
@pytest.mark.parametrize("name", list(E.nested_edge_keys(1)) + ["all"])
def test_nested_edge_leaves_and_level_nulls(name):
    """Edge leaves under LIST, STRUCT and LIST<STRUCT>, with LIST and STRUCT level nulls over rows that have
    children: xxhash64 and hive hash the children of a null list or struct, murmur3 skips them."""
    keys = E.nested_edge_keys(3001, seed=12)
    cols = list(keys.values()) if name == "all" else [keys[name]]
    kinds = ["xxhash64"]
    if all(c is not keys["list_of_struct"] for c in cols):
        kinds.append("murmur3")
    if all(E.nested_hive_ok(c) for c in cols):
        kinds.append("hive")
    run_all(cols, kinds=kinds, what=name)


def test_nested_partition_ids():
    """Partition ids of nested keys: pmod of their murmur3 hash, with the level-null rule of murmur3."""
    G = _gpu()
    from srj_b200.partitioning import HashPartitioner
    keys = E.nested_edge_keys(3001, seed=13)
    kc = [keys["struct_bool_double_string"], keys["list_list_string"], keys["list_decimal128"]]
    for P in (7, 200):
        ids = HashPartitioner.partitionIds([G.to_device(c) for c in kc], P).data.cpu().numpy().view(np.int32)
        want = O.partition_ids(kc, P)
        assert np.array_equal(ids, want), f"P={P}: rows {np.flatnonzero(ids != want)[:8].tolist()}"
        assert ids.tolist() == [M.pmod(int(h), P) for h in M.hash_rows("murmur3", kc, 42)]


def _nullable_lists(levels, n=256, seed=0):
    """`levels` nested nullable LIST levels over INT32 edge leaves; the null rows keep their children.  Few nulls per
    level, so that most leaves survive all the levels under murmur3."""
    rng = np.random.Generator(np.random.Philox(seed))
    def build(level, rows):
        if level == 0:
            return E.edge_col(O.INT32, rows, 0, 0.2, seed)
        lens = rng.choice(3, rows, p=[0.1, 0.8, 0.1]) if level < levels else np.full(rows, 2)
        offs = np.zeros(rows + 1, np.int32)
        np.cumsum(lens, out=offs[1:])
        return O.list_col(offs, build(level - 1, int(offs[-1])), valid=rng.random(rows) >= 0.04)
    return build(levels, n)


def test_murmur3_nullable_list_levels_limit():
    """murmur3 keeps one stack frame per nullable LIST level (plus one per STRUCT level and one leaf), at most
    2 * MAX_STACK_DEPTH + 2 = 18: 17 nullable levels still hash like the reference, 18 are refused with an error
    rather than hashed wrongly.  xxhash64 collapses list levels and has no such limit."""
    G = _gpu()
    import srj_b200 as S
    ok = _nullable_lists(17)
    assert np.array_equal(_device_hash("murmur3", [G.to_device(ok)], 42), M.hash_rows("murmur3", [ok], 42))
    deep = _nullable_lists(18)
    with pytest.raises(S.CudfException):
        S.Hash.murmurHash32(42, [G.to_device(deep)])
    assert np.array_equal(_device_hash("xxhash64", [G.to_device(deep)], 42), M.hash_rows("xxhash64", [deep], 42))


# ---------------------------------------------------------------- hash partitioning
@pytest.mark.parametrize("P", [1, 7, 200, 1024, 5000])
def test_partition_ids_of_edge_keys(P):
    G = _gpu()
    import srj_b200 as S
    from srj_b200.partitioning import HashPartitioner
    n = STREAM_MIN_ROWS + HS_ROWS - 1
    cols = E.edge_cols([O.DECIMAL128, O.BOOL8, O.FLOAT64, O.STRING], n, nulls=[0.2, None, 0.2, 0.1], seed=P)
    keys = cols[:3]
    pt = HashPartitioner.partition(S.Table([G.to_device(c) for c in cols]), [0, 1, 2], P)
    ids = pt.partition_ids.data.cpu().numpy().view(np.int32)
    want = O.spark_pmod(O.murmur_hash3_32(keys, 42), P)
    assert np.array_equal(ids, want), f"partition ids differ at rows {np.flatnonzero(ids != want)[:8].tolist()}"
    rows = model_rows(n, len(keys))
    m = [M.pmod(int(h), P) for h in M.hash_rows("murmur3", keys, 42, rows)]
    assert ids[rows].tolist() == m
    assert pt.getRowCounts() == np.bincount(want, minlength=P).tolist()
