"""GPU tests of HashPartitioning (csrc/partition.cu) at its dispatch edges, byte-exact against the independent model
(tests/shuffle_model.py): partition counts around the warp, tile-size and tile-kernel limits up to 16384, row counts
around each plan's tile, the refused partition counts, tables wider than one move launch (48 columns) and one mask round
(16 columns) on both the tile path and the per-row path, the width mixes of the staging groups, skew, keys of every
murmur3 type, Table.partition by the caller's ids, and the 8M-row permutation properties at 16384 partitions.

Every column is compared whole: values including null payload bytes, mask words including the tail bits, STRING offsets
and chars, and the null counts the library reports."""
import ctypes as C

import numpy as np
import pytest
import torch

import hash_edges as E
import shuffle_model as M
from oracle import oracle as O
from util import random_table

pytestmark = pytest.mark.gpu

TILE_EDGE_P = [1, 31, 32, 33, 512, 513, 1024, 1025, 2048, 2049, 5000, 8192, 16383, 16384]


def _gpu():
    import gpu_util
    gpu_util.require_cuda()
    return gpu_util


def part_tile_rows(P: int) -> int:
    t = 4096
    while t < 8 * P:
        t *= 2
    return t


def head(col, n: int) -> M.HostCol:
    """Rows [0, n) of a host column."""
    mask = None if col.mask is None else M.pack_valid(M._valid_bits(col)[:n])
    if col.type_id == O.STRING:
        offs = np.ascontiguousarray(col.offsets[:n + 1])
        return M.HostCol(O.STRING, col.data[:int(offs[-1])].copy(), mask, offs.copy(), col.scale, n)
    sz = O.size_of(col.type_id)
    return M.HostCol(col.type_id, np.ascontiguousarray(col.data).view(np.uint8)[:n * sz].copy(), mask, None, col.scale, n)


def assert_column_exact(g, want: M.MCol, what: str):
    """Device column g against a model column: every byte of data, offsets, mask words (tail bits included), null count."""
    G = _gpu()
    h = G.to_host(g)
    n = want.size
    assert h.size == n, f"{what}: rows"
    assert M._bytes(h.data)[:len(want.data)] == want.data and (h.data is None or h.data.nbytes >= len(want.data)), f"{what}: data"
    if want.type_id == O.STRING:
        assert h.offsets.tolist()[:n + 1] == want.offsets, f"{what}: offsets"
        assert int(h.offsets[n]) == len(want.data), f"{what}: chars"
    if want.valid is None:
        assert h.mask is None, f"{what}: unexpected mask"
    else:
        words = (n + 31) // 32
        assert M._bytes(h.mask)[:4 * words] == want.mask_words(), f"{what}: mask words"
    assert g.getNullCount() == want.null_count(), f"{what}: null count"


def check_hash_partition(cols, key_idx, P, seed=42, ids=None):
    """HashPartitioner.partition on the device against the model: ids, offsets, every column."""
    G = _gpu()
    from srj_b200.partitioning import HashPartitioner
    if ids is None:
        ids = M.partition_ids([cols[i] for i in key_idx], P, seed)
    offs, gather, _ = M.stable_partition(ids, P)
    pt = HashPartitioner.partition(G.table_to_device(cols), key_idx, P, seed)
    n = len(ids)
    assert pt.partition_ids.data.view(torch.int32)[:n].cpu().tolist() == ids, f"P={P}: ids"
    assert pt.getPartitions() == offs[:-1] and sum(pt.getRowCounts()) == n, f"P={P}: offsets"
    for i, (g, c) in enumerate(zip(pt.getTable().columns, cols)):
        assert_column_exact(g, M.take(c, gather), f"P={P} n={n} column {i}")
    return pt


def _schema_table(n: int, seed: int):
    """INT32 key with nulls, then INT64 (mask), STRING (mask), INT8 (no mask), DECIMAL128 (a mask with no null bit)."""
    cols = E.edge_cols([O.INT32], n, nulls=0.1, seed=seed) + random_table([O.INT64, O.STRING, O.INT8, O.DECIMAL128], n,
                                                                           seed=seed, all_valid_cols=(2, 3))
    cols[4].mask = O.pack_mask(np.ones(n, bool))
    return cols


_BIG = 2 * part_tile_rows(16384) + 31
_TABLE = None
_HASHES = None


def _table_and_hashes():
    """One table of 2 x 131072 + 31 rows and its murmur3 key hashes (the model's); smaller row counts take its head."""
    global _TABLE, _HASHES
    if _TABLE is None:
        _TABLE = _schema_table(_BIG, seed=5)
        _HASHES = [int(h) for h in M.H.hash_rows("murmur3", [_TABLE[0]], 42)]
    return _TABLE, _HASHES


@pytest.mark.parametrize("P", TILE_EDGE_P)
def test_partition_counts_at_every_tile_edge(P):
    t = part_tile_rows(P)
    table, hashes = _table_and_hashes()
    for n in (0, 1, t - 1, t, t + 1, 2 * t + 31):
        cols = [head(c, n) for c in table]
        check_hash_partition(cols, [0], P, ids=[M.H.pmod(h, P) for h in hashes[:n]])


def test_refused_partition_counts_launch_nothing():
    """P = 16385 and P = 0: refused before the keys are hashed (the ids buffer keeps its bytes), with the status and the
    message of the plan."""
    G = _gpu()
    import srj_b200 as S
    from srj_b200 import _native as N
    from srj_b200.partitioning import HashPartitioner, partition
    n = 1000
    key = G.to_device(E.edge_col(O.INT32, n))
    lib = N.lib()
    for P, rc_want in ((16385, N.SRJ_EUNSUPPORTED), (0, N.SRJ_EINVAL), (-3, N.SRJ_EINVAL)):
        ids = torch.full((n,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        offs = torch.zeros(max(P, 1) + 1, dtype=torch.int32, device="cuda")
        ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
        maps = torch.zeros(2 * n, dtype=torch.int32, device="cuda")
        arr = (N.SrjColumn * 1)(key._c())
        rc = lib.srj_hash_partition(arr, 1, n, C.c_uint32(42), P, ids.data_ptr(), offs.data_ptr(), maps.data_ptr(),
                                    maps[n:].data_ptr(), ws.data_ptr(), int(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert rc == rc_want, (P, rc)
        assert bool((ids == 0x5A5A5A5A).all()), f"P={P}: the keys were hashed"
        assert b"partition" in lib.srj_last_error()
    with pytest.raises(S.CudfException, match="16384"):
        HashPartitioner.partition(S.Table([key]), [0], 16385)
    with pytest.raises(ValueError):
        HashPartitioner.partition(S.Table([key]), [0], 0)
    pmap = S.ColumnVector(S.DType.INT32, n, torch.zeros(n, dtype=torch.int32, device="cuda").view(torch.uint8))
    with pytest.raises(S.CudfException, match="16384"):
        partition(S.Table([key]), pmap, 16385)


_WIDE_TYPES = [O.INT8, O.INT16, O.INT32, O.INT64, O.DECIMAL128, O.STRING, O.FLOAT32, O.BOOL8, O.DECIMAL64, O.UINT16, O.STRING]


def _wide(ncols: int, n: int, seed: int):
    """ncols columns cycling through every width and STRING; every third column has no mask, every fifth a mask with
    no null bit, the rest random nulls."""
    types = [_WIDE_TYPES[c % len(_WIDE_TYPES)] for c in range(ncols)]
    cols = random_table(types, n, seed=seed, all_valid_cols=range(1, ncols, 3))
    for c in range(0, ncols, 5):
        if cols[c].mask is not None:
            cols[c].mask = O.pack_mask(np.ones(n, bool))
    return cols


@pytest.mark.parametrize("P", [200, 2048])                       # tile path, per-row path
@pytest.mark.parametrize("ncols", [49, 97, 100])
def test_wide_tables(ncols, P):
    """More than one 48-column launch and more than one 16-column mask round; the per-row path counts each column's
    nulls on its own."""
    cols = _wide(ncols, 20_000, seed=ncols + P)
    check_hash_partition(cols, [2, 0], P)


@pytest.mark.parametrize("P", [7, 1025])
@pytest.mark.parametrize("mix", ["1,2,4,8,1", "8,8", "4,4,4,4,4", "1,16,2", "S,1,S,16,S"])
def test_width_mixes(mix, P):
    """Staging groups of <= 16 bytes: exact fits, a 16-byte column after narrow ones, STRING columns (width 0) with masks
    inside a mask round."""
    by_width = {"1": O.INT8, "2": O.INT16, "4": O.INT32, "8": O.INT64, "16": O.DECIMAL128, "S": O.STRING}
    types = [O.INT32] + [by_width[w] for w in mix.split(",")]
    cols = random_table(types, 9000, seed=len(mix) + P)
    check_hash_partition(cols, [0], P)


def test_skew():
    n = 30_000
    # every row in one partition
    const = M.HostCol(O.INT32, np.full(n, 77, np.int32).view(np.uint8), None, None, 0, n)
    vals = random_table([O.INT64, O.STRING], n, seed=3)
    check_hash_partition([const] + vals, [0], 1024)
    check_hash_partition([const] + vals, [0], 16384)
    # more partitions than rows
    small = random_table([O.INT32, O.STRING, O.DECIMAL128], 100, seed=4)
    check_hash_partition(small, [0], 5000)
    check_hash_partition(small, [0, 1], 16384)


def test_one_row_per_partition():
    """Table.partition with ids that are a permutation of 0 .. P - 1."""
    _check_partition_by_ids(1024, np.random.default_rng(1).permutation(1024).astype(np.int32))
    _check_partition_by_ids(16384, np.random.default_rng(2).permutation(16384).astype(np.int32))


@pytest.mark.parametrize("t", list(E.EDGES))
def test_keys_of_every_murmur3_type(t):
    keys = E.edge_cols([t, O.INT64], 3000, nulls=[0.2, None], seed=t)
    vals = random_table([O.STRING, O.INT16], 3000, seed=t)
    check_hash_partition(keys + vals, [0, 1], 1025)
    check_hash_partition(keys + vals, [0], 33)


def _check_partition_by_ids(P, ids):
    G = _gpu()
    import srj_b200 as S
    from srj_b200.partitioning import partition
    n = len(ids)
    cols = _wide(20, n, seed=P)
    offs, gather, _ = M.stable_partition(ids.tolist(), P)
    pmap = S.ColumnVector(S.DType.INT32, n, torch.from_numpy(ids).cuda().view(torch.uint8))
    pt = partition(G.table_to_device(cols), pmap, P)
    assert pt.getPartitions() == offs[:-1]
    for i, (g, c) in enumerate(zip(pt.getTable().columns, cols)):
        assert_column_exact(g, M.take(c, gather), f"P={P} column {i}")


@pytest.mark.parametrize("P", [1024, 1025, 16384])
def test_table_partition_by_caller_ids_uses_every_partition(P):
    n = 3 * P + 17
    ids = (np.random.default_rng(P).permutation(n) % P).astype(np.int32)
    assert len(set(ids.tolist())) == P
    _check_partition_by_ids(P, ids)


def test_partition_is_a_permutation_at_scale_with_16384_partitions():
    """8M rows at the partition limit: ids, offsets = histogram, grouped, stable, inverse maps."""
    _gpu()
    import srj_b200 as S
    from srj_b200 import _native as N
    n, P = 8_000_000, 16384
    g = torch.Generator(device="cuda").manual_seed(11)
    key = torch.randint(-2**31, 2**31 - 1, (n,), dtype=torch.int32, device="cuda", generator=g)
    kc = S.ColumnVector(S.DType.INT32, n, key.view(torch.uint8))
    lib = N.lib()
    ws = torch.empty(lib.srj_partition_workspace_bytes(n, P), dtype=torch.uint8, device="cuda")
    ids = torch.empty(n, dtype=torch.int32, device="cuda")
    offs = torch.empty(P + 1, dtype=torch.int32, device="cuda")
    smap = torch.empty(n, dtype=torch.int32, device="cuda")
    gmap = torch.empty(n, dtype=torch.int32, device="cuda")
    arr = (N.SrjColumn * 1)(kc._c())
    N.check(lib.srj_hash_partition(arr, 1, n, C.c_uint32(42), P, ids.data_ptr(), offs.data_ptr(), smap.data_ptr(), gmap.data_ptr(),
                                   ws.data_ptr(), int(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    h = S.Hash.murmurHash32(42, [kc]).data.view(torch.int32)
    assert torch.equal(ids, torch.remainder(h.to(torch.int64), P).to(torch.int32))
    assert torch.equal(offs[1:] - offs[:-1], torch.bincount(ids, minlength=P).to(torch.int32)) and int(offs[0]) == 0
    assert torch.equal(smap[gmap.long()], torch.arange(n, dtype=torch.int32, device="cuda"))
    pid_sorted = ids[gmap.long()]
    assert bool((pid_sorted[1:] >= pid_sorted[:-1]).all())
    same = pid_sorted[1:] == pid_sorted[:-1]
    assert bool((gmap[1:][same] > gmap[:-1][same]).all())
    # and a sample of rows against the model's hash
    rows = np.random.default_rng(3).integers(0, n, 2000)
    kh = key.cpu().numpy()
    want = [M.H.pmod(M.H.murmur_int(int(kh[r]), 42) - (1 << 32) * (M.H.murmur_int(int(kh[r]), 42) >> 31), P) for r in rows]
    assert ids.cpu().numpy()[rows].tolist() == want
