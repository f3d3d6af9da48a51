"""GPU tests of the Kudo split / assemble kernels (csrc/kudo.cu) at their dispatch and bit-offset edges, byte-exact
against the independent model (tests/shuffle_model.py) and the reference's flat shuffle cases (tests/golden/kudo_golden.py):
partition counts past one 1024-wide scan chunk up to 65535, 1 to 256 columns, chars sections at every offset mod 16,
buffers that start off 16-byte alignment, every validity slice assembled at every output bit offset, masked and unmasked
partitions in one assemble, hash partition -> split -> assemble, and the refused arguments.

Assembled columns are compared whole: values including null payload bytes, STRING offsets, mask words with their tail
bits, and null counts.  The host mirror gives every assembled column a mask, also when no partition carried validity (the
reference then gives the column none); such a column must come back with every bit set and no nulls."""
import numpy as np
import pytest
import torch

import shuffle_model as M
from golden import kudo_golden as KG
from oracle import kudo as K
from oracle import oracle as O
from util import random_table

pytestmark = pytest.mark.gpu

TYPES = [O.INT32, O.STRING, O.INT64, O.DECIMAL128, O.INT8, O.STRING, O.FLOAT64, O.INT16, O.BOOL8]


def _gpu():
    import gpu_util
    gpu_util.require_cuda()
    return gpu_util


def split_on_device(cols, splits):
    G = _gpu()
    from srj_b200.kudo import KudoGpuSerializer as KS
    buf, offs = KS.splitAndSerializeToDevice(G.table_to_device(cols), splits)
    return buf, offs


def check_split(cols, splits):
    """Device split == model split, byte for byte."""
    buf, offs = split_on_device(cols, splits)
    want, want_offs = M.split(cols, splits)
    assert offs.cpu().tolist() == want_offs
    got = buf.cpu().numpy().tobytes()
    if got != want:
        d = next(i for i in range(min(len(got), len(want))) if got[i] != want[i])
        raise AssertionError(f"split bytes differ first at {d} of {len(want)}")
    return buf, offs


def assemble_on_device(types, buf, offs):
    import srj_b200 as S
    from srj_b200.kudo import KudoGpuSerializer as KS
    if not isinstance(buf, torch.Tensor):
        buf = torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).cuda()
        offs = torch.tensor(list(offs), dtype=torch.int64, device="cuda")
    return KS.assembleFromDeviceRaw([S.DType(t) for t in types], buf, offs)


def check_assembled(tbl, want, what=""):
    G = _gpu()
    assert tbl.getRowCount() == (want[0].size if want else 0)
    for i, (g, w) in enumerate(zip(tbl.columns, want)):
        h = G.to_host(g)
        n = w.size
        assert M._bytes(h.data)[:len(w.data)] == w.data and (h.data is None or h.data.nbytes == len(w.data)), f"{what} column {i}: data"
        if w.type_id == O.STRING:
            assert h.offsets.tolist() == w.offsets, f"{what} column {i}: offsets"
        assert h.mask is not None, f"{what} column {i}: the mirror allocates a mask for every column"
        assert M._bytes(h.mask)[:4 * ((n + 31) // 32)] == w.mask_words(), f"{what} column {i}: mask words"
        assert g.getNullCount() == w.null_count(), f"{what} column {i}: null count"
        if not w.nullable:
            assert g.getNullCount() == 0 and all(w.valid), f"{what} column {i}: a column without validity has no nulls"


def round_trip(cols, splits, what=""):
    buf, offs = check_split(cols, splits)
    tbl = assemble_on_device([c.type_id for c in cols], buf, offs)
    check_assembled(tbl, M.assemble(buf.cpu().numpy().tobytes(), offs.cpu().tolist(), [c.type_id for c in cols]), what)
    check_assembled(tbl, M.concat_slices([cols], [(0, a, b - a) for a, b in zip(splits, splits[1:])]), what + " vs input")


# ---- the goldens ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", KG.CASES, ids=[c["name"] for c in KG.CASES])
def test_golden_cases_on_the_device(case):
    tables, parts, want = M.golden_tables(case)
    types = [c.type_id for c in tables[0]]
    buf, offs = M.write_parts(tables, parts)
    if len(tables) == 1 and [s for _, s, _ in parts] == [0] + [s + n for _, s, n in parts[:-1]] and len(parts) > 0:
        dbuf, doffs = check_split(tables[0], [0] + [s + n for _, s, n in parts])     # a split case: the device writes it
        assert dbuf.cpu().numpy().tobytes() == buf
    check_assembled(assemble_on_device(types, buf, offs), want, case["name"])


@pytest.mark.parametrize("name", list(KG.CONCAT_SCHEDULES))
def test_concat_validity_schedules_on_the_device(name):
    rng = np.random.Generator(np.random.Philox(len(name)))
    tables, parts = [], []
    for s, n in KG.CONCAT_SCHEDULES[name]:
        rows = (s or 0) + n
        bits = (rng.random(rows) < 0.5).tolist()
        vals = rng.integers(0, 256, rows, dtype=np.uint8)
        tables.append([M.HostCol(O.INT8, vals, None if s is None else M.pack_valid(bits), None, 0, rows)])
        parts.append((len(tables) - 1, s or 0, n))
    buf, offs = M.write_parts(tables, parts)
    check_assembled(assemble_on_device([O.INT8], buf, offs), M.concat_slices(tables, parts), name)


# ---- partition and column counts ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1023, 1024, 1025, 4097, 65535])
def test_many_partitions_most_empty(P):
    """The offsets and row bases scan P + 1 values in chunks of 1024 with a carry."""
    n = 5000
    cols = random_table(TYPES, n, seed=P)
    rng = np.random.default_rng(P)
    cuts = sorted(rng.integers(0, n + 1, 60).tolist())
    slots = sorted(rng.choice(np.arange(1, P), 60, replace=False).tolist())
    splits = [0] * (P + 1)
    for k in range(1, P + 1):
        j = np.searchsorted(slots, k, side="right")
        splits[k] = cuts[j - 1] if j else 0
    splits[P] = n
    round_trip(cols, splits, f"P={P}")


def test_partition_count_limit():
    import srj_b200 as S
    cols = random_table([O.INT32], 10, seed=1)
    with pytest.raises(S.CudfException, match="65535"):
        split_on_device(cols, [0] * 65536 + [10])
    buf, offs = M.split(cols, [0, 10])
    big = np.zeros(65537, np.int64)
    big[1:] = offs[1]
    with pytest.raises(S.CudfException, match="65535"):
        assemble_on_device([O.INT32], torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).cuda(), torch.from_numpy(big).cuda())


@pytest.mark.parametrize("ncols", [1, 7, 8, 9, 255, 256])
def test_column_counts(ncols):
    types = [TYPES[c % len(TYPES)] for c in range(ncols)]
    cols = random_table(types, 300, seed=ncols, all_valid_cols=range(0, ncols, 4))
    round_trip(cols, [0, 0, 1, 8, 9, 17, 100, 299, 300], f"ncols={ncols}")


def test_validity_padding_takes_every_value():
    """Masked column counts and slice lengths that put the zero padding after the validity buffers at 0, 1, 2 and 3
    bytes: the device writes every one of them as the model does."""
    seen = set()
    for ncols in M.PADDING_COLUMN_COUNTS:
        splits = [0]
        for n in M.PADDING_ROW_COUNTS:
            splits.append(splits[-1] + n)
        cols = random_table([O.INT32] * ncols, splits[-1], seed=ncols, null_frac=0.3)
        buf, offs = check_split(cols, splits)
        b, o = buf.cpu().numpy().tobytes(), offs.cpu().tolist()
        seen |= {M.validity_padding(b[o[p]:o[p + 1]]) for p in range(len(splits) - 1)}
        check_assembled(assemble_on_device([O.INT32] * ncols, buf, offs), M.concat_slices([cols], [(0, a, c - a) for a, c in zip(splits, splits[1:])]))
    assert seen == {0, 1, 2, 3}


def test_column_count_limit():
    import srj_b200 as S
    cols = random_table([O.INT8] * 257, 20, seed=2)
    with pytest.raises(S.CudfException, match="256"):
        split_on_device(cols, [0, 20])
    buf, offs = M.split(cols[:256], [0, 20])
    with pytest.raises(S.CudfException, match="256"):
        assemble_on_device([O.INT8] * 257, buf, offs)


# ---- alignment of the copies ---------------------------------------------------------------------------------------------------
def _strings(lens, seed):
    rng = np.random.default_rng(seed)
    offs = np.zeros(len(lens) + 1, np.int32)
    offs[1:] = np.cumsum(lens)
    return M.HostCol(O.STRING, rng.integers(0, 256, int(offs[-1]), dtype=np.uint8), None, offs, 0, len(lens))


def test_chars_at_every_offset_mod_16():
    """One-string partitions of 0 to 48 chars and of about 5 KB, whose chars start at every offset mod 16 of the input,
    behind a masked INT8 column that moves where the chars land in the partition."""
    lens = [L for k in range(3) for L in range(49)] + [5000, 5003, 4999, 5121] + list(range(17))
    s = _strings(lens, 1)
    cols = [random_table([O.INT8], len(lens), seed=3)[0], s]
    starts = s.offsets[:-1]
    assert {int(x) % 16 for x in starts} == set(range(16))
    round_trip(cols, list(range(len(lens) + 1)), "one string per partition")
    round_trip([s], [0, 3, 3, 50, 51, 100, 150, 152, len(lens) - 10, len(lens)], "a few partitions")


@pytest.mark.parametrize("shift", [4, 8, 12])
def test_assemble_from_a_buffer_off_16_byte_alignment(shift):
    cols = random_table(TYPES, 3000, seed=shift)
    splits = [0, 1, 700, 701, 2500, 3000]
    buf, offs = M.split(cols, splits)
    big = torch.zeros(len(buf) + 64, dtype=torch.uint8, device="cuda")
    assert big.data_ptr() % 16 == 0
    big[shift:shift + len(buf)] = torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).cuda()
    view = big[shift:shift + len(buf)]
    tbl = assemble_on_device(TYPES, view, torch.tensor(offs, dtype=torch.int64, device="cuda"))
    check_assembled(tbl, M.assemble(buf, offs, TYPES), f"+{shift}")


def test_strings_without_chars():
    s = M.HostCol(O.STRING, np.zeros(0, np.uint8), None, np.zeros(41, np.int32), 0, 40)
    masked = M.HostCol(O.STRING, np.zeros(0, np.uint8), M.pack_valid([i % 3 != 0 for i in range(40)]), np.zeros(41, np.int32), 0, 40)
    round_trip([s, masked], [0, 0, 13, 40], "no chars")
    round_trip([s], [0, 40], "no chars, one partition")


# ---- validity ---------------------------------------------------------------------------------------------------------------------
def test_every_validity_slice_at_every_output_bit_offset():
    """8 row offsets mod 8 x 40 lengths x 32 output offsets mod 32: 10,240 masked slices, each behind a slice of an
    unmasked table that moves the output row, in one assemble of 20,480 partitions; partitions of neighbouring slices
    share output words."""
    tables, parts = M.validity_slice_schedule(lambda rows: random_table([O.INT16], rows, seed=1, null_frac=0.5),
                                              lambda rows: random_table([O.INT16], rows, seed=2, null_frac=0.0))
    buf, offs = M.write_parts(tables, parts)
    want = M.concat_slices(tables, parts)
    check_assembled(assemble_on_device([O.INT16], buf, offs), want, "validity slices")


def test_masked_and_unmasked_partitions_in_one_assemble():
    a = random_table(TYPES, 3000, seed=7)
    b = random_table(TYPES, 2000, seed=8, null_frac=0.0)
    parts = [(0, 1234, 1766), (1, 0, 77), (0, 0, 1234), (1, 77, 1), (1, 78, 0), (0, 5, 33)]
    buf, offs = M.write_parts([a, b], parts)
    check_assembled(assemble_on_device(TYPES, buf, offs), M.concat_slices([a, b], parts), "mixed")
    # only unmasked partitions: the reference's column would not be nullable
    parts = [(1, 0, 1000), (1, 1000, 1000)]
    buf, offs = M.write_parts([a, b], parts)
    want = M.concat_slices([a, b], parts)
    assert not any(w.nullable for w in want)
    check_assembled(assemble_on_device(TYPES, buf, offs), want, "unmasked")


@pytest.mark.parametrize("P", [1025, 16384])
def test_hash_partition_split_assemble(P):
    G = _gpu()
    from srj_b200.partitioning import HashPartitioner
    n = 40_000
    cols = random_table(TYPES, n, seed=P)
    pt = HashPartitioner.partition(G.table_to_device(cols), [0, 2], P)
    splits = pt.getPartitions() + [n]
    ids = O.partition_ids([cols[0], cols[2]], P)
    want_cols, want_offs, _ = O.stable_partition(cols, ids, P)
    assert splits == want_offs.tolist()
    from srj_b200.kudo import KudoGpuSerializer as KS
    buf, offs = KS.splitAndSerializeToDevice(pt.getTable(), splits)
    wbuf, woffs = K.split(want_cols, want_offs)
    assert offs.cpu().tolist() == woffs.tolist() and buf.cpu().numpy().tobytes() == wbuf.tobytes()
    tbl = assemble_on_device(TYPES, buf, offs)
    check_assembled(tbl, M.concat_slices([want_cols], [(0, 0, n)]), f"P={P}")


# ---- refused arguments ----------------------------------------------------------------------------------------------------------
def test_splits_outside_the_table_are_refused():
    import srj_b200 as S
    cols = random_table([O.INT32, O.STRING], 100, seed=1)
    for splits in ([-1, 50, 100], [0, 50, 101], [0, 100, 200], [-8, -4, 100]):
        with pytest.raises(S.CudfException, match=r"\[0, 100\]"):
            split_on_device(cols, splits)
    with pytest.raises(S.CudfColumnSizeOverflowException):
        split_on_device(cols, [0, 60, 40, 100])
    check_split(cols, [0, 100])
