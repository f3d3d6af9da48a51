"""CPU checks of oracle/zorder.py against the independent model (tests/zorder_model.py), the reference's test inputs and
the hand-derived answers (tests/golden/zorder_golden.py), and the Hilbert curve's defining properties."""
import itertools

import numpy as np
import pytest

from golden import zorder_golden as G
from oracle import zorder as Z
import zorder_model as M

NP = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _col(values, width):
    """(raw little-endian bytes, cudf mask or None) of a list of Python ints / None"""
    rows = len(values)
    raw = b"".join(((v or 0) & ((1 << (8 * width)) - 1)).to_bytes(width, "little") for v in values)
    mask = None
    if any(v is None for v in values):
        bits = np.array([v is not None for v in values] + [False] * (-rows % 32), dtype=np.uint8)
        mask = np.packbits(bits, bitorder="little").view(np.uint32)
    return np.frombuffer(raw, dtype=np.uint8).copy(), mask


def _oracle_rows(columns, width, rows):
    offs, data = Z.interleave_bits([_col(c, width) for c in columns], width, rows)
    return offs, [data[offs[r]:offs[r + 1]].tobytes() for r in range(rows)]


@pytest.mark.parametrize("case", G.INTERLEAVE, ids=[c[0] for c in G.INTERLEAVE])
def test_interleave_golden_inputs_model_and_oracle_agree(case):
    _, width, rows, columns = case
    if not columns:                                    # the Java wrapper: numRows empty lists, no native call
        with pytest.raises(ValueError):
            Z.interleave_bits([], width, rows)
        return
    offs, got = _oracle_rows(columns, width, rows)
    assert offs.tolist() == [r * width * len(columns) for r in range(rows + 1)]
    for r in range(rows):
        assert got[r] == M.interleave_row([c[r] for c in columns], width)


@pytest.mark.parametrize("width,values,want", G.INTERLEAVE_KNOWN)
def test_interleave_known_answers(width, values, want):
    assert M.interleave_row(values, width) == want
    assert _oracle_rows([[v] for v in values], width, 1)[1][0] == want


def test_decimal128_single_column_is_its_bytes_reversed():
    v = int.from_bytes(G.DECIMAL128_BYTES, "little")
    assert M.interleave_row([v], 16) == G.DECIMAL128_BYTES[::-1]
    assert _oracle_rows([[v]], 16, 1)[1][0] == G.DECIMAL128_BYTES[::-1]


@pytest.mark.parametrize("width", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("ncols", [1, 2, 3, 5, 7, 9, 17, 33])
def test_interleave_oracle_matches_model_on_random_rows(width, ncols):
    rng = np.random.default_rng(width * 100 + ncols)
    rows = 40
    columns = [[None if rng.random() < 0.2 else int.from_bytes(rng.bytes(width), "little", signed=True) for _ in range(rows)]
               for _ in range(ncols)]
    _, got = _oracle_rows(columns, width, rows)
    for r in range(rows):
        assert got[r] == M.interleave_row([c[r] for c in columns], width)


def _hilbert_oracle(num_bits, columns, rows):
    return Z.hilbert_index(num_bits, [_col(c, 4) for c in columns], rows)


@pytest.mark.parametrize("case", G.HILBERT, ids=[c[0] for c in G.HILBERT])
def test_hilbert_golden_inputs_model_and_oracle_agree(case):
    _, num_bits, rows, columns = case
    if not columns:                                    # the Java wrapper: numRows zeros, no native call
        with pytest.raises(ValueError):
            Z.hilbert_index(num_bits, [], rows)
        return
    got = _hilbert_oracle(num_bits, columns, rows)
    want = [M.to_int64(M.hilbert_row([c[r] for c in columns], num_bits)) for r in range(rows)]
    assert got.tolist() == want


@pytest.mark.parametrize("num_bits,values,want", G.HILBERT_KNOWN)
def test_hilbert_known_answers(num_bits, values, want):
    assert M.hilbert_row(values, num_bits) == want
    assert _hilbert_oracle(num_bits, [[v] for v in values], 1).tolist() == [want]


@pytest.mark.parametrize("n,bits", [(2, b) for b in range(1, 7)] + [(3, b) for b in range(1, 5)] + [(4, b) for b in range(1, 4)])
def test_hilbert_curve_properties_exhaustive(n, bits):
    pts = list(itertools.product(range(1 << bits), repeat=n))
    idx = _hilbert_oracle(bits, [[p[c] for p in pts] for c in range(n)], len(pts)).astype(np.uint64)
    assert sorted(idx.tolist()) == list(range(1 << (n * bits)))             # a bijection onto [0, 2^(N * bits))
    assert idx[0] == 0                                                       # the origin comes first
    order = np.empty(len(pts), dtype=np.int64)
    order[idx.astype(np.int64)] = np.arange(len(pts))
    walk = np.array(pts)[order]
    assert (np.abs(np.diff(walk, axis=0)).sum(axis=1) == 1).all()            # consecutive indexes are neighbours
    sample = range(0, len(pts), max(1, len(pts) // 64))
    assert [M.hilbert_row(list(pts[i]), bits) for i in sample] == [int(idx[i]) for i in sample]


def test_hilbert_masks_values_and_nulls():
    vals = [[-1, 2**31 - 1, -2**31, 37, None], [5, None, 1 << 20, -7, 3]]
    for bits in (1, 5, 21, 32):
        got = _hilbert_oracle(bits, vals, 5).tolist()
        assert got == [M.to_int64(M.hilbert_row([c[r] for c in vals], bits)) for r in range(5)]


def test_hilbert_full_64_bit_shapes():
    rng = np.random.default_rng(7)
    for n in (1, 2, 4, 8, 16, 32, 64):
        bits = min(32, 64 // n) if n > 1 else 32
        cols = [[int(v) for v in rng.integers(-2**31, 2**31, 8)] for _ in range(n)]
        got = _hilbert_oracle(bits, cols, 8).tolist()
        assert got == [M.to_int64(M.hilbert_row([c[r] for c in cols], bits)) for r in range(8)]
