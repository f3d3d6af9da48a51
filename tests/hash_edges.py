"""Edge values of every hash key type, and tables tiled from them.

Random bytes almost never reach the values where the element rules of the row hashes branch: short DECIMAL128 byte
strings, BOOL8 bytes other than 0 / 1, NaN payloads, -0.0, subnormals, negative timestamps that are not whole seconds,
string tails with the high bit set.  Each list below holds those values for one type; `edge_cols` tiles them into
columns of any length, rotated per column so that a row mixes different edges.

The dispatch constants of csrc/hash.cu that the GPU edge tests size their tables from are kept here as well (and
checked against the source by test_hash_model.py)."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

# csrc/hash.cu: rows per streaming chunk, key columns per streaming launch, key columns per launch.  The streaming
# kernel takes tables from STREAM_MIN_ROWS rows on, if at least two stages of one chunk fit in STAGE_BUDGET bytes of
# shared memory.
HS_ROWS = 2048
HS_MAX_COLS = 16
HASH_COLS_PER_LAUNCH = 48
STREAM_MIN_ROWS = 4 * HS_ROWS
STAGE_BUDGET = 200 * 1024


def _ints(bits: int, signed: bool):
    if signed:
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        return [lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi]
    top = 1 << (bits - 1)
    return [0, 1, top - 1, top, top + 1, (1 << bits) - 1]


def _dec128():
    v = {0, 1, -1, (1 << 127) - 1, -(1 << 127)}
    for k in range(1, 17):
        p = 1 << (8 * k - 1)                     # every minimal BigInteger byte length, both signs
        v.update({p - 1, p, p + 1, -p - 1, -p, -p + 1})
    for p in (1 << 63, 1 << 64):                 # the two 64-bit halves of the value
        v.update({p - 1, p, p + 1, -p - 1, -p, -p + 1})
    return sorted(x for x in v if -(1 << 127) <= x < (1 << 127))


F32_BITS = [
    0x00000000, 0x80000000,                      # +-0
    0x7F800000, 0xFF800000,                      # +-inf
    0x7FC00000, 0x7FFFFFFF, 0xFFC00000, 0xFFFFFFFF,  # quiet NaN, both signs, lowest and highest payload
    0x7F800001, 0x7FBFFFFF, 0xFF800001, 0xFFBFFFFF,  # signalling NaN, both signs, lowest and highest payload
    0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF,  # smallest and largest subnormal
    0x00800000, 0x80800000, 0x7F7FFFFF, 0xFF7FFFFF,  # min normal, max
    0x3F800000, 0xBF800000,                      # +-1
]
F64_BITS = [
    0x0000000000000000, 0x8000000000000000,
    0x7FF0000000000000, 0xFFF0000000000000,
    0x7FF8000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFF8000000000000, 0xFFFFFFFFFFFFFFFF,
    0x7FF0000000000001, 0x7FF7FFFFFFFFFFFF, 0xFFF0000000000001, 0xFFF7FFFFFFFFFFFF,
    0x0000000000000001, 0x8000000000000001, 0x000FFFFFFFFFFFFF, 0x800FFFFFFFFFFFFF,
    0x0010000000000000, 0x8010000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF,
    0x3FF0000000000000, 0xBFF0000000000000,
]
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
TS_US = [0, 1, -1, 999_999, -999_999, 1_000_000, -1_000_000, 1_000_001, -1_000_001, -1_500_000, -123_456_789,
         -86_400_000_001, 1_700_000_000_123_456, -62_135_596_800_000_001, I64_MIN, I64_MIN + 1, I64_MAX]


def _string(n: int, k: int = 0) -> bytes:
    """n bytes: printable ASCII at the front, bytes >= 0x80 in the last seven positions (every tail murmur, hive and
    the XXH64 4- and 1-byte steps read sign-extended or byte by byte)."""
    return bytes((0x80 | ((i * 29 + n + k) & 0x7F)) if i >= n - 7 else 32 + (i * 37 + n + k) % 95 for i in range(n))


STRINGS = [_string(n) for n in range(81)] + [b"\xff" * 9, b"\x80" * 4, "é휠".encode()]

EDGES = {
    O.BOOL8: [0, 1, 2, 0x7F, 0x80, 0xFF],
    O.INT8: _ints(8, True), O.INT16: _ints(16, True), O.INT32: _ints(32, True), O.INT64: _ints(64, True),
    O.UINT8: _ints(8, False), O.UINT16: _ints(16, False), O.UINT32: _ints(32, False), O.UINT64: _ints(64, False),
    O.FLOAT32: F32_BITS, O.FLOAT64: F64_BITS,
    O.TIMESTAMP_DAYS: _ints(32, True),
    O.TIMESTAMP_SECONDS: _ints(64, True), O.TIMESTAMP_MILLISECONDS: _ints(64, True),
    O.TIMESTAMP_MICROSECONDS: TS_US, O.TIMESTAMP_NANOSECONDS: _ints(64, True),
    O.DECIMAL32: _ints(32, True), O.DECIMAL64: _ints(64, True), O.DECIMAL128: _dec128(),
    O.STRING: STRINGS,
}
FIXED_TYPES = [t for t in EDGES if t != O.STRING]
HIVE_TYPES = [O.BOOL8, O.INT8, O.INT16, O.INT32, O.INT64, O.FLOAT32, O.FLOAT64, O.TIMESTAMP_DAYS,
              O.TIMESTAMP_MICROSECONDS, O.STRING]
SIZE = {t: (0 if t == O.STRING else O.size_of(t)) for t in EDGES}


def edge_indices(nedges: int, nrows: int, ci: int) -> np.ndarray:
    """Which edge value row r of column ci holds: every pass over the list starts somewhere else, and neighbouring
    columns are rotated against each other."""
    r = np.arange(nrows, dtype=np.int64)
    return (r + 5 * ci + (r // nedges) * (2 * ci + 1)) % nedges


def null_mask(nrows: int, nulls, rng) -> np.ndarray | None:
    """nulls: None (no mask), "all", or a fraction of null rows.  A mask with no null bit is still a mask."""
    if nulls is None:
        return None
    if nulls == "all":
        return O.pack_mask(np.zeros(nrows, bool))
    return O.pack_mask(rng.random(nrows) >= float(nulls))


def edge_col(t: int, nrows: int, ci: int = 0, nulls=None, seed: int = 0) -> O.HCol:
    vals = EDGES[t]
    idx = edge_indices(len(vals), nrows, ci)
    mask = null_mask(nrows, nulls, np.random.Generator(np.random.Philox(seed * 1000 + ci)))
    if t == O.STRING:
        lens = np.array([len(v) for v in vals], np.int64)[idx]
        offs = np.zeros(nrows + 1, np.int32)
        np.cumsum(lens, out=offs[1:])
        chars = np.frombuffer(b"".join(vals[i] for i in idx), np.uint8).copy() if nrows else np.zeros(0, np.uint8)
        return O.HCol(t, chars, mask, offs, 0, nrows)
    sz = SIZE[t]
    table = np.frombuffer(b"".join(int(v).to_bytes(sz, "little", signed=v < 0) for v in vals), np.uint8).reshape(-1, sz)
    data = table[idx].reshape(-1).copy()
    return O.HCol(t, data, mask, None, -11 if t == O.DECIMAL128 else (-2 if t in (O.DECIMAL32, O.DECIMAL64) else 0), nrows)


def edge_cols(types, nrows: int, nulls=None, seed: int = 0) -> list:
    """One column per type id in `types`, tiled from the edge lists.  `nulls` is one pattern for every column or a
    list with one pattern per column (see null_mask)."""
    pats = nulls if isinstance(nulls, (list, tuple)) else [nulls] * len(types)
    return [edge_col(t, nrows, ci, pats[ci], seed) for ci, t in enumerate(types)]


def hive_ok(cols) -> list:
    return [c for c in cols if c.type_id in HIVE_TYPES]


def streams(cols) -> bool:
    """Whether launch_hash_stream (csrc/hash.cu) takes these key columns of one launch, given 16-byte aligned buffers:
    enough rows, at most HS_MAX_COLS fixed-width keys, and two stages of a chunk (values + 256-byte mask pieces,
    rounded up to 128 bytes) within STAGE_BUDGET."""
    if not cols or cols[0].size < STREAM_MIN_ROWS or len(cols) > HS_MAX_COLS or any(SIZE[c.type_id] == 0 for c in cols):
        return False
    stage = sum(HS_ROWS * SIZE[c.type_id] + (256 if c.mask is not None else 0) for c in cols)
    return STAGE_BUDGET // ((stage + 127) // 128 * 128) >= 2


# ---------------------------------------------------------------- nested keys with edge leaves
def _list(rng, nrows: int, child_builder, null_frac: float) -> O.HCol:
    """LIST column of 0-4 elements per row; a null row keeps its elements (a non-empty span under a null)."""
    lens = rng.integers(0, 5, nrows)
    offs = np.zeros(nrows + 1, np.int32)
    np.cumsum(lens, out=offs[1:])
    return O.list_col(offs, child_builder(int(offs[-1])), valid=rng.random(nrows) >= null_frac)


def nested_edge_keys(nrows: int, seed: int = 0) -> dict:
    """Nested key columns over edge leaves, with LIST and STRUCT level nulls set on rows that have children:
    name -> HCol.  "list_of_struct" is not hashable by murmur3."""
    rng = np.random.Generator(np.random.Philox(seed))
    leaf = lambda t, ci: (lambda n: edge_col(t, n, ci, 0.2, seed))   # noqa: E731

    def struct(fields, n, null_frac):
        return O.struct_col(*fields, valid=rng.random(n) >= null_frac)

    return {
        "list_decimal128": _list(rng, nrows, leaf(O.DECIMAL128, 1), 0.3),
        "list_list_string": _list(rng, nrows, lambda n: _list(rng, n, leaf(O.STRING, 2), 0.3), 0.2),
        "struct_bool_double_string": struct([edge_col(O.BOOL8, nrows, 3, 0.2, seed), edge_col(O.FLOAT64, nrows, 4, None, seed),
                                              edge_col(O.STRING, nrows, 5, 0.1, seed)], nrows, 0.3),
        "struct_of_struct_and_list": struct([edge_col(O.INT8, nrows, 6, None, seed),
                                             struct([edge_col(O.FLOAT32, nrows, 7, 0.2, seed)], nrows, 0.3),
                                             _list(rng, nrows, leaf(O.TIMESTAMP_MICROSECONDS, 8), 0.2)], nrows, 0.3),
        "list_of_struct": _list(rng, nrows, lambda n: struct([edge_col(O.FLOAT32, n, 9, 0.2, seed),
                                                              edge_col(O.INT64, n, 10, None, seed)], n, 0.3), 0.3),
    }


def nested_hive_ok(col: O.HCol) -> bool:
    """hive hashes only its own leaf types (no DECIMAL128)."""
    def ok(c):
        return all(ok(k) for k in c.children) if c.type_id in (O.LIST, O.STRUCT) else c.type_id in HIVE_TYPES
    return ok(col)
