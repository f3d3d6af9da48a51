"""JoinPrimitives goldens: the cases of the reference's JoinPrimitivesTest.java (sort-merge cases reused as hash-join cases,
since their pair sets are the same), plus hand-derived rows for NaN payloads, -0.0 against 0.0, null against the empty
string and the helpers' sentinels, duplicates and empty maps.

INNER: (name, left keys, right keys, nulls_equal, expected pairs as a sorted list of (left, right)); a key list is one
column, None a null.  HELPERS: (name, left map, right map, left size, right size) with the expected outputs of every
helper."""
INT32_MIN = -2 ** 31
NAN_A, NAN_B = 0x7ff8000000000000, 0x7ff8000000000123            # FLOAT64 bit patterns
NEG_ZERO = 0x8000000000000000

INNER = [
    ("inner_join", ("INT32", [0, 1, 2, 3]), ("INT32", [1, 2, 4]), True, [(1, 0), (2, 1)]),
    ("nulls_unequal", ("INT32", [None, 1, 2]), ("INT32", [None, 1, 3]), False, [(1, 1)]),
    ("nulls_equal", ("INT32", [None, 1, 2]), ("INT32", [None, 1, 3]), True, [(0, 0), (1, 1)]),
    ("no_match", ("INT32", [0, 1, 2]), ("INT32", [5, 6, 7]), True, []),
    ("left_outer_source", ("INT32", [1, 3]), ("INT32", [1, 5]), True, [(0, 0)]),
    ("semi_source", ("INT32", [1, 1, 2, 3]), ("INT32", [1, 2]), True, [(0, 0), (1, 0), (2, 1)]),
    ("matched_rows_source", ("INT32", [1, 2, 3, 4, 5, 6, 7]), ("INT32", [2, 4, 4, 6]), True, [(1, 0), (3, 1), (3, 2), (5, 3)]),
    # hand-derived
    ("nan_payloads", ("FLOAT64_BITS", [NAN_A, NAN_B, 0]), ("FLOAT64_BITS", [NAN_B, NEG_ZERO]), False, [(0, 0), (1, 0), (2, 1)]),
    ("null_vs_empty_string", ("STRING", [b"", None, b"a"]), ("STRING", [None, b""]), True, [(0, 1), (1, 0)]),
    ("null_vs_empty_string_unequal", ("STRING", [b"", None, b"a"]), ("STRING", [None, b""]), False, [(0, 1)]),
]

# (name, L, R, left size, right size, left outer, full outer, semi of L, anti of L, matched rows of R)
HELPERS = [
    ("left_outer", [1, 2], [0, 1], 4, 3, ([1, 2, 0, 3], [0, 1, INT32_MIN, INT32_MIN]),
     ([1, 2, 0, 3, INT32_MIN], [0, 1, INT32_MIN, INT32_MIN, 2]), [1, 2], [0, 3], [1, 1, 0]),
    ("full_outer", [0], [0], 2, 2, ([0, 1], [0, INT32_MIN]), ([0, 1, INT32_MIN], [0, INT32_MIN, 1]), [0], [1], [1, 0]),
    ("duplicates", [0, 1, 2], [0, 0, 1], 4, 2, ([0, 1, 2, 3], [0, 0, 1, INT32_MIN]), ([0, 1, 2, 3], [0, 0, 1, INT32_MIN]), [0, 1, 2], [3],
     [1, 1]),
    ("sentinels", [0, INT32_MIN, 2], [INT32_MIN, 0, -1], 3, 1, ([0, INT32_MIN, 2, 1], [INT32_MIN, 0, -1, INT32_MIN]),
     ([0, INT32_MIN, 2, 1], [INT32_MIN, 0, -1, INT32_MIN]), [0, 2], [1], [1]),
    ("empty_maps", [], [], 3, 3, ([0, 1, 2], [INT32_MIN] * 3), ([0, 1, 2] + [INT32_MIN] * 3, [INT32_MIN] * 3 + [0, 1, 2]), [], [0, 1, 2],
     [0, 0, 0]),
    ("empty_tables", [], [], 0, 0, ([], []), ([], []), [], [], []),
]
