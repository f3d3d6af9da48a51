"""Kudo split / assemble goldens: the reference's flat shuffle cases, transcribed as data.

Sources (the reference repository):
  CPP   src/main/cpp/tests/shuffle_split.cu         Simple, Strings, SimpleWithStrings, Nulls, ShortNulls, PurgeNulls,
                                                    EmptySplits, EmptyInputs, FixedPoint, MixedValidity
  JAVA  src/test/java/com/nvidia/spark/rapids/jni/kudo/KudoSerializerTest.java
                                                    testMergeTableWithDifferentValidity, testMergeString,
                                                    testSerializeValidity
  CONCAT src/test/java/com/nvidia/spark/rapids/jni/kudo/KudoConcatValidityTest.java
                                                    the (start row, length) schedules of cases 1-8, testConcatValidity
                                                    and testConcatValidityWithEmpty
Skipped, because they hold LIST or STRUCT columns, which this project's Kudo path does not carry: Lists, Struct,
EmptyOffsets, NestedTypes, Reshaping, NestedTerminatingEmptyPartition, EmptyPartitionsWithNulls (a LIST column) and
LargeBatchSimple (a 2^31-row batch) of shuffle_split.cu; testMergeList, testMergeComplexStructList and the struct / large
cases of KudoSerializerTest.java.

Split points.  cudf::split takes the interior cut points: {10} over n rows means the partitions [0, 10) and [10, n), and {}
means one partition [0, n).  This project takes all P + 1 boundaries, so {s1, ..., sk} over n rows is written here as
[0, s1, ..., sk, n]; a cut at 0 gives an empty first partition ({0} -> [0, 0, n]).

Every case is a list of `tables` and a list of `parts` (table index, first row, row count): each part is written as one
Kudo partition of its table, the partitions are laid back to back in that order and assembled.  `expected` is the
assembled table when the source states it; None means "the rows of the parts, concatenated" (for a split case, the input
table).

Columns are (type name, values, validity, scale):
  values    a list (None marks a null string), or ("seeded", seed, lo, hi, n): n integers drawn uniformly from [lo, hi]
  validity  None (no mask), a list of 0 / 1, ("mod", k): row i valid iff i % k != 0, or ("seeded", seed): a fair coin
            per row
Data the reference draws at random -- FixedPoint's values and validity (rand() after srand(31337)) and the validity bits of
KudoConcatValidityTest (java.util.Random(7863832)) -- are filled with seeded data of our own in the same shapes; the
shapes, scales, split sets and per-partition validity patterns are the reference's.
"""


def _splits(n, cuts):
    """cudf cut points -> [0, cuts..., n]"""
    return [0] + list(cuts) + [n]


def _split_case(name, src, cols, n, cut_sets):
    return [dict(name=f"{name}{list(c)}", src=src, tables=[cols], expected=None,
                 parts=[(0, a, b - a) for a, b in zip(_splits(n, c), _splits(n, c)[1:])]) for c in cut_sets]


def _iota(n):
    return list(range(n))


CASES = []

# shuffle_split.cu:169-195
_N = 10000
CASES += _split_case("Simple", "shuffle_split.cu:169-195",
                     [("INT32", _iota(_N), None, 0), ("FLOAT32", _iota(_N), None, 0), ("INT16", _iota(_N), None, 0),
                      ("INT8", [((i + 128) & 0xFF) - 128 for i in range(_N)], None, 0)],       # the int8 iota wraps
                     _N, [[10], [10, 100, 2756, 7777]])

# shuffle_split.cu:197-235
_NUMS = ["one", "two", "three", "four", "five", "six", "seven", "eight", "nine", "ten"]
_STR_CUTS = [[], [1], [1, 4]]
CASES += _split_case("Strings/one", "shuffle_split.cu:199-207", [("STRING", _NUMS, None, 0)], 10, _STR_CUTS)
CASES += _split_case("Strings/four", "shuffle_split.cu:209-234",
                     [("STRING", _NUMS, None, 0),
                      ("STRING", ["blue", "green", "yellow", "red", "black", "white", "gray", "aquamarine", "mauve",
                                  "ultraviolet"], None, 0),
                      ("STRING", ["left", "up", "right", "down", "", "space", "", "delete", "end", "insert"], None, 0),
                      ("STRING", ["a", "b", "c", "de", "fg", "h", "i", "jk", "lmn", "opq"], None, 0)], 10, _STR_CUTS)

# shuffle_split.cu:237-251 (0xF0, 0xAA as int8: -16, -86; the null strings carry no chars)
CASES += _split_case("SimpleWithStrings", "shuffle_split.cu:237-251",
                     [("INT8", [0, -16, 0x0F, -86, 0], [1, 0, 0, 0, 1], 0),
                      ("STRING", [None, "", None, None, None], [0, 1, 0, 0, 0], 0)],
                     5, [[], [1, 3], [0, 1, 2], [5]])

# shuffle_split.cu:343-353
CASES += _split_case("Nulls", "shuffle_split.cu:343-353", [("INT32", _iota(_N), ("mod", 3), 0)], _N, [[3]])

# shuffle_split.cu:355-415
_SN32 = [1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 0, 1, 1, 1, 1, 1, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 1, 1, 1, 1, 0, 1]
CASES += _split_case("ShortNulls/word", "shuffle_split.cu:357-382", [("INT32", _iota(32), _SN32, 0)], 32,
                     [[i] for i in range(32)] + [list(range(9)), list(range(32)), [], [2, 5, 18, 30], [8, 16, 24],
                                                 list(range(0, 31, 2))])
CASES += _split_case("ShortNulls/short", "shuffle_split.cu:384-398", [("INT32", _iota(7), [1, 1, 1, 0, 0, 0, 0], 0)], 7,
                     [[i] for i in range(7)] + [[], list(range(6)), [2, 5], [0, 2, 4]])
CASES += _split_case("ShortNulls/34", "shuffle_split.cu:400-414",
                     [("INT32", list(range(1, 35)), ([1, 1, 1, 1, 0, 0, 0, 0] * 5)[:34], 0)], 34, [[22]])

# shuffle_split.cu:417-436: a 0-row FLOAT32 column with a validity buffer; the assembled column is not nullable
CASES += _split_case("PurgeNulls", "shuffle_split.cu:417-436", [("FLOAT32", [], [], 0)], 0, [[]])

# shuffle_split.cu:471-501
_FOUR = lambda n: [("INT32", _iota(n), None, 0), ("FLOAT32", _iota(n), None, 0), ("INT16", _iota(n), None, 0),  # noqa: E731
                   ("INT8", [((i + 128) & 0xFF) - 128 for i in range(n)], None, 0)]
CASES += _split_case("EmptySplits", "shuffle_split.cu:471-485", _FOUR(100), 100, [[]])
CASES += _split_case("EmptyInputs", "shuffle_split.cu:487-501", _FOUR(0), 0, [[]])

# shuffle_split.cu:735-765: random int16 / int32 / int64 values as DECIMAL32 (scale 5) / DECIMAL64 (-5) / DECIMAL128 (-6),
# without and with a rand() % 2 validity; the iterator calls rand() again for every column, so each masked column has
# bits of its own (one seed each here)
_FP = 500_000
_V16, _V32, _V64 = ("seeded", 16, -2**15, 2**15 - 1, _FP), ("seeded", 32, -2**31, 2**31 - 1, _FP), ("seeded", 64, -2**63, 2**63 - 1, _FP)
CASES += _split_case("FixedPoint", "shuffle_split.cu:735-765",
                     [("DECIMAL32", _V16, None, 5), ("DECIMAL64", _V32, None, -5), ("DECIMAL128", _V64, None, -6),
                      ("DECIMAL32", _V16, ("seeded", 31337), 5), ("DECIMAL64", _V32, ("seeded", 31338), -5),
                      ("DECIMAL128", _V64, ("seeded", 31339), -6)],
                     _FP, [[], [100], [1000, _FP - 1000]])

# shuffle_split.cu:831-970: an INT32 iota cut at the split points; the pieces marked 1 get their own validity (i % 2 of
# the piece's rows), the others none; every piece is split on its own ({}) and the partitions are assembled together
for _n, _cuts, _has in [(256, [1], [0, 1]), (256, [1], [1, 0]), (256, [11, 32], [0, 1, 0]), (1024, [256, 512, 768], [1, 0, 1, 0]),
                        (1024, [256, 512, 768], [0, 1, 0, 1]), (1024, [62, 63], [1, 0, 1]), (1024, [62, 63], [0, 1, 0]),
                        (1024, [62, 97], [1, 0, 1]), (1024, [62, 97], [0, 1, 0]), (1024, [62, 500, 768, 901], [0, 1, 1, 0, 0])]:
    _b = _splits(_n, _cuts)
    CASES.append(dict(name=f"MixedValidity{_cuts}{_has}", src="shuffle_split.cu:831-970", expected=None,
                      tables=[[("INT32", list(range(a, b)), ("mod", 2) if h else None, 0)] for a, b, h in zip(_b, _b[1:], _has)],
                      parts=[(i, 0, b - a) for i, (a, b) in enumerate(zip(_b, _b[1:]))]))

# KudoSerializerTest.java:135-169
CASES.append(dict(name="testMergeTableWithDifferentValidity", src="KudoSerializerTest.java:135-169",
                  tables=[[("INT64", [-83182, 5822, 3389, 7384, 7297], None, 0), ("FLOAT64", [-2.06, -2.14, 8.04, 1.16, -1.0], None, 0)],
                          [("INT64", [-47, 0, -83, -166, -220, 470, 619, 803, 661], [1, 0, 1, 1, 1, 1, 1, 1, 1], 0),
                           ("FLOAT64", [-6.08, 1.6, 1.78, -8.01, 1.22, 1.43, 2.13, -1.65, 0.0], [1, 1, 1, 1, 1, 1, 1, 1, 0], 0)],
                          [("INT64", [8722, 8733], None, 0), ("FLOAT64", [2.51, 0.0], None, 0)]],
                  parts=[(0, 3, 2), (1, 7, 2), (2, 1, 1)],
                  expected=[("INT64", [7384, 7297, 803, 661, 8733], None, 0),
                            ("FLOAT64", [1.16, -1.0, -1.65, 0.0, 0.0], [1, 1, 1, 0, 1], 0)]))

# KudoSerializerTest.java:171-199
CASES.append(dict(name="testMergeString", src="KudoSerializerTest.java:171-199",
                  tables=[[("STRING", ["A", "B", "C", "D", None, "TESTING", "1", "2", "3", "4", "5", "6", "7", None, "9", "10",
                                       "11", "12", "13", None, "15"], [1, 1, 1, 1, 0] + [1] * 8 + [0] + [1] * 5 + [0, 1], 0)],
                          [("STRING", ["A", "A", "C", "C", "E", "TESTING", "1", "2", "3", "4", "5", "6", "7", "", "9", "10",
                                       "11", "12", "13", "", "15"], None, 0)]],
                  parts=[(0, 2, 13), (1, 3, 5)],
                  expected=[("STRING", ["C", "D", None, "TESTING", "1", "2", "3", "4", "5", "6", "7", None, "9", "C", "E",
                                        "TESTING", "1", "2"], [1, 1, 0] + [1] * 8 + [0] + [1] * 6, 0)]))

# KudoSerializerTest.java:270-291
CASES.append(dict(name="testSerializeValidity", src="KudoSerializerTest.java:270-291",
                  tables=[[("INT32", [0, 0] + list(range(2, 512)), [0, 0] + [1] * 510, 0)]],
                  parts=[(0, 509, 3)],
                  expected=[("INT32", [509, 510, 511], None, 0)]))

# KudoConcatValidityTest.java: (start row, row count) of every slice appended to one validity buffer, in order; a start
# of None is ValidityConcatArray(-1, n, null), appended with appendAllValid (a partition without validity)
CONCAT_SCHEDULES = {
    "Case1": [(0, 29), (7, 27)],                                               # :67-91
    "Case2": [(0, 29), (7, 127)],                                              # :93-117
    "Case3": [(0, 29), (7, 133)],                                              # :119-143
    "Case4": [(0, 29)],                                                        # :145-162
    "Case5": [(0, 29), (29, 105)],                                             # :164-188
    "Case6": [(0, 14), (17, 9)],                                               # :190-215
    "Case7": [(0, 14), (17, 87)],                                              # :217-242
    "Case8": [(0, 8), (12, 85)],                                               # :244-269
    "ConcatValidity": [(3, 129), (7, 79), (None, 129), (3, 70), (3, 62), (21, 79)],   # :271-317
    "WithEmpty": [(3, 512), (None, 0), (0, 0)],                                # :319-343
}
