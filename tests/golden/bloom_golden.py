"""Bloom filter goldens, transcribed as data from the reference's tests:
src/test/java/com/nvidia/spark/rapids/jni/BloomFilterTest.java:30-225 (JAVA) and src/main/cpp/tests/bloom_filter.cu:36-375
(CPP).  Each case builds one or more filters, optionally merges them, and probes; `expected` holds the probe result per
row, None where the probe row is null (its value is not part of the contract).

Plus KNOWN: single keys put into 64- and 128-bit filters with k = 3, pinning h1, the bit positions and the serialized
bytes (the reference's tests only pin present / absent answers on 2^22- and 2^26-bit filters).  They were derived from
Spark's definitions by hand-checkable integer arithmetic (tests/bloom_model.py spells it out); as one outside anchor,
Murmur3 hashLong(0, 42) = -1670924195 is Spark's well-known `hash(0L)`.  Example, V1 key 0 into 64 bits: positions 40,
43, 63 -> long 0 = 2^63 + 2^43 + 2^40 = 0x8000090000000000, written big-endian after the header {1, 3, 1}.
"""

BUILD = [20, 80, 100, 99, 47, -9, 234000000]
PROBE = [20, 80, 100, 99, 47, -9, 234000000, -10, 1, 2, 3]
MERGE_B = [100, 200, 300, 400]
MERGE_C = [-100, -200, -300, -400]
MERGE_PROBE = [-9, 200, 300, 6000, -2546, 99, 65535, 0, -100, -200, -300, -400]
ABSENT = [-10, 1, 2, 3, 5000, 999999, -77777]
T, F = True, False
JAVA_BITS = 4 * 1024 * 1024                 # BloomFilterTest.java: bloomFilterBits
CPP_BITS = 64 * 1024 * 1024                 # tests/bloom_filter.cu: bloom_filter_longs = 1024 * 1024


def _case(name, source, version, bits, puts, probe, expected, probe_valid=None, seed=0, merge=False, buffer=False, k=3):
    """puts: one list of (values, valid or None) per filter; merge: OR them first (else there is one filter)"""
    return dict(name=name, source=source, version=version, num_hashes=k, bits=bits, seed=seed, puts=puts, merge=merge,
                probe=probe, probe_valid=probe_valid, expected=expected, buffer=buffer)


CASES = []
for _v in (1, 2):
    CASES += [
        _case(f"java_build_probe_v{_v}", "BloomFilterTest.java:30-45", _v, JAVA_BITS, [[(BUILD, None)]], PROBE, [T] * 7 + [F] * 4),
        _case(f"java_build_probe_buffer_v{_v}", "BloomFilterTest.java:47-62", _v, JAVA_BITS, [[(BUILD, None)]], PROBE,
              [T] * 7 + [F] * 4, buffer=True),
        _case(f"java_build_with_nulls_v{_v}", "BloomFilterTest.java:64-79", _v, JAVA_BITS,
              [[(BUILD, [0, 1, 1, 0, 1, 1, 1])]], PROBE, [F, T, T, F, T, T, T, F, F, F, F]),
        _case(f"java_probe_with_nulls_v{_v}", "BloomFilterTest.java:81-96", _v, JAVA_BITS, [[(BUILD, None)]],
              [0, 0, 0, 99, 47, -9, 234000000, 0, 0, 2, 3], [None, None, None, T, T, T, T, None, None, F, F],
              probe_valid=[0, 0, 0, 1, 1, 1, 1, 0, 0, 1, 1]),
        _case(f"java_merge_probe_v{_v}", "BloomFilterTest.java:98-131", _v, JAVA_BITS,
              [[(BUILD, None)], [(MERGE_B, None)], [(MERGE_C, None)]], MERGE_PROBE, [T, T, T, F, F, T, F, F, T, T, T, T], merge=True),
        _case(f"java_trivial_merge_probe_v{_v}", "BloomFilterTest.java:133-152", _v, JAVA_BITS, [[(BUILD, None)]], MERGE_PROBE,
              [T, F, F, F, F, T, F, F, F, F, F, F], merge=True),
        _case(f"cpp_build_probe_v{_v}", f"tests/bloom_filter.cu:{'64-83' if _v == 1 else '232-248'}", _v, CPP_BITS,
              [[(BUILD, None)]], PROBE if _v == 1 else BUILD, [T] * 7 + [F] * 4 if _v == 1 else [T] * 7),
        _case(f"cpp_build_with_nulls_v{_v}", f"tests/bloom_filter.cu:{'85-105' if _v == 1 else '250-268'}", _v, CPP_BITS,
              [[(BUILD, [0, 1, 1, 1, 0, 1, 1])]], PROBE, [F, T, T, T, F, T, T, F, F, F, F]),
        _case(f"cpp_probe_with_nulls_v{_v}", f"tests/bloom_filter.cu:{'107-126' if _v == 1 else '270-289'}", _v, CPP_BITS,
              [[(BUILD, None)]], PROBE, [None, None, None, T, T, T, T, None, None, F, F], probe_valid=[0, 0, 0, 1, 1, 1, 1, 0, 0, 1, 1]),
        _case(f"cpp_probe_all_absent_v{_v}", f"tests/bloom_filter.cu:{'183-200' if _v == 1 else '334-351'}", _v, CPP_BITS,
              [[(BUILD, None)]], ABSENT, [F] * 7),
    ]
CASES += [
    _case("java_build_probe_v2_seed42", "BloomFilterTest.java:154-169", 2, JAVA_BITS, [[(BUILD, None)]], PROBE, [T] * 7 + [F] * 4, seed=42),
    _case("cpp_probe_merged_v1", "tests/bloom_filter.cu:133-181", 1, CPP_BITS, [[(BUILD, None)], [(MERGE_B, None)], [(MERGE_C, None)]],
          MERGE_PROBE, [T, T, T, F, F, T, F, F, T, T, T, T], merge=True),
    _case("cpp_probe_merged_v2", "tests/bloom_filter.cu:291-332", 2, CPP_BITS, [[(BUILD, None)], [(MERGE_B, None)], [(MERGE_C, None)]],
          BUILD + [200, 300, 400] + MERGE_C, [T] * 14, merge=True),
    _case("cpp_v2_seed0", "tests/bloom_filter.cu:353-375", 2, CPP_BITS, [[(BUILD, None)]], BUILD, [T] * 7, seed=0),
    _case("cpp_v2_seed42", "tests/bloom_filter.cu:353-375", 2, CPP_BITS, [[(BUILD, None)]], BUILD, [T] * 7, seed=42),
]

# Initialization tests: (version, num_hashes, num_longs, seed, serialized size); the bit array is all zero
# (tests/bloom_filter.cu:36-62, 204-230)
INIT = [(1, 3, 1, 0, 20), (1, 3, 2, 0, 28), (1, 3, 3, 0, 36), (2, 3, 1, 42, 24), (2, 3, 2, 42, 32), (2, 3, 3, 42, 40)]

# Expected failures (BloomFilterTest.java:171-225): ("create", version, num_hashes, bits, seed) must raise ValueError
# (IllegalArgumentException); ("merge", [(version, num_hashes, bits, seed), ...]) must raise CudfException
FAILURES = []
for _v in (1, 2):
    FAILURES += [("create", _v, 0, 64, 0), ("create", _v, 3, 0, 0),
                 ("merge", [(_v, 3, 1024, 0), (_v, 4, 1024, 0), (_v, 4, 1024, 0)]),
                 ("merge", [(_v, 3, 1024, 0), (_v, 3, 1024, 0), (_v, 3, 2048, 0)])]
FAILURES += [("create", 3, 3, 64, 0), ("merge", [(1, 3, 1024, 0), (2, 3, 1024, 0)])]

# (version, seed, bits, key, h1 = hashLong(key, V1 ? 0 : seed), positions, serialized filter hex) with k = 3
KNOWN = [
    (1, 0, 64, 0, 1669671676, (40, 43, 63), "0000000100000003000000018000090000000000"),
    (1, 0, 64, 234000000, -876378336, (27, 41, 17), "0000000100000003000000010000020008020000"),
    (1, 0, 128, 0, 1669671676, (40, 43, 127), "00000001000000030000000200000900000000008000000000000000"),
    (1, 0, 128, 234000000, -876378336, (91, 105, 81), "00000001000000030000000200000000000000000000020008020000"),
    (1, 42, 64, 0, 1669671676, (40, 43, 63), "0000000100000003000000018000090000000000"),
    (1, 42, 64, 234000000, -876378336, (27, 41, 17), "0000000100000003000000010000020008020000"),
    (1, 42, 128, 0, 1669671676, (40, 43, 127), "00000001000000030000000200000900000000008000000000000000"),
    (1, 42, 128, 234000000, -876378336, (91, 105, 81), "00000001000000030000000200000000000000000000020008020000"),
    (1, -1, 64, 0, 1669671676, (40, 43, 63), "0000000100000003000000018000090000000000"),
    (1, -1, 64, 234000000, -876378336, (27, 41, 17), "0000000100000003000000010000020008020000"),
    (1, -1, 128, 0, 1669671676, (40, 43, 127), "00000001000000030000000200000900000000008000000000000000"),
    (1, -1, 128, 234000000, -876378336, (91, 105, 81), "00000001000000030000000200000000000000000000020008020000"),
    (2, 0, 64, 0, 1669671676, (48, 28, 8), "000000020000000300000000000000010001000010000100"),
    (2, 0, 64, 234000000, -876378336, (36, 41, 46), "000000020000000300000000000000010000421000000000"),
    (2, 0, 128, 0, 1669671676, (48, 92, 8), "0000000200000003000000000000000200010000000001000000000010000000"),
    (2, 0, 128, 234000000, -876378336, (100, 41, 110), "0000000200000003000000000000000200000200000000000000401000000000"),
    (2, 42, 64, 0, -1670924195, (46, 0, 18), "00000002000000030000002a000000010000400000040001"),
    (2, 42, 64, 234000000, 1710090726, (55, 20, 49), "00000002000000030000002a000000010082000000100000"),
    (2, 42, 128, 0, -1670924195, (110, 0, 18), "00000002000000030000002a0000000200000000000400010000400000000000"),
    (2, 42, 128, 234000000, 1710090726, (119, 84, 49), "00000002000000030000002a0000000200020000000000000080000000100000"),
    (2, -1, 64, 0, -221081364, (28, 13, 62), "0000000200000003ffffffff000000014000000010002000"),
    (2, -1, 64, 234000000, -389737294, (8, 31, 54), "0000000200000003ffffffff000000010040000080000100"),
    (2, -1, 128, 0, -221081364, (92, 77, 62), "0000000200000003ffffffff0000000240000000000000000000000010002000"),
    (2, -1, 128, 234000000, -389737294, (72, 95, 118), "0000000200000003ffffffff0000000200000000000000000040000080000100"),
]
