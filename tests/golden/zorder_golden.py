"""ZOrder test data: the inputs of every case of the reference's InterleaveBitsTest.java and HilbertIndexTest.java (data
only), plus answers derived by hand from the contract.

INTERLEAVE cases: (name, width in bytes, rows, columns); each column a list of Python ints (None = null), values as the
Java tests write them (0xFFFFFFFF in an Integer[] is -1; the interleave reads the low 8W bits either way).
HILBERT cases: (name, num_bits, rows, columns).  The reference's expected Hilbert values come from a third-party
library; here the independent model and the curve's properties pin them.
"""

INTERLEAVE = [
    ("testInt0", 4, 10, []),
    ("testShort0", 2, 10, []),
    ("testByte0", 1, 10, []),
    ("testInt1NonNull", 4, 5, [[1, 2, 3, 4, 0x01020304]]),
    ("testShort1NonNull", 2, 5, [[1, 2, 3, 4, 0x0102]]),
    ("testByte1NonNull", 1, 5, [[1, 2, 3, 4, 5]]),
    ("testInt1Null", 4, 4, [[None, 7, None, 8]]),
    ("testShort1Null", 2, 4, [[None, 7, None, 8]]),
    ("testByte1Null", 1, 4, [[None, 7, None, 8]]),
    ("testInt2NonNull", 4, 4, [[0x01020304, 0x00000000, 0xFFFFFFFF, 0xFF00FF00],
                               [0x10203040, 0xFFFFFFFF, 0x00000000, 0x00FF00FF]]),
    ("testShort2NonNull", 2, 4, [[0x0102, 0x0000, 0xFFFF, 0xFF00], [0x1020, 0xFFFF, 0x0000, 0x00FF]]),
    ("testByte2NonNull", 1, 4, [[0x01, 0x00, 0xFF, 0x0F], [0x10, 0xFF, 0x00, 0xF0]]),
    ("testInt2Null", 4, 4, [[0x00000000, None, 0xFFFFFFFF, 0xFF00FF00], [0xFFFFFFFF, 0x00000000, 0x00FF00FF, None]]),
    ("testInt3NonNull", 4, 3, [[0x00000000, 0x44444444, 0x11111111], [0x11111111, 0x88888888, 0x22222222],
                               [0x22222222, 0x00000000, 0x44444444]]),
    ("testShort3NonNull", 2, 3, [[0x0000, 0x4444, 0x1111], [0x1111, 0x8888, 0x2222], [0x2222, 0x0000, 0x4444]]),
    ("testByte3NonNull", 1, 3, [[0x00, 0x44, 0x11], [0x11, 0x88, 0x22], [0x22, 0x00, 0x44]]),
]

HILBERT = [
    ("test0", 6, 10, []),
    ("test1NonNull", 3, 5, [[1, 2, 3, 4, 5]]),
    ("test1Null", 4, 4, [[None, 7, None, 8]]),
    ("testInt2NonNull", 10, 4, [[1, 500, 1000, 250], [500, 400, 300, 200]]),
    ("testInt2Null", 10, 4, [[0, None, 50, 1000], [200, 300, 100, 0]]),
    ("testInt3NonNull", 10, 6, [[0, 4, 1, 0, 1023, 512], [1, 8, 2, 0, 1023, 512], [2, 0, 4, 0, 1023, 512]]),
]

# Interleave answers derived by hand: (width, columns (one row each), row bytes)
INTERLEAVE_KNOWN = [
    # one column: the stream is the value's bits MSB first, i.e. its big-endian bytes
    (4, [0x01020304], bytes([0x01, 0x02, 0x03, 0x04])),
    # 0xFF then 0x00: every even position 1, every odd one 0
    (1, [0xFF, 0x00], bytes([0xAA, 0xAA])),
    # three INT16: position 0 = bit 15 of 0x8000; position 47 = bit 0 of the third column (1)
    (2, [0x8000, 0x0000, 0x0001], bytes([0x80, 0x00, 0x00, 0x00, 0x00, 0x01])),
    # testInt2NonNull row 0: 0x01020304 / 0x10203040; output byte k interleaves nibble k (MSB first) of each value,
    # e.g. byte 0 = nibbles 0x0 / 0x1 -> 00000001, byte 1 = nibbles 0x1 / 0x0 -> 00000010
    (4, [0x01020304, 0x10203040], bytes([0x01, 0x02, 0x04, 0x08, 0x05, 0x0A, 0x10, 0x20])),
]

# one DECIMAL128 column gives its 16 little-endian bytes reversed
DECIMAL128_BYTES = bytes(range(0x11, 0x21))

# Hilbert answers derived by hand: (num_bits, columns (one row each), index)
HILBERT_KNOWN = [
    (3, [1], 1), (3, [2], 2), (3, [3], 3), (3, [4], 4), (3, [5], 5),   # N = 1 is the identity
    (4, [None], 0), (4, [7], 7), (4, [8], 8),
    (1, [0, 0], 0), (1, [0, 1], 1), (1, [1, 1], 2), (1, [1, 0], 3),      # the 2-D curve of order 1
]
