"""Goldens of the radix casts, from the reference's tests (src/test/java/com/nvidia/spark/rapids/jni/):
NumberConverterTest (all seven overloads; isConvertOverflow is false in each) and CastStringsTest
(castFromLongToBinaryStringTest, the expected columns of baseDec2HexTestNoNulls / baseDec2HexTestMixed / baseHex2DecTest
read as UINT64 inputs of fromIntegersWithBase at bases 10 and 16, bytesToHexStringTest and bytesToHexBinaryTest).

A CONV case is (overload, input, fromBase, toBase, expected): input a list of strings or one scalar string, each base a
list of ints or one int, expected the rows (None: null).
"""
IN3 = ["Z1", "34", " azc "]
CONV = [
    ("CvCvCv", IN3, [36, 5, 34], [10, 10, 9], ["1261", "19", "11"]),
    ("CvCvS", IN3, [7, 36, 36], 27, ["0", "44", "JE3"]),
    ("CvSCv", IN3, 4, [7, 9, 36], ["0", "3", "0"]),
    ("CvSS", IN3, 9, 27, ["0", "14", "0"]),
    ("SCvCv", "-127", [10, 5, 34], [16, -10, 9], ["FFFFFFFFFFFFFF81", "-7", "145808576354216722140"]),
    ("SCvS", "-FF4D", [7, 35, 36], 27, ["0", "4EO8HFAM6EF567", "4EO8HFAM6EC6Q3"]),
    ("SSCv", "11223344FFTTZZ", 4, [7, 9, -36], ["4146", "1886", "14F"]),
]
CONV_OVERFLOW = {case[0]: False for case in CONV}

# castFromLongToBinaryStringTest
LONGS = [None, 0, 1, 10, -1, (1 << 63) - 1, -(1 << 63)]
LONGS_BINARY = [None, "0", "1", "1010", "1" * 64, "1" * 63, "1" + "0" * 63]

# (UINT64 input, base 10, base 16): the expected decimal column of the three conv tests as integers
UINT64_DEC_HEX = [
    (510, "510", "1FE"), (0, "0", "0"), (None, None, None),
    (18446744073709551106, "18446744073709551106", "FFFFFFFFFFFFFE02"),
    (15, "15", "F"), (18446744073709551526, "18446744073709551526", "FFFFFFFFFFFFFFA6"), (90, "90", "5A"),
]

# bytesToHexStringTest ("\0\1ÿ" is UTF-8 00 01 C3 BF) and bytesToHexBinaryTest
HEX_STRINGS = [b"AB", b"", b"Spark", None, b"\x00\x01\xc3\xbf"]
HEX_STRINGS_EXPECTED = ["4142", "", "537061726B", None, "0001C3BF"]
HEX_BINARY = [b"\x41\x42", b"\x00\xff", None, b""]
HEX_BINARY_EXPECTED = ["4142", "00FF", None, ""]
