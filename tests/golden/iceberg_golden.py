"""Iceberg transform test data: the hash vectors of the Iceberg table spec (Appendix B, "32-bit Hash Requirements"), the
standard MurmurHash3_x86_32 test vector, the spec's truncate examples, and date / time answers derived by hand.

HASH: (Iceberg type, value, expected signed 32-bit hash).  The value is what the column stores: an int / long, a
decimal's unscaled integer, days since 1970-01-01, microseconds since the epoch, UTF-8 text or raw bytes.
"""

# 2017-11-16 is day 17486: 47 years of 1970..2016 (12 leap years) = 17167 days, plus 319 days to November 16th
DATE_2017_11_16 = 17486
# 2017-11-16T22:31:08 in microseconds: (17486 * 86400 + 22 * 3600 + 31 * 60 + 8) * 10^6
TS_2017_11_16_22_31_08 = 1510871468000000

HASH = [
    ("int", 34, 2017239379),
    ("long", 34, 2017239379),
    ("decimal(9,2)", 1420, -500754589),               # 14.20
    ("date", DATE_2017_11_16, -653330422),
    ("timestamp", TS_2017_11_16_22_31_08, -2047944441),
    ("string", "iceberg", 1210000089),
    ("binary", bytes([0, 1, 2, 3]), -188683207),
]

# Appleby's MurmurHash3_x86_32 with seed 0
MURMUR3_FOX = (b"The quick brown fox jumps over the lazy dog", 0x2E4FF723)

# (Iceberg type, width, value, truncated value); decimals as unscaled integers (scale 2)
TRUNCATE = [
    ("int", 10, 1, 0),
    ("int", 10, -1, -10),
    ("long", 10, 1, 0),
    ("long", 10, -1, -10),
    ("decimal(9,2)", 50, 1065, 1050),                 # 10.65 -> 10.50
    ("string", 3, "iceberg", "ice"),
]

# (transform, input kind, value, expected)
DATETIME = [
    ("years", "date", DATE_2017_11_16, 47),
    ("months", "date", DATE_2017_11_16, 574),         # 47 * 12 + 10
    ("days", "date", DATE_2017_11_16, 17486),
    ("years", "timestamp", TS_2017_11_16_22_31_08, 47),
    ("months", "timestamp", TS_2017_11_16_22_31_08, 574),
    ("days", "timestamp", TS_2017_11_16_22_31_08, 17486),
    ("hours", "timestamp", TS_2017_11_16_22_31_08, 419686),   # 17486 * 24 + 22
    ("years", "timestamp", -1, -1),                   # 1969-12-31T23:59:59.999999
    ("months", "timestamp", -1, -1),
    ("days", "timestamp", -1, -1),
    ("hours", "timestamp", -1, -1),
]
