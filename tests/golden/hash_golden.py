"""Golden hash vectors transcribed (as DATA) from the reference's own tests.

Sources (paths relative to the reference repository's root):
  CPP  = src/main/cpp/tests/hash.cpp
  JAVA = src/test/java/com/nvidia/spark/rapids/jni/HashTest.java
The expected values there were produced by Apache Spark (see the Scala snippets in CPP:201-266,
CPP:616-679).  Each case: dict(name, src, kind in {"murmur","xxhash64","hive"}, seed,
cols=[(type, values[, scale])...], expected=[...]).  A value of None is a null row.
Strings are python str (UTF-8 encoded by the loader).  Floats given as ("bits32", int) /
("bits64", int) are raw IEEE bit patterns.
"""
INT8, INT16, INT32, INT64 = "INT8", "INT16", "INT32", "INT64"
FLOAT32, FLOAT64, BOOL8, STRING = "FLOAT32", "FLOAT64", "BOOL8", "STRING"
TS_DAYS, TS_MS, TS_US = "TIMESTAMP_DAYS", "TIMESTAMP_MILLISECONDS", "TIMESTAMP_MICROSECONDS"
DEC32, DEC64, DEC128 = "DECIMAL32", "DECIMAL64", "DECIMAL128"

I32_MIN, I32_MAX = -(2**31), 2**31 - 1
I64_MIN, I64_MAX = -(2**63), 2**63 - 1
F32_LOWEST = ("bits32", 0xFF7FFFFF)
F32_MAX = ("bits32", 0x7F7FFFFF)
F32_MIN_NORMAL = ("bits32", 0x00800000)
F32_MIN_VALUE = ("bits32", 0x00000001)
F32_NEG_QNAN = ("bits32", 0xFFC00000)
F32_INF, F32_NINF = ("bits32", 0x7F800000), ("bits32", 0xFF800000)
F64_LOWEST = ("bits64", 0xFFEFFFFFFFFFFFFF)
F64_MAX = ("bits64", 0x7FEFFFFFFFFFFFFF)
F64_MIN_NORMAL = ("bits64", 0x0010000000000000)
F64_NEG_QNAN = ("bits64", 0xFFF8000000000000)
F64_INF, F64_NINF = ("bits64", 0x7FF0000000000000), ("bits64", 0xFFF0000000000000)
# JAVA:43-52
PF_NAN_LO, PF_NAN_HI = ("bits32", 0x7F800001), ("bits32", 0x7FFFFFFF)
NF_NAN_LO, NF_NAN_HI = ("bits32", 0xFF800001), ("bits32", 0xFFFFFFFF)
PD_NAN_LO, PD_NAN_HI = ("bits64", 0x7FF0000000000001), ("bits64", 0x7FFFFFFFFFFFFFFF)
ND_NAN_LO, ND_NAN_HI = ("bits64", 0xFFF0000000000001), ("bits64", 0xFFFFFFFFFFFFFFFF)
NEG_ZERO32, NEG_ZERO64 = ("bits32", 0x80000000), ("bits64", 0x8000000000000000)

# CPP:312-317 / 814-823: the five canonical strings
S5 = ["", "The quick brown fox", "jumps over the lazy dog.",
      "All work and no play makes Jack a dull boy",
      "!\"#$%&'()*+,-./:;<=>?@[\\]^_`{|}~\ud720\ud721"]   # U+D720/U+D721 are BMP Hangul syllables

D128_A = (0xFFFFFFFFFCC4D1C3 << 64 | 0x602F7FC318000001) - (1 << 128)   # negative, CPP:341
D128_B = 0x0785EE10D5DA46D9 << 64 | 0x00F4369FFFFFFFFF                   # CPP:342

CASES = []


def _add(**kw):
    CASES.append(kw)


# ---------------------------------------------------------------- murmur, CPP:268-397 (seed 42)
_M = dict(kind="murmur", seed=42)
_add(name="cpp_mm_strings", src="CPP:271,312-317", cols=[(STRING, S5)],
     expected=[142593372, 1217302703, -715697185, -2061143941, -111635966], **_M)
_add(name="cpp_mm_doubles", src="CPP:273,318-319", cols=[(FLOAT64, [0.0, NEG_ZERO64, F64_NEG_QNAN, F64_LOWEST, F64_MAX])],
     expected=[-1670924195, -853646085, -1281358385, 1897734433, -508695674], **_M)
_add(name="cpp_mm_timestamps_ms", src="CPP:275,320-321",
     cols=[(TS_MS, [0, 100, -100, -9223372036854, 9223372036854])],
     expected=[-1670924195, 1114849490, 904948192, -1832979433, 1752430209], **_M)
_add(name="cpp_mm_decimal64", src="CPP:277,322-323",
     cols=[(DEC64, [0, 100, -100, -999999999999999999, 999999999999999999], -7)],
     expected=[-1670924195, 1114849490, 904948192, 1962370902, -1795328666], **_M)
_add(name="cpp_mm_longs", src="CPP:279,324-325", cols=[(INT64, [0, 100, -100, I64_MIN, I64_MAX])],
     expected=[-1670924195, 1114849490, 904948192, -853646085, -1604625029], **_M)
_add(name="cpp_mm_floats", src="CPP:281,326-327", cols=[(FLOAT32, [0.0, NEG_ZERO32, F32_NEG_QNAN, F32_LOWEST, F32_MAX])],
     expected=[933211791, 723455942, -349261430, -1225560532, -338752985], **_M)
_add(name="cpp_mm_dates", src="CPP:283,328-329",
     cols=[(TS_DAYS, [0, 100, -100, -21474836, 21474836])],   # int_limits::min()/100 truncates toward 0
     expected=[933211791, 751823303, -1080202046, -1906567553, -1503850410], **_M)
_add(name="cpp_mm_decimal32", src="CPP:285,330-331", cols=[(DEC32, [0, 100, -100, -999999999, 999999999], -3)],
     expected=[-1670924195, 1114849490, 904948192, -1454351396, -193774131], **_M)
_add(name="cpp_mm_ints", src="CPP:287,332-333", cols=[(INT32, [0, 100, -100, I32_MIN, I32_MAX])],
     expected=[933211791, 751823303, -1080202046, 723455942, 133916647], **_M)
_add(name="cpp_mm_shorts", src="CPP:289,334", cols=[(INT16, [0, 100, -100, -32768, 32767])],
     expected=[933211791, 751823303, -1080202046, -1871935946, 1249274084], **_M)
_add(name="cpp_mm_bytes", src="CPP:291,335", cols=[(INT8, [0, 100, -100, -128, 127])],
     expected=[933211791, 751823303, -1080202046, 1110053733, 1135925485], **_M)
_add(name="cpp_mm_bools1", src="CPP:293,336", cols=[(BOOL8, [0, 1, 1, 1, 0])],
     expected=[933211791, -559580957, -559580957, -559580957, 933211791], **_M)
_add(name="cpp_mm_bools2", src="CPP:293,337", cols=[(BOOL8, [0, 1, 2, 255, 0])],
     expected=[933211791, -559580957, -559580957, -559580957, 933211791], **_M)
_add(name="cpp_mm_decimal128", src="CPP:295,338-344", cols=[(DEC128, [0, 100, -1, D128_A, D128_B], -11)],
     expected=[-783713497, -295670906, 1398487324, -52622807, -1359749815], **_M)
# combined (CPP:297,378-396): struct column {a:int, b:string, c:{x:float, y:long}} has no nulls, so
# hashing it == hashing its leaves in order (murmur_hash.cu:119-144 chains the leaves).
_add(name="cpp_mm_structs_flattened", src="CPP:269,303-310",
     cols=[(INT32, [0, 100, -100, 0x12345678, -0x76543210]),
           (STRING, ["a", "bc", "def", "ghij", "klmno"]),
           (FLOAT32, [0.0, 100.0, -100.0, F32_INF, F32_NINF]),
           (INT64, [0, 100, -100, 0x0123456789ABCDEF, -0x0123456789ABCDEF])],
     expected=[-105406170, 90479889, -678041645, 1667387937, 301478567], **_M)
_add(name="cpp_mm_combined", src="CPP:297,378-396",
     cols=[(INT32, [0, 100, -100, 0x12345678, -0x76543210]),
           (STRING, ["a", "bc", "def", "ghij", "klmno"]),
           (FLOAT32, [0.0, 100.0, -100.0, F32_INF, F32_NINF]),
           (INT64, [0, 100, -100, 0x0123456789ABCDEF, -0x0123456789ABCDEF]),
           (STRING, S5),
           (FLOAT64, [0.0, NEG_ZERO64, F64_NEG_QNAN, F64_LOWEST, F64_MAX]),
           (TS_MS, [0, 100, -100, -9223372036854, 9223372036854]),
           (DEC64, [0, 100, -100, -999999999999999999, 999999999999999999], -7),
           (INT64, [0, 100, -100, I64_MIN, I64_MAX]),
           (FLOAT32, [0.0, NEG_ZERO32, F32_NEG_QNAN, F32_LOWEST, F32_MAX]),
           (TS_DAYS, [0, 100, -100, -21474836, 21474836]),
           (DEC32, [0, 100, -100, -999999999, 999999999], -3),
           (INT32, [0, 100, -100, I32_MIN, I32_MAX]),
           (INT16, [0, 100, -100, -32768, 32767]),
           (INT8, [0, 100, -100, -128, 127]),
           (BOOL8, [0, 1, 2, 255, 0]),
           (DEC128, [0, 100, -1, D128_A, D128_B], -11)],
     expected=[401603227, 588162166, 552160517, 1132537411, -326043017], **_M)
_add(name="cpp_mm_strings_seed314", src="CPP:411-412", kind="murmur", seed=314, cols=[(STRING, S5)],
     expected=[1467149710, 723257560, -1620282500, -2001858707, 1588473657])

# ---------------------------------------------------------------- murmur, JAVA:54-180
_JS1 = ["a", "B\nc", "dE\"Ā\tā \ud720\ud721\\Fg2'",
        "A very long (greater than 128 bytes/char string) to test a multi hash-step data point "
        "in the MD5 hash function. This string needed to be longer.A 60 character string to "
        "test MD5's message padding algorithm",
        "hiJ\ud720\ud721\ud720\ud721", None]
_add(name="java_mm_strings", src="JAVA:55-66", kind="murmur", seed=42, cols=[(STRING, _JS1)],
     expected=[1485273170, 1709559900, 1423943036, 176121990, 1199621434, 42])
_add(name="java_mm_ints", src="JAVA:69-76", kind="murmur", seed=42,
     cols=[(INT32, [0, 100, None, None, I32_MIN, None]), (INT32, [0, None, -100, None, None, I32_MAX])],
     expected=[59727262, 751823303, -1080202046, 42, 723455942, 133916647])
_add(name="java_mm_doubles", src="JAVA:79-90", kind="murmur", seed=0,
     cols=[(FLOAT64, [0.0, None, 100.0, -100.0, F64_MIN_NORMAL, F64_MAX, PD_NAN_HI, PD_NAN_LO, ND_NAN_HI,
                      ND_NAN_LO, F64_INF, F64_NINF])],
     expected=[1669671676, 0, -544903190, -1831674681, 150502665, 474144502, 1428788237, 1428788237,
               1428788237, 1428788237, 420913893, 1915664072])
_add(name="java_mm_timestamps_us", src="JAVA:93-102", kind="murmur", seed=42,
     cols=[(TS_US, [0, None, 100, -100, 0x123456789ABCDEF, None, -0x123456789ABCDEF])],
     expected=[-1670924195, 42, 1114849490, 904948192, 657182333, 42, -57193045])
_add(name="java_mm_decimal64", src="JAVA:105-114", kind="murmur", seed=42,
     cols=[(DEC64, [0, 100, -100, 0x123456789ABCDEF, -0x123456789ABCDEF], -7)],
     expected=[-1670924195, 1114849490, 904948192, 657182333, -57193045])
_add(name="java_mm_decimal32", src="JAVA:117-126", kind="murmur", seed=42,
     cols=[(DEC32, [0, 100, -100, 0x12345678, -0x12345678], -3)],
     expected=[-1670924195, 1114849490, 904948192, -958054811, -1447702630])
_add(name="java_mm_dates", src="JAVA:129-138", kind="murmur", seed=42,
     cols=[(TS_DAYS, [0, None, 100, -100, 0x12345678, None, -0x12345678])],
     expected=[933211791, 42, 751823303, -1080202046, -1721170160, 42, 1852996993])
_add(name="java_mm_floats", src="JAVA:141-152", kind="murmur", seed=411,
     cols=[(FLOAT32, [0.0, 100.0, -100.0, F32_MIN_NORMAL, F32_MAX, None, PF_NAN_LO, PF_NAN_HI, NF_NAN_LO,
                      NF_NAN_HI, F32_INF, F32_NINF])],
     expected=[-235179434, 1812056886, 2028471189, 1775092689, -1531511762, 411, -1053523253, -1053523253,
               -1053523253, -1053523253, -1526256646, 930080402])
_add(name="java_mm_bools", src="JAVA:155-162", kind="murmur", seed=0,
     cols=[(BOOL8, [None, 1, 0, 1, None, 0]), (BOOL8, [None, 1, 0, None, 0, 1])],
     expected=[0, -1589400010, -239939054, -68075478, 593689054, -1194558265])
_JMIX_S = ["a", "B\n", "dE\"Ā\tā \ud720\ud721",
           "A very long (greater than 128 bytes/char string) to test a multi hash-step data point "
           "in the MD5 hash function. This string needed to be longer.", None, None]
_JMIX = [(STRING, _JMIX_S),
         (INT32, [0, 100, -100, I32_MIN, I32_MAX, None]),
         (FLOAT64, [0.0, 100.0, -100.0, PD_NAN_LO, PD_NAN_HI, None]),
         (FLOAT32, [0.0, 100.0, -100.0, NF_NAN_LO, NF_NAN_HI, None]),
         (BOOL8, [1, 0, None, 0, 1, None])]
_add(name="java_mm_mixed", src="JAVA:165-180 (also the struct variants :183-225: structs hash as their leaves)",
     kind="murmur", seed=1868, cols=_JMIX,
     expected=[1936985022, 720652989, 339312041, 1400354989, 769988643, 1868])

# ---------------------------------------------------------------- xxhash64, CPP:686-957 (seed 42)
_X = dict(kind="xxhash64", seed=42)
_V8 = [1, 1, 1, 1, 1, 0, 1, 1]   # validity of the 8-row columns, CPP:824 etc.


def _nul(vals):
    return [v if ok else None for v, ok in zip(vals, _V8)]


_XS = _nul(S5 + ["", "abcdefgh", "abcdefghi"])
_add(name="cpp_xx_strings", src="CPP:686-694,814-824", cols=[(STRING, _XS)],
     expected=[-7444071767201028348, -3617261401988713833, 8198945020833482635, -5346617152005100141,
               6614298085531227868, 42, 2470326616177429180, -7093207067522615973], **_X)
_XD = _nul([0.0, NEG_ZERO64, F64_NEG_QNAN, F64_LOWEST, F64_MAX, 0.0, 100.0, 200.0])
_add(name="cpp_xx_doubles", src="CPP:695-703,825-833", cols=[(FLOAT64, _XD)],
     expected=[-5252525462095825812, -5252525462095825812, -3127944061524951246, 9065082843545458248,
               -4222314252576420879, 42, -7996023612001835843, -8838535416664833914], **_X)
_XT = _nul([0, 100, -100, -9223372036854, 9223372036854, 0, 200, 300])
_add(name="cpp_xx_timestamps_ms", src="CPP:704-712,834-837", cols=[(TS_MS, _XT)],
     expected=[-5252525462095825812, 8713583529807266080, 5675770457807661948, 7123048472642709644,
               -5141505295506489983, 42, -1244884446866925109, 1772389229253425430], **_X)
_XD64 = _nul([0, 100, -100, -999999999999999999, 999999999999999999, 0, 123, 432])
_add(name="cpp_xx_decimal64", src="CPP:713-721,838-841", cols=[(DEC64, _XD64, -7)],
     expected=[-5252525462095825812, 8713583529807266080, 5675770457807661948, 4265531446127695490,
               2162198894918931945, 42, -3178482946328430151, 4788666723486520022], **_X)
_XL = _nul([0, 100, -100, I64_MIN, I64_MAX, 0, 0x123456789ABCDEF, -0x123456789ABCDEF])
_add(name="cpp_xx_longs", src="CPP:722-730,842-850", cols=[(INT64, _XL)],
     expected=[-5252525462095825812, 8713583529807266080, 5675770457807661948, -8619748838626508300,
               -3246596055638297850, 42, 1941233597257011502, -1318946533059658749], **_X)
_XF = _nul([0.0, NEG_ZERO32, F32_NEG_QNAN, F32_LOWEST, F32_MAX, 0.0, F32_INF, F32_NINF])
_add(name="cpp_xx_floats", src="CPP:731-739,851-859", cols=[(FLOAT32, _XF)],
     expected=[3614696996920510707, 3614696996920510707, 2692338816207849720, -8545425418825163117,
               -1065250890878313112, 42, -5940311692336719973, -7580553461823983095], **_X)
_XDT = _nul([0, 100, -100, -21474836, 21474836, 0, -200, -300])
_add(name="cpp_xx_dates", src="CPP:740-748,860-862", cols=[(TS_DAYS, _XDT)],
     expected=[3614696996920510707, -7987742665087449293, 8990748234399402673, -8442426365007754391,
               -1447590449373190349, 42, -953008374380745918, 2895908635257747121], **_X)
_XD32 = _nul([0, 100, -100, -999999999, 999999999, 0, -200, -300])
_add(name="cpp_xx_decimal32", src="CPP:749-757,863-866", cols=[(DEC32, _XD32, -3)],
     expected=[-5252525462095825812, 8713583529807266080, 5675770457807661948, 8670643431269007867,
               6810183316718625826, 42, 7277994511003214036, 6264187449999859617], **_X)
_XI = _nul([0, 100, -100, I32_MIN, I32_MAX, 0, -200, -300])
_add(name="cpp_xx_ints", src="CPP:758-766,867-868", cols=[(INT32, _XI)],
     expected=[3614696996920510707, -7987742665087449293, 8990748234399402673, 2073849959933241805,
               1508894993788531228, 42, -953008374380745918, 2895908635257747121], **_X)
_XSH = _nul([0, 100, -100, -32768, 32767, 0, -200, -300])
_add(name="cpp_xx_shorts", src="CPP:767-775,869-870", cols=[(INT16, _XSH)],
     expected=[3614696996920510707, -7987742665087449293, 8990748234399402673, -904511417458573795,
               8952525448871805501, 42, -953008374380745918, 2895908635257747121], **_X)
_XB = _nul([0, 100, -100, -128, 127, 0, -90, -80])
_add(name="cpp_xx_bytes", src="CPP:776-784,871-872", cols=[(INT8, _XB)],
     expected=[3614696996920510707, -7987742665087449293, 8990748234399402673, 4160238337661960656,
               8632298611707923906, 42, -4008061843281999337, 6690883199412647955], **_X)
_XBO1 = _nul([0, 1, 1, 1, 0, 0, 0, 0])
_XBO2 = _nul([0, 1, 2, 255, 0, 0, 0, 0])
_XBOE = [3614696996920510707, -6698625589789238999, -6698625589789238999, -6698625589789238999,
         3614696996920510707, 42, 3614696996920510707, 3614696996920510707]
_add(name="cpp_xx_bools1", src="CPP:785-793,873-874", cols=[(BOOL8, _XBO1)], expected=_XBOE, **_X)
_add(name="cpp_xx_bools2", src="CPP:785-793,875-876", cols=[(BOOL8, _XBO2)], expected=_XBOE, **_X)
_XD128 = _nul([0, 100, -1, D128_A, D128_B, 0, D128_A, D128_B])
_add(name="cpp_xx_decimal128", src="CPP:794-802,877-889", cols=[(DEC128, _XD128, -11)],
     expected=[-8959994473701255385, 4409375254388155230, -4006032525457443936, -5423362182451591024,
               7041733194569950081, 42, -5423362182451591024, 7041733194569950081], **_X)
_add(name="cpp_xx_combined", src="CPP:803-811,938-957",
     cols=[(STRING, _XS), (FLOAT64, _XD), (TS_MS, _XT), (DEC64, _XD64, -7), (INT64, _XL), (FLOAT32, _XF),
           (TS_DAYS, _XDT), (DEC32, _XD32, -3), (INT32, _XI), (INT16, _XSH), (INT8, _XB), (BOOL8, _XBO2),
           (DEC128, _XD128, -11)],
     expected=[541735645035655239, 9011982951766246298, 3834379147931449211, -5406325166887725795,
               7797509897614041972, 42, -9032872913521304524, -604070008711895908], **_X)
_add(name="cpp_xx_strings2", src="CPP:971-990", cols=[(STRING, ["", None] + S5[1:])],
     expected=[-7444071767201028348, 42, -3617261401988713833, 8198945020833482635, -5346617152005100141,
               6614298085531227868], **_X)

# ---------------------------------------------------------------- xxhash64, JAVA:273-405
_add(name="java_xx_strings", src="JAVA:274-285", cols=[(STRING, _JS1)],
     expected=[-8582455328737087284, 2221214721321197934, 5798966295358745941, -4834097201550955483,
               -3782648123388245694, 42], **_X)
_add(name="java_xx_ints", src="JAVA:288-295",
     cols=[(INT32, [0, 100, None, None, I32_MIN, None]), (INT32, [0, None, -100, None, None, I32_MAX])],
     expected=[1151812168208346021, -7987742665087449293, 8990748234399402673, 42, 2073849959933241805,
               1508894993788531228], **_X)
_add(name="java_xx_doubles", src="JAVA:298-309",
     cols=[(FLOAT64, [0.0, None, 100.0, -100.0, F64_MIN_NORMAL, F64_MAX, PD_NAN_HI, PD_NAN_LO, ND_NAN_HI,
                      ND_NAN_LO, F64_INF, F64_NINF])],
     expected=[-5252525462095825812, 42, -7996023612001835843, 5695175288042369293, 6181148431538304986,
               -4222314252576420879, -3127944061524951246, -3127944061524951246, -3127944061524951246,
               -3127944061524951246, 5810986238603807492, 5326262080505358431], **_X)
_add(name="java_xx_timestamps_us", src="JAVA:312-321",
     cols=[(TS_US, [0, None, 100, -100, 0x123456789ABCDEF, None, -0x123456789ABCDEF])],
     expected=[-5252525462095825812, 42, 8713583529807266080, 5675770457807661948, 1941233597257011502, 42,
               -1318946533059658749], **_X)
_add(name="java_xx_decimal64", src="JAVA:324-333",
     cols=[(DEC64, [0, 100, -100, 0x123456789ABCDEF, -0x123456789ABCDEF], -7)],
     expected=[-5252525462095825812, 8713583529807266080, 5675770457807661948, 1941233597257011502,
               -1318946533059658749], **_X)
_add(name="java_xx_decimal32", src="JAVA:336-345", cols=[(DEC32, [0, 100, -100, 0x12345678, -0x12345678], -3)],
     expected=[-5252525462095825812, 8713583529807266080, 5675770457807661948, -7728554078125612835,
               3142315292375031143], **_X)
_add(name="java_xx_dates", src="JAVA:348-357", cols=[(TS_DAYS, [0, None, 100, -100, 0x12345678, None, -0x12345678])],
     expected=[3614696996920510707, 42, -7987742665087449293, 8990748234399402673, 6954428822481665164, 42,
               -4294222333805341278], **_X)
_add(name="java_xx_floats", src="JAVA:360-371",
     cols=[(FLOAT32, [0.0, 100.0, -100.0, F32_MIN_NORMAL, F32_MAX, None, PF_NAN_LO, PF_NAN_HI, NF_NAN_LO,
                      NF_NAN_HI, F32_INF, F32_NINF])],
     expected=[3614696996920510707, -8232251799677946044, -6625719127870404449, -6699704595004115126,
               -1065250890878313112, 42, 2692338816207849720, 2692338816207849720, 2692338816207849720,
               2692338816207849720, -5940311692336719973, -7580553461823983095], **_X)
_add(name="java_xx_bools", src="JAVA:374-381",
     cols=[(BOOL8, [None, 1, 0, 1, None, 0]), (BOOL8, [None, 1, 0, None, 0, 1])],
     expected=[42, 9083826852238114423, 1151812168208346021, -6698625589789238999, 3614696996920510707,
               7945966957015589024], **_X)
_add(name="java_xx_mixed", src="JAVA:384-401 (also struct variants :404-445)", cols=_JMIX,
     expected=[7451748878409563026, 6024043102550151964, 3380664624738534402, 8444697026100086329,
               -5888679192448042852, 42], **_X)

# ---------------------------------------------------------------- hive, JAVA:576-700
_H = dict(kind="hive", seed=0)
_add(name="java_hive_bools", src="JAVA:577-584", cols=[(BOOL8, [1, 0, None])], expected=[1, 0, 0], **_H)
_add(name="java_hive_ints", src="JAVA:587-596", cols=[(INT32, [I32_MIN, I32_MAX, -1, 1, -10, 10, None])],
     expected=[I32_MIN, I32_MAX, -1, 1, -10, 10, 0], **_H)
_add(name="java_hive_bytes", src="JAVA:599-608", cols=[(INT8, [-128, 127, -1, 1, -10, 10, None])],
     expected=[-128, 127, -1, 1, -10, 10, 0], **_H)
_add(name="java_hive_longs", src="JAVA:611-620", cols=[(INT64, [I64_MIN, I64_MAX, -1, 1, -10, 10, None])],
     expected=[I32_MIN, I32_MIN, 0, 1, 9, 10, 0], **_H)
_HS_LONG = ("This is a long string (greater than 128 bytes/char string) case to test this "
            "hash function. Just want an abnormal case here to see if any error may happen when"
            "doing the hive hashing")
_add(name="java_hive_strings", src="JAVA:623-634",
     cols=[(STRING, ["a", "B\n", "dE\"Ā\tā \ud720\ud721", None, _HS_LONG])],
     expected=[97, 2056, 745239896, 0, 2112075710], **_H)
_add(name="java_hive_floats", src="JAVA:637-649",
     cols=[(FLOAT32, [0.0, 100.0, -100.0, F32_MIN_NORMAL, F32_MAX, None, F32_MIN_VALUE, PF_NAN_LO, PF_NAN_HI,
                      NF_NAN_LO, NF_NAN_HI, F32_INF, F32_NINF])],
     expected=[0, 1120403456, -1027080192, 8388608, 2139095039, 0, 1, 2143289344, 2143289344, 2143289344,
               2143289344, 2139095040, -8388608], **_H)
_add(name="java_hive_doubles", src="JAVA:652-660", cols=[(FLOAT64, [0.0, 100.0, -100.0, PD_NAN_LO, PD_NAN_HI, None])],
     expected=[0, 1079574528, -1067909120, 2146959360, 2146959360, 0], **_H)
_add(name="java_hive_dates", src="JAVA:663-671", cols=[(TS_DAYS, [0, None, 100, -100, 0x12345678, None, -0x12345678])],
     expected=[0, 0, 100, -100, 0x12345678, 0, -0x12345678], **_H)
_add(name="java_hive_timestamps", src="JAVA:674-682",
     cols=[(TS_US, [0, None, 100, -100, 0x123456789ABCDEF, None, -0x123456789ABCDEF])],
     expected=[0, 0, 100000, 99999, -660040456, 0, 486894999], **_H)
_add(name="java_hive_mixed", src="JAVA:685-706 (also struct variants :709-758: structs fold like columns)",
     cols=[(STRING, ["a", "B\n", "dE\"Ā\tā \ud720\ud721", _HS_LONG, None, None]),
           (INT32, [0, 100, -100, I32_MIN, I32_MAX, None]),
           (FLOAT64, [0.0, 100.0, -100.0, PD_NAN_LO, PD_NAN_HI, None]),
           (FLOAT32, [0.0, 100.0, -100.0, NF_NAN_LO, NF_NAN_HI, None]),
           (BOOL8, [1, 0, None, 0, 1, None])],
     expected=[89581538, 363542820, 413439036, 1272817854, 1513589666, 0], **_H)
