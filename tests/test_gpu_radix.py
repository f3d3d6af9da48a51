"""GPU checks of the radix casts (srj_b200.radix.NumberConverter and srj_b200.cast.CastStrings' fromLongToBinary,
fromIntegersWithBase and bytesToHex over libsrj_b200.so, csrc/radix.cu) against oracle/radix.py, which
tests/test_oracle_radix.py pins to the reference's tests and a model of Spark's intent.  Offsets, chars, masks and null
counts are compared bit for bit, and the overflow flag of every isConvertOverflow overload."""
import random
import threading

import numpy as np
import pytest

from golden import radix_golden as G
from oracle import radix as R

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1
OVERLOADS = ["CvCvCv", "CvCvS", "CvSCv", "CvSS", "SCvCv", "SCvS", "SSCv"]


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200.bloom import Scalar
    from srj_b200.cast import CastStrings
    from srj_b200.radix import NumberConverter
    return S, Scalar, CastStrings, NumberConverter


def _mask(valid):
    if valid is None or all(valid):
        return None
    v = np.concatenate([np.asarray(valid, bool), np.zeros(-len(valid) % 32, bool)])
    return np.packbits(v, bitorder="little").view(np.uint32)


def strcol(rows, pad=0):
    """a STRING column of `rows` (None: null); pad > 0 puts pad bytes before the first row, so the offsets start there"""
    S = _s()[0]
    data = b"x" * pad + b"".join(r for r in rows if r is not None)
    offs = [pad]
    for r in rows:
        offs.append(offs[-1] + (0 if r is None else len(r)))
    return S.ColumnVector.from_numpy(S.DType.STRING, np.frombuffer(data or b"\0", np.uint8), _mask([r is not None for r in rows]),
                                     np.array(offs, np.int32), size=len(rows))


def intcol(vals, type_id=None, np_type=np.int32):
    S = _s()[0]
    valid = [v is not None for v in vals]
    arr = np.array([0 if v is None else v for v in vals], dtype=np_type)
    return S.ColumnVector.from_numpy(S.DType.INT32 if type_id is None else type_id, arr, _mask(valid), size=len(vals))


def check(got, rows):
    """got (a STRING column) holds exactly `rows`: offsets, chars, mask and null count"""
    offs, chars, valid = R.to_column(rows)
    assert got.size == len(rows)
    assert got.offsets.cpu().numpy().tolist() == offs
    assert bytes(got.data.cpu().numpy().tobytes()) == chars
    nulls = valid.count(False)
    assert got.getNullCount() == nulls
    if nulls:
        bits = np.unpackbits(got.mask.cpu().numpy().view(np.uint8), bitorder="little")[:len(rows)].astype(bool)
        assert bits.tolist() == valid
    else:
        assert got.mask is None


def _conv_call(kind, NC, Scalar, name, inp, fb, tb):
    """the overload `name` on python arguments: the input rows or scalar bytes, each base a list or an int"""
    args = [Scalar.fromString(inp) if name[0] == "S" else strcol(inp)]
    rest = name[1:] if name[0] == "S" else name[2:]
    for b in (fb, tb):
        if rest.startswith("Cv"):
            args.append(intcol(b))
            rest = rest[2:]
        else:
            args.append(int(b))
            rest = rest[1:]
    return getattr(NC, kind + name)(*args)


@pytest.mark.parametrize("case", G.CONV, ids=[c[0] for c in G.CONV])
def test_conv_goldens(case):
    S, Scalar, CS, NC = _s()
    name, inp, fb, tb, want = case
    inp = [s.encode() for s in inp] if isinstance(inp, list) else inp.encode()
    check(_conv_call("convert", NC, Scalar, name, inp, fb, tb), [w.encode() for w in want])
    assert _conv_call("isConvertOverflow", NC, Scalar, name, inp, fb, tb) is G.CONV_OVERFLOW[name]


EDGES = [b"0", b"1", str(2**63 - 1).encode(), str(2**63).encode(), str(M64).encode(), str(2**64).encode(), b"-", b"-0",
         b"12 34", b"  -42  ", b"99xyz", b"abcXYZ", b"AbCdEf", b"\xff12", b"12\xc3\xa9", b"   ", b"", b"--5", b"-9223372036854775808",
         b"-18446744073709551616", b"ffffffffffffffff", b"10000000000000000", b"zzzzzzzzzzzzz", b"1" * 64, b"1" * 65, b"-zz", None]


def _rows(n, seed):
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        k = rng.random()
        if k < 0.15:
            out.append(rng.choice(EDGES))
            continue
        alphabet = rng.choice(["0123456789", "0123456789abcdefABCDEF", "01", "0123456789abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"])
        s = ("-" if rng.random() < 0.3 else "") + "".join(rng.choice(alphabet) for _ in range(rng.randint(0, 22)))
        if rng.random() < 0.1:
            s = " " * rng.randint(1, 3) + s + " " * rng.randint(0, 2)
        out.append(s.encode())
    return out


def _bases(n, seed, lo, hi, signed):
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        k = rng.random()
        if k < 0.03:
            out.append(None)
        elif k < 0.06:
            out.append(rng.choice([0, 1, 37, -1, 100, -(2**31)]))
        else:
            out.append(rng.randint(lo, hi) * (rng.choice([1, -1]) if signed else 1))
    return out


@pytest.mark.parametrize("name", OVERLOADS)
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000])
def test_conv_every_overload(name, n):
    S, Scalar, CS, NC = _s()
    rows = _rows(n, n)
    scalar = b"  -7fffffffffffffffZ"
    fbs, tbs = _bases(n, 2 * n, 2, 36, False), _bases(n, 3 * n, 2, 36, True)
    inp = scalar if name[0] == "S" else rows
    rest = name[1:] if name[0] == "S" else name[2:]
    fb = fbs if rest.startswith("Cv") else 16
    tb = tbs if rest.endswith("Cv") else -10
    check(_conv_call("convert", NC, Scalar, name, inp, fb, tb), R.conv(inp, fb, tb))
    assert _conv_call("isConvertOverflow", NC, Scalar, name, inp, fb, tb) == R.conv_overflow(inp, fb, tb)


@pytest.mark.parametrize("name", OVERLOADS)
def test_conv_overflow_flag_per_overload(name):
    S, Scalar, CS, NC = _s()
    big = str(2**64).encode()
    inp = big if name[0] == "S" else [b"1", None, big, b"5"]
    rest = name[1:] if name[0] == "S" else name[2:]
    fb = [10, 10, 10, 10] if rest.startswith("Cv") else 10
    tb = [16, 16, 16, 16] if rest.endswith("Cv") else 16
    assert _conv_call("isConvertOverflow", NC, Scalar, name, inp, fb, tb) is True
    check(_conv_call("convert", NC, Scalar, name, inp, fb, tb), R.conv(inp, fb, tb))
    # the overflowing row's base null: no overflow
    if rest.startswith("Cv"):
        assert _conv_call("isConvertOverflow", NC, Scalar, name, inp, [10, 10, None, 10] if name[0] != "S" else [None] * 4, tb) is False


def test_conv_every_base_pair():
    S, Scalar, CS, NC = _s()
    rows = [e for e in EDGES if e is not None]
    pairs = [(f, t) for f in range(2, 37) for t in list(range(2, 37)) + list(range(-36, -1))]
    inp = [r for _ in pairs for r in rows]
    fb = [f for f, _ in pairs for _ in rows]
    tb = [t for _, t in pairs for _ in rows]
    check(NC.convertCvCvCv(strcol(inp), intcol(fb), intcol(tb)), R.conv(inp, fb, tb))


@pytest.mark.parametrize("fb,tb", [(1, 10), (10, 37), (37, -2), (10, -1), (0, 0)])
def test_conv_invalid_scalar_bases(fb, tb):
    S, Scalar, CS, NC = _s()
    rows = [b"12", None, b"99"]
    check(NC.convertCvSS(strcol(rows), fb, tb), [None, None, None])
    assert NC.isConvertOverflowCvSS(strcol([str(2**64).encode()]), fb, tb) is False


def test_conv_sliced_input_and_grid_stride_edges():
    S, Scalar, CS, NC = _s()
    import torch
    sweep = 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256   # rows of one grid sweep
    for n in (sweep - 1, sweep, sweep + 33):
        rows = _rows(n, n)
        check(NC.convertCvSS(strcol(rows, pad=7), 36, -16), R.conv(rows, 36, -16))
        assert NC.isConvertOverflowCvSS(strcol(rows, pad=7), 36, -16) == R.conv_overflow(rows, 36, -16)


def test_conv_zero_rows():
    S, Scalar, CS, NC = _s()
    check(NC.convertCvSS(strcol([]), 10, 16), [])
    assert NC.isConvertOverflowCvSS(strcol([]), 10, 16) is False


INT_TYPES = [(1, np.int8, 8, True), (2, np.int16, 16, True), (3, np.int32, 32, True), (4, np.int64, 64, True),
             (5, np.uint8, 8, False), (6, np.uint16, 16, False), (7, np.uint32, 32, False), (8, np.uint64, 64, False)]


@pytest.mark.parametrize("type_id,np_type,bits,signed", INT_TYPES)
@pytest.mark.parametrize("base", [10, 16])
def test_from_integers_with_base(type_id, np_type, bits, signed, base):
    S, Scalar, CS, NC = _s()
    lo, hi = (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if signed else (0, (1 << bits) - 1)
    rng = random.Random(bits + base)
    vals = [lo, hi, 0, 1, None, 15, 16, lo + 1, hi - 1] + [rng.randint(lo, hi) >> rng.randint(0, bits - 1) if rng.random() > 0.1 else None
                                                           for _ in range(4099)]
    got = CS.fromIntegersWithBase(intcol(vals, type_id, np_type), base)
    check(got, R.integers_to_string([v or 0 for v in vals], [v is not None for v in vals], bits, signed, base))


def test_from_integers_with_base_other_base_is_a_cast_error():
    S, Scalar, CS, NC = _s()
    from srj_b200.cast import CastException
    with pytest.raises(CastException, match="Bases supported 10, 16; Actual: 8") as e:
        CS.fromIntegersWithBase(intcol([1]), 8)
    assert e.value.getRowWithError() == 0


def test_integer_goldens():
    S, Scalar, CS, NC = _s()
    check(CS.fromLongToBinary(intcol(G.LONGS, S.DType.INT64, np.int64)), [None if w is None else w.encode() for w in G.LONGS_BINARY])
    vals = [v for v, _, _ in G.UINT64_DEC_HEX]
    col = intcol(vals, S.DType.UINT64, np.uint64)
    check(CS.fromIntegersWithBase(col, 10), [None if d is None else d.encode() for _, d, _ in G.UINT64_DEC_HEX])
    check(CS.fromIntegersWithBase(col, 16), [None if h is None else h.encode() for _, _, h in G.UINT64_DEC_HEX])


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 100_003])
def test_long_to_binary(n):
    S, Scalar, CS, NC = _s()
    rng = random.Random(n)
    vals = [None if rng.random() < 0.1 else rng.randint(-(2**63), 2**63 - 1) >> rng.randint(0, 63) for _ in range(n)]
    check(CS.fromLongToBinary(intcol(vals, S.DType.INT64, np.int64)), R.long_to_binary([v or 0 for v in vals], [v is not None for v in vals]))


def _hex_check(got, data, offs, valid):
    w_offs, w_chars = R.bytes_to_hex(data, offs)
    assert got.offsets.cpu().numpy().tolist() == w_offs
    assert bytes(got.data.cpu().numpy().tobytes()) == w_chars
    if all(valid):
        assert got.mask is None
    else:
        bits = np.unpackbits(got.mask.cpu().numpy().view(np.uint8), bitorder="little")[:len(valid)].astype(bool)
        assert bits.tolist() == list(valid) and got.getNullCount() == list(valid).count(False)


def test_bytes_to_hex_goldens():
    S, Scalar, CS, NC = _s()
    got = CS.bytesToHex(strcol(G.HEX_STRINGS))
    check(got, [None if w is None else w.encode() for w in G.HEX_STRINGS_EXPECTED])
    import torch
    data = b"".join(r for r in G.HEX_BINARY if r is not None)
    offs = np.array([0, 2, 4, 4, 4], np.int32)
    child = S.ColumnVector.from_numpy(S.DType.UINT8, np.frombuffer(data, np.uint8))
    lst = S.ColumnView.makeListView(torch.from_numpy(offs).cuda(), child, torch.from_numpy(_mask([True, True, False, True]).view(np.int32)).cuda())
    check(CS.bytesToHex(lst), [None if w is None else w.encode() for w in G.HEX_BINARY_EXPECTED])


@pytest.mark.parametrize("n", [1, 31, 32, 33, 20_011])
@pytest.mark.parametrize("binary", [False, True])
def test_bytes_to_hex_null_rows_keep_their_span(n, binary):
    S, Scalar, CS, NC = _s()
    import torch
    rng = random.Random(n)
    lens = [rng.choice([0, 1, 3, 4, 5, 40, 300]) for _ in range(n)]
    pad = 5
    data = bytes(rng.getrandbits(8) for _ in range(pad + sum(lens)))
    offs = np.concatenate([[pad], pad + np.cumsum(lens)]).astype(np.int32)     # a slice: offsets start at 5
    valid = [rng.random() > 0.2 for _ in range(n)]
    m = _mask(valid)
    mt = None if m is None else torch.from_numpy(m.view(np.int32).copy()).cuda()
    if binary:
        child = S.ColumnVector.from_numpy(S.DType.UINT8, np.frombuffer(data, np.uint8))
        col = S.ColumnView.makeListView(torch.from_numpy(offs).cuda(), child, mt)
    else:
        col = S.ColumnVector.from_numpy(S.DType.STRING, np.frombuffer(data, np.uint8), m, offs, size=n)
    _hex_check(CS.bytesToHex(col), data, offs.tolist(), valid)


def test_bytes_to_hex_rejects_a_list_of_other_bytes():
    S, Scalar, CS, NC = _s()
    import torch
    child = S.ColumnVector.from_numpy(S.DType.INT8, np.zeros(4, np.int8))
    with pytest.raises(S.CudfException):
        CS.bytesToHex(S.ColumnView.makeListView(torch.tensor([0, 4], dtype=torch.int32, device="cuda"), child))


def test_results_near_the_int32_chars_limit():
    """bytesToHex of 2^30 - 1 bytes (2^31 - 2 chars) succeeds; 2^30 + 1 bytes overflow.  conv of INT64_MIN to base -2 (65
    chars a row) over 33,038,209 rows (2^31 - 63 chars) succeeds; one row more overflows."""
    S, Scalar, CS, NC = _s()
    import torch
    table = torch.tensor([ord(c) for b in range(256) for c in "%02X" % b], dtype=torch.uint8, device="cuda").view(256, 2)
    for nbytes, ok in ((2**30 - 1, True), (2**30 + 1, False)):
        data = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda")
        offs = torch.tensor([0, nbytes], dtype=torch.int32, device="cuda")
        col = S.ColumnVector(S.DType(S.DType.STRING), 1, data, None, offs)
        if ok:
            got = CS.bytesToHex(col)
            assert got.offsets.cpu().tolist() == [0, 2 * nbytes]
            assert torch.equal(got.data, table[data.long()].view(-1))
            del got
        else:
            with pytest.raises(S.CudfColumnSizeOverflowException):
                CS.bytesToHex(col)
        del data, col
        torch.cuda.empty_cache()
    want = R.conv(b"-9223372036854775808", [10], -2)[0]
    assert len(want) == 65
    row = torch.tensor(list(want), dtype=torch.uint8, device="cuda")
    for n, ok in ((33_038_209, True), (33_038_210, False)):
        bases = S.ColumnVector(S.DType(S.DType.INT32), n, torch.full((n,), 10, dtype=torch.int32, device="cuda").view(torch.uint8))
        if ok:
            got = NC.convertSCvS(Scalar.fromString(b"-9223372036854775808"), bases, -2)
            assert torch.equal(got.offsets, torch.arange(0, 65 * (n + 1), 65, dtype=torch.int64, device="cuda").to(torch.int32))
            assert torch.equal(got.data.view(n, 65), row.expand(n, 65)) and got.mask is None
            del got
        else:
            with pytest.raises(S.CudfColumnSizeOverflowException):
                NC.convertSCvS(Scalar.fromString(b"-9223372036854775808"), bases, -2)
        del bases
        torch.cuda.empty_cache()


def test_four_threads_on_their_own_streams():
    S, Scalar, CS, NC = _s()
    import torch
    errors = []

    def work(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for k in range(3):
                    rows = _rows(5000 + 17 * i + k, 100 * i + k)
                    got = NC.convertCvSS(strcol(rows), 10 + i, -(16 + i))
                    torch.cuda.current_stream().synchronize()
                    check(got, R.conv(rows, 10 + i, -(16 + i)))
                    vals = list(range(-2000 * i, 3000))
                    check(CS.fromIntegersWithBase(intcol(vals, S.DType.INT64, np.int64), 16), R.integers_to_string(vals, None, 64, True, 16))
        except Exception as e:   # noqa: BLE001 - reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
