"""CPU checks of oracle/radix.py: the reference's test cases (tests/golden/radix_golden.py), and agreement with the
independent model of Spark's intent (tests/radix_model.py) on the named edges, every (fromBase, toBase) pair with toBase
of both signs, and 10^6 random rows per native."""
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import radix as R          # noqa: E402
import radix_model as M                # noqa: E402
from golden import radix_golden as G   # noqa: E402

M64 = (1 << 64) - 1
ROWS = 1_000_000


def _enc(x):
    return None if x is None else x.encode()


@pytest.mark.parametrize("case", G.CONV, ids=[c[0] for c in G.CONV])
def test_conv_goldens(case):
    name, inp, fb, tb, want = case
    ins = [_enc(s) for s in inp] if isinstance(inp, list) else inp.encode()
    assert R.conv(ins, fb, tb) == [_enc(w) for w in want]
    assert R.conv_overflow(ins, fb, tb) == G.CONV_OVERFLOW[name]


def test_integer_goldens():
    assert R.long_to_binary([v or 0 for v in G.LONGS], [v is not None for v in G.LONGS]) == [_enc(w) for w in G.LONGS_BINARY]
    vals = [v or 0 for v, _, _ in G.UINT64_DEC_HEX]
    valid = [v is not None for v, _, _ in G.UINT64_DEC_HEX]
    assert R.integers_to_string(vals, valid, 64, False, 10) == [_enc(d) for _, d, _ in G.UINT64_DEC_HEX]
    assert R.integers_to_string(vals, valid, 64, False, 16) == [_enc(h) for _, _, h in G.UINT64_DEC_HEX]


@pytest.mark.parametrize("rows,want", [(G.HEX_STRINGS, G.HEX_STRINGS_EXPECTED), (G.HEX_BINARY, G.HEX_BINARY_EXPECTED)])
def test_bytes_to_hex_goldens(rows, want):
    data = b"".join(r for r in rows if r is not None)
    offs = [0]
    for r in rows:
        offs.append(offs[-1] + (0 if r is None else len(r)))
    out_offs, chars = R.bytes_to_hex(data, offs)
    got = [chars[out_offs[i]:out_offs[i + 1]].decode() for i in range(len(rows))]
    assert [g if r is not None else None for g, r in zip(got, rows)] == want


def _model_row(s, fb, tb):
    if s is None or fb is None or tb is None or not (2 <= fb <= 36 and 2 <= abs(tb) <= 36):
        return None
    r = M.conv(s, fb, tb)[0]
    return None if r is None else r.encode()


EDGES = [b"0", b"1", str(2**63 - 1).encode(), str(2**63).encode(), str(M64).encode(), str(2**64).encode(), b"-", b"-0",
         b"12 34", b"  -42  ", b"99xyz", b"abcXYZ", b"AbCdEf", b"\xff12", b"12\xc3\xa9", b"   ", b"", b"--5", b"-9223372036854775808",
         b"-18446744073709551615", b"-18446744073709551616", b"ffffffffffffffff", b"10000000000000000", b"zzzzzzzzzzzzz", b"1" * 64,
         b"1" * 65, b"7777777777777777777777", b"2000000000000000000000", b"+5", b"\t5", b"0x1F", b"-zz"]


@pytest.mark.parametrize("fb", range(2, 37))
def test_conv_every_base_pair_on_the_edges(fb):
    for tb in list(range(2, 37)) + list(range(-36, -1)):
        for s in EDGES:
            assert R.conv([s], fb, tb) == [_model_row(s, fb, tb)], (s, fb, tb)
            want = M.conv(s, fb, tb, ansi=True)[1]
            assert (R.convert_row(s, fb, tb, True)[0] == R.OVERFLOW) == want, (s, fb, tb)


def test_conv_edges_by_hand():
    assert R.conv([b"-0"], 10, -10) == [b"-0"]
    assert R.conv([b"-9223372036854775808"], 10, -10) == [b"-9223372036854775808"]
    assert R.conv([b"-"], 10, 16) == [b"0"] and R.conv([b"xyz"], 10, 16) == [b"0"]
    assert R.conv([str(2**64).encode()], 10, 16) == [b"FFFFFFFFFFFFFFFF"]
    assert R.conv_overflow([str(2**64).encode()], 10, 16) and not R.conv_overflow([str(M64).encode()], 10, 16)
    assert R.conv([b" ", b"", None], 10, 16) == [None, None, None]
    assert R.conv([b"5"], 1, 10) == [None] and not R.conv_overflow([str(2**64).encode()], 37, 10)
    assert R.conv([b"5", b"5"], [10, None], [10, 10]) == [b"5", None]


def _rand_string(rng):
    k = rng.random()
    if k < 0.05:
        return None
    if k < 0.1:
        return rng.choice(EDGES)
    alphabet = rng.choice(["0123456789", "0123456789abcdefABCDEF", "01", "0123456789abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"])
    body = "".join(rng.choice(alphabet) for _ in range(rng.randint(0, 24)))
    s = ("-" if rng.random() < 0.3 else "") + body
    if rng.random() < 0.1:
        s = " " * rng.randint(1, 3) + s + " " * rng.randint(0, 3)
    if rng.random() < 0.1:
        s += rng.choice([" 12", "x", "é", "-3"])
    return s.encode()


def test_conv_random_rows_against_the_model():
    rng = random.Random(11)
    for _ in range(ROWS):
        s = _rand_string(rng)
        fb = rng.randint(2, 36) if rng.random() < 0.97 else rng.choice([None, 0, 1, 37, -10])
        tb = rng.choice([1, -1]) * rng.randint(2, 36) if rng.random() < 0.97 else rng.choice([None, 0, 1, -1, 37, -37])
        assert R.conv([s], [fb], [tb]) == [_model_row(s, fb, tb)], (s, fb, tb)
        if s is not None and fb is not None and tb is not None and 2 <= fb <= 36 and 2 <= abs(tb) <= 36:
            assert R.conv_overflow([s], fb, tb) == M.conv(s, fb, tb, ansi=True)[1], (s, fb, tb)


INT_TYPES = [(8, True), (16, True), (32, True), (64, True), (8, False), (16, False), (32, False), (64, False)]


@pytest.mark.parametrize("bits,signed", INT_TYPES)
def test_integers_random_rows_against_the_model(bits, signed):
    rng = random.Random(bits * 2 + signed)
    lo, hi = (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if signed else (0, (1 << bits) - 1)
    vals = [lo, hi, 0, 1, -1 if signed else 2, 15, 16, 255 if hi >= 255 else hi] + [rng.randint(lo, hi) >> rng.randint(0, bits - 1)
                                                                                      for _ in range(ROWS // 8)]
    for base in (10, 16):
        got = R.integers_to_string(vals, None, bits, signed, base)
        assert got == [M.integer_to_string(v, bits, base).encode() for v in vals]


def test_long_to_binary_random_rows_against_the_model():
    rng = random.Random(3)
    vals = [0, 1, -1, 2**63 - 1, -(2**63)] + [rng.randint(-(2**63), 2**63 - 1) >> rng.randint(0, 63) for _ in range(ROWS)]
    assert R.long_to_binary(vals) == [M.long_to_binary(v).encode() for v in vals]


def test_bytes_to_hex_random_rows_against_the_model():
    rng = random.Random(4)
    data = bytes(rng.getrandbits(8) for _ in range(ROWS))
    offs = sorted({0, ROWS} | {rng.randrange(ROWS) for _ in range(ROWS // 20)})
    start = len(offs) // 3                                       # a slice: offsets that do not start at 0
    out_offs, chars = R.bytes_to_hex(data, offs[start:])
    assert out_offs[0] == 0 and chars.decode() == M.bytes_to_hex(data[offs[start]:])
    for i in range(0, len(out_offs) - 1, 97):
        a, b = offs[start + i], offs[start + i + 1]
        assert chars[out_offs[i]:out_offs[i + 1]].decode() == M.bytes_to_hex(data[a:b])
