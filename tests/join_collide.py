"""An invertible model of the hash join's row hash (csrc/join.cu row_hash), for building keys that collide on purpose.

The join decides that two rows match in two steps: the 32-bit row hash in the slot equals the probe's, then keys_equal
compares the keys.  The second step only decides anything for unequal keys with the same hash, which random keys almost
never produce.  Every step of the row hash is a bijection on the 32-bit state, and mm_mix is a bijection in its word as
well, so one free 32-bit word of a row can be solved for any target hash: run the steps forward up to the free word,
backward from the target to just after it, and solve mm_mix for the word.

A row is a list of (type_id, value) pairs, one per key column.  value is None for a null, the raw unsigned bits for a
fixed-width value (width * 8 bits; DECIMAL128 as one 128-bit int, low half first in memory), or bytes for a STRING.

The row hash (join.cu row_hash), with seed 0 and the running hash as the next column's seed:
  1-, 2- and 4-byte values: mm_u32 of the canonical bits, zero-extended (BOOL8 as 0 / 1; FLOAT32 with every NaN one NaN
  and -0.0 as 0.0); 8-byte values: mm_u64 (FLOAT64 canonical likewise); DECIMAL128: mm_u64(hi, mm_u64(lo, h));
  STRING: mm_bytes with Spark's sign-extended tail bytes; a null: mm_mix(h, kNullKeyWord) with no fmix.

The Murmur3 primitives come from spark_hash_model; only their inverses are written here.
"""
from __future__ import annotations

import os
import re

from spark_hash_model import (BOOL8, DECIMAL32, DECIMAL64, DECIMAL128, DURATION_DAYS, DURATION_MICROSECONDS,
                              DURATION_MILLISECONDS, DURATION_NANOSECONDS, DURATION_SECONDS, FLOAT32, FLOAT64, INT8,
                              INT16, INT32, INT64, M32, STRING, TIMESTAMP_DAYS, TIMESTAMP_MICROSECONDS,
                              TIMESTAMP_MILLISECONDS, TIMESTAMP_NANOSECONDS, TIMESTAMP_SECONDS, UINT8, UINT16, UINT32,
                              UINT64, _f32, _f64, _fmix, _mix_h1, _mix_k1)

JOIN_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "spark-rapids-jni_b200", "csrc", "join.cu")

NULL_KEY_WORD = 0x9E3779B9          # join.cu kNullKeyWord; test_join_collide.py ties it to the source

# join.cu join_key_width: bytes of each key type, 0 for STRING
WIDTH = {INT8: 1, UINT8: 1, BOOL8: 1, INT16: 2, UINT16: 2, DECIMAL128: 16, STRING: 0}
WIDTH.update({t: 4 for t in (INT32, UINT32, FLOAT32, TIMESTAMP_DAYS, DURATION_DAYS, DECIMAL32)})
WIDTH.update({t: 8 for t in (INT64, UINT64, FLOAT64, DECIMAL64, TIMESTAMP_SECONDS, TIMESTAMP_MILLISECONDS,
                             TIMESTAMP_MICROSECONDS, TIMESTAMP_NANOSECONDS, DURATION_SECONDS, DURATION_MILLISECONDS,
                             DURATION_MICROSECONDS, DURATION_NANOSECONDS)})
FIXED_TYPES = [t for t in WIDTH if WIDTH[t] > 0]


# ---------------------------------------------------------------- inverses of the Murmur3 steps
def _rotr32(x: int, r: int) -> int:
    return ((x >> r) | (x << (32 - r))) & M32


_INV5 = pow(5, -1, 1 << 32)
_INV_C1 = pow(0xCC9E2D51, -1, 1 << 32)
_INV_C2 = pow(0x1B873593, -1, 1 << 32)
_INV_F1 = pow(0x85EBCA6B, -1, 1 << 32)
_INV_F2 = pow(0xC2B2AE35, -1, 1 << 32)


def unmix_k1(x: int) -> int:
    """k with _mix_k1(k) == x"""
    return (_rotr32((x * _INV_C2) & M32, 15) * _INV_C1) & M32


def unmix_h1(h: int, k1: int) -> int:
    """h0 with _mix_h1(h0, k1) == h"""
    return _rotr32(((h - 0xE6546B64) * _INV5) & M32, 13) ^ k1


def _unxorshift(h: int, s: int) -> int:
    """x with x ^ (x >> s) == h"""
    x = h
    for _ in range(32 // s + 1):
        x = h ^ (x >> s)
    return x


def unfmix(h: int, length: int) -> int:
    """h0 with _fmix(h0, length) == h"""
    h = _unxorshift(h, 16)
    h = (h * _INV_F2) & M32
    h = _unxorshift(h, 13)
    h = (h * _INV_F1) & M32
    h = _unxorshift(h, 16)
    return h ^ (length & M32)


def mm_mix(h: int, k: int) -> int:
    """hash_device.cuh mm_mix: one block into the running hash"""
    return _mix_h1(h, _mix_k1(k & M32))


def unmm_mix(h: int, k: int) -> int:
    """h0 with mm_mix(h0, k) == h"""
    return unmix_h1(h, _mix_k1(k & M32))


def solve_mix(h0: int, h1: int) -> int:
    """the word k with mm_mix(h0, k) == h1"""
    return unmix_k1(_rotr32(((h1 - 0xE6546B64) * _INV5) & M32, 13) ^ h0)


def step(kind: str, arg: int, h: int) -> int:
    return mm_mix(h, arg) if kind == "mix" else _fmix(h, arg)


def unstep(kind: str, arg: int, h: int) -> int:
    return unmm_mix(h, arg) if kind == "mix" else unfmix(h, arg)


# ---------------------------------------------------------------- the row hash as a list of 32-bit steps
def canon(t: int, v: int) -> int:
    """join.cu canon: the bits a fixed-width value hashes and compares by"""
    if t == BOOL8:
        return int(v != 0)
    if t == FLOAT32:
        return _f32(v, True)
    if t == FLOAT64:
        return _f64(v, True)
    return v


def column_steps(t: int, v, c: int):
    """[(kind, arg, addr)] of one key column c: kind "mix" (arg the word) or "fmix" (arg the length); addr names the value
    word a "mix" step reads, (c, j), or is None for a word the row cannot change on its own (a sub-word value, a tail
    byte, the null word)"""
    if v is None:
        return [("mix", NULL_KEY_WORD, None)]
    w = WIDTH[t]
    if w == 0:
        n4 = len(v) // 4
        out = [("mix", int.from_bytes(v[4 * j:4 * j + 4], "little"), (c, j)) for j in range(n4)]
        out += [("mix", (x - 256 if x >= 128 else x) & M32, None) for x in v[4 * n4:]]
        return out + [("fmix", len(v), None)]
    b = canon(t, v)
    if w <= 4:
        return [("mix", b, (c, 0) if w == 4 else None), ("fmix", 4, None)]
    if w == 8:
        return [("mix", b & M32, (c, 0)), ("mix", b >> 32, (c, 1)), ("fmix", 8, None)]
    return [("mix", b & M32, (c, 0)), ("mix", (b >> 32) & M32, (c, 1)), ("fmix", 8, None),
            ("mix", (b >> 64) & M32, (c, 2)), ("mix", b >> 96, (c, 3)), ("fmix", 8, None)]


def steps(row):
    out = []
    for c, (t, v) in enumerate(row):
        out += column_steps(t, v, c)
    return out


def row_hash(row) -> int:
    """the join's 32-bit row hash, unsigned"""
    h = 0
    for kind, arg, _ in steps(row):
        h = step(kind, arg, h)
    return h


def signed(h: int) -> int:
    return h - (1 << 32) if h >> 31 else h


# ---------------------------------------------------------------- free words
def free_words(row):
    """every (column, word) the solver may rewrite: a 4-byte value, either half of an 8-byte value, any of a
    DECIMAL128's four words, any whole 4-byte block of a string"""
    return [a for _, _, a in steps(row) if a is not None]


def get_word(row, addr) -> int:
    c, j = addr
    t, v = row[c]
    if WIDTH[t] == 0:
        return int.from_bytes(v[4 * j:4 * j + 4], "little")
    return (v >> (32 * j)) & M32


def set_word(row, addr, w: int):
    """a copy of row with word addr set to w (raw bits)"""
    c, j = addr
    t, v = row[c]
    if WIDTH[t] == 0:
        nv = v[:4 * j] + (w & M32).to_bytes(4, "little") + v[4 * j + 4:]
    else:
        nv = (v & ~(M32 << (32 * j))) | ((w & M32) << (32 * j))
    out = list(row)
    out[c] = (t, nv)
    return out


def _canonical_word(row, addr) -> bool:
    """the value around addr hashes by its own bits (a solved FLOAT32 / FLOAT64 word may make a NaN or a -0.0)"""
    t, v = row[addr[0]]
    return t not in (FLOAT32, FLOAT64) or canon(t, v) == v


def solve(row, free, target: int, filler=None):
    """a copy of row, with word `free` rewritten, whose row hash is target.  When the solved word would make a float
    that the join canonicalises, word `filler` is stepped and the solve repeated (ValueError without a filler)."""
    for attempt in range(64):
        st = steps(row)
        i = next(n for n, s in enumerate(st) if s[2] == free)
        h0 = 0
        for kind, arg, _ in st[:i]:
            h0 = step(kind, arg, h0)
        h1 = target & M32
        for kind, arg, _ in reversed(st[i + 1:]):
            h1 = unstep(kind, arg, h1)
        out = set_word(row, free, solve_mix(h0, h1))
        if _canonical_word(out, free):
            assert row_hash(out) == target & M32
            return out
        if filler is None:
            raise ValueError(f"the solved word at {free} is not canonical")
        row = set_word(row, filler, get_word(row, filler) + 0x9E3779B1 * (attempt + 1))
    raise ValueError("no canonical solution")


# ---------------------------------------------------------------- collisions in string tail bytes
# A pair of rows that differ only in a string's 1-3 tail bytes cannot be made to collide by solving a block: the block
# would differ too.  Two tail bytes have 65,536 value pairs, so trying them all finds a colliding pair for about two
# base rows in five (birthday bound over 32 bits).
def _byte_step(row, pos) -> int:
    c, i = pos
    t, v = row[c]
    assert t == STRING and v is not None and 4 * (len(v) // 4) <= i < len(v), f"{pos} is not a tail byte"
    return sum(len(column_steps(tt, vv, cc)) for cc, (tt, vv) in enumerate(row[:c])) + len(v) // 4 + i - 4 * (len(v) // 4)


def set_byte(row, pos, x: int):
    c, i = pos
    t, v = row[c]
    out = list(row)
    out[c] = (t, v[:i] + bytes([x]) + v[i + 1:])
    return out


def tail_collision(row, p1, p2):
    """two copies of row that differ only in the tail bytes p1 and p2 ((column, byte index), p1 hashed first) and share
    a row hash, or None when no pair of values collides for this row"""
    st = steps(row)
    i1, i2 = _byte_step(row, p1), _byte_step(row, p2)
    assert i1 < i2
    h = 0
    for kind, arg, _ in st[:i1]:
        h = step(kind, arg, h)
    k2 = [_mix_k1((x - 256 if x >= 128 else x) & M32) for x in range(256)]
    seen = {}
    for x1 in range(256):
        g = mm_mix(h, x1 - 256 if x1 >= 128 else x1)
        for kind, arg, _ in st[i1 + 1:i2]:
            g = step(kind, arg, g)
        for x2 in range(256):
            s = _mix_h1(g, k2[x2])                    # the state after byte p2; every later step is the same for both
            if s in seen:
                y1, y2 = seen[s]
                return set_byte(set_byte(row, p1, y1), p2, y2), set_byte(set_byte(row, p1, x1), p2, x2)
            seen[s] = (x1, x2)
    return None


# ---------------------------------------------------------------- the build table
def buckets(right_rows: int) -> int:
    """join.cu join_buckets: the power-of-two count of 4-slot buckets, at least 2 * right_rows slots"""
    b = 1
    while 4 * b < 2 * right_rows:
        b <<= 1
    return b


# ---------------------------------------------------------------- the source this models
def join_source() -> str:
    with open(JOIN_CU) as f:
        return f.read()


def source_null_key_word(src: str) -> int:
    m = re.search(r"constexpr\s+uint32_t\s+kNullKeyWord\s*=\s*(0x[0-9a-fA-F]+)u?\s*;", src)
    assert m, "kNullKeyWord not found in join.cu"
    return int(m.group(1), 16)
