"""CPU tests of tests/join_collide.py, the invertible model of the hash join's row hash: the forward model against
spark_hash_model's Murmur3 where the two definitions agree, every inverse step, the solver on random rows over every
free-word kind and position, and a guard that ties the model to csrc/join.cu (the null word and the row hash's steps)."""
import os
import re
from collections import namedtuple

import numpy as np
import pytest

import join_collide as JC
import spark_hash_model as SH
from join_collide import (BOOL8, DECIMAL128, FLOAT32, FLOAT64, INT8, INT16, INT32, INT64, M32, STRING, TIMESTAMP_DAYS,
                          UINT8, UINT16, UINT32)

HCol = namedtuple("HCol", "type_id data mask offsets size children")

# the types whose join hash is Spark's Murmur3 of the same value (INT8 / INT16 and DECIMAL32 / DECIMAL128 are hashed
# differently by Spark: sign-extended, as a long, as BigInteger bytes; Spark's murmur3 does not fold -0.0)
AGREE_4 = [UINT8, UINT16, INT32, UINT32, TIMESTAMP_DAYS, SH.DURATION_DAYS, BOOL8]
AGREE_8 = [t for t in JC.FIXED_TYPES if JC.WIDTH[t] == 8 and t != FLOAT64]


def _host(t, v):
    """a one-row host column of value v (raw bits / bytes) for spark_hash_model"""
    if t == STRING:
        return HCol(t, np.frombuffer(v, np.uint8), None, np.array([0, len(v)], np.int32), 1, [])
    return HCol(t, np.frombuffer(v.to_bytes(JC.WIDTH[t], "little"), np.uint8), None, None, 1, [])


def _random_value(t, rng, finite_nonzero=False):
    if t == STRING:
        return rng.bytes(int(rng.integers(0, 70)))
    if t == FLOAT32:
        return int(np.float32(rng.standard_normal() * 1e3 + 0.5).view(np.uint32)) if finite_nonzero else int(rng.integers(0, 1 << 32))
    if t == FLOAT64:
        return int(np.float64(rng.standard_normal() * 1e9 + 0.5).view(np.uint64)) if finite_nonzero else int(rng.integers(0, 1 << 63)) * 2 + int(rng.integers(0, 2))
    w = JC.WIDTH[t]
    return int.from_bytes(rng.bytes(w), "little") if t != BOOL8 else int(rng.integers(0, 4))


def test_forward_model_matches_spark_murmur3():
    rng = np.random.default_rng(1)
    types = AGREE_4 + AGREE_8 + [STRING, FLOAT32, FLOAT64]
    for it in range(3000):
        ts = [types[int(i)] for i in rng.integers(0, len(types), 1 + it % 5)]
        row = [(t, _random_value(t, rng, finite_nonzero=True)) for t in ts]
        want = SH.row_hash("murmur3", [_host(t, v) for t, v in row], 0, seed=0)
        assert JC.row_hash(row) == want & M32, row
    for n in (0, 1, 2, 3, 4, 5, 7, 8, 4099, 4100, 4103):
        s = rng.bytes(n)
        assert JC.row_hash([(STRING, s)]) == SH.murmur_bytes(s, 0)


def test_forward_model_where_the_join_differs_from_spark():
    rng = np.random.default_rng(2)
    for _ in range(500):
        h = int(rng.integers(0, 1 << 32))
        lead = (UINT32, h)                                          # any running hash is reached from some leading word
        h = JC.row_hash([lead])
        b1, b2, dec = int(rng.integers(0, 256)), int(rng.integers(0, 1 << 16)), int.from_bytes(rng.bytes(16), "little")
        assert JC.row_hash([lead, (INT8, b1)]) == SH.murmur_int(b1, h)                   # zero-extended, not sign-extended
        assert JC.row_hash([lead, (INT16, b2)]) == SH.murmur_int(b2, h)
        assert JC.row_hash([lead, (SH.DECIMAL32, b2 << 16)]) == SH.murmur_int(b2 << 16, h)  # as an int, not a long
        assert JC.row_hash([lead, (DECIMAL128, dec)]) == SH.murmur_long(dec >> 64, SH.murmur_long(dec & ((1 << 64) - 1), h))
        assert JC.row_hash([lead, (INT32, None)]) == SH._mix_h1(h, SH._mix_k1(JC.NULL_KEY_WORD))   # no fmix
        assert JC.row_hash([lead, (BOOL8, b1)]) == SH.murmur_int(int(b1 != 0), h)
    for nan in (0x7FC00001, 0xFFC00000, 0x7F800001):
        assert JC.row_hash([(FLOAT32, nan)]) == SH.murmur_int(0x7FC00000, 0)
    assert JC.row_hash([(FLOAT32, 0x80000000)]) == JC.row_hash([(FLOAT32, 0)])
    assert JC.row_hash([(FLOAT64, 0x8000000000000000)]) == JC.row_hash([(FLOAT64, 0)])
    assert JC.row_hash([(FLOAT64, 0xFFF0000000000001)]) == SH.murmur_long(0x7FF8000000000000, 0)


def test_inverse_steps_round_trip():
    rng = np.random.default_rng(3)
    hs, ks = rng.integers(0, 1 << 32, 10_000), rng.integers(0, 1 << 32, 10_000)
    for h, k in zip(hs.tolist(), ks.tolist()):
        assert JC.unmix_k1(SH._mix_k1(k)) == k
        assert JC.unmix_h1(SH._mix_h1(h, k), k) == h
        assert JC.unmm_mix(JC.mm_mix(h, k), k) == h
        assert JC.solve_mix(h, JC.mm_mix(h, k)) == k
        for n in (4, 8, k & 0xFFF):
            assert JC.unfmix(SH._fmix(h, n), n) == h
    for h in (0, M32, 0x80000000, 1):
        assert JC.unfmix(SH._fmix(h, 4), 4) == h and JC.solve_mix(h, JC.mm_mix(h, h)) == h


SOLVE_TYPES = [t for t in JC.FIXED_TYPES] + [STRING, STRING, STRING]


def _random_row(rng, ncols):
    row = []
    for _ in range(ncols):
        t = SOLVE_TYPES[int(rng.integers(0, len(SOLVE_TYPES)))]
        if rng.random() < 0.1:
            row.append((t, None))
        elif t == STRING:
            row.append((t, rng.bytes(int(rng.integers(0, 41)) if rng.random() < 0.995 else int(rng.integers(4090, 4110)))))
        else:
            row.append((t, int(JC.canon(t, _random_value(t, rng)))))
    return row


def test_solver_collides_on_every_free_word():
    rng = np.random.default_rng(4)
    kinds, solved = set(), 0
    specials = [0, M32, 0x80000000] + [(1 << b) - 1 for b in range(1, 24)]       # buckets - 1 for every table size
    while solved < 10_000:
        row = _random_row(rng, int(rng.integers(1, 7)))
        free = JC.free_words(row)
        if len(free) < 2:
            continue
        fi = int(rng.integers(0, len(free)))
        addr, filler = free[fi], free[(fi + 1) % len(free)]
        target = specials[solved % len(specials)] if solved % 2 else int(rng.integers(0, 1 << 32))
        out = JC.solve(row, addr, target, filler)
        assert JC.row_hash(out) == target
        assert out != row
        t = row[addr[0]][0]
        kinds.add((t if t in (STRING, FLOAT32, FLOAT64) else JC.WIDTH[t], addr[1] if t != STRING else min(addr[1], 2)))
        solved += 1
    # every free-word kind was solved for: 4-byte values, both halves of 8-byte values, DECIMAL128's four words, the
    # first, second and later blocks of strings, and both float widths (whose solutions must stay canonical)
    assert kinds >= {(4, 0), (8, 0), (8, 1), (16, 0), (16, 1), (16, 2), (16, 3), (STRING, 0), (STRING, 1), (STRING, 2),
                     (FLOAT32, 0), (FLOAT64, 0), (FLOAT64, 1)}


def test_solver_steps_the_filler_past_non_canonical_floats():
    # targets whose solution is a NaN payload or -0.0: the join would hash those as the canonical NaN / 0.0
    for t, row, free, filler, bad in ((FLOAT64, [(FLOAT64, 5)], (0, 1), (0, 0), 0x7FF80001),
                                      (FLOAT64, [(FLOAT64, 0)], (0, 1), None, 0x80000000),
                                      (FLOAT32, [(FLOAT32, 0), (INT32, 7)], (0, 0), (1, 0), 0x80000000),
                                      (FLOAT32, [(INT32, 7), (FLOAT32, 0)], (1, 0), (0, 0), 0xFFC00001)):
        raw = JC.set_word(row, free, bad)
        target = 0
        for kind, arg, _ in [s for c, (tt, v) in enumerate(raw) for s in JC.column_steps(INT64 if tt == FLOAT64 else INT32 if tt == FLOAT32 else tt, v, c)]:
            target = JC.step(kind, arg, target)                  # the hash of the raw bits, as if not canonicalised
        with pytest.raises(ValueError):
            JC.solve(row, free, target)
        if filler is not None:
            out = JC.solve(row, free, target, filler)
            assert JC.row_hash(out) == target and JC.canon(t, out[free[0]][1]) == out[free[0]][1]


def test_solver_long_strings_and_extreme_targets():
    rng = np.random.default_rng(5)
    for n in (4, 5, 8, 4096, 4100, 4103):
        s = rng.bytes(n)
        for target in (0, M32, 0x80000000, 0x7FFFF):
            for j in (0, n // 4 - 1):
                out = JC.solve([(STRING, s)], (0, j), target)
                assert JC.row_hash(out) == target and out[0][1] != s and len(out[0][1]) == n
                assert out[0][1][:4 * j] == s[:4 * j] and out[0][1][4 * j + 4:] == s[4 * j + 4:]


def test_tail_collisions_differ_only_in_the_tail():
    rng = np.random.default_rng(6)
    found = 0
    for it in range(40):
        la, lb = 4 * int(rng.integers(0, 4)) + 1 + it % 3, 4 * int(rng.integers(0, 4)) + 1 + (it // 3) % 3
        if it % 2:
            row = [(STRING, rng.bytes(la)), (INT32, 7), (STRING, rng.bytes(lb))]
            p1, p2 = (0, la - 1), (2, lb - 1)
        else:
            la = la if la % 4 >= 2 else la + 1
            row = [(STRING, rng.bytes(la)), (INT64, 9)]
            p1, p2 = (0, la - 2), (0, la - 1)
        pair = JC.tail_collision(row, p1, p2)
        if pair is None:
            continue
        a, b = pair
        found += 1
        assert a != b and JC.row_hash(a) == JC.row_hash(b)
        for (t, x), (_, y) in zip(a, b):
            if t == STRING:
                n4 = len(x) // 4 * 4
                assert len(x) == len(y) and x[:n4] == y[:n4]
            else:
                assert x == y
    assert found >= 8


def test_model_matches_join_cu_and_type_width():
    src = JC.join_source()
    assert JC.source_null_key_word(src) == JC.NULL_KEY_WORD
    body = re.search(r"uint32_t row_hash\(.*?\n}\n", src, re.S)
    assert body, "row_hash not found in join.cu"
    flat = re.sub(r"\s+", " ", body.group(0))
    for piece in ("uint32_t h = 0;",
                  "if (!valid_at(k.mask, r)) { any = true; h = mm_mix(h, kNullKeyWord); }",
                  "h = mm_bytes(k.data + b, __ldg(k.offsets + r + 1) - b, h);",
                  "h = k.width <= 4 ? mm_u32(static_cast<uint32_t>(v), h) : k.width == 8 ? mm_u64(v, h) : mm_u64(hi, mm_u64(v, h));"):
        assert piece in flat, piece
    canon_src = re.sub(r"\s+", " ", re.search(r"uint64_t canon\(.*?\n}\n", src, re.S).group(0))
    for piece in ("return c.type == SRJ_BOOL8 ? uint64_t{v != 0} : v;", "return c.type == SRJ_FLOAT32 ? norm_f32(v, true) : v;",
                  "return c.type == SRJ_FLOAT64 ? norm_f64(v, true) : v;", "hi = __ldg(p + 1); return __ldg(p);"):
        assert piece in canon_src, piece
    # the table the chain tests wrap around: empty slots all ones, buckets a power of two with 2 x right_rows slots
    assert re.search(r"constexpr uint64_t kEmptySlot\s*=\s*~0ull;", src)
    assert re.search(r"while \(4 \* b < 2 \* static_cast<uint64_t>\(right_rows\)\) b <<= 1;", src)
    assert [JC.buckets(n) for n in (0, 1, 2, 3, 1000, 1 << 20)] == [1, 1, 1, 2, 512, 1 << 19]
    # the widths the model steps by are type_width's (check.hpp), which join.cu reads its key widths from
    assert "d.width             = s.type_id == SRJ_STRING ? 0 : type_width(s.type_id);" in src
    check_hpp = open(os.path.join(os.path.dirname(JC.JOIN_CU), "check.hpp")).read()
    for t, w in JC.WIDTH.items():
        if w:
            cases = re.search(r"int type_width\(int32_t type_id\)\s*{(.*?)\n}", check_hpp, re.S).group(1)
            name = {v: k for k, v in vars(SH).items() if k.isupper() and isinstance(v, int) and k not in ("M32", "M64")}[t]
            arm = re.search(r"case SRJ_" + name + r":[^;]*?return (\d+);", cases)
            assert arm and int(arm.group(1)) == w, name
