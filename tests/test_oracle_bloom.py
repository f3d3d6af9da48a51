"""CPU checks of the bloom filter oracle (oracle/bloom.py): it reproduces every transcribed golden of the reference's
tests and the hand-derived known answers, and agrees with the independent model (tests/bloom_model.py) on random keys.
Also checks the modulo the kernels use (bloom_filter.cu: mod_v1 / mod_v2 with the host's bloom_reciprocal) through a
host mirror of the device arithmetic against Python's %."""
import random

import numpy as np
import pytest

import bloom_model as M
from golden import bloom_golden as G
from oracle import bloom as B

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def _build(case):
    filters = []
    for puts in case["puts"]:
        f = B.create(case["version"], case["num_hashes"], case["bits"], case["seed"])
        for values, valid in puts:
            f = B.put(f, np.array(values, np.int64), None if valid is None else np.array(valid, bool))
        filters.append(f)
    return B.merge(filters) if case["merge"] else filters[0]


@pytest.mark.parametrize("case", G.CASES, ids=[c["name"] for c in G.CASES])
def test_oracle_matches_golden(case):
    got = B.probe(_build(case), np.array(case["probe"], np.int64))
    for g, e in zip(got, case["expected"]):
        if e is not None:
            assert bool(g) == e
    assert len(got) == len(case["expected"])


@pytest.mark.parametrize("version,k,longs,seed,size", G.INIT)
def test_oracle_initialization(version, k, longs, seed, size):
    f = B.create(version, k, 64 * longs, seed)
    assert len(f) == size and not f[B.header_bytes(version):].any()
    assert B.parse(f) == (version, k, seed if version == 2 else 0, longs)


@pytest.mark.parametrize("failure", G.FAILURES, ids=[str(i) for i in range(len(G.FAILURES))])
def test_oracle_expected_failures(failure):
    with pytest.raises(ValueError):
        if failure[0] == "create":
            B.create(*failure[1:])
        else:
            B.merge([B.create(*p) for p in failure[1]])


@pytest.mark.parametrize("known", G.KNOWN, ids=[f"v{k[0]}_seed{k[1]}_bits{k[2]}_key{k[3]}" for k in G.KNOWN])
def test_known_answers(known):
    version, seed, bits, key, h1, pos, hexbytes = known
    assert int(B.hash_long(np.array([key]), seed if version == 2 else 0)[0]) == h1 & 0xFFFFFFFF
    assert M.hash_long(key, seed if version == 2 else 0) == h1
    assert tuple(B.positions(version, 3, seed, bits, np.array([key]))[:, 0]) == pos
    assert tuple(M.positions(version, 3, seed, bits, key)) == pos
    assert B.put(B.create(version, 3, bits, seed), np.array([key])).tobytes().hex() == hexbytes
    f = M.Filter(version, 3, bits // 64, seed)
    f.put(key)
    assert f.serialize().hex() == hexbytes


def _keys(n, seed):
    r = random.Random(seed)
    return [INT64_MIN, INT64_MAX, 0, -1, 1] + [r.randrange(INT64_MIN, INT64_MAX + 1) for _ in range(n)]


@pytest.mark.parametrize("version", [1, 2])
@pytest.mark.parametrize("seed", [0, 42, -1])
@pytest.mark.parametrize("k,bits", [(1, 64), (3, 65), (5, 4096), (12, 29_193_763), (30, 2**22)])
def test_oracle_agrees_with_model(version, seed, k, bits):
    keys = _keys(300, seed=k * 7 + version)
    nbits = 64 * B.num_longs(bits)
    got = B.positions(version, k, seed, nbits, np.array(keys, np.int64))
    for j, key in enumerate(keys):
        assert got[:, j].tolist() == M.positions(version, k, seed, nbits, key)
    f = B.put(B.create(version, k, bits, seed), np.array(keys[:150], np.int64))
    m = M.Filter(version, k, B.num_longs(bits), seed)
    for key in keys[:150]:
        m.put(key)
    assert f.tobytes() == m.serialize()
    assert B.probe(f, np.array(keys, np.int64)).tolist() == [m.might_contain(x) for x in keys]


def test_v2_positions_reach_above_2_pow_32():
    nbits = 2**33
    keys = _keys(200, seed=3)
    got = B.positions(2, 5, 42, nbits, np.array(keys, np.int64))
    assert (got >= 2**32).any()
    for j, key in enumerate(keys[:40]):
        assert got[:, j].tolist() == M.positions(2, 5, 42, nbits, key)


def test_merge_is_the_or_of_the_bit_arrays():
    a = B.put(B.create(2, 4, 1000, 7), np.array([1, 2, 3]))
    b = B.put(B.create(2, 4, 1000, 7), np.array([4, 5]))
    m = B.merge([a, b])
    assert m[:16].tobytes() == a[:16].tobytes()
    assert np.array_equal(m[16:], a[16:] | b[16:])
    assert B.probe(m, np.array([1, 2, 3, 4, 5])).all()


# ---- the modulo of the put / probe kernels: host mirror of mod_v1 / mod_v2 and bloom_reciprocal (bloom_filter.cu)
M32, M64 = 2**32 - 1, 2**64 - 1
V1_MAX = 2**31 - 64                       # the largest V1 modulus (numLongs * 64 <= INT32_MAX)
V2_MAX = (2**31 - 1) * 64                 # numLongs <= INT32_MAX
DIVISORS = [64, 128, 29_193_792, V1_MAX, 2**32, 2**34 + 64, V2_MAX]


def reciprocal(version, d):
    return M32 // d if version == 1 else M64 // d


def mod_v1(x, d, m):
    r = (x - ((x * m) >> 32) * d) & M32
    return r - d if r >= d else r


def mod_v2(x, d, m):
    r = (x - ((x * m) >> 64) * d) & M64
    return r - d if r >= d else r


def _mulhi64_np(a, b):
    """floor(a * b / 2^64) of uint64 arrays, from 32-bit halves"""
    lo = np.uint64(M32)
    s = np.uint64(32)
    a0, a1, b0, b1 = a & lo, a >> s, b & lo, b >> s
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> s) + (p01 & lo) + (p10 & lo)
    return p11 + (p01 >> s) + (p10 >> s) + (mid >> s)


def _edge_dividends(d, top):
    return sorted(x for x in {0, 1, d - 1, d, d + 1, 2 * d - 1, 2 * d, top - 1, top - d, top - d - 1, (top - 1) // d * d,
                              (top - 1) // d * d - 1} if 0 <= x < top)


@pytest.mark.parametrize("d", [d for d in DIVISORS if d <= V1_MAX])
def test_v1_modulo_exact(d):
    m = reciprocal(1, d)
    for x in _edge_dividends(d, 2**31):
        assert mod_v1(x, d, m) == x % d, x
    x = np.random.default_rng(d).integers(0, 2**31, 1_000_000, dtype=np.uint64)
    q = (x * np.uint64(m)) >> np.uint64(32)
    r = (x - q * np.uint64(d)) & np.uint64(M32)
    r = np.where(r >= d, r - np.uint64(d), r)
    assert np.array_equal(r, x % np.uint64(d))


@pytest.mark.parametrize("d", DIVISORS)
def test_v2_modulo_exact(d):
    m = reciprocal(2, d)
    for x in _edge_dividends(d, 2**63):
        assert mod_v2(x, d, m) == x % d, x
    x = np.random.default_rng(d).integers(0, 2**63, 1_000_000, dtype=np.uint64)
    with np.errstate(over="ignore"):
        r = x - _mulhi64_np(x, np.uint64(m)) * np.uint64(d)
    r = np.where(r >= d, r - np.uint64(d), r)
    assert np.array_equal(r, x % np.uint64(d))
