"""GPU checks of BloomFilter (srj_b200.bloom over libsrj_b200.so): serialized bytes after create / put / merge are compared
byte for byte with oracle/bloom.py, which tests/test_oracle_bloom.py pins to the reference's goldens, to hand-derived known
answers and to an independent model; probe values on valid rows, the output mask and the null count are compared too."""
import threading

import numpy as np
import pytest

from golden import bloom_golden as G
from oracle import bloom as B

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    from srj_b200 import bloom
    return S, bloom


def _mask_words(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)


def _col(values, valid=None):
    S, _ = _s()
    v = np.asarray(values, dtype=np.int64)
    return S.ColumnVector.from_numpy(S.DType.INT64, v, None if valid is None else _mask_words(valid), size=len(v))


def _bytes(f) -> np.ndarray:
    return f.data.cpu().numpy()


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    k = rng.integers(INT64_MIN, INT64_MAX, n, dtype=np.int64, endpoint=True)
    k[: min(n, 4)] = [INT64_MIN, INT64_MAX, 0, -1][: min(n, 4)]
    return k


def _check_probe(filter_or_buffer, values, valid, want_filter_bytes):
    import torch
    _, bloom = _s()
    col = _col(values, valid)
    out = bloom.BloomFilter.probe(filter_or_buffer, col)
    torch.cuda.synchronize()
    want = B.probe(want_filter_bytes, np.asarray(values, np.int64))
    got = out.data.cpu().numpy().astype(bool)
    assert out.dtype.type_id == 11 and out.size == len(values)
    ok = np.ones(len(values), bool) if valid is None else np.asarray(valid, bool)
    assert np.array_equal(got[ok], want[ok])
    if valid is None:
        assert out.mask is None
    else:
        assert torch.equal(out.mask, col.mask)
    nulls = int((~ok).sum())
    assert out.getNullCount() == nulls
    out._null_count = None
    assert out.getNullCount() == nulls
    return got


# ---- the reference's goldens, through probe and probebuffer
@pytest.mark.parametrize("case", G.CASES, ids=[c["name"] for c in G.CASES])
def test_goldens(case):
    _, bloom = _s()
    BF = bloom.BloomFilter
    filters, want = [], []
    for puts in case["puts"]:
        f = BF.create(case["version"], case["num_hashes"], case["bits"], case["seed"])
        w = B.create(case["version"], case["num_hashes"], case["bits"], case["seed"])
        for values, valid in puts:
            BF.put(f, _col(values, valid))
            w = B.put(w, np.array(values, np.int64), None if valid is None else np.array(valid, bool))
        assert np.array_equal(_bytes(f), w)
        filters.append(f)
        want.append(w)
    if case["merge"]:
        f = BF.merge(bloom.list_column(filters))
        w = B.merge(want)
        assert np.array_equal(_bytes(f), w)
    else:
        f, w = filters[0], want[0]
    for target in (f, f.data):                                  # probe(Scalar) and probe(device buffer)
        got = _check_probe(target, case["probe"], case["probe_valid"], w)
        for g, e in zip(got, case["expected"]):
            if e is not None:
                assert bool(g) == e
    got = BF.probebuffer(f.data.data_ptr(), f.data.numel(), _col(case["probe"], case["probe_valid"])).data.cpu().numpy()
    assert [bool(g) for g, e in zip(got, case["expected"]) if e is not None] == [e for e in case["expected"] if e is not None]


@pytest.mark.parametrize("version,k,longs,seed,size", G.INIT)
def test_initialization(version, k, longs, seed, size):
    _, bloom = _s()
    f = bloom.BloomFilter.create(version, k, 64 * longs, seed)
    assert f.data.numel() == size
    assert np.array_equal(_bytes(f), B.create(version, k, 64 * longs, seed))


@pytest.mark.parametrize("failure", G.FAILURES, ids=[str(i) for i in range(len(G.FAILURES))])
def test_expected_failures(failure):
    S, bloom = _s()
    BF = bloom.BloomFilter
    if failure[0] == "create":
        with pytest.raises(ValueError):
            BF.create(*failure[1:])
    else:
        col = bloom.list_column([BF.create(*p) for p in failure[1]])
        with pytest.raises(S.CudfException):
            BF.merge(col)


@pytest.mark.parametrize("known", G.KNOWN, ids=[f"v{k[0]}_seed{k[1]}_bits{k[2]}_key{k[3]}" for k in G.KNOWN])
def test_known_answers(known):
    _, bloom = _s()
    version, seed, bits, key, _, _, hexbytes = known
    f = bloom.BloomFilter.create(version, 3, bits, seed)
    bloom.BloomFilter.put(f, _col([key]))
    assert _bytes(f).tobytes().hex() == hexbytes


def test_deprecated_create_is_v1_with_the_default_seed():
    _, bloom = _s()
    with pytest.warns(DeprecationWarning):
        f = bloom.BloomFilter.create(3, 1000)
    assert np.array_equal(_bytes(f), B.create(1, 3, 1000, 0))


# ---- serialized bytes over the parameter matrix: create, put twice into the same filter, merge, probe
@pytest.mark.parametrize("bits", [1, 64, 65, 4096, 2**22, 29_193_763])
@pytest.mark.parametrize("k", [1, 3, 5, 12, 30])
@pytest.mark.parametrize("seed", [0, 42, -1])
@pytest.mark.parametrize("version", [1, 2])
def test_bytes_match_oracle(version, seed, k, bits):
    _, bloom = _s()
    BF = bloom.BloomFilter
    a, b = _keys(33, seed=k * 1000 + bits % 997), _keys(31, seed=k * 1000 + bits % 997 + 1)
    va = np.arange(33) % 5 != 2
    f = BF.create(version, k, bits, seed)
    w = B.create(version, k, bits, seed)
    assert np.array_equal(_bytes(f), w)
    BF.put(f, _col(a, va))
    w = B.put(w, a, va)
    assert np.array_equal(_bytes(f), w)
    BF.put(f, _col(b))
    w = B.put(w, b)
    assert np.array_equal(_bytes(f), w)
    g = BF.create(version, k, bits, seed)
    BF.put(g, _col(_keys(40, seed=bits)))
    wg = B.put(B.create(version, k, bits, seed), _keys(40, seed=bits))
    m = BF.merge(bloom.list_column([f, g]))
    wm = B.merge([w, wg])
    assert np.array_equal(_bytes(m), wm)
    probe = np.concatenate([a, b, _keys(100, seed=bits + 5)])
    ok = np.arange(len(probe)) % 7 != 3
    got = _check_probe(m, probe, ok, wm)
    assert got[33:64][ok[33:64]].all()                            # every key put unmasked is found


# ---- row counts and null patterns, including a 10M-row column
@pytest.mark.parametrize("n", [0, 1, 31, 33, 10_000_000])
@pytest.mark.parametrize("nulls", ["none", "some", "all"])
@pytest.mark.parametrize("version", [1, 2])
def test_row_counts_and_nulls(version, nulls, n):
    _, bloom = _s()
    BF = bloom.BloomFilter
    keys = _keys(n, seed=n + version)
    valid = None if nulls == "none" else (np.zeros(n, bool) if nulls == "all" else np.random.default_rng(n).random(n) > 0.3)
    f = BF.create(version, 5, 29_193_763, 42)
    BF.put(f, _col(keys, valid))
    w = B.put(B.create(version, 5, 29_193_763, 42), keys, valid)
    assert np.array_equal(_bytes(f), w)
    probe = np.concatenate([keys[: n // 2], _keys(n - n // 2, seed=n + 77)])
    _check_probe(f, probe, valid, w)


def test_unaligned_keys_and_output_take_the_scalar_path():
    import torch
    S, bloom = _s()
    BF = bloom.BloomFilter
    keys = _keys(1001, seed=9)
    f = BF.create(2, 7, 100_000, 3)
    w = B.put(B.create(2, 7, 100_000, 3), keys[1:])
    raw = torch.from_numpy(keys.view(np.uint8).copy()).cuda()
    col = S.ColumnVector(S.DType.INT64, 1000, raw[8:])                  # keys 8 bytes past a 16-byte boundary
    BF.put(f, col)
    assert np.array_equal(_bytes(f), w)
    out = BF.probe(f, col)
    assert np.array_equal(out.data.cpu().numpy().astype(bool), B.probe(w, keys[1:]))


# ---- large filters: V1 at its 2^31 - 64 bit limit, V2 over 2^32 bits
def _popcount(t):
    import torch
    lut = torch.tensor([bin(i).count("1") for i in range(256)], dtype=torch.int64, device=t.device)
    return int(sum(lut[t[o:o + (1 << 28)].long()].sum() for o in range(0, t.numel(), 1 << 28)))


def _touched(version, k, seed, nbits, keys):
    """(sorted unique positions, unique bytes of the bit array they touch, the OR of their bits per byte)"""
    p = np.unique(B.positions(version, k, seed, nbits, keys).ravel())
    byte, bit = B.byte_bit(p)
    order = np.argsort(byte, kind="stable")
    byte, bit = byte[order], bit[order]
    ub, start = np.unique(byte, return_index=True)
    return p, ub, np.bitwise_or.reduceat(bit, start)


@pytest.mark.parametrize("version,bits,seed", [(1, 2**31 - 64, 0), (2, 2**33, 42)])
def test_large_filters(version, bits, seed):
    import torch
    _, bloom = _s()
    BF = bloom.BloomFilter
    k = 5
    keys = _keys(1_000_000, seed=bits % 1009)
    f = BF.create(version, k, bits, seed)
    BF.put(f, _col(keys))
    torch.cuda.synchronize()
    hdr = B.header_bytes(version)
    assert f.data[:hdr].cpu().numpy().tobytes() == (B.create(version, k, 64, seed)[:hdr - 4].tobytes()       # numLongs is last
                                                    + np.array([B.num_longs(bits)], ">i4").tobytes())
    p, ub, ubits = _touched(version, k, seed, bits, keys)
    if version == 2:
        assert (p >= 2**32).any()
    arr = f.data[hdr:]
    got = arr[torch.from_numpy(ub).cuda()].cpu().numpy()
    assert np.array_equal(got, ubits)                              # every byte the oracle touches, exactly
    assert _popcount(arr) == len(p)                                # and no other bit is set
    absent = _keys(1_000_000, seed=bits % 1009 + 1)
    out = BF.probe(f, _col(np.concatenate([keys, absent])))
    got = out.data.cpu().numpy().astype(bool)
    assert got[: len(keys)].all()
    want = np.all(np.isin(B.positions(version, k, seed, bits, absent), p), axis=0)
    assert np.array_equal(got[len(keys):], want)


# ---- merge: 1, 3 and 200 filters, the child at every 4-byte alignment; 16-, 8- and 4-byte access paths
@pytest.mark.parametrize("pad", [0, 4, 8, 12])
@pytest.mark.parametrize("nfilters", [1, 3, 200])
@pytest.mark.parametrize("version,bits", [(1, 4096), (2, 4096), (2, 4096 + 64)])
def test_merge_alignment(version, bits, nfilters, pad):
    import torch
    S, bloom = _s()
    BF = bloom.BloomFilter
    want = []
    for i in range(nfilters):
        keys = _keys(5, seed=1000 * nfilters + i)
        want.append(B.put(B.create(version, 4, bits, 11), keys))
    child = np.concatenate(want)
    raw = torch.zeros(pad + len(child), dtype=torch.uint8, device="cuda")
    raw[pad:] = torch.from_numpy(child).cuda()
    size = len(want[0])
    offs = torch.arange(0, nfilters + 1, dtype=torch.int32, device="cuda") * size
    col = S.ColumnVector(S.DType.LIST, nfilters, None, None, offs, S.ColumnVector(S.DType.UINT8, len(child), raw[pad:]))
    m = BF.merge(col)
    assert np.array_equal(_bytes(m), B.merge(want))


# ---- errors
def _merge_raises(filters):
    S, bloom = _s()
    with pytest.raises(S.CudfException):
        bloom.BloomFilter.merge(bloom.list_column(filters))


@pytest.mark.parametrize("base,other", [((1, 3, 1024, 0), (1, 4, 1024, 0)), ((2, 3, 1024, 0), (2, 4, 1024, 0)),     # k
                                        ((1, 3, 1024, 0), (1, 3, 2048, 0)), ((2, 3, 1024, 0), (2, 3, 2048, 0)),     # size
                                        ((1, 3, 1024, 0), (2, 3, 1024, 0)), ((2, 3, 1024, 0), (1, 3, 1024, 0)),     # version
                                        ((2, 3, 1024, 0), (2, 3, 1024, 42))])                                        # seed
def test_merge_mismatch(base, other):
    _, bloom = _s()
    BF = bloom.BloomFilter
    _merge_raises([BF.create(*base), BF.create(*base), BF.create(*other)])


def test_merge_wrong_child_size_and_truncated_header():
    import torch
    S, bloom = _s()
    BF = bloom.BloomFilter
    a = BF.create(2, 3, 1024, 0)
    cut = bloom.Scalar(a.data[:-8].clone())
    _merge_raises([a, cut])
    one = bloom.list_column([a])
    one.child = S.ColumnVector(S.DType.UINT8, a.data.numel() - 8, a.data[:-8].clone())
    with pytest.raises(S.CudfException):
        BF.merge(one)
    for nbytes in (8, 14):                                             # V2 header is 16 bytes
        with pytest.raises(S.CudfException):
            BF.merge(bloom.list_column([bloom.Scalar(a.data[:nbytes].clone())]))
        with pytest.raises(S.CudfException):
            BF.probe(a.data[:nbytes].clone(), _col([1, 2]))
    with pytest.raises(S.CudfException):
        BF.probe(torch.cat([a.data, a.data[:8]]), _col([1, 2]))        # buffer size != header + bit array


def test_v1_over_int32_max_bits_is_rejected_by_put_and_probe():
    S, bloom = _s()
    BF = bloom.BloomFilter
    f = BF.create(1, 3, 2**31, 0)                                      # created like the reference; not usable as V1
    with pytest.raises(S.CudfException):
        BF.put(f, _col([1]))
    with pytest.raises(S.CudfException):
        BF.probe(f, _col([1]))


def test_non_int64_input_is_rejected():
    S, bloom = _s()
    BF = bloom.BloomFilter
    f = BF.create(2, 3, 1024, 0)
    c = S.ColumnVector.from_numpy(S.DType.INT32, np.arange(4, dtype=np.int32))
    with pytest.raises(S.CudfException):
        BF.put(f, c)
    with pytest.raises(S.CudfException):
        BF.probe(f, c)


# ---- concurrency: 8 threads, each on its own stream, build and probe their own filters
def test_threads_on_their_own_streams():
    import torch
    _, bloom = _s()
    BF = bloom.BloomFilter
    errors, results = [], {}

    def work(t):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                version = 1 + t % 2
                keys = _keys(200_000, seed=500 + t)
                f = BF.create(version, 3 + t, 1_000_000 + 64 * t, t)
                BF.put(f, _col(keys))
                out = BF.probe(f, _col(np.concatenate([keys, _keys(50_000, seed=900 + t)])))
                s.synchronize()
                results[t] = (version, keys, _bytes(f), out.data.cpu().numpy().astype(bool))
        except Exception as e:             # noqa: BLE001 -- reported below
            errors.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
    for t, (version, keys, got, hits) in results.items():
        w = B.put(B.create(version, 3 + t, 1_000_000 + 64 * t, t), keys)
        assert np.array_equal(got, w)
        assert np.array_equal(hits, B.probe(w, np.concatenate([keys, _keys(50_000, seed=900 + t)])))
