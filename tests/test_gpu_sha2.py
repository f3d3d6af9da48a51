"""GPU checks of Hash.sha{224,256,384,512}NullsPreserved: every output (offsets, chars, mask, null count) is compared byte
for byte with python's hashlib, which tests/test_oracle_sha2_golden.py pins to the FIPS 180-4 examples."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from golden import sha2_golden as GOLD

pytestmark = pytest.mark.gpu

BITS = (224, 256, 384, 512)


def _s():
    import gpu_util
    gpu_util.require_cuda()
    import srj_b200 as S
    return S


def _mask_words(valid):
    b = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view(np.uint32)    # ceil(n / 32) words


def _column(values, with_mask=True):
    """Device STRING column of `values` (bytes or None = null row); without a mask every row must be valid."""
    S = _s()
    lens = np.array([0 if v is None else len(v) for v in values], np.int64)
    offs = np.zeros(len(values) + 1, np.int32)
    np.cumsum(lens, out=offs[1:])
    chars = np.frombuffer(b"".join(v for v in values if v is not None), np.uint8)
    mask = _mask_words([v is not None for v in values]) if with_mask else None
    if not with_mask:
        assert all(v is not None for v in values)
    return S.ColumnView.from_numpy(S.DType.STRING, chars, mask, offs)


def _expect(values, bits):
    width = bits // 4
    digests = [None if v is None else hashlib.new(f"sha{bits}", v).hexdigest().encode() for v in values]
    offs = np.zeros(len(values) + 1, np.int32)
    np.cumsum([0 if d is None else width for d in digests], out=offs[1:])
    return offs, b"".join(d for d in digests if d is not None)


def _hash(col, bits):
    S = _s()
    return getattr(S.Hash, f"sha{bits}NullsPreserved")(col)


def _check(values, bits, with_mask=True):
    import torch
    col = _column(values, with_mask)
    out = _hash(col, bits)
    torch.cuda.synchronize()
    want_offs, want_chars = _expect(values, bits)
    assert out.dtype.type_id == 23 and out.size == len(values)
    assert np.array_equal(out.offsets.cpu().numpy(), want_offs)
    assert out.data.cpu().numpy().tobytes() == want_chars
    nulls = sum(v is None for v in values)
    if with_mask:
        assert torch.equal(out.mask, col.mask)
    else:
        assert out.mask is None
    assert out.getNullCount() == nulls
    out._null_count = None                      # recount from the output mask itself
    assert out.getNullCount() == nulls
    return out


@pytest.mark.parametrize("bits", BITS)
def test_goldens(bits):
    values = [None if s is None else s.encode("utf-8") for s in GOLD.JAVA_INPUTS]
    out = _check(values, bits)
    o = out.offsets.cpu().numpy()
    chars = out.data.cpu().numpy().tobytes()
    got = [None if not (out.mask.cpu().numpy().view(np.uint32)[i // 32] >> (i % 32)) & 1 else chars[o[i]:o[i + 1]].decode()
           for i in range(len(values))]
    assert got == GOLD.JAVA_DIGESTS[bits]
    nist = [c["input"].encode() for c in GOLD.NIST]
    out = _check(nist, bits, with_mask=False)
    chars = out.data.cpu().numpy().tobytes()
    w = bits // 4
    assert [chars[i * w:(i + 1) * w].decode() for i in range(len(nist))] == [c["digests"][bits] for c in GOLD.NIST]


@pytest.mark.parametrize("bits", BITS)
def test_every_length_0_to_300(bits):
    """covers the 55/56/63/64 (SHA-224/256) and 111/112/127/128 (SHA-384/512) padding boundaries"""
    rng = np.random.default_rng(bits)
    values = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in range(301)]
    _check(values, bits, with_mask=False)
    _check(values, bits, with_mask=True)


@pytest.mark.parametrize("bits", BITS)
def test_random_strings_with_nulls_and_all_null(bits):
    rng = np.random.default_rng(100 + bits)
    values = [None if rng.random() < 0.3 else rng.integers(0, 256, int(rng.integers(0, 200)), dtype=np.uint8).tobytes()
              for _ in range(5003)]
    _check(values, bits)
    _check([None] * 77, bits)
    _check([v for v in values if v is not None][:1000], bits, with_mask=False)


@pytest.mark.parametrize("bits", BITS)
def test_every_start_alignment(bits):
    """each hashed string is preceded by a filler of 0..15 bytes, so strings start at every alignment modulo 16"""
    rng = np.random.default_rng(7)
    values = []
    for a in range(16):
        for n in (0, 1, 3, 4, 5, 31, 55, 56, 63, 64, 65, 111, 112, 127, 128, 129, 200):
            values.append(b"x" * a)
            values.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    _check(values, bits)


@pytest.mark.parametrize("bits", BITS)
def test_one_long_string_among_short_ones(bits):
    rng = np.random.default_rng(11)
    values = [rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8).tobytes() for _ in range(3000)]
    values[1234] = rng.integers(0, 256, (1 << 20) + 3, dtype=np.uint8).tobytes()    # 1 MiB + 3 bytes
    values[17] = None
    _check(values, bits)


@pytest.mark.parametrize("bits", BITS)
def test_multibyte_utf8(bits):
    rng = np.random.default_rng(3)
    alphabet = "aé¼³⅝中文字符😀𝄞ßЖ"
    values = ["".join(rng.choice(list(alphabet), int(rng.integers(0, 60)))).encode("utf-8") for _ in range(500)]
    _check(values, bits)


@pytest.mark.parametrize("bits", BITS)
def test_zero_rows(bits):
    out = _check([], bits, with_mask=False)
    assert out.offsets.cpu().numpy().tolist() == [0]
    _check([], bits, with_mask=True)


def test_non_string_column_is_rejected():
    S = _s()
    from srj_b200 import _native as N
    import torch
    col = S.ColumnVector(S.DType.INT32, 4, torch.zeros(16, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        S.Hash.sha256NullsPreserved(col)
    offs = torch.zeros(5, dtype=torch.int32, device="cuda")
    total = C.c_int64(0)
    cin = col._c()
    assert N.lib().srj_sha2_sizes(256, C.byref(cin), offs.data_ptr(), C.byref(total), None, None) == N.SRJ_EUNSUPPORTED


@pytest.mark.parametrize("bits", (256, 512))
def test_non_default_stream(bits):
    import torch
    rng = np.random.default_rng(9)
    values = [None if rng.random() < 0.2 else rng.integers(0, 256, int(rng.integers(0, 150)), dtype=np.uint8).tobytes()
              for _ in range(20000)]
    col = _column(values)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = _hash(col, bits)
    s.synchronize()
    want_offs, want_chars = _expect(values, bits)
    assert np.array_equal(out.offsets.cpu().numpy(), want_offs)
    assert out.data.cpu().numpy().tobytes() == want_chars
    assert torch.equal(out.mask, col.mask)


def test_20m_rows_sha256_sample():
    """20M rows: full offsets and mask, digests on a seeded sample of rows"""
    import torch
    S = _s()
    n = 20_000_000
    rng = np.random.default_rng(2024)
    valid = rng.random(n) >= 0.2
    lens = rng.integers(0, 33, n).astype(np.int64) * valid
    offs = np.zeros(n + 1, np.int32)
    np.cumsum(lens, out=offs[1:])
    chars = rng.integers(0, 256, int(offs[-1]), dtype=np.uint8)
    mask = _mask_words(valid)
    col = S.ColumnView.from_numpy(S.DType.STRING, chars, mask, offs)
    out = S.Hash.sha256NullsPreserved(col)
    torch.cuda.synchronize()
    want_offs = np.zeros(n + 1, np.int64)
    np.cumsum(valid.astype(np.int64) * 64, out=want_offs[1:])
    got_offs = out.offsets.cpu().numpy()
    assert np.array_equal(got_offs, want_offs)
    assert torch.equal(out.mask, col.mask)
    assert out.getNullCount() == int((~valid).sum())
    out_chars = out.data.cpu().numpy()
    for r in np.sort(rng.integers(0, n, 4000)):
        if valid[r]:
            want = hashlib.sha256(chars[offs[r]:offs[r + 1]].tobytes()).hexdigest().encode()
            assert out_chars[got_offs[r]:got_offs[r + 1]].tobytes() == want, r
        else:
            assert got_offs[r] == got_offs[r + 1]


@pytest.mark.parametrize("with_mask", [False, True])
def test_sizes_overflow_writes_nothing(with_mask):
    """16,777,216 valid empty rows at SHA-512 need 2^31 chars: SRJ_EOVERFLOW from the sizes call, offsets untouched"""
    import torch
    S = _s()
    from srj_b200 import _native as N
    n = 1 << 24
    col = S.ColumnVector(S.DType.STRING, n, None, torch.full(((n + 31) // 32,), -1, dtype=torch.int32, device="cuda") if with_mask else None,
                         torch.zeros(n + 1, dtype=torch.int32, device="cuda"))
    lib = N.lib()
    out_offs = torch.full((n + 1,), 7, dtype=torch.int32, device="cuda")
    ws = torch.empty(max(lib.srj_sha2_workspace_bytes(n), 8), dtype=torch.uint8, device="cuda")
    total = C.c_int64(0)
    cin = col._c()
    st = int(torch.cuda.current_stream().cuda_stream)
    assert lib.srj_sha2_sizes(512, C.byref(cin), out_offs.data_ptr(), C.byref(total), ws.data_ptr(), st) == N.SRJ_EOVERFLOW
    torch.cuda.synchronize()
    assert total.value == 128 * n
    assert bool((out_offs == 7).all())
    with pytest.raises(S.CudfColumnSizeOverflowException):
        S.Hash.sha512NullsPreserved(col)
    # one row fewer fits
    assert lib.srj_sha2_sizes(512, C.byref(cin), out_offs.data_ptr(), C.byref(total), ws.data_ptr(), st) == N.SRJ_EOVERFLOW
    cin.size = n - 1
    assert lib.srj_sha2_sizes(512, C.byref(cin), out_offs.data_ptr(), C.byref(total), ws.data_ptr(), st) == N.SRJ_OK
    torch.cuda.synchronize()
    assert total.value == 128 * (n - 1) and int(out_offs[n - 1]) == 128 * (n - 1) and int(out_offs[1]) == 128
