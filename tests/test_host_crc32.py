"""Hash.hostCrc32 (srj_host_crc32): zlib's crc32 of a host buffer, restating HashTest.java:964-1028 of the reference
against python's zlib (the same function as java.util.zip.CRC32), plus the argument checks of HashJni.cpp:146-150."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest


def _lib():
    from srj_b200 import _native as N
    return N, N.lib()


def _crc(crc, data: bytes):
    N, lib = _lib()
    buf = C.create_string_buffer(data, len(data)) if data else None
    out = C.c_uint32(0)
    assert lib.srj_host_crc32(crc, buf, len(data), C.byref(out)) == N.SRJ_OK
    return out.value


@pytest.mark.parametrize("size", [0, 1, 10, 100, 256, 1000, 4096])
def test_crc32_matches_zlib(size):
    data = random.Random(17).randbytes(size)
    assert _crc(0, data) == zlib.crc32(data)


def test_crc32_chained_update():
    rng = random.Random(17)
    a, b = rng.randbytes(rng.randrange(1024)), rng.randbytes(rng.randrange(1024))
    assert _crc(_crc(0, a), b) == zlib.crc32(a + b) == zlib.crc32(b, zlib.crc32(a))


def test_crc32_every_length_and_alignment():
    data = random.Random(5).randbytes(300)
    for start in range(9):
        for n in range(0, 70):
            assert _crc(0xDEADBEEF, data[start:start + n]) == zlib.crc32(data[start:start + n], 0xDEADBEEF)


def test_crc32_null_buffer_and_bad_lengths():
    N, lib = _lib()
    out = C.c_uint32(7)
    assert lib.srj_host_crc32(1234, None, 0, C.byref(out)) == N.SRJ_OK and out.value == 1234   # NULL with len 0: unchanged
    buf = C.create_string_buffer(b"abc", 3)
    assert lib.srj_host_crc32(0, None, 5, C.byref(out)) == N.SRJ_EINVAL
    assert lib.srj_host_crc32(0, buf, -1, C.byref(out)) == N.SRJ_EINVAL


def test_python_mirror_host_buffers():
    import torch
    import srj_b200 as S
    data = random.Random(3).randbytes(1000)
    want = zlib.crc32(data)
    assert S.Hash.hostCrc32(0, data) == want
    assert S.Hash.hostCrc32(0, bytearray(data)) == want
    assert S.Hash.hostCrc32(0, np.frombuffer(data, np.uint8)) == want
    assert S.Hash.hostCrc32(0, torch.frombuffer(bytearray(data), dtype=torch.uint8)) == want
    assert S.Hash.hostCrc32(S.Hash.hostCrc32(0, data[:300]), data[300:]) == want
    assert S.Hash.hostCrc32(99, b"") == 99
