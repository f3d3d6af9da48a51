"""Spark's runtime-join bloom filter, restated in numpy: the serialized bytes of create / put / merge and the probe.

Reference lines (src/main/cpp/src/ of the reference unless noted):
  - format: bloom_filter.hpp:32-49 (V1 header {version, numHashes, numLongs}, 12 B; V2 {version, numHashes, seed,
    numLongs}, 16 B), bloom_filter.cu:154-172 (big-endian header), 288-331 (create: zeroed bit array);
    numLongs = ceil(bits / 64) (BloomFilterJni.cpp:47); the modulus is numLongs * 64 (bloom_filter.cu:226).
  - bit p = bit p % 64 of the big-endian long p / 64 (Spark's BitArray), i.e. byte 8 * (p / 64) + 7 - (p % 64) / 8,
    bit p % 8 of the serialized bit array (bloom_filter.cu:60-66 says the same in 32-bit words).
  - hashes (bloom_filter.cu:70-152): h1 = Murmur3_x86_32.hashLong(x, s), h2 = hashLong(x, h1), s = 0 (V1) or the seed
    (V2); V1: for i = 1..k, c = (int32)(h1 + i * h2), p = (c < 0 ? ~c : c) % bits; V2: c = (int64)h1 * INT32_MAX, for
    i = 0..k-1: c += h2, p = (c < 0 ? ~c : c) % bits.
  - put skips null rows (bloom_filter.cu:80-82); probe is true when all k bits are set (bloom_filter.cu:117-152).
  - merge: the first header, then the OR of the bit arrays; every header must equal the first and the child must hold
    exactly F filters (bloom_filter.cu:374-449).
Every function takes and returns host numpy arrays; the filter is the uint8 array of its serialized bytes.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

INT32_MAX = 2**31 - 1
U32 = np.uint64(0xFFFFFFFF)


def header_bytes(version: int) -> int:
    return 16 if version == 2 else 12


def num_longs(bits: int) -> int:
    return (int(bits) + 63) // 64


def create(version: int, num_hashes: int, bits: int, seed: int = 0) -> np.ndarray:
    """bloom_filter_create (bloom_filter.cu:298-331) with the JNI's rounding of the bit count."""
    if version not in (1, 2) or num_hashes <= 0 or bits <= 0 or bits > INT32_MAX * 64:
        raise ValueError("bad bloom filter parameters")
    L = num_longs(bits)
    hdr = [1, num_hashes, L] if version == 1 else [2, num_hashes, seed, L]
    head = np.array(hdr, dtype=">i4").view(np.uint8)
    return np.concatenate([head, np.zeros(8 * L, np.uint8)])


def parse(buf: np.ndarray) -> Tuple[int, int, int, int]:
    """(version, numHashes, seed, numLongs) of a serialized filter (bloom_filter.cu:189-236)."""
    if len(buf) < 12:
        raise ValueError("Encountered truncated bloom filter")
    w = np.frombuffer(np.ascontiguousarray(buf[:min(16, len(buf))]).tobytes() + b"\0" * 4, dtype=">i4")
    version = int(w[0])
    if version not in (1, 2):
        raise ValueError("Unexpected bloom filter version")
    if len(buf) < header_bytes(version):
        raise ValueError("Encountered truncated bloom filter header")
    if version == 1:
        return 1, int(w[1]), 0, int(w[2])
    return 2, int(w[1]), int(w[2]), int(w[3])


# ---- Murmur3_x86_32.hashLong, vectorised over keys and per-row seeds (uint64 arrays holding 32-bit values)
def _rotl(x, r):
    return ((x << np.uint64(r)) | (x >> np.uint64(32 - r))) & U32


def _mix(h, k):
    k = (k * np.uint64(0xCC9E2D51)) & U32
    k = _rotl(k, 15)
    k = (k * np.uint64(0x1B873593)) & U32
    h = _rotl(h ^ k, 13)
    return (h * np.uint64(5) + np.uint64(0xE6546B64)) & U32


def _fmix(h, length):
    h = h ^ np.uint64(length)
    h ^= h >> np.uint64(16)
    h = (h * np.uint64(0x85EBCA6B)) & U32
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xC2B2AE35)) & U32
    return h ^ (h >> np.uint64(16))


def hash_long(keys: np.ndarray, seed) -> np.ndarray:
    """Murmur3_x86_32.hashLong(key, seed): low word, then high word, length 8 -> uint64 array of 32-bit values"""
    k = np.asarray(keys, dtype=np.int64).view(np.uint64)
    s = np.asarray(seed, dtype=np.int64).astype(np.uint64) & U32
    h = _mix(np.broadcast_to(s, k.shape).copy(), k & U32)
    h = _mix(h, k >> np.uint64(32))
    return _fmix(h, 8)


def positions(version: int, num_hashes: int, seed: int, nbits: int, keys: np.ndarray) -> np.ndarray:
    """int64 [k, n]: the bit positions of every key, in the order the reference visits them"""
    keys = np.asarray(keys, dtype=np.int64)
    h1 = hash_long(keys, seed if version == 2 else 0)
    h2 = hash_long(keys, h1)
    out = np.empty((max(num_hashes, 0), len(keys)), np.int64)
    with np.errstate(over="ignore"):
        if version == 1:
            a, b = h1.astype(np.uint32), h2.astype(np.uint32)
            for i in range(1, num_hashes + 1):
                c = (a + np.uint32(i) * b).view(np.int32)                   # Java int arithmetic
                out[i - 1] = np.where(c < 0, ~c, c).astype(np.int64) % nbits
        else:
            c = h1.astype(np.uint32).view(np.int32).astype(np.int64) * INT32_MAX
            s = h2.astype(np.uint32).view(np.int32).astype(np.int64)
            for i in range(num_hashes):
                c = c + s                                                     # Java long arithmetic (wraps)
                out[i] = np.where(c < 0, ~c, c) % nbits
    return out


def byte_bit(p: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(byte offset in the bit array, bit mask) of positions p: bit p % 64 of the big-endian long p / 64"""
    p = np.asarray(p, dtype=np.int64)
    return (p >> 6) * 8 + 7 - ((p & 63) >> 3), (np.uint8(1) << (p & 7).astype(np.uint8))


def put(buf: np.ndarray, keys: np.ndarray, valid: Optional[np.ndarray] = None) -> np.ndarray:
    """bloom_filter_put: a new filter with the bits of every valid key set"""
    version, k, seed, L = parse(buf)
    out = np.array(buf, dtype=np.uint8, copy=True)
    keys = np.asarray(keys, dtype=np.int64)
    if valid is not None:
        keys = keys[np.asarray(valid, dtype=bool)]
    if len(keys) == 0 or k <= 0:
        return out
    byte, bit = byte_bit(positions(version, k, seed, 64 * L, keys).ravel())
    bits = out[header_bytes(version):]
    np.bitwise_or.at(bits, byte, bit)
    return out


def probe(buf: np.ndarray, keys: np.ndarray) -> np.ndarray:
    """bloom_filter_probe on the values (the mask of the result is the input's): bool per key"""
    version, k, seed, L = parse(buf)
    keys = np.asarray(keys, dtype=np.int64)
    if k <= 0:
        return np.ones(len(keys), bool)
    byte, bit = byte_bit(positions(version, k, seed, 64 * L, keys))
    bits = np.asarray(buf, dtype=np.uint8)[header_bytes(version):]
    return np.all((bits[byte] & bit) != 0, axis=0)


def merge(filters: Sequence[np.ndarray]) -> np.ndarray:
    """bloom_filter_merge of the rows of a LIST<UINT8> column (each a serialized filter)"""
    if not filters:
        raise ValueError("Encountered truncated bloom filter")
    child = np.concatenate([np.asarray(f, dtype=np.uint8) for f in filters])
    version, k, seed, L = parse(child)
    hdr = header_bytes(version)
    size = hdr + 8 * L
    if L <= 0:
        raise ValueError("Invalid empty bloom filter size")
    if len(child) != size * len(filters):
        raise ValueError("Encountered invalid/mismatched bloom filter buffer data")
    rows = child.reshape(len(filters), size)
    if not np.all(rows[:, :hdr] == rows[0, :hdr]):
        raise ValueError("Mismatch of bloom filter parameters")
    return np.concatenate([rows[0, :hdr], np.bitwise_or.reduce(rows[:, hdr:], axis=0)])
