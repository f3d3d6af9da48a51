"""An independent model of Spark's bloom filter, one key at a time in Python integers.

Written from Spark's org.apache.spark.util.sketch sources as the reference's comments link them (BloomFilterImpl.putLong /
mightContainLong for V1, BloomFilterImplV2 for V2, BitArray.set / writeTo), not from the CUDA kernels or oracle/bloom.py,
and imports neither.  Murmur3_x86_32.hashLong is spelled out again here.

  V1: int h1 = hashLong(item, 0), h2 = hashLong(item, h1);
      for (int i = 1; i <= k; i++) { int c = h1 + i * h2; if (c < 0) c = ~c; bits.set(c % bitSize); }
  V2: int h1 = hashLong(item, seed), h2 = hashLong(item, h1); long c = (long) h1 * Integer.MAX_VALUE;
      for (int i = 0; i < k; i++) { c += h2; long idx = c < 0 ? ~c : c; bits.set(idx % bitSize); }
  BitArray.set(i): data[(int) (i >>> 6)] |= 1L << i   (a Java long shift takes i mod 64)
  writeTo: the int header fields, then every long with DataOutputStream.writeLong (big-endian).
"""
from __future__ import annotations

M32, M64 = (1 << 32) - 1, (1 << 64) - 1


def _s32(x: int) -> int:
    x &= M32
    return x - (1 << 32) if x >> 31 else x


def _s64(x: int) -> int:
    x &= M64
    return x - (1 << 64) if x >> 63 else x


def _rotl(x: int, r: int) -> int:
    return ((x << r) | (x >> (32 - r))) & M32


def _mix(h: int, k: int) -> int:
    k = _rotl((k * 0xCC9E2D51) & M32, 15) * 0x1B873593 & M32
    return (_rotl(h ^ k, 13) * 5 + 0xE6546B64) & M32


def hash_long(v: int, seed: int) -> int:
    """Murmur3_x86_32.hashLong(v, seed) as a Java int"""
    v &= M64
    h = _mix(_mix(seed & M32, v & M32), v >> 32) ^ 8
    h ^= h >> 16
    h = h * 0x85EBCA6B & M32
    h ^= h >> 13
    h = h * 0xC2B2AE35 & M32
    return _s32(h ^ (h >> 16))


def positions(version: int, k: int, seed: int, bit_size: int, item: int) -> list:
    """the bit indices putLong / mightContainLong visit for `item`, in order"""
    h1 = hash_long(item, seed if version == 2 else 0)
    h2 = hash_long(item, h1)
    out = []
    if version == 1:
        for i in range(1, k + 1):
            c = _s32(h1 + i * h2)
            out.append((~c if c < 0 else c) % bit_size)
    else:
        c = h1 * 0x7FFFFFFF
        for _ in range(k):
            c = _s64(c + h2)
            out.append((~c if c < 0 else c) % bit_size)
    return out


class Filter:
    """BloomFilterImpl / BloomFilterImplV2 with a BitArray of num_longs longs"""

    def __init__(self, version: int, k: int, num_longs: int, seed: int = 0):
        self.version, self.k, self.seed = version, k, seed if version == 2 else 0
        self.data = [0] * num_longs

    def put(self, item: int):
        for p in positions(self.version, self.k, self.seed, 64 * len(self.data), item):
            self.data[p >> 6] |= 1 << (p & 63)

    def might_contain(self, item: int) -> bool:
        return all((self.data[p >> 6] >> (p & 63)) & 1 for p in positions(self.version, self.k, self.seed, 64 * len(self.data), item))

    def serialize(self) -> bytes:
        head = [1, self.k, len(self.data)] if self.version == 1 else [2, self.k, self.seed, len(self.data)]
        return b"".join((h & M32).to_bytes(4, "big") for h in head) + b"".join(d.to_bytes(8, "big") for d in self.data)
