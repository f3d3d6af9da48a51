// hash_device.cuh -- Spark-compatible element hashes, in registers.
//   xxhash64   : standard XXH64 chained across columns        (reference hash/xxhash64.cu:73-273)
//   murmur3_32 : Murmur3_x86_32 with Spark's sign-extending tail (reference hash/murmur_hash.cuh:67-205)
//   hive       : Hive hashCode, h = 31*h + x                    (reference hash/hive_hash.cu:42-152)
// Fixed-width values are hashed straight from registers with the byte loops of the reference
// unrolled away (a 4/8-byte key is a handful of multiplies); variable-length inputs (strings,
// DECIMAL128's minimal big-endian bytes) go through the *_bytes functions.
#pragma once
#include <stdint.h>

#include "../../include/srj_b200.h"

namespace srj {
namespace hash {

// ---------------------------------------------------------------- XXH64
constexpr uint64_t XP1 = 0x9E3779B185EBCA87ull;
constexpr uint64_t XP2 = 0xC2B2AE3D27D4EB4Full;
constexpr uint64_t XP3 = 0x165667B19E3779F9ull;
constexpr uint64_t XP4 = 0x85EBCA77C2B2AE63ull;
constexpr uint64_t XP5 = 0x27D4EB2F165667C5ull;

__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

__device__ __forceinline__ uint64_t xx_finalize(uint64_t h)
{
  h ^= h >> 33;
  h *= XP2;
  h ^= h >> 29;
  h *= XP3;
  h ^= h >> 32;
  return h;
}
__device__ __forceinline__ uint64_t xx_step8(uint64_t h, uint64_t v)
{
  h ^= rotl64(v * XP2, 31) * XP1;
  return rotl64(h, 27) * XP1 + XP4;
}
__device__ __forceinline__ uint64_t xx_step4(uint64_t h, uint32_t v)
{
  h ^= static_cast<uint64_t>(v) * XP1;
  return rotl64(h, 23) * XP2 + XP3;
}
__device__ __forceinline__ uint64_t xx_step1(uint64_t h, uint8_t v)
{
  h ^= static_cast<uint64_t>(v) * XP5;
  return rotl64(h, 11) * XP1;
}
// XXH64 of exactly 4 / 8 bytes (xxhash64.cu:174-178 with nbytes < 32)
__device__ __forceinline__ uint64_t xx_u32(uint32_t v, uint64_t seed) { return xx_finalize(xx_step4(seed + XP5 + 4, v)); }
__device__ __forceinline__ uint64_t xx_u64(uint64_t v, uint64_t seed) { return xx_finalize(xx_step8(seed + XP5 + 8, v)); }

__device__ __forceinline__ uint64_t ld_u64_bytes(const uint8_t* p)
{
  uint64_t v = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) v |= static_cast<uint64_t>(p[i]) << (8 * i);
  return v;
}
__device__ __forceinline__ uint32_t ld_u32_bytes(const uint8_t* p)
{
  return p[0] | (p[1] << 8) | (p[2] << 16) | (static_cast<uint32_t>(p[3]) << 24);
}

// general XXH64 over unaligned bytes (strings)
__device__ inline uint64_t xx_bytes(const uint8_t* d, int32_t n, uint64_t seed)
{
  int32_t off = 0;
  uint64_t h;
  if (n >= 32) {
    uint64_t v1 = seed + XP1 + XP2, v2 = seed + XP2, v3 = seed, v4 = seed - XP1;
    const int32_t limit = n - 32;
    do {
      v1 = rotl64(v1 + ld_u64_bytes(d + off) * XP2, 31) * XP1;
      v2 = rotl64(v2 + ld_u64_bytes(d + off + 8) * XP2, 31) * XP1;
      v3 = rotl64(v3 + ld_u64_bytes(d + off + 16) * XP2, 31) * XP1;
      v4 = rotl64(v4 + ld_u64_bytes(d + off + 24) * XP2, 31) * XP1;
      off += 32;
    } while (off <= limit);
    h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = (h ^ (rotl64(v1 * XP2, 31) * XP1)) * XP1 + XP4;
    h = (h ^ (rotl64(v2 * XP2, 31) * XP1)) * XP1 + XP4;
    h = (h ^ (rotl64(v3 * XP2, 31) * XP1)) * XP1 + XP4;
    h = (h ^ (rotl64(v4 * XP2, 31) * XP1)) * XP1 + XP4;
  } else {
    h = seed + XP5;
  }
  h += static_cast<uint64_t>(n);
  for (; off + 8 <= n; off += 8) h = xx_step8(h, ld_u64_bytes(d + off));
  if (off + 4 <= n) {
    h = xx_step4(h, ld_u32_bytes(d + off));
    off += 4;
  }
  for (; off < n; ++off) h = xx_step1(h, d[off]);
  return xx_finalize(h);
}

// ---------------------------------------------------------------- Murmur3 (Spark tail)
constexpr uint32_t MC1 = 0xcc9e2d51u, MC2 = 0x1b873593u, MC3 = 0xe6546b64u;
__device__ __forceinline__ uint32_t mm_mix(uint32_t h, uint32_t k1)
{
  k1 *= MC1;
  k1 = __funnelshift_l(k1, k1, 15);
  k1 *= MC2;
  h ^= k1;
  h = __funnelshift_l(h, h, 13);
  return h * 5 + MC3;
}
__device__ __forceinline__ uint32_t mm_fmix(uint32_t h, uint32_t len)
{
  h ^= len;
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}
__device__ __forceinline__ uint32_t mm_u32(uint32_t v, uint32_t seed) { return mm_fmix(mm_mix(seed, v), 4); }
__device__ __forceinline__ uint32_t mm_u64(uint64_t v, uint32_t seed)
{
  return mm_fmix(mm_mix(mm_mix(seed, static_cast<uint32_t>(v)), static_cast<uint32_t>(v >> 32)), 8);
}
__device__ inline uint32_t mm_bytes(const uint8_t* d, int32_t len, uint32_t seed)
{
  uint32_t h = seed;
  const int32_t nb = len >> 2;
  for (int32_t i = 0; i < nb; ++i) h = mm_mix(h, ld_u32_bytes(d + 4 * i));
  for (int32_t i = nb * 4; i < len; ++i)
    h = mm_mix(h, static_cast<uint32_t>(static_cast<int32_t>(static_cast<int8_t>(d[i]))));  // murmur_hash.cuh:72-93
  return mm_fmix(h, static_cast<uint32_t>(len));
}
// Standard MurmurHash3_x86_32 (Iceberg's bucket hash, Guava's murmur3_32): the 4-byte blocks are mm_mix, but the 1-3 tail
// bytes are folded into one little-endian word k1 (upper bytes zero), scrambled and XORed into h without the
// rotate-multiply-add of a block.  iceberg.cu feeds the blocks and that tail word from registers.
__device__ __forceinline__ uint32_t mm_tail_std(uint32_t h, uint32_t k1)
{
  k1 *= MC1;
  k1 = __funnelshift_l(k1, k1, 15);
  k1 *= MC2;
  return h ^ k1;
}

// ---------------------------------------------------------------- float canonicalisation (hash.cuh:34-57)
__device__ __forceinline__ uint32_t norm_f32(uint32_t bits, bool zeros)
{
  const float f = __uint_as_float(bits);
  if (zeros && f == 0.0f) return 0u;
  if (f != f) return 0x7fc00000u;
  return bits;
}
__device__ __forceinline__ uint64_t norm_f64(uint64_t bits, bool zeros)
{
  const double d = __longlong_as_double(static_cast<long long>(bits));
  if (zeros && d == 0.0) return 0ull;
  if (d != d) return 0x7ff8000000000000ull;
  return bits;
}

// ---------------------------------------------------------------- DECIMAL128 -> Java BigInteger bytes
// hash.cuh:64-107: minimal big-endian two's complement.  lo/hi are the little-endian halves.
__device__ inline int dec128_java_bytes(uint64_t lo, uint64_t hi, uint8_t out[16])
{
  uint8_t le[16];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    le[i]     = static_cast<uint8_t>(lo >> (8 * i));
    le[8 + i] = static_cast<uint8_t>(hi >> (8 * i));
  }
  const bool neg     = (hi >> 63) != 0;
  const uint8_t zero = neg ? 0xff : 0x00;
  int length         = 16;
  while (length > 0 && le[length - 1] == zero) --length;
  if (length < 1) length = 1;
  if (length < 16 && (neg != ((le[length - 1] & 0x80) != 0))) ++length;
  for (int i = 0; i < length; ++i) out[i] = le[length - 1 - i];
  return length;
}

// ---------------------------------------------------------------- per-type element hashing
// `v` holds the raw little-endian value bits (up to 8 bytes; DECIMAL128 passes lo in v, hi in v2).
// Type rules: xxhash64.cu:201-273 / murmur_hash.cuh:130-205.
__device__ __forceinline__ uint64_t xx_fixed(int32_t type, uint64_t v, uint64_t v2, uint64_t h)
{
  switch (type) {
    case SRJ_BOOL8: return xx_u32((v & 0xff) != 0, h);
    case SRJ_INT8: return xx_u32(static_cast<uint32_t>(static_cast<int32_t>(static_cast<int8_t>(v))), h);
    case SRJ_UINT8: return xx_u32(static_cast<uint32_t>(v & 0xff), h);
    case SRJ_INT16: return xx_u32(static_cast<uint32_t>(static_cast<int32_t>(static_cast<int16_t>(v))), h);
    case SRJ_UINT16: return xx_u32(static_cast<uint32_t>(v & 0xffff), h);
    case SRJ_FLOAT32: return xx_u32(norm_f32(static_cast<uint32_t>(v), true), h);
    case SRJ_FLOAT64: return xx_u64(norm_f64(v, true), h);
    case SRJ_DECIMAL32: return xx_u64(static_cast<uint64_t>(static_cast<int64_t>(static_cast<int32_t>(v))), h);
    case SRJ_DECIMAL128: {
      uint8_t b[16];
      const int n = dec128_java_bytes(v, v2, b);
      return xx_bytes(b, n, h);
    }
    case SRJ_INT32:
    case SRJ_UINT32:
    case SRJ_TIMESTAMP_DAYS:
    case SRJ_DURATION_DAYS: return xx_u32(static_cast<uint32_t>(v), h);
    default: return xx_u64(v, h);  // 8-byte integers, timestamps, durations, DECIMAL64
  }
}

__device__ __forceinline__ uint32_t mm_fixed(int32_t type, uint64_t v, uint64_t v2, uint32_t h)
{
  switch (type) {
    case SRJ_BOOL8: return mm_u32((v & 0xff) != 0, h);
    case SRJ_INT8: return mm_u32(static_cast<uint32_t>(static_cast<int32_t>(static_cast<int8_t>(v))), h);
    case SRJ_UINT8: return mm_u32(static_cast<uint32_t>(v & 0xff), h);
    case SRJ_INT16: return mm_u32(static_cast<uint32_t>(static_cast<int32_t>(static_cast<int16_t>(v))), h);
    case SRJ_UINT16: return mm_u32(static_cast<uint32_t>(v & 0xffff), h);
    case SRJ_FLOAT32: return mm_u32(norm_f32(static_cast<uint32_t>(v), false), h);
    case SRJ_FLOAT64: return mm_u64(norm_f64(v, false), h);
    case SRJ_DECIMAL32: return mm_u64(static_cast<uint64_t>(static_cast<int64_t>(static_cast<int32_t>(v))), h);
    case SRJ_DECIMAL128: {
      uint8_t b[16];
      const int n = dec128_java_bytes(v, v2, b);
      return mm_bytes(b, n, h);
    }
    case SRJ_INT32:
    case SRJ_UINT32:
    case SRJ_TIMESTAMP_DAYS:
    case SRJ_DURATION_DAYS: return mm_u32(static_cast<uint32_t>(v), h);
    default: return mm_u64(v, h);
  }
}

// hive_hash.cu:42-152.  Returns false for unsupported types (the reference hits CUDF_UNREACHABLE;
// the host API rejects those schemas up front).
__device__ __forceinline__ int32_t hive_long(uint64_t k) { return static_cast<int32_t>((k >> 32) ^ k); }
__device__ __forceinline__ int32_t hive_fixed(int32_t type, uint64_t v)
{
  switch (type) {
    case SRJ_BOOL8: return (v & 0xff) != 0;
    case SRJ_INT8: return static_cast<int8_t>(v);
    case SRJ_INT16: return static_cast<int16_t>(v);
    case SRJ_INT32:
    case SRJ_TIMESTAMP_DAYS: return static_cast<int32_t>(v);
    case SRJ_INT64: return hive_long(v);
    case SRJ_FLOAT32: return static_cast<int32_t>(norm_f32(static_cast<uint32_t>(v), false));
    case SRJ_FLOAT64: return hive_long(norm_f64(v, false));
    case SRJ_TIMESTAMP_MICROSECONDS: {
      const int64_t t   = static_cast<int64_t>(v);
      const int64_t ts  = t / 1000000;
      const int64_t tns = (t % 1000000) * 1000;
      const uint64_t r  = (static_cast<uint64_t>(ts) << 30) | static_cast<uint64_t>(tns);
      return hive_long(r);
    }
    default: return 0;
  }
}
__device__ inline int32_t hive_bytes(const uint8_t* d, int32_t len)
{
  uint32_t h = 0;
  for (int32_t i = 0; i < len; ++i) h = h * 31u + static_cast<uint32_t>(static_cast<int32_t>(static_cast<int8_t>(d[i])));
  return static_cast<int32_t>(h);
}

__host__ __device__ inline bool hive_supported(int32_t t)
{
  return t == SRJ_BOOL8 || t == SRJ_INT8 || t == SRJ_INT16 || t == SRJ_INT32 || t == SRJ_INT64 || t == SRJ_FLOAT32 ||
         t == SRJ_FLOAT64 || t == SRJ_TIMESTAMP_DAYS || t == SRJ_TIMESTAMP_MICROSECONDS || t == SRJ_STRING;
}

}  // namespace hash
}  // namespace srj
