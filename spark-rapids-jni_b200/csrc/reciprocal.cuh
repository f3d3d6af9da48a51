// reciprocal.cuh -- the remainder by a per-call constant divisor d through a host-computed reciprocal, so that no division
// instruction or subroutine is left in a kernel's row loop (bloom_filter.cu, iceberg.cu).
//
// m = floor((2^N - 1) / d) with N = 32 (mod_v1) or 64 (mod_v2).  For a dividend x <= 2^(N-1), q = mulhi(x, m) is floor(x / d)
// or one less: x / d - x * m / 2^N = x * (2^N - d * m) / (d * 2^N) with 2^N - d * m in [1, d + 1] (1 for d = 1), which is
// below 1.  So r = x - q * d < 2d needs at most one conditional subtraction.  Divisors up to 2^(N-1) keep 2d within N bits.
#pragma once
#include <stdint.h>

namespace srj {

inline uint32_t reciprocal_v1(uint32_t d) { return 0xffffffffu / d; }
inline uint64_t reciprocal_v2(uint64_t d) { return ~uint64_t{0} / d; }

// x % d for x <= 2^31, 1 <= d <= 2^31, m = reciprocal_v1(d)
__device__ __forceinline__ uint32_t mod_v1(uint32_t x, uint32_t d, uint32_t m)
{
  uint32_t r = x - __umulhi(x, m) * d;
  return r >= d ? r - d : r;
}

// x % d for x <= 2^63, 1 <= d <= 2^63, m = reciprocal_v2(d)
__device__ __forceinline__ uint64_t mod_v2(uint64_t x, uint64_t d, uint64_t m)
{
  uint64_t r = x - __umul64hi(x, m) * d;
  return r >= d ? r - d : r;
}

}  // namespace srj
