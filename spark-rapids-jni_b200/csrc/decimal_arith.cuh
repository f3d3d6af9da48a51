// decimal_arith.cuh -- the 256-bit integer arithmetic of DecimalUtils (decimal.cu), usable on the host as well: the host
// computes the reciprocals of a call's fixed powers of ten with the same code the device uses for per-row divisors, and
// a CPU test compiles this header with a plain C++ compiler to check the division against exact integers.
//
// Values are 256-bit two's complement in four 64-bit limbs.  Division is by a 128-bit magnitude d != 0, normalised to
// D = d << s with its top bit set, through the 3-by-2 reciprocal v = floor((2^192 - 1) / D) - 2^64 (N. Möller and
// T. Granlund, "Improved division by invariant integers", IEEE Trans. Computers 60(2), 2011: Algorithms 2, 5 and 6).
// No '/' or '%' of a 64- or 128-bit operand appears, so the device code calls no division subroutine; the one 32-bit
// division (the 11-bit seed of the reciprocal) compiles to inline instructions.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

namespace srj {
namespace dec {

using u128 = unsigned __int128;

struct U256 {
  uint64_t w[4];   // little-endian limbs
};

__host__ __device__ __forceinline__ int clz64(uint64_t x)   // x != 0
{
#ifdef __CUDA_ARCH__
  return __clzll(static_cast<long long>(x));
#else
  return __builtin_clzll(x);
#endif
}

__host__ __device__ __forceinline__ U256 sext(u128 v)   // a signed 128-bit value widened
{
  const uint64_t s = static_cast<uint64_t>(static_cast<int64_t>(static_cast<uint64_t>(v >> 64)) >> 63);
  return U256{{static_cast<uint64_t>(v), static_cast<uint64_t>(v >> 64), s, s}};
}

__host__ __device__ __forceinline__ bool is_neg(const U256& x) { return static_cast<int64_t>(x.w[3]) < 0; }

__host__ __device__ __forceinline__ U256 add(const U256& a, const U256& b)
{
  U256 r;
  u128 c = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    c += static_cast<u128>(a.w[i]) + b.w[i];
    r.w[i] = static_cast<uint64_t>(c);
    c >>= 64;
  }
  return r;
}

__host__ __device__ __forceinline__ U256 neg(const U256& a)
{
  U256 r;
  u128 c = 1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    c += static_cast<uint64_t>(~a.w[i]);
    r.w[i] = static_cast<uint64_t>(c);
    c >>= 64;
  }
  return r;
}

__host__ __device__ __forceinline__ U256 abs256(const U256& a) { return is_neg(a) ? neg(a) : a; }

__host__ __device__ __forceinline__ U256 add_small(const U256& a, int64_t k) { return add(a, sext(static_cast<u128>(static_cast<__int128>(k)))); }

// the low 256 bits of a * b (the reference's chunked256 multiply)
__host__ __device__ __forceinline__ U256 mul(const U256& a, const U256& b)
{
  U256 r{{0, 0, 0, 0}};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint64_t carry = 0;
#pragma unroll
    for (int i = 0; i + j < 4; ++i) {
      const u128 t = static_cast<u128>(a.w[i]) * b.w[j] + r.w[i + j] + carry;
      r.w[i + j]   = static_cast<uint64_t>(t);
      carry        = static_cast<uint64_t>(t >> 64);
    }
  }
  return r;
}

// the exact product of two signed 128-bit values: |a| * |b| <= 2^254, negated when the signs differ
__host__ __device__ __forceinline__ U256 mul128(u128 a, u128 b)
{
  const bool an = static_cast<int64_t>(static_cast<uint64_t>(a >> 64)) < 0, bn = static_cast<int64_t>(static_cast<uint64_t>(b >> 64)) < 0;
  const u128 x = an ? u128(0) - a : a, y = bn ? u128(0) - b : b;
  const uint64_t x0 = static_cast<uint64_t>(x), x1 = static_cast<uint64_t>(x >> 64);
  const uint64_t y0 = static_cast<uint64_t>(y), y1 = static_cast<uint64_t>(y >> 64);
  const u128 p00 = static_cast<u128>(x0) * y0, p01 = static_cast<u128>(x0) * y1, p10 = static_cast<u128>(x1) * y0,
             p11 = static_cast<u128>(x1) * y1;
  const u128 mid = (p00 >> 64) + static_cast<uint64_t>(p01) + static_cast<uint64_t>(p10);
  const u128 hi  = p11 + (p01 >> 64) + (p10 >> 64) + (mid >> 64);
  const U256 r{{static_cast<uint64_t>(p00), static_cast<uint64_t>(mid), static_cast<uint64_t>(hi), static_cast<uint64_t>(hi >> 64)}};
  return an != bn ? neg(r) : r;
}

// unsigned a >= b
__host__ __device__ __forceinline__ bool ge(const U256& a, const U256& b)
{
  for (int i = 3; i >= 0; --i)
    if (a.w[i] != b.w[i]) return a.w[i] > b.w[i];
  return true;
}

// floor((2^128 - 1) / d) - 2^64 for d >= 2^63 (Möller-Granlund Algorithm 2)
__host__ __device__ __forceinline__ uint64_t reciprocal_word(uint64_t d)
{
  const uint64_t d0  = d & 1;
  const uint32_t d9  = static_cast<uint32_t>(d >> 55);                 // [256, 511]
  const uint64_t d40 = (d >> 24) + 1;
  const uint64_t d63 = (d >> 1) + d0;                                  // ceil(d / 2)
  const uint64_t v0  = 523520u / d9;                                   // (2^19 - 3 * 2^8) / d9, 11 bits
  const uint64_t v1  = (v0 << 11) - ((v0 * v0 * d40) >> 40) - 1;
  const uint64_t v2  = (v1 << 13) + ((v1 * ((uint64_t{1} << 60) - v1 * d40)) >> 47);
  const uint64_t e   = ((v2 >> 1) & (uint64_t{0} - d0)) - v2 * d63;
  const uint64_t v3  = static_cast<uint64_t>((static_cast<u128>(v2) * e) >> 65) + (v2 << 31);
  const u128 t       = static_cast<u128>(v3) * d + d;
  return v3 - static_cast<uint64_t>(t >> 64) - d;
}

// 10^0 .. 10^76 in little-endian 64-bit limbs; the low limb of 10^k is also 10^k mod 2^64 (k < 64)
constexpr int kMaxPow = 76;

struct PowTable {
  uint64_t w[kMaxPow + 1][4];
};

// each power the previous times 10 in 32-bit halves (a constant expression, so one definition serves the host and the
// __constant__ copies of decimal.cu and float_to_decimal.cu)
constexpr PowTable make_pow10()
{
  PowTable t{};
  t.w[0][0] = 1;
  for (int k = 1; k <= kMaxPow; ++k) {
    uint64_t carry = 0;
    for (int i = 0; i < 4; ++i) {
      const uint64_t lo = (t.w[k - 1][i] & 0xffffffffu) * 10 + carry;
      const uint64_t hi = (t.w[k - 1][i] >> 32) * 10 + (lo >> 32);
      t.w[k][i]         = (hi << 32) | (lo & 0xffffffffu);
      carry             = hi >> 32;
    }
  }
  return t;
}

static_assert(make_pow10().w[19][0] == 10000000000000000000ull && make_pow10().w[20][1] == 5 &&
                make_pow10().w[76][3] == 0x161bcca7119915b5ull,
              "powers of ten");

// A divisor: D = (d1, d0) = d << s with the top bit set, and its 3-by-2 reciprocal v.  zero: d == 0, which divides as the
// reference's bit-serial loop does (every quotient bit set, the remainder the dividend's low 128 bits).
struct Div {
  uint64_t d1, d0, v;
  int32_t s;
  bool zero;
};

// Möller-Granlund Algorithm 6
__host__ __device__ __forceinline__ Div make_div(u128 d)
{
  Div r{};
  if (d == 0) {
    r.zero = true;
    return r;
  }
  const uint64_t hi = static_cast<uint64_t>(d >> 64), lo = static_cast<uint64_t>(d);
  r.s              = hi ? clz64(hi) : 64 + clz64(lo);
  const u128 D     = d << r.s;
  const uint64_t d1 = static_cast<uint64_t>(D >> 64), d0 = static_cast<uint64_t>(D);
  uint64_t v       = reciprocal_word(d1);
  uint64_t p       = d1 * v + d0;
  if (p < d0) {
    --v;
    if (p >= d1) {
      --v;
      p -= d1;
    }
    p -= d1;
  }
  const u128 t = static_cast<u128>(v) * d0;
  const uint64_t t1 = static_cast<uint64_t>(t >> 64), t0 = static_cast<uint64_t>(t);
  p += t1;
  if (p < t1) {
    --v;
    if (p > d1 || (p == d1 && t0 >= d0)) --v;
  }
  r.d1 = d1;
  r.d0 = d0;
  r.v  = v;
  return r;
}

// (u2, u1, u0) / (d1, d0) with (u2, u1) < (d1, d0): one quotient limb, the remainder in *r (Algorithm 5)
__host__ __device__ __forceinline__ uint64_t div_3by2(uint64_t u2, uint64_t u1, uint64_t u0, const Div& D, u128* r)
{
  const u128 q  = static_cast<u128>(D.v) * u2 + ((static_cast<u128>(u2) << 64) | u1);
  uint64_t q1   = static_cast<uint64_t>(q >> 64);
  const uint64_t q0 = static_cast<uint64_t>(q);
  const uint64_t r1 = u1 - q1 * D.d1;
  const u128 DD = (static_cast<u128>(D.d1) << 64) | D.d0;
  u128 rr       = ((static_cast<u128>(r1) << 64) | u0) - static_cast<u128>(D.d0) * q1 - DD;
  ++q1;
  if (static_cast<uint64_t>(rr >> 64) >= q0) {
    --q1;
    rr += DD;
  }
  if (rr >= DD) {
    ++q1;
    rr -= DD;
  }
  *r = rr;
  return q1;
}

__host__ __device__ __forceinline__ uint64_t shl_in(uint64_t hi, uint64_t lo, int b) { return b ? (hi << b) | (lo >> (64 - b)) : hi; }

// n / d and n % d for an unsigned 256-bit n
__host__ __device__ __forceinline__ U256 udivrem(const U256& n, const Div& D, u128* rem)
{
  if (D.zero) {
    *rem = (static_cast<u128>(n.w[1]) << 64) | n.w[0];
    return U256{{~uint64_t{0}, ~uint64_t{0}, ~uint64_t{0}, ~uint64_t{0}}};
  }
  const int b = D.s & 63;
  const uint64_t y0 = n.w[0] << b, y1 = shl_in(n.w[1], n.w[0], b), y2 = shl_in(n.w[2], n.w[1], b), y3 = shl_in(n.w[3], n.w[2], b),
                 y4 = b ? n.w[3] >> (64 - b) : 0;
  const bool wide = D.s >= 64;                                         // shift one more limb
  const uint64_t x0 = wide ? 0 : y0, x1 = wide ? y0 : y1, x2 = wide ? y1 : y2, x3 = wide ? y2 : y3, x4 = wide ? y3 : y4,
                 x5 = wide ? y4 : 0;
  u128 r = (static_cast<u128>(x5) << 64) | x4;                          // < 2^s <= D
  U256 q;
  q.w[3] = div_3by2(static_cast<uint64_t>(r >> 64), static_cast<uint64_t>(r), x3, D, &r);
  q.w[2] = div_3by2(static_cast<uint64_t>(r >> 64), static_cast<uint64_t>(r), x2, D, &r);
  q.w[1] = div_3by2(static_cast<uint64_t>(r >> 64), static_cast<uint64_t>(r), x1, D, &r);
  q.w[0] = div_3by2(static_cast<uint64_t>(r >> 64), static_cast<uint64_t>(r), x0, D, &r);
  *rem = r >> D.s;
  return q;
}

// n / d for n < 2^128: udivrem's two low quotient limbs (its two high ones are 0), all ones for d == 0 as udivrem
__host__ __device__ __forceinline__ u128 udiv128(u128 n, const Div& D)
{
  if (D.zero) return ~u128(0);
  const int b        = D.s & 63;
  const uint64_t n0  = static_cast<uint64_t>(n), n1 = static_cast<uint64_t>(n >> 64);
  const uint64_t y0  = n0 << b, y1 = shl_in(n1, n0, b), y2 = b ? n1 >> (64 - b) : 0;
  const bool wide    = D.s >= 64;                                     // (y2, y1) < 2^s <= D: the high limbs are 0
  u128 r             = wide ? (static_cast<u128>(y2) << 64) | y1 : static_cast<u128>(y2);
  const uint64_t q1  = div_3by2(static_cast<uint64_t>(r >> 64), static_cast<uint64_t>(r), wide ? y0 : y1, D, &r);
  const uint64_t q0  = div_3by2(static_cast<uint64_t>(r >> 64), static_cast<uint64_t>(r), wide ? 0 : y0, D, &r);
  return (static_cast<u128>(q1) << 64) | q0;
}

// The reference's signed divide (decimal_utils.cu:163-183): quotient truncated toward zero, negated when the signs of n
// (256-bit) and d differ; *rmag = |remainder|; *round_down = the signs differ.
struct Quot {
  U256 q;
  u128 rmag;
  bool neg;        // the quotient's sign: n's sign != d's sign
};

__host__ __device__ __forceinline__ Quot sdivrem(const U256& n, bool d_neg, const Div& D)
{
  Quot r;
  const bool n_neg = is_neg(n);
  r.q   = udivrem(n_neg ? neg(n) : n, D, &r.rmag);
  r.neg = n_neg != d_neg;
  if (r.neg) r.q = neg(r.q);
  return r;
}

// HALF_UP from the remainder: one unit away from zero when 2 |r| >= |d| (decimal_utils.cu:185-217 for |d| < 2^127)
__host__ __device__ __forceinline__ U256 round_half_up(const Quot& r, u128 dmag)
{
  return r.rmag >= dmag - r.rmag ? add_small(r.q, r.neg ? -1 : 1) : r.q;
}

}  // namespace dec
}  // namespace srj
