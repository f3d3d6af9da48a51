/*
 * float_to_decimal.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE) of DecimalUtils.floatingPointToDecimal.
 *
 * A restatement of src/main/cpp/src/decimal_utils.cu:1193-1336 (scaled_round, floating_point_to_decimal_fn) over cudf's
 * fixed_point/detail/floating_conversion.hpp (FC) with FloatingType = double, at the width of each step's C++ type,
 * so that its wraps are kept; oracle/float_to_decimal.py restates the same steps in Python integers and builds and
 * loads this file.  u128 stands for every unsigned type of the reference and is masked to the step's width (32, 64 or
 * 128 bits).  Paths are relative to the reference repository's root.  OpenMP runs the rows in parallel, for the tests'
 * sweeps of 2^32 rows.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

enum { T_DEC32 = 25, T_DEC64 = 26, T_DEC128 = 27 };   /* cudf type ids: thirdparty/cudf/cpp/include/cudf/types.hpp */

typedef unsigned __int128 u128;

static int is_valid(const uint32_t* m, int64_t i) { return !m || ((m[i >> 5] >> (i & 31)) & 1u); }

static u128 f2d_mask(int bits) { return bits >= 128 ? ~(u128)0 : (((u128)1 << bits) - 1); }

static u128 f2d_ipow10(int k, int bits)          /* fixed_point.hpp:78-97 mod 2^bits; k < 0 gives 10 */
{
  if (k == 0) return 1;
  u128 extra = 1, square = 10, m = f2d_mask(bits);
  while (k > 1) {
    if (k & 1) extra = (extra * square) & m;
    k >>= 1;
    square = (square * square) & m;
  }
  return (square * extra) & m;
}

static u128 f2d_pow10_exact(int k) { u128 r = 1; while (k-- > 0) r *= 10; return r; }

static u128 f2d_mul_pow10(u128 v, int k, int rep_bits, int t_bits)   /* FC:402-472 */
{
  if (rep_bits == 32) return (k >= 0 && k <= 9) ? (v * f2d_pow10_exact(k)) & f2d_mask(t_bits) : 0;
  return (v * f2d_ipow10(k, rep_bits)) & f2d_mask(t_bits);
}

static u128 f2d_div_pow10(u128 v, int k, int rep_bits, int t_bits)   /* FC:324-391, 487-498 */
{
  if (rep_bits == 32) return (k >= 0 && k <= 9) ? v / f2d_pow10_exact(k) : 0;
  u128 d = f2d_ipow10(k, rep_bits);
  return d ? v / d : f2d_mask(t_bits);       /* 10^k = 0 mod 2^64: undefined in C++, all ones here */
}

static u128 f2d_gls(u128 v, int s, int bits) { return s <= bits - 1 ? (v << s) & f2d_mask(bits) : f2d_mask(bits); }   /* FC:509-515 */
static u128 f2d_grs(u128 v, int s, int bits) { return s <= bits - 1 ? v >> s : 0; }                                    /* FC:526-531 */

static u128 f2d_pospow(uint64_t base2, int pow2, int p, int ub)       /* FC:687-759 */
{
  u128 sr = base2;
  if (pow2 <= 70) return f2d_div_pow10(sr << pow2, p, 128, 128) & f2d_mask(ub);
  sr <<= 70;
  pow2 -= 70;
  while (p > 18) {
    sr /= f2d_pow10_exact(18);
    p -= 18;
    if (pow2 <= 60) return f2d_div_pow10(sr << pow2, p, 128, 128) & f2d_mask(ub);
    sr <<= 60;
    pow2 -= 60;
  }
  sr = f2d_div_pow10(sr, p, 64, 128);
  return f2d_gls(sr & f2d_mask(ub), pow2, ub);
}

static u128 f2d_negpow(uint64_t base2, int pow2, int p, int ub)       /* FC:774-845 */
{
  u128 sr = base2;
  int p10 = -p, p2 = -pow2;
  if (p10 > 18) {
    sr <<= 14;
    p2 += 14;
    do {
      sr *= f2d_pow10_exact(18);
      p10 -= 18;
      if (p2 <= 60) return f2d_mul_pow10((sr >> p2) & f2d_mask(ub), p10, ub, ub);
      sr >>= 60;
      p2 -= 60;
    } while (p10 > 18);
  }
  return f2d_grs(sr * f2d_ipow10(p10, 64), p2, 128) & f2d_mask(ub);
}

static u128 f2d_convert(uint64_t base2, int p, int pow2, int ub)      /* FC:860-898 */
{
  if (p == 0) return pow2 >= 0 ? f2d_gls(base2 & f2d_mask(ub), pow2, ub) : f2d_grs(base2, -pow2, 64) & f2d_mask(ub);
  if (p > 0) {
    if (pow2 <= 0) return f2d_div_pow10(f2d_grs(base2, -pow2, 64), p, 64, 64) & f2d_mask(ub);
    return f2d_pospow(base2, pow2, p, ub);
  }
  if (pow2 >= 0) return f2d_mul_pow10(f2d_gls(base2 & f2d_mask(ub), pow2, ub), -p, ub, ub);
  return f2d_negpow(base2, pow2, p, ub);
}

/* scaled_round (decimal_utils.cu:1193-1309) of a finite x: the IntType result as a 128-bit two's complement value */
static u128 f2d_scaled_round(double x, int is_f32, int width, int pow10, double scale_factor)
{
  uint64_t bits;
  memcpy(&bits, &x, 8);
  if ((bits & ~(1ull << 63)) == 0) return 0;
  int neg = (int)(bits >> 63);
  uint64_t mant = bits & ((1ull << 52) - 1);
  int e = (int)((bits >> 52) & 0x7ff), fp2;
  if (e == 0) {
    int shift = 53 - (64 - __builtin_clzll(mant));
    mant <<= shift;
    fp2 = 1 - 1023 - shift;
  } else {
    fp2 = e - 1023;
    mant |= 1ull << 52;
  }
  int pow2 = fp2 - 52;
  double uf = fabs(x);
  double max_rep = width == 32 ? 2147483647.0 : width == 64 ? 9223372036854775808.0 : 170141183460469231731687303715884105728.0;
  volatile double prod = 10.0 * uf;          /* two roundings, as the reference's double expression */
  int rwo = prod * scale_factor < max_rep;
  int can_round = width == 128 ? rwo : 1;
  int sp = can_round ? pow10 - 1 : pow10;
  int whole = floor(x) == x;
  uint64_t base2 = (mant << 1) + (uint64_t)(!is_f32 && !whole);
  pow2 -= 1;
  int ub = width == 32 ? (rwo ? 32 : 64) : 128, tb = width == 32 ? 64 : 128;
  u128 mag = f2d_convert(base2, sp, pow2, ub), mt = f2d_mask(tb);
  int fp = (3 * pow2 - 10 * pow10 + (is_f32 ? 0 : 9 * (uf > 9223372036854775807.0))) / 10;   /* C division truncates */
  if (can_round) {
    if (fp < 0) {
      mag = ((mag + 5) & mt) / 10;
    } else {
      if (is_f32 || whole) mag = (mag + f2d_mul_pow10(5, fp, width, tb)) & mt;
      mag = f2d_mul_pow10(f2d_div_pow10(mag, fp + 1, width, tb), fp, width, tb);
    }
  } else if (fp > 0) {
    mag = f2d_mul_pow10(f2d_div_pow10(mag, fp, width, tb), fp, width, tb);
  }
  u128 s = mag & f2d_mask(width);
  if (neg) s = (0 - s) & f2d_mask(width);
  if (width < 128 && (s >> (width - 1)) & 1) s |= ~f2d_mask(width);   /* sign-extend to 128 bits */
  return s;
}

/* The cast of n rows (in: float or double by is_f32; in_mask NULL = all valid) to the DECIMAL type out_type (25, 26,
 * 27) of `precision` at cudf scale `scale`: out gets n values of the type's width, valid[i] the row's validity;
 * *failure_row the smallest row outside the bound, or -1.  The caller checks the domain (float_to_decimal.py:f2d_check). */
int f2d_float_to_decimal(const void* in, int32_t is_f32, const uint32_t* in_mask, int64_t n, int32_t out_type, int32_t precision,
                         int32_t scale, void* out, uint8_t* valid, int64_t* failure_row)
{
  int width = out_type == T_DEC32 ? 32 : out_type == T_DEC64 ? 64 : 128;
  u128 sf_int = f2d_mul_pow10(1, -scale, width, width);
  double sf = (double)sf_int;
  __int128 bound = (__int128)f2d_mul_pow10(1, precision, width, width);
  int64_t first = INT64_MAX;
#pragma omp parallel for schedule(static) reduction(min : first)
  for (int64_t i = 0; i < n; ++i) {
    double x = is_f32 ? (double)((const float*)in)[i] : ((const double*)in)[i];
    __int128 v = 0;
    int ok = is_valid(in_mask, i) && isfinite(x);
    if (ok) {
      v = (__int128)f2d_scaled_round(x, is_f32, width, scale, sf);
      if (-bound >= v || v >= bound) {
        ok = 0;
        v = 0;
        if (i < first) first = i;
      }
    }
    valid[i] = (uint8_t)ok;
    if (width == 32) ((int32_t*)out)[i] = (int32_t)v;
    else if (width == 64) ((int64_t*)out)[i] = (int64_t)v;
    else memcpy((uint8_t*)out + 16 * i, &v, 16);
  }
  *failure_row = first == INT64_MAX ? -1 : first;
  return 0;
}
