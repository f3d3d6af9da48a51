// float_to_decimal.cu -- DecimalUtils.floatingPointToDecimal on the device: FLOAT32 / FLOAT64 to DECIMAL32 / 64 / 128
// with Spark's rounding (reference decimal_utils.cu:1174-1417, scaled_round and floating_point_to_decimal_fn, over cudf's
// fixed_point/detail/floating_conversion.hpp, "FC" below, instantiated with FloatingType = double).
//
// Each row restates the reference's integer steps at the width of the C++ type that holds them, so that its wraps are
// kept: values are carried in 128 bits and masked to 32 or 64 where the reference's type is narrower.  Which power-of-ten
// helper a step uses decides what 10^k is there: the 32-bit one is 10^k for k in 0..9 and 0 otherwise; the 64- and
// 128-bit ones are ipow (fixed_point.hpp:78-97) modulo 2^64 or 2^128, which is 10 for k < 0.  A division by such a
// value is a division by it, not by 10^k.  One division the reference leaves undefined, by 10^64 mod 2^64 = 0 (DECIMAL64
// rows whose floor_pow10 is 63), gives an all-ones quotient here (dec::udiv128), so those rows fail.
//
// No '/' or '%' of a 64- or 128-bit operand by a row value appears: divisions by 10^k and by the wrapped powers go through
// the 3-by-2 reciprocal of decimal_arith.cuh (dec::udiv128), the divisor's reciprocal computed in the row unless it is the
// call's 10.  Per-call constants come from the host: the double scale factor of rounding_wont_overflow, its threshold,
// the bound 10^precision and the scale.
//
// f2d_kernel<F, W> (F float / double, W the output's bits) is grid-stride with 64-bit indices; a lane owns one row of a
// 32-row step, so the warp's ballot is the output's mask word.  The null count and the smallest failing row leave each
// CTA with one atomic each (row_counters.cuh), read back together once per call.
#include <cmath>
#include <type_traits>

#include "check.hpp"
#include "common.cuh"
#include "decimal_arith.cuh"
#include "kernels.hpp"
#include "row_counters.cuh"

namespace srj {
namespace {

using dec::Div;
using dec::u128;

constexpr int kF2dThreads  = 256;
constexpr int kF2dBlocksSm = 8;   // grid cap per multiprocessor: one full-occupancy wave

__constant__ dec::PowTable c_f2d_pow10 = dec::make_pow10();

struct F2dParams {
  double scale_factor;   // double(multiply_power10<IntType>(1, -scale)), decimal_utils.cu:1206-1207
  double max_rep;        // double(numeric_limits<IntType>::max())
  u128 bound;            // 10^precision: a valid result lies strictly inside (-bound, bound)
  Div ten;               // 10, the last digit's divisor
  int32_t pow10;         // the cudf scale
};

template <int B>
__device__ __forceinline__ u128 trunc_to(u128 v)
{
  if constexpr (B == 128) return v;
  else return v & ((u128(1) << B) - 1);
}

__device__ __forceinline__ u128 pow10_lo(int k)   // 10^k mod 2^128, k in 0..76
{
  return (static_cast<u128>(c_f2d_pow10.w[k][1]) << 64) | c_f2d_pow10.w[k][0];
}

// ipow<uint64_t / __uint128_t, BASE_10>(k) (fixed_point.hpp:78-97): 10 for k < 0 (its assert is compiled out and the
// loop never runs), 10^k mod 2^B otherwise, which is 0 from k = B on
template <int B>
__device__ __forceinline__ u128 ipow10(int k)
{
  if (k < 0) return 10;
  if (k >= B) return 0;
  if constexpr (B == 64) return c_f2d_pow10.w[k][0];
  else return k <= dec::kMaxPow ? pow10_lo(k) : pow10_lo(dec::kMaxPow) * pow10_lo(k - dec::kMaxPow);
}

// multiply_power10<Rep>(v, k) on a T of TB bits (FC:402-472)
template <int Rep, int TB>
__device__ __forceinline__ u128 mul_pow10(u128 v, int k)
{
  if constexpr (Rep == 32) return k >= 0 && k <= 9 ? trunc_to<TB>(v * c_f2d_pow10.w[k][0]) : u128(0);
  else return trunc_to<TB>(v * ipow10<Rep>(k));
}

// divide_power10<Rep>(v, k) on a T of TB bits (FC:324-391, 487-498)
template <int Rep, int TB>
__device__ __forceinline__ u128 div_pow10(u128 v, int k)
{
  if constexpr (Rep == 32) return k >= 0 && k <= 9 ? dec::udiv128(v, dec::make_div(c_f2d_pow10.w[k][0])) : u128(0);
  else return trunc_to<TB>(dec::udiv128(v, dec::make_div(ipow10<Rep>(k))));
}

template <int B>
__device__ __forceinline__ u128 guarded_left_shift(u128 v, int s)   // FC:509-515
{
  return s <= B - 1 ? trunc_to<B>(v << s) : trunc_to<B>(~u128(0));
}

template <int B>
__device__ __forceinline__ u128 guarded_right_shift(u128 v, int s)   // FC:526-531
{
  return s <= B - 1 ? v >> s : u128(0);
}

// FC:687-759, pow2 > 0 and p > 0 (p <= 38): shift up by 2s and divide by 10s, at most two 18-digit steps
template <int UB>
__device__ __forceinline__ u128 shift_pospow(uint64_t base2, int pow2, int p)
{
  u128 sr = base2;
  if (pow2 <= 70) return trunc_to<UB>(dec::udiv128(sr << pow2, dec::make_div(pow10_lo(p))));   // 70: 124 - 54 bits
  sr <<= 70;
  pow2 -= 70;
  while (p > 18) {
    sr = dec::udiv128(sr, dec::make_div(pow10_lo(18)));
    p -= 18;
    if (pow2 <= 60) return trunc_to<UB>(dec::udiv128(sr << pow2, dec::make_div(pow10_lo(p))));
    sr <<= 60;
    pow2 -= 60;
  }
  sr = dec::udiv128(sr, dec::make_div(pow10_lo(p)));
  return guarded_left_shift<UB>(trunc_to<UB>(sr), pow2);
}

// FC:774-845, pow2 < 0 and p < 0 (p >= -39): multiply by 10s and shift down by 2s, at most two 18-digit steps
template <int UB>
__device__ __forceinline__ u128 shift_negpow(uint64_t base2, int pow2, int p)
{
  u128 sr = base2;
  int p10 = -p, p2 = -pow2;
  if (p10 > 18) {
    sr <<= 14;   // (128 - 60) - 54 bits
    p2 += 14;
    do {
      sr *= pow10_lo(18);
      p10 -= 18;
      if (p2 <= 60) return mul_pow10<UB, UB>(trunc_to<UB>(sr >> p2), p10);
      sr >>= 60;
      p2 -= 60;
    } while (p10 > 18);
  }
  return trunc_to<UB>(guarded_right_shift<128>(sr * pow10_lo(p10), p2));
}

// convert_floating_to_integral_shifting<Rep, double> (FC:860-898); UB is the width of make_unsigned_t<Rep>
template <int UB>
__device__ __forceinline__ u128 convert(uint64_t base2, int p, int pow2)
{
  if (p == 0) return pow2 >= 0 ? guarded_left_shift<UB>(trunc_to<UB>(base2), pow2) : trunc_to<UB>(guarded_right_shift<64>(base2, -pow2));
  if (p > 0) {
    if (pow2 <= 0) return trunc_to<UB>(div_pow10<64, 64>(guarded_right_shift<64>(base2, -pow2), p));
    return shift_pospow<UB>(base2, pow2, p);
  }
  if (pow2 >= 0) return mul_pow10<UB, UB>(guarded_left_shift<UB>(trunc_to<UB>(base2), pow2), -p);
  return shift_negpow<UB>(base2, pow2, p);
}

// scaled_round<F, IntType> (decimal_utils.cu:1193-1309) of a finite x: the IntType result's W bits
template <bool kF32, int W>
__device__ __forceinline__ u128 scaled_round(double x, const F2dParams& prm)
{
  constexpr int TB = W == 32 ? 64 : 128;   // the intermediate magnitude: uint64 for DECIMAL32, unsigned __int128 otherwise
  const uint64_t bits = static_cast<uint64_t>(__double_as_longlong(x));
  if ((bits << 1) == 0) return 0;
  uint64_t mant = bits & ((uint64_t{1} << 52) - 1);
  const int e   = static_cast<int>((bits >> 52) & 0x7ff);
  int pow2;
  if (e == 0) {                            // FC:187-200: a denormal lined up to the understood bit
    const int sh = __clzll(static_cast<long long>(mant)) - 11;
    mant <<= sh;
    pow2 = -1022 - sh - 52;
  } else {
    mant |= uint64_t{1} << 52;
    pow2 = e - 1023 - 52;
  }
  const double uf       = fabs(x);
  const bool rwo        = __dmul_rn(__dmul_rn(10.0, uf), prm.scale_factor) < prm.max_rep;   // :1205-1210
  const bool can_round  = W == 128 ? rwo : true;
  const int sp          = can_round ? prm.pow10 - 1 : prm.pow10;
  const bool whole      = floor(x) == x;
  const uint64_t base2  = (mant << 1) + ((!kF32 && !whole) ? 1u : 0u);   // :1223-1236
  pow2 -= 1;
  u128 mag;
  if constexpr (W == 32) mag = rwo ? convert<32>(base2, sp, pow2) : convert<64>(base2, sp, pow2);   // :1239-1253
  else mag = convert<128>(base2, sp, pow2);
  const int fp = (3 * pow2 - 10 * prm.pow10 + (kF32 ? 0 : 9 * (uf > 9223372036854775807.0))) / 10;   // :1259-1270, truncating
  if (can_round) {                         // :1273-1303
    if (fp < 0) {
      if constexpr (TB == 64) mag = static_cast<uint64_t>(mag + 5) / 10u;
      else mag = dec::udiv128(mag + 5, prm.ten);
    } else {
      if (kF32 || whole) mag = trunc_to<TB>(mag + mul_pow10<W, TB>(5, fp));
      mag = mul_pow10<W, TB>(div_pow10<W, TB>(mag, fp + 1), fp);
    }
  } else if (fp > 0) {
    mag = mul_pow10<W, TB>(div_pow10<W, TB>(mag, fp), fp);
  }
  const u128 s = trunc_to<W>(mag);         // :1307-1308: the cast and the negation wrap
  return (bits >> 63) ? trunc_to<W>(u128(0) - s) : s;
}

template <int W>
__device__ __forceinline__ __int128 sign_extend(u128 v)
{
  if constexpr (W == 128) return static_cast<__int128>(v);
  else return static_cast<__int128>(v << (128 - W)) >> (128 - W);
}

template <int W>   // the output's element: DECIMAL128 as two little-endian longs (8-byte alignment suffices)
using Rep = typename std::conditional<W == 32, int32_t, typename std::conditional<W == 64, int64_t, uint64_t>::type>::type;

// One warp step covers 32 rows, lane l row base + l.  A null, NaN or infinite input is a null 0; a result outside the
// bound is a null 0 and a failure (decimal_utils.cu:1321-1334).
template <class F, int W>
__global__ void __launch_bounds__(kF2dThreads) f2d_kernel(const F* __restrict__ in, const uint32_t* __restrict__ in_mask, int64_t n,
                                                          const F2dParams prm, Rep<W>* __restrict__ out, uint32_t* __restrict__ out_mask,
                                                          unsigned long long* __restrict__ counters)
{
  const int lane = threadIdx.x & 31;
  const __int128 bound = static_cast<__int128>(prm.bound);
  unsigned long long nulls = 0, first = kNoRow;
  const int64_t step = static_cast<int64_t>(gridDim.x) * kF2dThreads;
  for (int64_t base = (static_cast<int64_t>(blockIdx.x) * kF2dThreads + threadIdx.x) & ~int64_t{31}; base < n; base += step) {
    const int64_t row = base + lane;
    const bool live   = row < n;
    const double x    = live ? static_cast<double>(in[row]) : 0.0;
    bool ok           = live && isfinite(x) && (!in_mask || ((__ldg(in_mask + (base >> 5)) >> lane) & 1u));
    __int128 v        = 0;
    if (ok) {
      v = sign_extend<W>(scaled_round<std::is_same<F, float>::value, W>(x, prm));
      if (-bound >= v || v >= bound) {
        ok    = false;
        v     = 0;
        first = tmin<unsigned long long>(first, static_cast<unsigned long long>(row));
      }
    }
    if (live) {
      if constexpr (W == 128) {
        out[2 * row]     = static_cast<uint64_t>(v);
        out[2 * row + 1] = static_cast<uint64_t>(static_cast<u128>(v) >> 64);
      } else {
        out[row] = static_cast<Rep<W>>(v);
      }
    }
    const uint32_t word = __ballot_sync(0xffffffffu, ok);
    nulls += live && !ok;
    if (lane == 0) out_mask[base >> 5] = word;
  }
  flush_counters(nulls, first, counters);
}

unsigned f2d_grid(int64_t rows)
{
  const int64_t blocks = (rows + kF2dThreads - 1) / kF2dThreads;
  return static_cast<unsigned>(tmax<int64_t>(1, tmin<int64_t>(blocks, int64_t{kF2dBlocksSm} * sm_count())));
}

// ipow<Rep, BASE_10>(k) wrapped to `bits`, or the 32-bit helper's switch (0 outside 0..9), on the host
u128 host_pow10(int k, int bits)
{
  if (bits == 32) return k >= 0 && k <= 9 ? dec::make_pow10().w[k][0] : 0;
  if (k < 0) return 10;
  u128 r = 1;
  for (int i = 0; i < k; ++i) r *= 10;
  return bits == 64 ? static_cast<uint64_t>(r) : r;
}

template <class F, int W>
int launch_f2d_t(const srj_column& in, const F2dParams& prm, void* out, uint32_t* out_mask, unsigned long long* counters, cudaStream_t stream)
{
  f2d_kernel<F, W><<<f2d_grid(in.size), kF2dThreads, 0, stream>>>(static_cast<const F*>(in.data), in.null_mask, in.size, prm,
                                                                  static_cast<Rep<W>*>(out), out_mask, counters);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

template <class F>
int launch_f2d_f(const srj_column& in, int w, const F2dParams& prm, void* out, uint32_t* out_mask, unsigned long long* counters, cudaStream_t stream)
{
  if (w == 32) return launch_f2d_t<F, 32>(in, prm, out, out_mask, counters, stream);
  if (w == 64) return launch_f2d_t<F, 64>(in, prm, out, out_mask, counters, stream);
  return launch_f2d_t<F, 128>(in, prm, out, out_mask, counters, stream);
}

}  // namespace

// n > 0 rows of a checked call
static int launch_float_to_decimal(const srj_column& in, int32_t out_type, int32_t precision, int32_t scale, void* out, uint32_t* out_mask,
                                   int64_t* null_count, int64_t* failure_row, cudaStream_t stream)
{
  const int w = 8 * type_width(out_type);
  F2dParams prm{};
  prm.scale_factor = static_cast<double>(host_pow10(-scale, w));   // multiply_power10<IntType>(1, decimal_places)
  prm.max_rep      = w == 32 ? 2147483647.0 : w == 64 ? 9223372036854775808.0 : 170141183460469231731687303715884105728.0;
  prm.bound        = host_pow10(precision, w);
  prm.ten          = dec::make_div(10);
  prm.pow10        = scale;
  unsigned long long* counters = nullptr;
  int rc = counters_reset(&counters, stream);
  if (rc != SRJ_OK) return rc;
  rc = in.type_id == SRJ_FLOAT32 ? launch_f2d_f<float>(in, w, prm, out, out_mask, counters, stream)
                                 : launch_f2d_f<double>(in, w, prm, out, out_mask, counters, stream);
  if (rc != SRJ_OK) return rc;
  return counters_read(counters, null_count, failure_row, stream);
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

// decimal_utils.cu:1384-1417 and DecimalUtilsJni.cpp:118-137; the domain checks are this library's (srj_b200.h)
int srj_float_to_fixed_point(const srj_column* input, int32_t out_type_id, int32_t precision, int32_t scale, void* out, uint32_t* out_mask,
                             int64_t* null_count, int64_t* failure_row, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "floatingPointToDecimal";
  if (!input || !null_count || !failure_row) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *null_count  = 0;
  *failure_row = -1;
  if (input->type_id != SRJ_FLOAT32 && input->type_id != SRJ_FLOAT64) {
    set_error("%s: Unsupported input type %d (FLOAT32 or FLOAT64)", what, input->type_id);
    return SRJ_EUNSUPPORTED;
  }
  if (out_type_id != SRJ_DECIMAL32 && out_type_id != SRJ_DECIMAL64 && out_type_id != SRJ_DECIMAL128) {
    set_error("%s: Unsupported output type %d (DECIMAL32, DECIMAL64 or DECIMAL128)", what, out_type_id);
    return SRJ_EUNSUPPORTED;
  }
  const int max_precision = out_type_id == SRJ_DECIMAL32 ? 9 : out_type_id == SRJ_DECIMAL64 ? 18 : 38;
  if (precision < 1 || precision > max_precision) {
    set_error("%s: precision %d outside 1..%d for the output type", what, precision, max_precision);
    return SRJ_EINVAL;
  }
  if (scale < -precision || scale > 38) {
    set_error("%s: scale %d outside [-precision, 38] (Spark scale -38 .. precision)", what, scale);
    return SRJ_EINVAL;
  }
  if (input->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (input->size == 0) return SRJ_OK;
  int rc;
  if ((rc = check_data(what, "input", *input)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output", out, std::min(type_width(out_type_id), 8))) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output mask", out_mask, 4)) != SRJ_OK) return rc;
  return launch_float_to_decimal(*input, out_type_id, precision, scale, out, out_mask, null_count, failure_row,
                                 static_cast<cudaStream_t>(stream));
}

}  // extern "C"
