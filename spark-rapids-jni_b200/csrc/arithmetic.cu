// arithmetic.cu -- Spark's multiply with ANSI and try overflow handling, and round / bround (HALF_UP / HALF_EVEN) of
// integers, floats and decimals on the device (reference multiply.cu, round_float.cu, and cudf's round/round.cu, which
// round_float.cu calls for every type that is not floating point).
//
// multiply: the exact product decides overflow (INT8 / INT16 in int32, INT32 in int64, INT64 through __mul64hi: the product
// fits when its high word is the sign of its low word).  Default mode wraps; try mode gives a null row; ANSI mode keeps the
// smallest overflowing row with both operands valid.  Floats are __fmul_rn / __dmul_rn in every mode.  A null on either
// side, or a null scalar, gives a null row holding 0.  A scalar's value and validity are read on the device.
// round, floats: the reference's recipe operation for operation, each rounded to nearest with no contraction.  The one
// division, by n = 10^|dp|, is div_n below: two Markstein corrections of e * RN(1 / n), so no division subroutine is called.
// round, integers and decimals: |v| = q * 10^k + r through a host-computed reciprocal (reciprocal.cuh; DECIMAL128: the
// 3-by-2 division of decimal_arith.cuh), then q + 1 when r > 10^k - r, or on a tie under HALF_UP or with q odd under
// HALF_EVEN.  Integers return the exact q * 10^k wrapped to the type, decimals the exact quotient.
//
// Every kernel is grid-stride with 64-bit indices.  A thread owns 16 bytes of consecutive rows per step (one DECIMAL128,
// two INT64, ..., sixteen INT8), loaded and stored with 16-byte accesses when the buffers are 16-byte aligned; the rows
// share one mask word.  mul_kernel assembles each output mask word across the lanes that own it.  The null count and the
// first error row leave each CTA with one atomicAdd and one atomicMin into the two counters of null_counter().
#include <cmath>
#include <cstdlib>
#include <limits>
#include <type_traits>

#include "check.hpp"
#include "common.cuh"
#include "decimal_arith.cuh"
#include "kernels.hpp"
#include "reciprocal.cuh"
#include "row_counters.cuh"

namespace srj {
namespace {

constexpr int kArThreads  = 256;
constexpr int kArBlocksSm = 8;        // grid cap per multiprocessor: one full-occupancy wave

enum MulMode { kMulWrap, kMulTry, kMulAnsi };

struct I128 {                         // DECIMAL128 storage: little-endian halves (8-byte alignment suffices)
  uint64_t lo, hi;
};

// the rows a thread owns per step: 16 bytes
template <class T>
struct Pack {
  static constexpr int V = 16 / sizeof(T);
  union {
    T v[V];
    uint4 u;
  };
};

template <class T>
__device__ __forceinline__ void ld_pack(Pack<T>& p, const T* __restrict__ src, int64_t r0, int cnt, bool vec)
{
  if (vec && cnt == Pack<T>::V) {
    p.u = __ldg(reinterpret_cast<const uint4*>(src + r0));
  } else {
#pragma unroll
    for (int j = 0; j < Pack<T>::V; ++j) p.v[j] = j < cnt ? src[r0 + j] : T{};
  }
}

template <class T>
__device__ __forceinline__ void st_pack(const Pack<T>& p, T* __restrict__ dst, int64_t r0, int cnt, bool vec)
{
  if (vec && cnt == Pack<T>::V) {
    *reinterpret_cast<uint4*>(dst + r0) = p.u;
  } else {
#pragma unroll
    for (int j = 0; j < Pack<T>::V; ++j)
      if (j < cnt) dst[r0 + j] = p.v[j];
  }
}

__device__ __forceinline__ uint32_t low_bits(int cnt) { return cnt >= 32 ? ~0u : (1u << cnt) - 1u; }

// the validity of rows [r0, r0 + cnt) (r0 a multiple of cnt's pack size, which divides 32), bit j for row r0 + j
__device__ __forceinline__ uint32_t valid_bits(const uint32_t* __restrict__ mask, int64_t r0, int cnt)
{
  if (cnt <= 0) return 0;
  if (!mask) return low_bits(cnt);
  return (__ldg(mask + (r0 >> 5)) >> (r0 & 31)) & low_bits(cnt);
}

__device__ __forceinline__ int64_t grid_threads() { return static_cast<int64_t>(gridDim.x) * kArThreads; }
__device__ __forceinline__ int64_t thread_index() { return static_cast<int64_t>(blockIdx.x) * kArThreads + threadIdx.x; }

// ---- multiply -------------------------------------------------------------------------------------------------------
// *r = x * y wrapped; true when the exact product is outside T
__device__ __forceinline__ bool mul_ovf(int8_t x, int8_t y, int8_t* r)
{
  const int32_t p = static_cast<int32_t>(x) * y;
  *r = static_cast<int8_t>(p);
  return p != *r;
}
__device__ __forceinline__ bool mul_ovf(int16_t x, int16_t y, int16_t* r)
{
  const int32_t p = static_cast<int32_t>(x) * y;
  *r = static_cast<int16_t>(p);
  return p != *r;
}
__device__ __forceinline__ bool mul_ovf(int32_t x, int32_t y, int32_t* r)
{
  const int64_t p = static_cast<int64_t>(x) * y;
  *r = static_cast<int32_t>(p);
  return p != *r;
}
__device__ __forceinline__ bool mul_ovf(int64_t x, int64_t y, int64_t* r)
{
  const uint64_t lo = static_cast<uint64_t>(x) * static_cast<uint64_t>(y);
  const int64_t hi  = __mul64hi(static_cast<long long>(x), static_cast<long long>(y));
  *r = static_cast<int64_t>(lo);
  return hi != (static_cast<int64_t>(lo) >> 63);
}
__device__ __forceinline__ bool mul_ovf(float x, float y, float* r)
{
  *r = __fmul_rn(x, y);
  return false;
}
__device__ __forceinline__ bool mul_ovf(double x, double y, double* r)
{
  *r = __dmul_rn(x, y);
  return false;
}

// One warp step covers 32 * V rows: lane l owns rows [base + l * V, + V), and the 32 / V lanes of one mask word OR their
// bits together.  a_valid / b_valid non-NULL: that operand is a scalar (its one value broadcast, validity a device byte).
// counters NULL: neither the null count nor the error row is wanted.
template <class T, int Mode>
__global__ void __launch_bounds__(kArThreads) mul_kernel(const T* __restrict__ a, const uint32_t* __restrict__ a_mask,
                                                         const uint8_t* __restrict__ a_valid, const T* __restrict__ b,
                                                         const uint32_t* __restrict__ b_mask, const uint8_t* __restrict__ b_valid,
                                                         int64_t n, bool vec, T* __restrict__ out, uint32_t* __restrict__ out_mask,
                                                         unsigned long long* __restrict__ counters)
{
  constexpr int V = Pack<T>::V;
  constexpr int G = 32 / V;                                   // lanes per mask word
  const int lane  = threadIdx.x & 31;
  const T sa = a_valid ? a[0] : T{}, sb = b_valid ? b[0] : T{};
  const bool sa_ok = !a_valid || *a_valid, sb_ok = !b_valid || *b_valid;
  unsigned long long nulls = 0, first = kNoRow;
  const int64_t step = grid_threads() * V;                    // rows per grid step (whole warps)
  for (int64_t base = (thread_index() & ~int64_t{31}) * V; base < n; base += step) {
    const int64_t r0 = base + static_cast<int64_t>(lane) * V;
    const int cnt    = static_cast<int>(tmax<int64_t>(0, tmin<int64_t>(V, n - r0)));
    Pack<T> pa, pb, po;
    uint32_t valid = low_bits(cnt);
    if (a_valid) {
#pragma unroll
      for (int j = 0; j < V; ++j) pa.v[j] = sa;
      if (!sa_ok) valid = 0;
    } else {
      ld_pack(pa, a, r0, cnt, vec);
      valid &= valid_bits(a_mask, r0, cnt);
    }
    if (b_valid) {
#pragma unroll
      for (int j = 0; j < V; ++j) pb.v[j] = sb;
      if (!sb_ok) valid = 0;
    } else {
      ld_pack(pb, b, r0, cnt, vec);
      valid &= valid_bits(b_mask, r0, cnt);
    }
#pragma unroll
    for (int j = 0; j < V; ++j) {
      T r;
      const bool ovf = mul_ovf(pa.v[j], pb.v[j], &r);
      const bool ok  = (valid >> j) & 1u;
      if (Mode != kMulWrap && ok && ovf) {
        valid &= ~(1u << j);
        if (Mode == kMulAnsi) first = tmin<unsigned long long>(first, static_cast<unsigned long long>(r0 + j));
      }
      po.v[j] = ((valid >> j) & 1u) ? r : T{};
    }
    st_pack(po, out, r0, cnt, vec);
    nulls += static_cast<unsigned>(cnt - __popc(valid));
    if (out_mask) {
      uint32_t word = valid << ((lane * V) & 31);
#pragma unroll
      for (int o = 1; o < G; o <<= 1) word |= __shfl_xor_sync(0xffffffffu, word, o);
      if (lane % G == 0 && cnt > 0) out_mask[r0 >> 5] = word;
    }
  }
  if (counters) flush_counters(nulls, first, counters);
}

// ---- round: floats --------------------------------------------------------------------------------------------------
__device__ __forceinline__ float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ double fma_rn(double a, double b, double c) { return __fma_rn(a, b, c); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float round_half(float x, bool even) { return even ? rintf(x) : roundf(x); }
__device__ __forceinline__ double round_half(double x, bool even) { return even ? rint(x) : ::round(x); }
__device__ __forceinline__ float modf_t(float x, float* ip) { return modff(x, ip); }
__device__ __forceinline__ double modf_t(double x, double* ip) { return modf(x, ip); }

// RN(e / n) for n = pow(10, k) >= 10 or +inf, y = RN(1 / n).  For finite e and n: q0 = RN(e * y) is within 1.5 ulp of
// e / n, the first correction RN(q0 + (e - q0 n) y) (the remainder exact through the FMA) makes it faithful, and the
// second is correctly rounded (Markstein's theorem: y within half an ulp of 1 / n, the quotient faithful).  From n > 2^126
// (float, dp >= 38) or 2^1022 (double, dp >= 308) y is subnormal and carries fewer bits, so the theorem's premise fails;
// and the dp > 0 branch returns m / n itself (|m| <= n), which is subnormal for m = +-1 (float, dp = 38) and m = +-1, +-2
// (double, dp = 308).  That the result still equals IEEE e / n there is measured, not proved: test_gpu_round_exhaustive.py
// checks every float32 input at every dp, and double quotients at the smallest distance from a rounding midpoint that
// their numerators reach, the subnormal ones included.  The dp < 0 branch rounds its quotient to an integer, where any
// subnormal gives the same +-0.  The sign is e's, as for 0 / n.  e infinite or NaN, or n infinite: e * y is e / n (inf,
// NaN, or +-0 from y = 0).
template <class T>
__device__ __forceinline__ T div_n(T e, T n, T y)
{
  if (!isfinite(e) || isinf(n)) return mul_rn(e, y);
  T q = mul_rn(e, y);
  q   = fma_rn(fma_rn(-q, n, e), y, q);
  q   = fma_rn(fma_rn(-q, n, e), y, q);
  return copysign(q, e);
}

template <class T, bool kEven, int kSign>
struct RoundFloat {
  T n, y;
  __device__ __forceinline__ T operator()(T e) const
  {
    if constexpr (kSign == 0) {
      return round_half(e, kEven);
    } else if constexpr (kSign > 0) {
      T ip;
      const T frac = modf_t(e, &ip);
      return add_rn(ip, div_n(round_half(mul_rn(frac, n), kEven), n, y));
    } else {
      return mul_rn(round_half(div_n(e, n, y), kEven), n);
    }
  }
};

template <class T, bool kEven, int kSign>
__global__ void __launch_bounds__(kArThreads) round_float_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t n, bool vec,
                                                                 const RoundFloat<T, kEven, kSign> op)
{
  constexpr int V = Pack<T>::V;
  for (int64_t r0 = thread_index() * V; r0 < n; r0 += grid_threads() * V) {
    const int cnt = static_cast<int>(tmin<int64_t>(V, n - r0));
    Pack<T> p;
    ld_pack(p, in, r0, cnt, vec);
#pragma unroll
    for (int j = 0; j < V; ++j) p.v[j] = op(p.v[j]);
    st_pack(p, out, r0, cnt, vec);
  }
}

// ---- round: integers and decimals -----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mulhi(uint32_t a, uint32_t b) { return __umulhi(a, b); }
__device__ __forceinline__ uint64_t mulhi(uint64_t a, uint64_t b) { return __umul64hi(a, b); }

// round(x / d) half up or half even, for x <= 2^(N-1) and d <= 2^(N-1) (or, for N = 64, any d > x with m = 1); m is the
// reciprocal of reciprocal.cuh.  r is compared with d - r, so 2r never overflows.
template <class U>
__device__ __forceinline__ U round_quot(U x, U d, U m, bool even)
{
  U q = mulhi(x, m);
  U r = x - q * d;
  if (r >= d) {
    r -= d;
    ++q;
  }
  const U h = d - r;
  if (r > h || (r == h && (!even || (q & 1u)))) ++q;
  return q;
}

template <class T>
struct IntRound {
  using U = typename std::conditional<sizeof(T) == 8, uint64_t, uint32_t>::type;
  U d, m;
  bool even;
};

// dp < 0 on INT8..INT64: the exact q * 10^k (below 2^N, see launch_round) wrapped to T; with counters, the smallest valid
// row whose exact result is outside T goes to counters[1]
template <class T>
__global__ void __launch_bounds__(kArThreads) round_int_kernel(const T* __restrict__ in, const uint32_t* __restrict__ mask, T* __restrict__ out,
                                                               int64_t n, bool vec, const IntRound<T> op, unsigned long long* __restrict__ counters)
{
  using U         = typename IntRound<T>::U;
  constexpr int V = Pack<T>::V;
  constexpr U kMax = static_cast<U>(std::numeric_limits<T>::max());
  unsigned long long first = kNoRow;
  for (int64_t r0 = thread_index() * V; r0 < n; r0 += grid_threads() * V) {
    const int cnt = static_cast<int>(tmin<int64_t>(V, n - r0));
    Pack<T> p;
    ld_pack(p, in, r0, cnt, vec);
    const uint32_t valid = counters ? valid_bits(mask, r0, cnt) : 0u;
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const T v    = p.v[j];
      const bool neg = v < 0;
      const U x    = neg ? U(0) - static_cast<U>(v) : static_cast<U>(v);
      const U mag  = round_quot<U>(x, op.d, op.m, op.even) * op.d;
      if (((valid >> j) & 1u) && mag > kMax + (neg ? 1u : 0u))
        first = tmin<unsigned long long>(first, static_cast<unsigned long long>(r0 + j));
      p.v[j] = static_cast<T>(neg ? U(0) - mag : mag);
    }
    st_pack(p, out, r0, cnt, vec);
  }
  if (counters) flush_counters(0, first, counters);
}

// DECIMAL32 / 64 (T = int32_t / int64_t) and DECIMAL128 (T = I128).  kUp: v * p wrapped (a rescale to a smaller scale,
// p = 10^k mod 2^N); otherwise the exact quotient of |v| by 10^k rounded, with v's sign.
template <class T>
struct DecRound {
  using U = typename std::conditional<sizeof(T) == 4, uint32_t, uint64_t>::type;
  U d, m, p;                        // DECIMAL32 / 64: 10^k, its reciprocal, the scale-up factor
  dec::Div div;                     // DECIMAL128: 10^k as a divisor, and its value
  dec::u128 d128, p128;             // DECIMAL128: 10^k, the scale-up factor
  bool even;
};

template <class T, bool kUp>
__device__ __forceinline__ T dec_round(T v, const DecRound<T>& op)
{
  using U = typename DecRound<T>::U;
  if constexpr (std::is_same<T, I128>::value) {
    const dec::u128 u = (static_cast<dec::u128>(v.hi) << 64) | v.lo;
    dec::u128 r;
    if constexpr (kUp) {
      r = u * op.p128;
    } else {
      const bool neg = static_cast<int64_t>(v.hi) < 0;
      dec::u128 rem;
      const dec::U256 q = dec::udivrem(dec::abs256(dec::sext(u)), op.div, &rem);
      dec::u128 qq      = (static_cast<dec::u128>(q.w[1]) << 64) | q.w[0];
      const dec::u128 h = op.d128 - rem;
      if (rem > h || (rem == h && (!op.even || (qq & 1u)))) ++qq;
      r = neg ? dec::u128(0) - qq : qq;
    }
    return I128{static_cast<uint64_t>(r), static_cast<uint64_t>(r >> 64)};
  } else {
    if constexpr (kUp) return static_cast<T>(static_cast<U>(v) * op.p);
    const bool neg = v < 0;
    const U q      = round_quot<U>(neg ? U(0) - static_cast<U>(v) : static_cast<U>(v), op.d, op.m, op.even);
    return static_cast<T>(neg ? U(0) - q : q);
  }
}

template <class T, bool kUp>
__global__ void __launch_bounds__(kArThreads) round_decimal_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t n, bool vec,
                                                                   const DecRound<T> op)
{
  constexpr int V = Pack<T>::V;
  for (int64_t r0 = thread_index() * V; r0 < n; r0 += grid_threads() * V) {
    const int cnt = static_cast<int>(tmin<int64_t>(V, n - r0));
    Pack<T> p;
    ld_pack(p, in, r0, cnt, vec);
#pragma unroll
    for (int j = 0; j < V; ++j) p.v[j] = dec_round<T, kUp>(p.v[j], op);
    st_pack(p, out, r0, cnt, vec);
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

unsigned grid_for(int64_t rows, int per_thread)
{
  const int64_t blocks = (rows + int64_t{kArThreads} * per_thread - 1) / (int64_t{kArThreads} * per_thread);
  return static_cast<unsigned>(tmax<int64_t>(1, tmin<int64_t>(blocks, int64_t{kArBlocksSm} * sm_count())));
}

int copy_mask(const srj_column& in, uint32_t* out_mask, cudaStream_t stream)
{
  if (!out_mask) return SRJ_OK;
  const size_t bytes = static_cast<size_t>((in.size + 31) / 32) * 4;
  if (in.null_mask) SRJ_CUDA_TRY(cudaMemcpyAsync(out_mask, in.null_mask, bytes, cudaMemcpyDeviceToDevice, stream));
  else SRJ_CUDA_TRY(cudaMemsetAsync(out_mask, 0xff, bytes, stream));
  return SRJ_OK;
}

// 10^k wrapped to N bits (N = 8 * sizeof(U)), by squaring
template <class U>
U pow10_wrapped(int64_t k)
{
  U r = 1, b = 10;
  for (; k > 0; k >>= 1, b *= b)
    if (k & 1) r *= b;
  return r;
}

struct Operand {
  const void* data;
  const uint32_t* mask;
  const uint8_t* scalar_valid;
};

template <class T, int Mode>
int launch_mul_t(const Operand& a, const Operand& b, int64_t n, void* out, uint32_t* out_mask, unsigned long long* counters,
                 cudaStream_t stream)
{
  const bool vec = (a.scalar_valid || aligned16(a.data)) && (b.scalar_valid || aligned16(b.data)) && aligned16(out);
  mul_kernel<T, Mode><<<grid_for(n, Pack<T>::V), kArThreads, 0, stream>>>(
    static_cast<const T*>(a.data), a.mask, a.scalar_valid, static_cast<const T*>(b.data), b.mask, b.scalar_valid, n, vec,
    static_cast<T*>(out), out_mask, counters);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

template <class T>
int launch_mul_mode(int mode, const Operand& a, const Operand& b, int64_t n, void* out, uint32_t* out_mask, unsigned long long* counters,
                    cudaStream_t stream)
{
  if constexpr (std::is_floating_point<T>::value) {
    return launch_mul_t<T, kMulWrap>(a, b, n, out, out_mask, counters, stream);   // floats ignore the mode
  } else {
    if (mode == kMulWrap) return launch_mul_t<T, kMulWrap>(a, b, n, out, out_mask, counters, stream);
    if (mode == kMulTry) return launch_mul_t<T, kMulTry>(a, b, n, out, out_mask, counters, stream);
    return launch_mul_t<T, kMulAnsi>(a, b, n, out, out_mask, counters, stream);
  }
}

}  // namespace

// n rows (n > 0).  need_nulls: count the null rows (the result can hold nulls); need_error: find the first overflow (ANSI
// on an integer type).  Neither: asynchronous, *null_count 0, *error_row -1.
static int launch_multiply(int32_t type_id, const Operand& a, const Operand& b, int64_t n, int mode, bool need_nulls, bool need_error,
                           void* out, uint32_t* out_mask, int64_t* null_count, int64_t* error_row, cudaStream_t stream)
{
  unsigned long long* counters = nullptr;
  if (need_nulls || need_error) {
    const int rc = counters_reset(&counters, stream);
    if (rc != SRJ_OK) return rc;
  }
  int rc = SRJ_OK;
  switch (type_id) {
    case SRJ_INT8: rc = launch_mul_mode<int8_t>(mode, a, b, n, out, out_mask, counters, stream); break;
    case SRJ_INT16: rc = launch_mul_mode<int16_t>(mode, a, b, n, out, out_mask, counters, stream); break;
    case SRJ_INT32: rc = launch_mul_mode<int32_t>(mode, a, b, n, out, out_mask, counters, stream); break;
    case SRJ_INT64: rc = launch_mul_mode<int64_t>(mode, a, b, n, out, out_mask, counters, stream); break;
    case SRJ_FLOAT32: rc = launch_mul_mode<float>(mode, a, b, n, out, out_mask, counters, stream); break;
    default: rc = launch_mul_mode<double>(mode, a, b, n, out, out_mask, counters, stream); break;
  }
  if (rc != SRJ_OK || !counters) return rc;
  return counters_read(counters, need_nulls ? null_count : nullptr, error_row, stream);
}

template <class T, bool kEven, int kSign>
static int launch_round_float_t(const srj_column& in, T n, void* out, cudaStream_t stream)
{
  const RoundFloat<T, kEven, kSign> op{n, static_cast<T>(T(1) / n)};
  round_float_kernel<T, kEven, kSign><<<grid_for(in.size, Pack<T>::V), kArThreads, 0, stream>>>(
    static_cast<const T*>(in.data), static_cast<T*>(out), in.size, aligned16(in.data) && aligned16(out), op);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

template <class T>
static int launch_round_float(const srj_column& in, int32_t dp, bool even, void* out, cudaStream_t stream)
{
  const T n = static_cast<T>(std::pow(10.0, static_cast<double>(std::llabs(static_cast<long long>(dp)))));   // as std::pow computes it
  if (dp == 0) return even ? launch_round_float_t<T, true, 0>(in, n, out, stream) : launch_round_float_t<T, false, 0>(in, n, out, stream);
  if (dp > 0) return even ? launch_round_float_t<T, true, 1>(in, n, out, stream) : launch_round_float_t<T, false, 1>(in, n, out, stream);
  return even ? launch_round_float_t<T, true, -1>(in, n, out, stream) : launch_round_float_t<T, false, -1>(in, n, out, stream);
}

// dp < 0.  k = -dp: when 10^k is above twice the type's largest magnitude every value rounds to 0 (INT8 k >= 3, INT16
// k >= 5, INT32 k >= 10, INT64 k >= 20); INT64 k = 19 rounds to 0 or +-10^19 (wrapped), with d = 10^19 and m = 1.
template <class T>
static int launch_round_int(const srj_column& in, int64_t k, bool even, bool ansi, void* out, int64_t* error_row, cudaStream_t stream)
{
  using U                = typename IntRound<T>::U;
  constexpr int kZeroAt  = sizeof(T) == 1 ? 3 : sizeof(T) == 2 ? 5 : sizeof(T) == 4 ? 10 : 20;
  const int64_t n        = in.size;
  if (k >= kZeroAt) {
    SRJ_CUDA_TRY(cudaMemsetAsync(out, 0, static_cast<size_t>(n) * sizeof(T), stream));
    return SRJ_OK;
  }
  const U d = pow10_wrapped<U>(k);
  const IntRound<T> op{d, sizeof(T) == 8 ? static_cast<U>(reciprocal_v2(d)) : static_cast<U>(reciprocal_v1(static_cast<uint32_t>(d))), even};
  unsigned long long* counters = nullptr;
  if (ansi) {
    const int rc = counters_reset(&counters, stream);
    if (rc != SRJ_OK) return rc;
  }
  round_int_kernel<T><<<grid_for(n, Pack<T>::V), kArThreads, 0, stream>>>(static_cast<const T*>(in.data), in.null_mask, static_cast<T*>(out), n,
                                                                           aligned16(in.data) && aligned16(out), op, counters);
  SRJ_CUDA_TRY(cudaGetLastError());
  if (!ansi) return SRJ_OK;
  return counters_read(counters, nullptr, error_row, stream);
}

template <class T, bool kUp>
static int launch_round_decimal_t(const srj_column& in, const DecRound<T>& op, void* out, cudaStream_t stream)
{
  round_decimal_kernel<T, kUp><<<grid_for(in.size, Pack<T>::V), kArThreads, 0, stream>>>(static_cast<const T*>(in.data), static_cast<T*>(out),
                                                                                        in.size, aligned16(in.data) && aligned16(out), op);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// k = -dp - scale: 0 copies, < 0 rescales up (wrapping), above the type's digits (9 / 18 / 38) zero-fills, else rounds
template <class T>
static int launch_round_decimal(const srj_column& in, int64_t k, bool even, void* out, cudaStream_t stream)
{
  constexpr int kDigits = sizeof(T) == 4 ? 9 : sizeof(T) == 8 ? 18 : 38;
  const size_t bytes    = static_cast<size_t>(in.size) * sizeof(T);
  if (k > kDigits) {
    SRJ_CUDA_TRY(cudaMemsetAsync(out, 0, bytes, stream));
    return SRJ_OK;
  }
  DecRound<T> op{};
  op.even = even;
  using U = typename DecRound<T>::U;
  if (k < 0) {
    if constexpr (std::is_same<T, I128>::value) op.p128 = pow10_wrapped<dec::u128>(-k);
    else op.p = pow10_wrapped<U>(-k);
    return launch_round_decimal_t<T, true>(in, op, out, stream);
  }
  if constexpr (std::is_same<T, I128>::value) {
    op.d128 = pow10_wrapped<dec::u128>(k);
    op.div  = dec::make_div(op.d128);
  } else {
    op.d = pow10_wrapped<U>(k);
    op.m = sizeof(T) == 8 ? static_cast<U>(reciprocal_v2(op.d)) : static_cast<U>(reciprocal_v1(static_cast<uint32_t>(op.d)));
  }
  return launch_round_decimal_t<T, false>(in, op, out, stream);
}

// n > 0 rows; *error_row is set by the integer ANSI path only
static int launch_round(const srj_column& in, int32_t dp, bool even, bool ansi, void* out, uint32_t* out_mask, int64_t* error_row,
                        cudaStream_t stream)
{
  int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  const int64_t k = -static_cast<int64_t>(dp);
  const int w     = type_width(in.type_id);
  switch (in.type_id) {
    case SRJ_FLOAT32: return launch_round_float<float>(in, dp, even, out, stream);
    case SRJ_FLOAT64: return launch_round_float<double>(in, dp, even, out, stream);
    case SRJ_DECIMAL32:
    case SRJ_DECIMAL64:
    case SRJ_DECIMAL128: {
      const int64_t kd = k - in.scale;
      if (kd == 0) break;
      if (in.type_id == SRJ_DECIMAL32) return launch_round_decimal<int32_t>(in, kd, even, out, stream);
      if (in.type_id == SRJ_DECIMAL64) return launch_round_decimal<int64_t>(in, kd, even, out, stream);
      return launch_round_decimal<I128>(in, kd, even, out, stream);
    }
    default:
      if (k <= 0) break;
      if (in.type_id == SRJ_INT8) return launch_round_int<int8_t>(in, k, even, ansi, out, error_row, stream);
      if (in.type_id == SRJ_INT16) return launch_round_int<int16_t>(in, k, even, ansi, out, error_row, stream);
      if (in.type_id == SRJ_INT32) return launch_round_int<int32_t>(in, k, even, ansi, out, error_row, stream);
      return launch_round_int<int64_t>(in, k, even, ansi, out, error_row, stream);
  }
  SRJ_CUDA_TRY(cudaMemcpyAsync(out, in.data, static_cast<size_t>(in.size) * w, cudaMemcpyDeviceToDevice, stream));   // a copy
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

static bool mul_type(int32_t t)
{
  return t == SRJ_INT8 || t == SRJ_INT16 || t == SRJ_INT32 || t == SRJ_INT64 || t == SRJ_FLOAT32 || t == SRJ_FLOAT64;
}

// multiply.cu:38-50 (the checks, in order), ArithmeticJni.cpp:56-58 (two scalars)
int srj_multiply(const srj_column* left, const uint8_t* left_scalar_valid, const srj_column* right, const uint8_t* right_scalar_valid,
                 int32_t is_ansi_mode, int32_t is_try_mode, void* out, uint32_t* out_mask, int64_t* null_count, int64_t* error_row,
                 void* stream)
{
  SRJ_API_RANGE();
  const char* what = "multiply";
  if (!left || !right || !null_count || !error_row) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *null_count = 0;
  *error_row  = -1;
  const bool ls = left_scalar_valid != nullptr, rs = right_scalar_valid != nullptr;
  if (ls && rs) { set_error("%s: Unsupported: Both left and right are scalars", what); return SRJ_EINVAL; }
  if (left->type_id != right->type_id) { set_error("%s: Input columns must have the same data type", what); return SRJ_EINVAL; }
  if (!mul_type(left->type_id)) { set_error("%s: Unsupported data type for multiplication. (type id %d)", what, left->type_id); return SRJ_EUNSUPPORTED; }
  if (!ls && !rs && left->size != right->size) { set_error("%s: Input columns must have the same size", what); return SRJ_EINVAL; }
  if (is_ansi_mode && is_try_mode) { set_error("%s: Cannot enable both ANSI mode and TRY mode at the same time", what); return SRJ_EINVAL; }
  const int64_t n = ls ? right->size : left->size;
  if (n < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (n == 0) return SRJ_OK;
  const int w = type_width(left->type_id);
  int rc;
  srj_column l = *left, r = *right;
  if (ls) l.size = 1, l.null_mask = nullptr;                   // a scalar is its one value; its validity is the device byte
  if (rs) r.size = 1, r.null_mask = nullptr;
  if ((rc = check_data(what, "left", l)) != SRJ_OK || (rc = check_data(what, "right", r)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output", out, w)) != SRJ_OK) return rc;
  const bool integer   = left->type_id != SRJ_FLOAT32 && left->type_id != SRJ_FLOAT64;
  const bool can_null  = ls || rs || l.null_mask || r.null_mask || (is_try_mode && integer);
  if ((rc = check_out(what, "output mask", out_mask, 4, can_null)) != SRJ_OK) return rc;
  const int mode = is_ansi_mode ? kMulAnsi : is_try_mode ? kMulTry : kMulWrap;
  return launch_multiply(left->type_id, Operand{l.data, l.null_mask, left_scalar_valid}, Operand{r.data, r.null_mask, right_scalar_valid}, n, mode,
                         can_null, is_ansi_mode && integer, out, out_mask, null_count, error_row, static_cast<cudaStream_t>(stream));
}

// round_float.cu:306-341 and round/round.cu:397-417
int srj_round(const srj_column* input, int32_t decimal_places, int32_t method, int32_t is_ansi_mode, void* out, uint32_t* out_mask,
              int64_t* error_row, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "round";
  if (!input || !error_row) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *error_row = -1;
  if (input->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (input->size == 0) return SRJ_OK;                        // before any check, as the reference's empty_like
  switch (input->type_id) {
    case SRJ_INT8: case SRJ_INT16: case SRJ_INT32: case SRJ_INT64: case SRJ_FLOAT32: case SRJ_FLOAT64:
    case SRJ_DECIMAL32: case SRJ_DECIMAL64: case SRJ_DECIMAL128: break;
    default: set_error("%s: Only integral/floating point/fixed point currently supported (type id %d)", what, input->type_id); return SRJ_EUNSUPPORTED;
  }
  if (method != SRJ_ROUND_HALF_UP && method != SRJ_ROUND_HALF_EVEN) { set_error("%s: Undefined rounding method %d", what, method); return SRJ_EINVAL; }
  int rc;
  if ((rc = check_data(what, "input", *input)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output", out, std::min(type_width(input->type_id), 8))) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output mask", out_mask, 4, input->null_mask != nullptr)) != SRJ_OK) return rc;
  return launch_round(*input, decimal_places, method == SRJ_ROUND_HALF_EVEN, is_ansi_mode != 0, out, out_mask, error_row,
                      static_cast<cudaStream_t>(stream));
}

}  // extern "C"
