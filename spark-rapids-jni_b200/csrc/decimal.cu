// decimal.cu -- DecimalUtils' DECIMAL128 arithmetic on the device (reference decimal_utils.cu:529-949): multiply (with
// Spark's interim cast to 38 digits), divide, integral divide, remainder, add and subtract, each with the reference's
// HALF_UP rounding and its |result| >= 10^38 overflow flag.
//
// Every row is computed from the bits under it, null or not, in 256-bit two's complement (decimal_arith.cuh), following
// the reference's steps so that its wrap-arounds are kept.  Divisions use a normalised limb division with a 3-by-2
// reciprocal: a per-row divisor's reciprocal is computed in the row; a call's fixed power of ten has its reciprocal
// computed on the host; the multiply's row-dependent powers (10^(precision10 - 38) of the interim cast) come from a
// 39-entry table in shared memory, next to 10^0 .. 10^76 for precision10, which guesses the digit count from the bit
// length and settles it with one compare.
//
// dec_map_kernel: a thread owns kDecRows consecutive rows, loaded with 16-byte accesses when a, b and out are 16-byte
// aligned (8 bytes suffice otherwise); the rows' overflow flags go out as one 4-byte store when that is aligned.
#include <algorithm>
#include <map>
#include <type_traits>

#include "check.hpp"
#include "common.cuh"
#include "decimal_arith.cuh"
#include "kernels.hpp"

namespace srj {
namespace {

using dec::Div;
using dec::Quot;
using dec::U256;
using dec::u128;

constexpr int kDecThreads = 256;
constexpr int kDecRows    = 4;
using dec::kMaxPow;
using dec::PowTable;
using dec::make_pow10;

__constant__ PowTable c_pow10 = make_pow10();
constexpr PowTable h_pow10    = make_pow10();

U256 host_pow(int k) { return U256{{h_pow10.w[k][0], h_pow10.w[k][1], h_pow10.w[k][2], h_pow10.w[k][3]}}; }
Div host_div(int k) { return dec::make_div((static_cast<u128>(h_pow10.w[k][1]) << 64) | h_pow10.w[k][0]); }   // k <= 38

struct Tables {            // the multiply's shared-memory tables
  U256 pow[kMaxPow + 1];   // 10^0 .. 10^76
  Div div[39];             // 10^0 .. 10^38
};

__device__ __forceinline__ u128 lo128(const U256& x) { return (static_cast<u128>(x.w[1]) << 64) | x.w[0]; }
__device__ __forceinline__ bool i128_neg(u128 v) { return static_cast<int64_t>(static_cast<uint64_t>(v >> 64)) < 0; }
__device__ __forceinline__ u128 i128_abs(u128 v) { return i128_neg(v) ? u128(0) - v : v; }

__device__ __forceinline__ bool ge_pow38(const U256& x)   // is_greater_than_decimal_38
{
  const U256 p{{c_pow10.w[38][0], c_pow10.w[38][1], 0, 0}};
  return dec::ge(dec::abs256(x), p);
}

// the reference's precision10 (decimal_utils.cu:512-527): the smallest i in [0, 76] with 10^i >= |x|, else -1.  With L
// the bit length of |x| >= 2, g = ceil((L - 1) log10 2) = floor((L - 1) * 1233 / 4096) + 1 (exact for L <= 256), and
// 10^(g-1) < 2^(L-1) <= |x| < 2^L <= 10^(g+1), so the answer is g or g + 1.
__device__ __forceinline__ int precision10(const U256& x, const U256* pow)
{
  const U256 a = dec::abs256(x);
  const int lz = a.w[3] ? dec::clz64(a.w[3]) : a.w[2] ? 64 + dec::clz64(a.w[2]) : a.w[1] ? 128 + dec::clz64(a.w[1])
               : a.w[0] ? 192 + dec::clz64(a.w[0]) : 256;
  const int L = 256 - lz;
  if (L <= 1) return 0;
  const int g = (((L - 1) * 1233) >> 12) + 1;
  const int i = g > kMaxPow || !dec::ge(pow[g > kMaxPow ? kMaxPow : g], a) ? g + 1 : g;
  return i > kMaxPow ? -1 : i;
}

__device__ __forceinline__ U256 div_round(const U256& n, const Div& D, u128 dmag) { return dec::round_half_up(dec::sdivrem(n, false, D), dmag); }

__device__ __forceinline__ u128 pow_lo(int k) { return (static_cast<u128>(c_pow10.w[k][1]) << 64) | c_pow10.w[k][0]; }

struct Res {
  u128 v;
  bool ovf;
};

// ---- multiply (decimal_utils.cu:667-714) ------------------------------------------------------------------------------
template <bool kCast>
struct MulOp {
  static constexpr bool kTables = true;
  using Out = u128;
  int32_t e0;                  // product_scale - (a_scale + b_scale), clamped to [-40, 38]
  Div d0;                      // 10^e0 when e0 > 0
  __device__ __forceinline__ Res operator()(u128 a, u128 b, const Tables* t) const
  {
    U256 p = dec::mul128(a, b);
    int e  = e0;
    if constexpr (kCast) {
      const int k = precision10(p, t->pow) - 38;                    // <= 38
      if (k > 0) {
        p = div_round(p, t->div[k], pow_lo(k));
        e -= k;
      }
    }
    if (e < 0) {
      if (precision10(p, t->pow) - e > 38) return Res{0, true};     // the reference leaves the value unwritten: 0 here
      p = dec::mul(p, t->pow[-e > kMaxPow ? kMaxPow : -e]);         // -e <= 39 on every row that gets here
    } else if (e > 0) {
      const Div D = e == e0 ? d0 : t->div[e];
      p            = div_round(p, D, pow_lo(e));
    }
    return Res{lo128(p), ge_pow38(p)};
  }
};

// ---- divide / integral divide (decimal_utils.cu:754-833) ----------------------------------------------------------------
// The per-call path is a template parameter, so that each instantiation holds only the code its calls run (and its SASS
// count is that path's instruction count): kPath 0: x > 0, 1: x < -38, 2: -38 <= x <= 0.
template <bool kInt, int kPath>
struct DivOp {
  static constexpr bool kTables = false;
  using Out = typename std::conditional<kInt, uint64_t, u128>::type;
  int32_t x;                   // quot_scale - (a_scale - b_scale), in [-114, 38]
  Div dx;                      // 10^x when x > 0
  U256 m;                      // 10^-x when -38 <= x < 0; 10^(-x - 38) when x < -38
  __device__ __forceinline__ Res operator()(u128 a, u128 b, const Tables*) const
  {
    if (b == 0) return Res{0, true};
    const bool bneg = i128_neg(b);
    const u128 bmag = i128_abs(b);
    const Div D     = dec::make_div(bmag);
    U256 n          = dec::sext(a);
    U256 res;
    if constexpr (kPath == 0) {
      const U256 q1 = dec::sdivrem(n, bneg, D).q;
      const Quot q  = dec::sdivrem(q1, false, dx);
      res           = kInt ? q.q : dec::round_half_up(q, pow_lo(x));
    } else if constexpr (kPath == 1) {
      n               = dec::mul(n, U256{{c_pow10.w[38][0], c_pow10.w[38][1], 0, 0}});
      const Quot q1   = dec::sdivrem(n, bneg, D);
      const bool nneg = dec::is_neg(n);
      const U256 r1   = dec::sext(nneg ? u128(0) - q1.rmag : q1.rmag);
      res             = dec::mul(q1.q, m);
      const U256 sdr  = dec::mul(r1, m);
      Quot q2         = dec::sdivrem(sdr, bneg, D);
      q2.q            = dec::add(res, q2.q);
      res             = kInt ? q2.q : dec::round_half_up(q2, bmag);
    } else {
      if (x < 0) n = dec::mul(n, m);
      const Quot q = dec::sdivrem(n, bneg, D);
      res          = kInt ? q.q : dec::round_half_up(q, bmag);
    }
    return Res{lo128(res), ge_pow38(res)};
  }
};

// ---- remainder (decimal_utils.cu:862-949) -------------------------------------------------------------------------------
template <bool kRoundDivisor, bool kDivideTwice>   // ds > 0; ns > 0
struct RemOp {
  static constexpr bool kTables = false;
  using Out = u128;
  int32_t ds, ns;              // rem_scale - b_scale; the dividend's shift after the divisor's (decimal_utils.cu:890-914)
  Div dds, dns;                // 10^ds when ds > 0, 10^ns when ns > 0
  U256 mns, mds;               // 10^-ns when ns < 0, 10^-ds when ds < 0
  __device__ __forceinline__ Res operator()(u128 a, u128 b, const Tables*) const
  {
    if (b == 0) return Res{0, true};
    const bool nneg = i128_neg(a);
    u128 d          = i128_abs(b);                                 // the reference's abs_d, a signed 128-bit value
    if constexpr (kRoundDivisor) d = lo128(div_round(dec::sext(d), dds, pow_lo(ds)));   // may round to 0
    const bool dneg = i128_neg(d);
    const Div D     = dec::make_div(i128_abs(d));                  // d == 0 divides as the reference's loop does
    U256 n          = dec::abs256(dec::sext(a));
    U256 idr;
    if constexpr (kDivideTwice) {
      const U256 q1 = dec::sdivrem(n, dneg, D).q;
      idr           = dec::sdivrem(q1, false, dns).q;
    } else {
      if (ns < 0) n = dec::mul(n, mns);
      idr = dec::sdivrem(n, dneg, D).q;
    }
    U256 less = dec::mul(idr, dec::sext(d));
    if (!kRoundDivisor && ds < 0) less = dec::mul(less, mds);
    n               = dec::add(n, dec::neg(less));
    const u128 v    = lo128(n);
    return Res{nneg ? u128(0) - v : v, ge_pow38(n)};
  }
};

// ---- add / subtract (decimal_utils.cu:536-588) --------------------------------------------------------------------------
template <bool kSub, int kT>   // the sign of kt
struct AddOp {
  static constexpr bool kTables = false;
  using Out = u128;
  int32_t ka, kb, kt;          // 10^ka scales a, 10^kb scales b up to the common scale; kt < 0: scale up, kt > 0: round
  U256 ma, mb, mt;
  Div dt;
  __device__ __forceinline__ Res operator()(u128 a, u128 b, const Tables*) const
  {
    U256 x = dec::sext(a), y = dec::sext(b);
    if (ka > 0) x = dec::mul(x, ma);
    if (kb > 0) y = dec::mul(y, mb);
    x = dec::add(x, kSub ? dec::neg(y) : y);
    if constexpr (kT < 0) x = dec::mul(x, mt);
    else if constexpr (kT > 0) x = div_round(x, dt, pow_lo(kt));
    return Res{lo128(x), ge_pow38(x)};
  }
};

// ---- the row map --------------------------------------------------------------------------------------------------------
template <class Op>
__global__ void __launch_bounds__(kDecThreads) dec_map_kernel(const uint64_t* __restrict__ a, const uint64_t* __restrict__ b,
                                                              uint8_t* __restrict__ ovf, typename Op::Out* __restrict__ out, int64_t n,
                                                              bool vec, bool ovf_vec, const Op op)
{
  using Out = typename Op::Out;
  const Tables* t = nullptr;
  if constexpr (Op::kTables) {
    __shared__ Tables w;
    for (int i = threadIdx.x; i <= kMaxPow; i += kDecThreads) w.pow[i] = U256{{c_pow10.w[i][0], c_pow10.w[i][1], c_pow10.w[i][2], c_pow10.w[i][3]}};
    if (threadIdx.x < 39) w.div[threadIdx.x] = dec::make_div(pow_lo(threadIdx.x));
    __syncthreads();
    t = &w;
  }
  const int64_t r0 = (static_cast<int64_t>(blockIdx.x) * kDecThreads + threadIdx.x) * kDecRows;
  if (r0 >= n) return;
  const int cnt = static_cast<int>(tmin<int64_t>(kDecRows, n - r0));
  const bool full = cnt == kDecRows;
  uint64_t av[2 * kDecRows], bv[2 * kDecRows];
  if (vec && full) {
#pragma unroll
    for (int i = 0; i < kDecRows; ++i) {
      const ulonglong2 x = __ldg(reinterpret_cast<const ulonglong2*>(a) + r0 + i);
      const ulonglong2 y = __ldg(reinterpret_cast<const ulonglong2*>(b) + r0 + i);
      av[2 * i] = x.x, av[2 * i + 1] = x.y, bv[2 * i] = y.x, bv[2 * i + 1] = y.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 2 * kDecRows; ++i) {
      const bool in = i / 2 < cnt;
      av[i] = in ? __ldg(reinterpret_cast<const unsigned long long*>(a) + 2 * r0 + i) : 0;
      bv[i] = in ? __ldg(reinterpret_cast<const unsigned long long*>(b) + 2 * r0 + i) : 0;
    }
  }
  Out res[kDecRows];
  uint32_t flags = 0;
#pragma unroll
  for (int j = 0; j < kDecRows; ++j) {
    const Res r = op((static_cast<u128>(av[2 * j + 1]) << 64) | av[2 * j], (static_cast<u128>(bv[2 * j + 1]) << 64) | bv[2 * j], t);
    res[j]      = static_cast<Out>(r.v);
    flags |= static_cast<uint32_t>(r.ovf) << (8 * j);
  }
  if (ovf_vec && full) {
    *reinterpret_cast<uint32_t*>(ovf + r0) = flags;
  } else {
    for (int j = 0; j < cnt; ++j) ovf[r0 + j] = static_cast<uint8_t>(flags >> (8 * j));
  }
  if constexpr (sizeof(Out) == 16) {
#pragma unroll
    for (int j = 0; j < kDecRows; ++j) {
      if (j >= cnt) break;
      const ulonglong2 v = make_ulonglong2(static_cast<uint64_t>(res[j]), static_cast<uint64_t>(res[j] >> 64));
      if (vec) reinterpret_cast<ulonglong2*>(out)[r0 + j] = v;
      else {
        reinterpret_cast<uint64_t*>(out)[2 * (r0 + j)]     = v.x;
        reinterpret_cast<uint64_t*>(out)[2 * (r0 + j) + 1] = v.y;
      }
    }
  } else {
    if (vec && full) {
      reinterpret_cast<ulonglong2*>(out + r0)[0] = make_ulonglong2(res[0], res[1]);
      reinterpret_cast<ulonglong2*>(out + r0)[1] = make_ulonglong2(res[2], res[3]);
    } else {
#pragma unroll
      for (int j = 0; j < kDecRows; ++j)
        if (j < cnt) out[r0 + j] = res[j];
    }
  }
}

// out = ma & mb (a NULL mask is all valid); *nulls += the cleared bits among the first n
__global__ void __launch_bounds__(kDecThreads) dec_mask_and_kernel(const uint32_t* __restrict__ ma, const uint32_t* __restrict__ mb,
                                                                   uint32_t* __restrict__ out, int64_t n, unsigned long long* nulls)
{
  const int64_t words = (n + 31) / 32;
  const int64_t i     = static_cast<int64_t>(blockIdx.x) * kDecThreads + threadIdx.x;
  int cleared         = 0;
  if (i < words) {
    const uint32_t w = (ma ? __ldg(ma + i) : ~0u) & (mb ? __ldg(mb + i) : ~0u);
    out[i]           = w;
    const int bits   = static_cast<int>(tmin<int64_t>(32, n - 32 * i));
    cleared          = __popc(~w & (bits == 32 ? ~0u : (1u << bits) - 1u));
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) cleared += __shfl_xor_sync(0xffffffffu, cleared, o);
  if ((threadIdx.x & 31) == 0 && cleared) atomicAdd(nulls, static_cast<unsigned long long>(cleared));
}

unsigned grid_for(int64_t threads) { return static_cast<unsigned>((threads + kDecThreads - 1) / kDecThreads); }

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

template <class Op>
int launch(const srj_column& a, const srj_column& b, uint8_t* ovf, void* out, const Op& op, cudaStream_t stream)
{
  const int64_t n = a.size;
  const bool vec  = aligned(a.data, 16) && aligned(b.data, 16) && aligned(out, 16);
  dec_map_kernel<Op><<<grid_for((n + kDecRows - 1) / kDecRows), kDecThreads, 0, stream>>>(
    static_cast<const uint64_t*>(a.data), static_cast<const uint64_t*>(b.data), ovf, static_cast<typename Op::Out*>(out), n, vec,
    aligned(ovf, 4), op);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

U256 pow_or_one(int k) { return host_pow(k < 0 || k > kMaxPow ? 0 : k); }
Div div_or_one(int k) { return host_div(k < 1 || k > 38 ? 0 : k); }

}  // namespace

// The counters of the calling host thread on the current device (two words: the null count here, and arithmetic.cu's
// first error row beside its null count), allocated once.  A call reads them back before it returns, and one host thread makes one call at a time, so a counter per (thread, device) is never shared by two calls
// in flight.
struct NullCounters {
  std::map<int, unsigned long long*> by_device;
  ~NullCounters()
  {
    for (auto& kv : by_device) cudaFree(kv.second);   // at thread exit; errors ignored (the context may be gone)
  }
};

int null_counter(unsigned long long** out)
{
  thread_local NullCounters counters;
  int dev = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  unsigned long long*& p = counters.by_device[dev];
  if (!p) {
    unsigned long long* q = nullptr;
    SRJ_CUDA_TRY(cudaMalloc(&q, 2 * sizeof(*q)));
    p = q;
  }
  *out = p;
  return SRJ_OK;
}

static int launch_decimal128_binary(int32_t op, const srj_column& a, const srj_column& b, int32_t out_scale, bool interim_cast, uint8_t* ovf,
                             void* out, uint32_t* out_mask, int64_t* null_count, cudaStream_t stream)
{
  const int64_t n = a.size;
  if (null_count) *null_count = 0;
  if (n == 0) return SRJ_OK;
  if (a.null_mask || b.null_mask) {
    unsigned long long* d_nulls = nullptr;
    int rc = null_counter(&d_nulls);
    if (rc != SRJ_OK) return rc;
    unsigned long long h_nulls = 0;
    SRJ_CUDA_TRY(cudaMemsetAsync(d_nulls, 0, sizeof(*d_nulls), stream));
    dec_mask_and_kernel<<<grid_for((n + 31) / 32), kDecThreads, 0, stream>>>(a.null_mask, b.null_mask, out_mask, n, d_nulls);
    SRJ_CUDA_TRY(cudaGetLastError());
    SRJ_CUDA_TRY(cudaMemcpyAsync(&h_nulls, d_nulls, sizeof(h_nulls), cudaMemcpyDeviceToHost, stream));
    SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
    if (null_count) *null_count = static_cast<int64_t>(h_nulls);
  }
  const int64_t sa = a.scale, sb = b.scale, so = out_scale;
  switch (op) {
    case SRJ_DECIMAL_MULTIPLY: {
      // e0 <= 38 (checked).  Below -40 every row takes the early exit (precision10 >= -1, so precision10 - e > 38), as
      // it does at -40 itself; clamping there keeps e0 - k (k <= 38) far from int32's range for any pair of int32 scales.
      const int32_t e0 = static_cast<int32_t>(std::max<int64_t>(so - (sa + sb), -40));
      const Div d0     = div_or_one(e0);
      return interim_cast ? launch(a, b, ovf, out, MulOp<true>{e0, d0}, stream) : launch(a, b, ovf, out, MulOp<false>{e0, d0}, stream);
    }
    case SRJ_DECIMAL_DIVIDE:
    case SRJ_DECIMAL_INTEGER_DIVIDE: {
      const int32_t x = static_cast<int32_t>(so - (sa - sb));
      const U256 m    = pow_or_one(x < -38 ? -x - 38 : -x);
      const Div dx    = div_or_one(x);
      if (op == SRJ_DECIMAL_DIVIDE) {
        if (x > 0) return launch(a, b, ovf, out, DivOp<false, 0>{x, dx, m}, stream);
        if (x < -38) return launch(a, b, ovf, out, DivOp<false, 1>{x, dx, m}, stream);
        return launch(a, b, ovf, out, DivOp<false, 2>{x, dx, m}, stream);
      }
      if (x > 0) return launch(a, b, ovf, out, DivOp<true, 0>{x, dx, m}, stream);
      if (x < -38) return launch(a, b, ovf, out, DivOp<true, 1>{x, dx, m}, stream);
      return launch(a, b, ovf, out, DivOp<true, 2>{x, dx, m}, stream);
    }
    case SRJ_DECIMAL_REMAINDER: {
      const int32_t ds = static_cast<int32_t>(so - sb);
      const int32_t ns = static_cast<int32_t>(ds > 0 ? so - sa : sb - sa);
      const Div dds = div_or_one(ds), dns = div_or_one(ns);
      const U256 mns = pow_or_one(-ns), mds = pow_or_one(-ds);
      if (ds > 0) {
        if (ns > 0) return launch(a, b, ovf, out, RemOp<true, true>{ds, ns, dds, dns, mns, mds}, stream);
        return launch(a, b, ovf, out, RemOp<true, false>{ds, ns, dds, dns, mns, mds}, stream);
      }
      if (ns > 0) return launch(a, b, ovf, out, RemOp<false, true>{ds, ns, dds, dns, mns, mds}, stream);
      return launch(a, b, ovf, out, RemOp<false, false>{ds, ns, dds, dns, mns, mds}, stream);
    }
    default: {
      const int64_t inter = sa < sb ? sa : sb;
      const int32_t ka = static_cast<int32_t>(sa - inter), kb = static_cast<int32_t>(sb - inter), kt = static_cast<int32_t>(so - inter);
      const U256 ma = pow_or_one(ka), mb = pow_or_one(kb), mt = pow_or_one(-kt);
      const Div dt  = div_or_one(kt);
      if (op == SRJ_DECIMAL_ADD) {
        if (kt < 0) return launch(a, b, ovf, out, AddOp<false, -1>{ka, kb, kt, ma, mb, mt, dt}, stream);
        if (kt > 0) return launch(a, b, ovf, out, AddOp<false, 1>{ka, kb, kt, ma, mb, mt, dt}, stream);
        return launch(a, b, ovf, out, AddOp<false, 0>{ka, kb, kt, ma, mb, mt, dt}, stream);
      }
      if (kt < 0) return launch(a, b, ovf, out, AddOp<true, -1>{ka, kb, kt, ma, mb, mt, dt}, stream);
      if (kt > 0) return launch(a, b, ovf, out, AddOp<true, 1>{ka, kb, kt, ma, mb, mt, dt}, stream);
      return launch(a, b, ovf, out, AddOp<true, 0>{ka, kb, kt, ma, mb, mt, dt}, stream);
    }
  }
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

// The scale combinations whose rows would reach pow_ten's CUDF_UNREACHABLE (k > 76) or divide by a truncated
// pow_ten(k).as_128_bits() (k > 38) in the reference, path by path; multiply keeps the reference's own
// check_scale_divisor (decimal_utils.cu:505-510).  Spark's type rules never produce them.
static const char* decimal_scale_error(int32_t op, int64_t sa, int64_t sb, int64_t so)
{
  switch (op) {
    case SRJ_DECIMAL_MULTIPLY: return so - (sa + sb) > 38 ? "divisor too big" : nullptr;
    case SRJ_DECIMAL_DIVIDE:
    case SRJ_DECIMAL_INTEGER_DIVIDE: {
      const int64_t x = so - (sa - sb);                 // > 0: round by 10^x; < -38: 10^38, then 10^(-x - 38)
      return x > 38 || x < -38 - 76 ? "the quotient scale needs a power of ten beyond 10^38 (divisor) or 10^76 (multiplier)" : nullptr;
    }
    case SRJ_DECIMAL_REMAINDER: {
      const int64_t ds = so - sb, ns = ds > 0 ? so - sa : sb - sa;
      return ds > 38 || ds < -76 || ns > 38 || ns < -76 ? "the remainder scale needs a power of ten beyond 10^38 (divisor) or 10^76 (multiplier)"
                                                        : nullptr;
    }
    default: {
      const int64_t inter = std::min(sa, sb), d = sa - sb;
      return d > 76 || d < -76 || inter - so > 76 || so - inter > 38 ? "the intermediate scale needs a power of ten beyond 10^38 (divisor) or 10^76 (multiplier)"
                                                                     : nullptr;
    }
  }
}

// decimal_utils.cu:967-1167 (multiply_decimal128 .. sub_decimal128)
int srj_decimal128_binary(int32_t op, const srj_column* a, const srj_column* b, int32_t out_scale, int32_t interim_cast, uint8_t* overflow,
                          void* out, uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "decimal128_binary";
  if (!a || !b) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (op < SRJ_DECIMAL_MULTIPLY || op > SRJ_DECIMAL_SUBTRACT) { set_error("%s: unknown op %d", what, op); return SRJ_EINVAL; }
  if (a->type_id != SRJ_DECIMAL128 || b->type_id != SRJ_DECIMAL128) { set_error("%s: not a DECIMAL128 column", what); return SRJ_EUNSUPPORTED; }
  if (a->size < 0 || a->size != b->size) { set_error("%s: inputs have mismatched row counts", what); return SRJ_EINVAL; }
  if (const char* e = decimal_scale_error(op, a->scale, b->scale, out_scale)) {
    set_error("%s: scales (%d, %d) -> %d: %s", what, a->scale, b->scale, out_scale, e);
    return SRJ_EINVAL;
  }
  if (a->size == 0) {
    if (null_count) *null_count = 0;
    return SRJ_OK;
  }
  int rc = check_data(what, "first input", *a);
  if (rc == SRJ_OK) rc = check_data(what, "second input", *b);
  if (rc == SRJ_OK) rc = check_out(what, "overflow output", overflow, 1);
  if (rc == SRJ_OK) rc = check_out(what, "result output", out, 8);
  if (rc == SRJ_OK) rc = check_out_mask(what, a->null_mask || b->null_mask, out_mask);
  if (rc != SRJ_OK) return rc;
  if ((a->null_mask || b->null_mask) && !null_count) { set_error("%s: an input has a null mask but no null count was given", what); return SRJ_EINVAL; }
  return launch_decimal128_binary(op, *a, *b, out_scale, interim_cast != 0, overflow, out, out_mask, null_count, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
