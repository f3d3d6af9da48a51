// radix.cu -- integers written as digit strings on the device: Spark's conv() (NumberConverter, reference
// number_converter.cu, a port of Spark 3.5's NumberConverter), bin() (CastStrings.fromLongToBinary,
// cast_long_to_binary_string.cu), hex() / decimal strings of integers (CastStrings.fromIntegersWithBase: cudf's
// from_integers and integers_to_hex, CastStringJni.cpp's leading-zero extract) and hex() of strings and binary
// (CastStrings.bytesToHex, hex.cu).
//
// Every output is a STRING column.  conv, bin and fromIntegersWithBase are sizes -> scan -> write: a sizes kernel writes
// each row's length (0 for a null row), launch_i32_exclusive_scan (partition.cu) turns the lengths into offsets, and a
// write kernel fills each row from its end.  The int32 scan wraps, so each sizes kernel also sums the lengths in 64 bits
// (the workspace's first word, one atomic per warp) and the sizes call returns SRJ_EOVERFLOW when that total passes
// INT32_MAX.  bytesToHex needs no scan: its offsets are twice the input's, rebased to 0, and its chars are a byte -> two
// digit map over the input's whole chars span.
//
// One digit writer (radix_write) serves every base.  Bases 2, 4, 8, 16 and 32 take shifts, their lengths from __clzll.
// Other bases divide through a reciprocal m = floor((2^64 - 1) / b): 2^64 - b * m lies in [1, b], so for any 64-bit x the
// estimate mulhi(x, m) is floor(x / b) or one less (the error x * (2^64 - b * m) / (b * 2^64) is below x / 2^64 < 1), and
// one conditional step corrects quotient and remainder.  This covers values with the top bit set, which reciprocal.cuh's
// remainder-only form leaves out.  Per-row bases read their reciprocal from a 37-entry table.
//
// conv's sizes kernel trims and parses each row once and keeps the final 64-bit value in the workspace; the write kernel
// only emits digits.  A row whose length exceeds its digit count gets the '-' in front.  Its null count and, for
// isConvertOverflow (the same parse under Spark's ANSI rule), the smallest overflowing row leave each CTA through
// row_counters.cuh.  Every kernel is grid-stride with 64-bit indices; conv's output mask words are warp ballots.
#include <type_traits>

#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"
#include "row_counters.cuh"

namespace srj {
namespace {

constexpr int kRadixThreads  = 256;
constexpr int kRadixBlocksSm = 8;   // grid cap per multiprocessor: one full-occupancy wave
constexpr int kMinBase = 2, kMaxBase = 36;

struct Radix {
  uint64_t m;       // floor((2^64 - 1) / b); unused when shift != 0
  uint32_t b;
  uint32_t shift;   // log2(b) for a power of two, else 0
};

struct RadixTable {
  Radix r[kMaxBase + 1];
};

constexpr Radix make_radix(uint32_t b)
{
  uint32_t s = 0;
  while ((1u << s) < b) ++s;
  return Radix{~uint64_t{0} / b, b, (1u << s) == b ? s : 0u};
}

constexpr RadixTable make_radix_table()
{
  RadixTable t{};
  for (uint32_t b = kMinBase; b <= kMaxBase; ++b) t.r[b] = make_radix(b);
  return t;
}

__constant__ RadixTable c_radix = make_radix_table();

// number_converter.cu:55-59
__host__ __device__ __forceinline__ bool bases_ok(int32_t from, int32_t to)
{
  const int64_t ta = to < 0 ? -int64_t{to} : to;
  return from >= kMinBase && from <= kMaxBase && ta >= kMinBase && ta <= kMaxBase;
}

__device__ __forceinline__ bool bit_of(const uint32_t* mask, int64_t row)
{
  return !mask || ((__ldg(mask + (row >> 5)) >> (row & 31)) & 1u);
}

// digits of v in base r.b ("0" for zero)
__device__ __forceinline__ uint32_t radix_len(uint64_t v, const Radix& r)
{
  if (r.shift) {
    const uint32_t bits = 64 - __clzll(static_cast<long long>(v));
    return bits ? (bits + r.shift - 1) / r.shift : 1;
  }
  uint32_t n = 1;
  uint64_t p = r.b;   // b^n
  while (v >= p) {
    ++n;
    if (__umul64hi(p, r.b)) break;   // b^n overflows: v < b^n
    p *= r.b;
  }
  return n;
}

// out[start, end) <- the upper-case digits of v in base r.b, right-aligned at end, and '-' at start when a place is left
__device__ __forceinline__ void radix_write(uint8_t* __restrict__ out, int64_t start, int64_t end, uint64_t v, const Radix& r)
{
  int64_t pos = end;
  do {
    uint32_t d;
    if (r.shift) {
      d = static_cast<uint32_t>(v) & (r.b - 1);
      v >>= r.shift;
    } else {
      uint64_t q   = __umul64hi(v, r.m);
      uint64_t rem = v - q * r.b;
      if (rem >= r.b) {
        ++q;
        rem -= r.b;
      }
      d = static_cast<uint32_t>(rem);
      v = q;
    }
    out[--pos] = static_cast<uint8_t>(d < 10 ? '0' + d : 'A' - 10 + d);
  } while (v);
  if (pos > start) out[start] = '-';
}

// the lengths' 64-bit total: one atomic per warp
__device__ __forceinline__ void flush_total(unsigned long long t, unsigned long long* total)
{
#pragma unroll
  for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0 && t) atomicAdd(total, t);
}

unsigned radix_grid(int64_t rows)
{
  const int64_t blocks = (rows + kRadixThreads - 1) / kRadixThreads;
  return static_cast<unsigned>(tmax<int64_t>(1, tmin<int64_t>(blocks, int64_t{kRadixBlocksSm} * sm_count())));
}

// ---- conv --------------------------------------------------------------------------------------------------------------
struct ConvArgs {
  const uint8_t* chars;      // the input column's chars, or the scalar's bytes
  const int32_t* offsets;    // NULL: every row is the scalar of s_len bytes
  const uint32_t* in_mask;
  const int32_t* from_col;   // NULL: from
  const uint32_t* from_mask;
  const int32_t* to_col;     // NULL: to
  const uint32_t* to_mask;
  int32_t s_len, from, to;
  Radix to_r;                // a scalar `to`'s |to| when in range
};

// number_converter.cu:117-128: the digit's value, 36 or more for a byte that is no digit
__device__ __forceinline__ uint32_t digit_of(uint32_t c)
{
  const uint32_t d = c - '0';
  if (d < 10) return d;
  const uint32_t l = (c | 0x20u) - 'a';
  return l < 26 ? l + 10 : 99u;
}

enum : int { kConvOk = 0, kConvNull = 1, kConvOverflow = 2 };

// number_converter.cu:148-243 (convert): the value the digits are written from, and whether a '-' goes in front.  The
// reference's bound tests (v < 0 before a digit, or v >= (2^64 - 1 - b) / b and (2^64 - 1 - d) / b < v) together say
// v * b + d >= 2^64, which the 128-bit product decides here without a division.
__device__ __forceinline__ int conv_parse(const uint8_t* p, int32_t len, uint32_t fb, int32_t tb, uint64_t& out, bool& minus)
{
  int32_t i = 0;
  while (i < len && p[i] == ' ') ++i;   // trailing spaces end the digits anyway; only the all-space row matters
  if (i == len) return kConvNull;
  const bool neg = p[i] == '-';
  i += neg;
  uint64_t v = 0;
  int rc     = kConvOk;
  for (; i < len; ++i) {
    const uint32_t d = digit_of(p[i]);
    if (d >= fb) break;
    const uint64_t lo = v * fb, nv = lo + d;
    if (__umul64hi(v, fb) | (nv < lo)) {
      rc = kConvOverflow;
      v  = ~uint64_t{0};   // Spark's non-ANSI result: -1
      break;
    }
    v = nv;
  }
  if (neg && tb > 0) v = static_cast<int64_t>(v) < 0 ? ~uint64_t{0} : uint64_t{0} - v;
  minus = false;
  if (tb < 0) {
    minus = neg || static_cast<int64_t>(v) < 0;
    if (static_cast<int64_t>(v) < 0) v = uint64_t{0} - v;
  }
  out = v;
  return rc;
}

// kSizes: lengths, output mask words, kept values, null count and the lengths' total.  Otherwise (isConvertOverflow)
// only the smallest row that overflows.
template <bool kSizes>
__global__ void __launch_bounds__(kRadixThreads) conv_parse_kernel(const ConvArgs a, int64_t n, int32_t* __restrict__ sizes,
                                                                   uint32_t* __restrict__ out_mask, uint64_t* __restrict__ values,
                                                                   unsigned long long* __restrict__ total,
                                                                   unsigned long long* __restrict__ counters)
{
  const int lane = threadIdx.x & 31;
  unsigned long long nulls = 0, first = kNoRow, chars = 0;
  const int64_t step = static_cast<int64_t>(gridDim.x) * kRadixThreads;
  for (int64_t base = (static_cast<int64_t>(blockIdx.x) * kRadixThreads + threadIdx.x) & ~int64_t{31}; base < n; base += step) {
    const int64_t row = base + lane;
    const bool live   = row < n;
    bool ok           = live;
    int32_t fb = a.from, tb = a.to;
    if (ok && a.offsets) ok = bit_of(a.in_mask, row);
    if (ok && a.from_col) {
      ok = bit_of(a.from_mask, row);
      fb = __ldg(a.from_col + row);
    }
    if (ok && a.to_col) {
      ok = bit_of(a.to_mask, row);
      tb = __ldg(a.to_col + row);
    }
    ok = ok && bases_ok(fb, tb);
    int32_t len = 0;
    if (ok) {
      const uint8_t* p = a.chars;
      int32_t sl       = a.s_len;
      if (a.offsets) {
        const int32_t o0 = __ldg(a.offsets + row);
        p += o0;
        sl = __ldg(a.offsets + row + 1) - o0;
      }
      uint64_t v;
      bool minus;
      const int rc = conv_parse(p, sl, static_cast<uint32_t>(fb), tb, v, minus);
      if (rc == kConvNull) {
        ok = false;
      } else if (kSizes) {
        const Radix r = a.to_col ? c_radix.r[tb < 0 ? -tb : tb] : a.to_r;
        len           = static_cast<int32_t>(radix_len(v, r)) + minus;
        values[row]   = v;
      } else if (rc == kConvOverflow) {
        first = tmin<unsigned long long>(first, static_cast<unsigned long long>(row));
      }
    }
    if constexpr (kSizes) {
      if (live) sizes[row] = len;
      const uint32_t word = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) out_mask[base >> 5] = word;
      nulls += live && !ok;
      chars += static_cast<unsigned long long>(len);
    }
  }
  if constexpr (kSizes) flush_total(chars, total);
  flush_counters(nulls, first, counters);
}

__global__ void __launch_bounds__(kRadixThreads) conv_write_kernel(const int32_t* __restrict__ to_col, const Radix to_r, int64_t n,
                                                                   const uint64_t* __restrict__ values, const int32_t* __restrict__ offsets,
                                                                   uint8_t* __restrict__ out)
{
  const int64_t step = static_cast<int64_t>(gridDim.x) * kRadixThreads;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * kRadixThreads + threadIdx.x; row < n; row += step) {
    const int64_t s = __ldg(offsets + row), e = __ldg(offsets + row + 1);
    if (e == s) continue;   // a null row
    if (to_col) {
      const int32_t tb = __ldg(to_col + row);
      radix_write(out, s, e, __ldg(values + row), c_radix.r[tb < 0 ? -tb : tb]);
    } else {
      radix_write(out, s, e, __ldg(values + row), to_r);
    }
  }
}

// ---- bin and fromIntegersWithBase --------------------------------------------------------------------------------------
// the value written and its sign: base 10 writes |v| after a '-'; bases 2 and 16 write the bits of the value's own width
template <class T>
__device__ __forceinline__ uint64_t int_value(T v, bool dec, bool& minus)
{
  using U = typename std::make_unsigned<T>::type;
  minus   = std::is_signed<T>::value && dec && v < 0;
  if (minus) return uint64_t{0} - static_cast<uint64_t>(static_cast<int64_t>(v));
  return static_cast<uint64_t>(static_cast<U>(v));
}

template <class T>
__global__ void __launch_bounds__(kRadixThreads) int_sizes_kernel(const T* __restrict__ in, const uint32_t* __restrict__ in_mask, int64_t n,
                                                                  const Radix r, int32_t* __restrict__ sizes,
                                                                  unsigned long long* __restrict__ total)
{
  unsigned long long chars = 0;
  const int64_t step = static_cast<int64_t>(gridDim.x) * kRadixThreads;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * kRadixThreads + threadIdx.x; row < n; row += step) {
    int32_t len = 0;
    if (bit_of(in_mask, row)) {
      bool minus;
      const uint64_t v = int_value<T>(__ldg(in + row), r.b == 10, minus);
      len              = static_cast<int32_t>(radix_len(v, r)) + minus;
    }
    sizes[row] = len;
    chars += static_cast<unsigned long long>(len);
  }
  flush_total(chars, total);
}

template <class T>
__global__ void __launch_bounds__(kRadixThreads) int_write_kernel(const T* __restrict__ in, int64_t n, const Radix r,
                                                                  const int32_t* __restrict__ offsets, uint8_t* __restrict__ out)
{
  const int64_t step = static_cast<int64_t>(gridDim.x) * kRadixThreads;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * kRadixThreads + threadIdx.x; row < n; row += step) {
    const int64_t s = __ldg(offsets + row), e = __ldg(offsets + row + 1);
    if (e == s) continue;   // a null row
    bool minus;
    radix_write(out, s, e, int_value<T>(__ldg(in + row), r.b == 10, minus), r);
  }
}

// ---- bytesToHex --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRadixThreads) hex_offsets_kernel(const int32_t* __restrict__ in_off, int64_t n, int32_t* __restrict__ out_off)
{
  const int32_t base = __ldg(in_off);
  const int64_t step = static_cast<int64_t>(gridDim.x) * kRadixThreads;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kRadixThreads + threadIdx.x; i <= n; i += step)
    out_off[i] = 2 * (__ldg(in_off + i) - base);
}

__device__ __forceinline__ uint32_t hex_pair(uint32_t b)   // the two digits of byte b, first digit in the low byte
{
  const uint32_t hi = b >> 4, lo = b & 15u;
  return (hi < 10 ? '0' + hi : 'A' - 10 + hi) | ((lo < 10 ? '0' + lo : 'A' - 10 + lo) << 8);
}

// out[0 .. 2 * span) from the input's chars span [in_off[0], in_off[n]): each thread turns 4 bytes into one 8-byte store
// (byte stores when out is not 8-byte aligned, and for the tail)
__global__ void __launch_bounds__(kRadixThreads) hex_chars_kernel(const uint8_t* __restrict__ in, const int32_t* __restrict__ in_off, int64_t n,
                                                                  uint8_t* __restrict__ out, bool vec)
{
  const int64_t first = __ldg(in_off), bytes = __ldg(in_off + n) - first;
  const uint8_t* src  = in + first;
  const int64_t step  = static_cast<int64_t>(gridDim.x) * kRadixThreads;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kRadixThreads + threadIdx.x; 4 * i < bytes; i += step) {
    const int64_t j = 4 * i;
    if (vec && j + 4 <= bytes) {
      const uint32_t lo = hex_pair(__ldg(src + j)) | (hex_pair(__ldg(src + j + 1)) << 16);
      const uint32_t hi = hex_pair(__ldg(src + j + 2)) | (hex_pair(__ldg(src + j + 3)) << 16);
      reinterpret_cast<uint2*>(out)[i] = make_uint2(lo, hi);
    } else {
      for (int64_t k = j; k < j + 4 && k < bytes; ++k) {
        const uint32_t p = hex_pair(__ldg(src + k));
        out[2 * k]       = static_cast<uint8_t>(p);
        out[2 * k + 1]   = static_cast<uint8_t>(p >> 8);
      }
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------------
// the workspace: [0, 8) the lengths' 64-bit total, then (conv) the kept values, then the scan's chunk sums
int64_t scan_ws_bytes(int64_t n) { return 4 * tmax<int64_t>(1, i32_scan_nchunks(n)); }
int64_t conv_ws_bytes(int64_t n) { return 8 + 8 * n + scan_ws_bytes(n); }
int64_t int_ws_bytes(int64_t n) { return 8 + scan_ws_bytes(n); }

// scan the lengths in d_offsets[0 .. n) into offsets, then read the 64-bit total (one synchronisation, with `extra` read
// beside it when given)
int scan_and_total(int32_t* d_offsets, int64_t n, void* ws, int32_t* sums, int64_t* h_total, const unsigned long long* d_extra,
                   unsigned long long* h_extra, cudaStream_t stream)
{
  int rc = launch_i32_exclusive_scan(d_offsets, n, sums, d_offsets + n, stream);
  if (rc != SRJ_OK) return rc;
  unsigned long long t = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(&t, ws, 8, cudaMemcpyDeviceToHost, stream));
  if (d_extra) SRJ_CUDA_TRY(cudaMemcpyAsync(h_extra, d_extra, 16, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  if (t > static_cast<unsigned long long>(INT32_MAX)) {
    set_error("the result's %llu chars exceed the int32 offsets limit", t);
    return SRJ_EOVERFLOW;
  }
  *h_total = static_cast<int64_t>(t);
  return SRJ_OK;
}

}  // namespace

static int launch_conv_sizes(const ConvArgs& a, int64_t n, int32_t* d_offsets, uint32_t* out_mask, int64_t* null_count, int64_t* h_total,
                             void* ws, cudaStream_t stream)
{
  if (!a.from_col && !a.to_col && !bases_ok(a.from, a.to)) {   // number_converter.cu:378-385: every row null
    SRJ_CUDA_TRY(cudaMemsetAsync(d_offsets, 0, static_cast<size_t>(n + 1) * 4, stream));
    SRJ_CUDA_TRY(cudaMemsetAsync(out_mask, 0, static_cast<size_t>((n + 31) / 32) * 4, stream));
    *null_count = n;
    *h_total    = 0;
    return SRJ_OK;
  }
  unsigned long long* counters = nullptr;
  int rc = counters_reset(&counters, stream);
  if (rc != SRJ_OK) return rc;
  auto* total = static_cast<unsigned long long*>(ws);
  SRJ_CUDA_TRY(cudaMemsetAsync(total, 0, 8, stream));
  conv_parse_kernel<true><<<radix_grid(n), kRadixThreads, 0, stream>>>(a, n, d_offsets, out_mask, static_cast<uint64_t*>(ws) + 1, total, counters);
  SRJ_CUDA_TRY(cudaGetLastError());
  unsigned long long h[2];
  rc = scan_and_total(d_offsets, n, ws, reinterpret_cast<int32_t*>(static_cast<uint64_t*>(ws) + 1 + n), h_total, counters, h, stream);
  if (rc != SRJ_OK) return rc;
  *null_count = static_cast<int64_t>(h[0]);
  return SRJ_OK;
}

static int launch_conv_write(const ConvArgs& a, int64_t n, const int32_t* d_offsets, uint8_t* out, const void* ws, cudaStream_t stream)
{
  if (!a.from_col && !a.to_col && !bases_ok(a.from, a.to)) return SRJ_OK;
  conv_write_kernel<<<radix_grid(n), kRadixThreads, 0, stream>>>(a.to_col, a.to_r, n, static_cast<const uint64_t*>(ws) + 1, d_offsets, out);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_conv_overflow(const ConvArgs& a, int64_t n, int32_t* overflow, cudaStream_t stream)
{
  *overflow = 0;
  if (!a.from_col && !a.to_col && !bases_ok(a.from, a.to)) return SRJ_OK;   // number_converter.cu:461-467
  unsigned long long* counters = nullptr;
  int rc = counters_reset(&counters, stream);
  if (rc != SRJ_OK) return rc;
  conv_parse_kernel<false><<<radix_grid(n), kRadixThreads, 0, stream>>>(a, n, nullptr, nullptr, nullptr, nullptr, counters);
  SRJ_CUDA_TRY(cudaGetLastError());
  int64_t row = -1;
  rc = counters_read(counters, nullptr, &row, stream);
  if (rc != SRJ_OK) return rc;
  *overflow = row >= 0;
  return SRJ_OK;
}

template <class T>
static int int_sizes_t(const srj_column& in, const Radix& r, int32_t* d_offsets, void* ws, cudaStream_t stream)
{
  int_sizes_kernel<T><<<radix_grid(in.size), kRadixThreads, 0, stream>>>(static_cast<const T*>(in.data), in.null_mask, in.size, r, d_offsets,
                                                                          static_cast<unsigned long long*>(ws));
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

template <class T>
static int int_write_t(const srj_column& in, const Radix& r, const int32_t* d_offsets, uint8_t* out, cudaStream_t stream)
{
  int_write_kernel<T><<<radix_grid(in.size), kRadixThreads, 0, stream>>>(static_cast<const T*>(in.data), in.size, r, d_offsets, out);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// the integer types of fromIntegersWithBase (bin is INT64 at base 2)
template <template <class> class F, class... Args>
static int int_dispatch(int32_t type_id, Args&&... args)
{
  switch (type_id) {
    case SRJ_INT8: return F<int8_t>::run(args...);
    case SRJ_INT16: return F<int16_t>::run(args...);
    case SRJ_INT32: return F<int32_t>::run(args...);
    case SRJ_INT64: return F<int64_t>::run(args...);
    case SRJ_UINT8: return F<uint8_t>::run(args...);
    case SRJ_UINT16: return F<uint16_t>::run(args...);
    case SRJ_UINT32: return F<uint32_t>::run(args...);
    default: return F<uint64_t>::run(args...);
  }
}

template <class T>
struct IntSizes {
  static int run(const srj_column& in, const Radix& r, int32_t* d, void* ws, cudaStream_t s) { return int_sizes_t<T>(in, r, d, ws, s); }
};
template <class T>
struct IntWrite {
  static int run(const srj_column& in, const Radix& r, const int32_t* d, uint8_t* o, cudaStream_t s) { return int_write_t<T>(in, r, d, o, s); }
};

static int launch_int_sizes(const srj_column& in, uint32_t base, int32_t* d_offsets, int64_t* h_total, void* ws, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(d_offsets, 0, 4, stream));
    *h_total = 0;
    return SRJ_OK;
  }
  SRJ_CUDA_TRY(cudaMemsetAsync(ws, 0, 8, stream));
  int rc = int_dispatch<IntSizes>(in.type_id, in, make_radix(base), d_offsets, ws, stream);
  if (rc != SRJ_OK) return rc;
  return scan_and_total(d_offsets, n, ws, reinterpret_cast<int32_t*>(static_cast<uint64_t*>(ws) + 1), h_total, nullptr, nullptr, stream);
}

static int copy_mask(const srj_column& in, uint32_t* out_mask, cudaStream_t stream)
{
  if (in.null_mask && out_mask && in.size > 0)
    SRJ_CUDA_TRY(cudaMemcpyAsync(out_mask, in.null_mask, static_cast<size_t>((in.size + 31) / 32) * 4, cudaMemcpyDeviceToDevice, stream));
  return SRJ_OK;
}

static int launch_int_write(const srj_column& in, uint32_t base, const srj_column& out, cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  int rc = copy_mask(in, out.null_mask, stream);
  if (rc != SRJ_OK) return rc;
  return int_dispatch<IntWrite>(in.type_id, in, make_radix(base), out.offsets, static_cast<uint8_t*>(out.data), stream);
}

static const uint8_t* hex_input_bytes(const srj_column& c)
{
  return static_cast<const uint8_t*>(c.type_id == SRJ_LIST ? c.children[0].data : c.data);
}

static int launch_hex_sizes(const srj_column& in, int32_t* d_offsets, int64_t* h_total, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(d_offsets, 0, 4, stream));
    *h_total = 0;
    return SRJ_OK;
  }
  int32_t ends[2];
  SRJ_CUDA_TRY(cudaMemcpyAsync(ends, in.offsets, 4, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaMemcpyAsync(ends + 1, in.offsets + n, 4, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  const int64_t chars = 2 * (static_cast<int64_t>(ends[1]) - ends[0]);
  if (chars > INT32_MAX) {
    set_error("bytesToHex: the result's %lld chars exceed the int32 offsets limit", static_cast<long long>(chars));
    return SRJ_EOVERFLOW;
  }
  hex_offsets_kernel<<<radix_grid(n + 1), kRadixThreads, 0, stream>>>(in.offsets, n, d_offsets);
  SRJ_CUDA_TRY(cudaGetLastError());
  *h_total = chars;
  return SRJ_OK;
}

static int launch_hex_write(const srj_column& in, const srj_column& out, cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  int rc = copy_mask(in, out.null_mask, stream);
  if (rc != SRJ_OK) return rc;
  // one thread per 4 input bytes: the grid covers the largest span an int32 offsets column allows, capped per SM
  hex_chars_kernel<<<radix_grid(int64_t{1} << 29), kRadixThreads, 0, stream>>>(hex_input_bytes(in), in.offsets, in.size,
                                                                                static_cast<uint8_t*>(out.data), aligned_to(out.data, 8));
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

// NumberConverter's arguments (number_converter.cu:478-508 and the row count of convert_impl's callers): a STRING input
// column or a valid scalar, INT32 base columns of the input's rows, not three scalars.  *a and *rows on success.
static int conv_args(const char* what, const srj_column* input, const uint8_t* scalar, int32_t scalar_len, const srj_column* from_base,
                     int32_t from, const srj_column* to_base, int32_t to, ConvArgs* a, int64_t* rows)
{
  if (input && input->type_id != SRJ_STRING) { set_error("%s: Input column must be of type STRING", what); return SRJ_EUNSUPPORTED; }
  if (from_base && from_base->type_id != SRJ_INT32) { set_error("%s: From base column must be of type INT32", what); return SRJ_EUNSUPPORTED; }
  if (to_base && to_base->type_id != SRJ_INT32) { set_error("%s: To base column must be of type INT32", what); return SRJ_EUNSUPPORTED; }
  if (!input) {
    if (scalar_len < 0) { set_error("%s: Input scalar must be valid", what); return SRJ_EINVAL; }
    if (scalar_len > 0 && !scalar) { set_error("%s: the input scalar's bytes are missing", what); return SRJ_EINVAL; }
    if (!from_base && !to_base) { set_error("%s: Input is string scalar, from base is int scalar, to base is int scalar", what); return SRJ_EINVAL; }
  }
  const srj_column* lead = input ? input : from_base ? from_base : to_base;
  const int64_t n        = lead->size;
  if (n < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  for (const srj_column* b : {from_base, to_base})
    if (b && b->size != n) {
      set_error("%s: a base column has %lld rows, the input %lld", what, static_cast<long long>(b->size), static_cast<long long>(n));
      return SRJ_EINVAL;
    }
  int rc;
  if (n > 0) {
    if (input && (rc = check_offsets(what, "input", *input)) != SRJ_OK) return rc;
    if (from_base && (rc = check_data(what, "from base", *from_base)) != SRJ_OK) return rc;
    if (to_base && (rc = check_data(what, "to base", *to_base)) != SRJ_OK) return rc;
  }
  *a = ConvArgs{};
  if (input) {
    a->chars   = static_cast<const uint8_t*>(input->data);
    a->offsets = input->offsets;
    a->in_mask = input->null_mask;
  } else {
    a->chars = scalar;
    a->s_len = scalar_len;
  }
  if (from_base) {
    a->from_col  = static_cast<const int32_t*>(from_base->data);
    a->from_mask = from_base->null_mask;
  }
  if (to_base) {
    a->to_col  = static_cast<const int32_t*>(to_base->data);
    a->to_mask = to_base->null_mask;
  }
  a->from = from;
  a->to   = to;
  if (!to_base && bases_ok(kMinBase, to)) a->to_r = make_radix(static_cast<uint32_t>(to < 0 ? -to : to));
  *rows   = n;
  return SRJ_OK;
}

int64_t srj_conv_workspace_bytes(int64_t num_rows) { return conv_ws_bytes(std::max<int64_t>(0, num_rows)); }

int srj_conv_sizes(const srj_column* input, const uint8_t* scalar, int32_t scalar_len, const srj_column* from_base, int32_t from,
                   const srj_column* to_base, int32_t to, int32_t* d_out_offsets, uint32_t* out_mask, int64_t* null_count, int64_t* total_chars,
                   void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "NumberConverter.convert";
  if (!null_count || !total_chars) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *null_count = *total_chars = 0;
  ConvArgs a;
  int64_t n;
  int rc = conv_args(what, input, scalar, scalar_len, from_base, from, to_base, to, &a, &n);
  if (rc != SRJ_OK) return rc;
  if ((rc = check_out(what, "output offsets", d_out_offsets, 4)) != SRJ_OK) return rc;
  if (n == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(d_out_offsets, 0, 4, static_cast<cudaStream_t>(stream)));
    return SRJ_OK;
  }
  if ((rc = check_out(what, "output mask", out_mask, 4)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "workspace", workspace, 8)) != SRJ_OK) return rc;
  return launch_conv_sizes(a, n, d_out_offsets, out_mask, null_count, total_chars, workspace, static_cast<cudaStream_t>(stream));
}

int srj_conv(const srj_column* input, const uint8_t* scalar, int32_t scalar_len, const srj_column* from_base, int32_t from,
             const srj_column* to_base, int32_t to, const int32_t* d_out_offsets, uint8_t* out_chars, const void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "NumberConverter.convert";
  ConvArgs a;
  int64_t n;
  int rc = conv_args(what, input, scalar, scalar_len, from_base, from, to_base, to, &a, &n);
  if (rc != SRJ_OK || n == 0) return rc;
  if ((rc = check_out(what, "output offsets", d_out_offsets, 4)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "workspace", workspace, 8)) != SRJ_OK) return rc;
  return launch_conv_write(a, n, d_out_offsets, out_chars, workspace, static_cast<cudaStream_t>(stream));
}

int srj_conv_overflow(const srj_column* input, const uint8_t* scalar, int32_t scalar_len, const srj_column* from_base, int32_t from,
                      const srj_column* to_base, int32_t to, int32_t* overflow, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "NumberConverter.isConvertOverflow";
  if (!overflow) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *overflow = 0;
  ConvArgs a;
  int64_t n;
  int rc = conv_args(what, input, scalar, scalar_len, from_base, from, to_base, to, &a, &n);
  if (rc != SRJ_OK || n == 0) return rc;
  return launch_conv_overflow(a, n, overflow, static_cast<cudaStream_t>(stream));
}

static bool radix_int_type(int32_t t) { return t >= SRJ_INT8 && t <= SRJ_UINT64; }

// the input of the integer casts: its type, its data, and an output mask when it has a null mask
static int int_input(const char* what, const srj_column* input, bool int64_only)
{
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (int64_only ? input->type_id != SRJ_INT64 : !radix_int_type(input->type_id)) {
    set_error(int64_only ? "%s: Input column must be long type" : "%s: Values for from_integers function must be an integer type.", what);
    return SRJ_EUNSUPPORTED;
  }
  if (input->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  return check_data(what, "input", *input);
}

static int int_sizes_call(const char* what, const srj_column* input, bool int64_only, uint32_t base, int32_t* d_out_offsets, int64_t* total_chars,
                          void* workspace, void* stream)
{
  if (!total_chars) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *total_chars = 0;
  int rc = int_input(what, input, int64_only);
  if (rc != SRJ_OK) return rc;
  if ((rc = check_out(what, "output offsets", d_out_offsets, 4)) != SRJ_OK) return rc;
  if (input->size > 0 && (rc = check_out(what, "workspace", workspace, 8)) != SRJ_OK) return rc;
  return launch_int_sizes(*input, base, d_out_offsets, total_chars, workspace, static_cast<cudaStream_t>(stream));
}

static int int_write_call(const char* what, const srj_column* input, bool int64_only, uint32_t base, const srj_column* out, void* stream)
{
  if (!out) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  int rc = int_input(what, input, int64_only);
  if (rc != SRJ_OK || input->size == 0) return rc;
  if ((rc = check_out(what, "output offsets", out->offsets, 4)) != SRJ_OK) return rc;
  if ((rc = check_out_mask(what, input->null_mask != nullptr, out->null_mask)) != SRJ_OK) return rc;
  return launch_int_write(*input, base, *out, static_cast<cudaStream_t>(stream));
}

// CastStringJni.cpp:263-280: the base is checked before the type
static int int_base(const char* what, int32_t base)
{
  if (base == 10 || base == 16) return SRJ_OK;
  set_error("%s: Bases supported 10, 16; Actual: %d", what, base);
  return SRJ_EINVAL;
}

int64_t srj_long_to_binary_workspace_bytes(int64_t num_rows) { return int_ws_bytes(std::max<int64_t>(0, num_rows)); }

int srj_long_to_binary_sizes(const srj_column* input, int32_t* d_out_offsets, int64_t* total_chars, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  return int_sizes_call("CastStrings.fromLongToBinary", input, true, 2, d_out_offsets, total_chars, workspace, stream);
}

int srj_long_to_binary(const srj_column* input, const srj_column* out, void* stream)
{
  SRJ_API_RANGE();
  return int_write_call("CastStrings.fromLongToBinary", input, true, 2, out, stream);
}

int64_t srj_integers_to_string_workspace_bytes(int64_t num_rows) { return int_ws_bytes(std::max<int64_t>(0, num_rows)); }

int srj_integers_to_string_sizes(const srj_column* input, int32_t base, int32_t* d_out_offsets, int64_t* total_chars, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "CastStrings.fromIntegersWithBase";
  if (total_chars) *total_chars = 0;
  const int rc = int_base(what, base);
  if (rc != SRJ_OK) return rc;
  return int_sizes_call(what, input, false, static_cast<uint32_t>(base), d_out_offsets, total_chars, workspace, stream);
}

int srj_integers_to_string(const srj_column* input, int32_t base, const srj_column* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "CastStrings.fromIntegersWithBase";
  const int rc     = int_base(what, base);
  if (rc != SRJ_OK) return rc;
  return int_write_call(what, input, false, static_cast<uint32_t>(base), out, stream);
}

// CastStringJni.cpp:294-315: STRING, or LIST<UINT8> read as its child's bytes
static int hex_input(const char* what, const srj_column* input)
{
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (input->type_id == SRJ_LIST) {
    if (input->num_children < 1 || !input->children || input->children[0].type_id != SRJ_UINT8) {
      set_error("%s: LIST child must be UINT8 (BinaryType)", what);
      return SRJ_EUNSUPPORTED;
    }
  } else if (input->type_id != SRJ_STRING) {
    set_error("%s: unsupported input type, expected STRING or LIST<UINT8>", what);
    return SRJ_EUNSUPPORTED;
  }
  if (input->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  return input->size > 0 ? check_offsets(what, "input", *input) : SRJ_OK;
}

int srj_bytes_to_hex_sizes(const srj_column* input, int32_t* d_out_offsets, int64_t* total_chars, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "CastStrings.bytesToHex";
  if (!total_chars) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *total_chars = 0;
  int rc = hex_input(what, input);
  if (rc != SRJ_OK) return rc;
  if ((rc = check_out(what, "output offsets", d_out_offsets, 4)) != SRJ_OK) return rc;
  return launch_hex_sizes(*input, d_out_offsets, total_chars, static_cast<cudaStream_t>(stream));
}

int srj_bytes_to_hex(const srj_column* input, const srj_column* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "CastStrings.bytesToHex";
  if (!out) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  int rc = hex_input(what, input);
  if (rc != SRJ_OK || input->size == 0) return rc;
  if ((rc = check_out_mask(what, input->null_mask != nullptr, out->null_mask)) != SRJ_OK) return rc;
  return launch_hex_write(*input, *out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
