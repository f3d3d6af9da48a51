// iceberg.cu -- Iceberg's partition transforms on the device (reference iceberg/iceberg_bucket.cu, iceberg_truncate.cu,
// iceberg_datetime_util.cu): bucket[N], truncate[W] and year / month / day / hour.
//
// bucket: (murmur3_x86_32(bytes, seed 0) & INT32_MAX) % N, standard MurmurHash3 (hash_device.cuh: mm_mix for the 4-byte
// blocks, mm_tail_std for the 1-3 tail bytes).  The bytes are an int widened to 8 little-endian bytes, a long's 8 bytes,
// a decimal's unscaled value as Java's BigInteger.toByteArray() (minimal big-endian two's complement, built in
// registers), or a string's / binary row's bytes.  The % N is mod_v1 with a host-computed reciprocal (reciprocal.cuh).
// truncate[W]: v - (((v % W) + W) % W) in the storage type, wrapping; the % W is a remainder of |v| by |W| through a
// host-computed reciprocal (DECIMAL128: limb by limb), then C's truncated sign rule.  STRING keeps the bytes before the
// (W+1)-th byte that is not a UTF-8 continuation byte; binary keeps min(len, W) bytes.
// year / month / day / hour: floor divisions of microseconds by constant divisors, and the day -> civil-date conversion
// of H. Hinnant's "chrono-Compatible Low-Level Date Algorithms" (days_from_civil's inverse, integer arithmetic, no table).
//
// Fixed-width kernels (ice_map_kernel): a thread owns kIceRows consecutive rows, loaded and stored with 16-byte accesses
// when both buffers are 16-byte aligned; the rows share one mask word.  Bytes kernels: one lane per row, the row's bytes
// read as 4-byte aligned words funnel-shifted to its start (as sha2.cu does); only aligned words holding a byte of the row
// are loaded.
#include <type_traits>

#include "civil_date.cuh"
#include "check.hpp"
#include "common.cuh"
#include "hash_device.cuh"
#include "kernels.hpp"
#include "map_rows.cuh"
#include "reciprocal.cuh"

namespace srj {
namespace {

constexpr int kIceThreads = 256;
constexpr int kIceRows    = kMapRows;
constexpr int kLaneCopy   = 16;   // truncate: rows of up to this many output bytes are copied by their own lane

struct I128 {                     // DECIMAL128 storage: little-endian halves (8-byte alignment suffices)
  uint64_t lo, hi;
};

__device__ __forceinline__ I128 ld_elem(const I128* p)
{
  const auto* q = reinterpret_cast<const unsigned long long*>(p);
  return I128{__ldg(q), __ldg(q + 1)};
}

// ---- bucket ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t bswap32(uint64_t v) { return __byte_perm(static_cast<uint32_t>(v), 0, 0x0123); }   // of the low word

// murmur3 of the n <= 8 bytes of S (little-endian: byte 0 is the first byte hashed)
__device__ __forceinline__ uint32_t mm_le8(uint64_t S, int n)
{
  uint32_t h = 0;
  const uint32_t w0 = static_cast<uint32_t>(S), w1 = static_cast<uint32_t>(S >> 32);
  if (n >= 4) h = hash::mm_mix(h, w0);
  if (n == 8) h = hash::mm_mix(h, w1);
  if (n & 3) h = hash::mm_tail_std(h, n < 4 ? w0 : w1);
  return hash::mm_fmix(h, static_cast<uint32_t>(n));
}

// BigInteger.toByteArray() of a value that fits in 64 bits: n = 1 + (significant bits) / 8 bytes, big-endian.  The byte
// stream is the byte-reversed value shifted down to its last n bytes, so it is hashed straight from registers.
__device__ __forceinline__ uint32_t mm_decimal64(int64_t v)
{
  const uint64_t x = static_cast<uint64_t>(v ^ (v >> 63));             // v < 0 ? ~v : v
  const int n      = (64 - __clzll(static_cast<long long>(x))) / 8 + 1;   // 1 .. 8
  const uint64_t R = (static_cast<uint64_t>(bswap32(static_cast<uint64_t>(v))) << 32) | bswap32(static_cast<uint64_t>(v) >> 32);
  return mm_le8(R >> (64 - 8 * n), n);
}

// the same for DECIMAL128: 1 .. 16 bytes, the stream in four words
__device__ __forceinline__ uint32_t mm_decimal128(I128 v)
{
  const uint64_t s  = static_cast<uint64_t>(static_cast<int64_t>(v.hi) >> 63);
  const uint64_t xh = v.hi ^ s, xl = v.lo ^ s;
  const int lz      = xh ? __clzll(static_cast<long long>(xh)) : 64 + __clzll(static_cast<long long>(xl));
  const int n       = (128 - lz) / 8 + 1;
  // byte-reversed value: Rlo = bswap(hi), Rhi = bswap(lo); the stream is R >> (128 - 8n)
  const uint64_t Rlo = (static_cast<uint64_t>(bswap32(v.hi)) << 32) | bswap32(v.hi >> 32);
  const uint64_t Rhi = (static_cast<uint64_t>(bswap32(v.lo)) << 32) | bswap32(v.lo >> 32);
  const int sh       = 128 - 8 * n;                                      // 0 .. 120, a multiple of 8
  uint64_t Slo, Shi;
  if (sh >= 64) {
    Slo = Rhi >> (sh - 64);
    Shi = 0;
  } else {
    Slo = sh ? (Rlo >> sh) | (Rhi << (64 - sh)) : Rlo;
    Shi = Rhi >> sh;
  }
  const uint32_t w[4] = {static_cast<uint32_t>(Slo), static_cast<uint32_t>(Slo >> 32), static_cast<uint32_t>(Shi),
                         static_cast<uint32_t>(Shi >> 32)};
  uint32_t h = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (4 * k + 4 <= n) h = hash::mm_mix(h, w[k]);
  const int t = n >> 2;                                                  // the tail word, if any
  if (n & 3) h = hash::mm_tail_std(h, t == 0 ? w[0] : t == 1 ? w[1] : t == 2 ? w[2] : w[3]);
  return hash::mm_fmix(h, static_cast<uint32_t>(n));
}

enum BucketKind { kLong32, kLong64, kDec32, kDec64, kDec128 };

template <BucketKind K>
struct BucketOp {
  using In                       = typename std::conditional<K == kLong32 || K == kDec32, int32_t,
                                                             typename std::conditional<K == kDec128, I128, int64_t>::type>::type;
  using Out                      = int32_t;
  static constexpr bool kNullsZero = true;
  uint32_t d, m;                                                         // N and reciprocal_v1(N)
  __device__ __forceinline__ int32_t operator()(In v) const
  {
    uint32_t h;
    if constexpr (K == kDec128) h = mm_decimal128(v);
    else if constexpr (K == kDec32 || K == kDec64) h = mm_decimal64(static_cast<int64_t>(v));
    else h = hash::mm_u64(static_cast<uint64_t>(static_cast<int64_t>(v)), 0u);   // an int is hashed as its long
    return static_cast<int32_t>(mod_v1(h & 0x7fffffffu, d, m));
  }
};

// ---- truncate (integral) --------------------------------------------------------------------------------------------
// r1 = v % W (sign of v), s = r1 + W (wrapping), r2 = s % W, out = v - r2.  |s| < 2|W| always: without wrap-around
// |s| <= |r1| + |W|; an INT32 sum that wraps has |r1 + W| > 2^31 - 1, so |W| > 2^30 and |s| = 2^32 - |r1 + W| <= 2^31.
// So r2 is one compare-subtract on |s|.
template <class U>
__device__ __forceinline__ U second_mod(U s, U d, bool s_neg)
{
  U a = s_neg ? U(0) - s : s;
  a   = a >= d ? a - d : a;
  return s_neg ? U(0) - a : a;
}

struct Trunc32 {
  using In = int32_t;
  using Out = int32_t;
  static constexpr bool kNullsZero = true;
  uint32_t w, d, m;                                                      // W's bits, |W|, reciprocal_v1(|W|)
  __device__ __forceinline__ int32_t operator()(int32_t v) const
  {
    const uint32_t u  = static_cast<uint32_t>(v);
    const uint32_t ra = mod_v1(v < 0 ? 0u - u : u, d, m);
    const uint32_t s  = (v < 0 ? 0u - ra : ra) + w;
    return static_cast<int32_t>(u - second_mod<uint32_t>(s, d, static_cast<int32_t>(s) < 0));
  }
};

struct Trunc64 {
  using In = int64_t;
  using Out = int64_t;
  static constexpr bool kNullsZero = true;
  uint64_t w, d, m;                                                      // W sign-extended, |W|, reciprocal_v2(|W|)
  __device__ __forceinline__ int64_t operator()(int64_t v) const
  {
    const uint64_t u  = static_cast<uint64_t>(v);
    const uint64_t ra = mod_v2(v < 0 ? 0ull - u : u, d, m);
    const uint64_t s  = (v < 0 ? 0ull - ra : ra) + w;
    return static_cast<int64_t>(u - second_mod<uint64_t>(s, d, static_cast<int64_t>(s) < 0));
  }
};

struct Trunc128 {
  using In = I128;
  using Out = I128;
  static constexpr bool kNullsZero = true;
  uint64_t w, d, m;
  __device__ __forceinline__ I128 operator()(I128 v) const
  {
    using U128       = unsigned __int128;
    const U128 u     = (static_cast<U128>(v.hi) << 64) | v.lo;
    const bool neg   = static_cast<int64_t>(v.hi) < 0;
    const U128 a     = neg ? U128(0) - u : u;
    // |v| % |W| limb by limb: each step's dividend (r << 32 | limb) is below |W| * 2^32 <= 2^63
    uint64_t r = 0;
#pragma unroll
    for (int k = 3; k >= 0; --k) r = mod_v2((r << 32) | static_cast<uint32_t>(a >> (32 * k)), d, m);
    const U128 wide = static_cast<U128>(static_cast<__int128>(static_cast<int64_t>(w)));
    const U128 s    = (neg ? U128(0) - U128(r) : U128(r)) + wide;
    const bool sneg = static_cast<int64_t>(static_cast<uint64_t>(s >> 64)) < 0;
    const U128 out  = u - second_mod<U128>(s, d, sneg);
    return I128{static_cast<uint64_t>(out), static_cast<uint64_t>(out >> 64)};
  }
};

// ---- year / month / day / hour ----------------------------------------------------------------------------------------
template <int T, bool kMicros>   // T: SRJ_ICEBERG_YEARS / MONTHS / DAYS / HOURS
struct DateOp {
  using In  = typename std::conditional<kMicros, int64_t, int32_t>::type;
  using Out = int32_t;
  static constexpr bool kNullsZero = false;   // rows under nulls are computed from their bits, as in the reference
  __device__ __forceinline__ int32_t operator()(In v) const
  {
    if constexpr (T == SRJ_ICEBERG_HOURS) return static_cast<int32_t>(floor_div_const<kMicrosPerHour>(v));   // wraps
    const int32_t days = kMicros ? static_cast<int32_t>(floor_div_const<kMicrosPerDay>(v)) : static_cast<int32_t>(v);
    if constexpr (T == SRJ_ICEBERG_DAYS) return days;
    int32_t y, mo;
    civil_year_month(days, &y, &mo);
    if constexpr (T == SRJ_ICEBERG_YEARS) return y - 1970;
    return (y - 1970) * 12 + (mo - 1);
  }
};

// ---- the fixed-width map ---------------------------------------------------------------------------------------------
template <class Op>
__global__ void __launch_bounds__(kIceThreads) ice_map_kernel(const typename Op::In* __restrict__ in, const uint32_t* __restrict__ mask,
                                                              typename Op::Out* __restrict__ out, int64_t n, bool vec, const Op op)
{
  map_rows<kIceThreads>(in, mask, out, n, vec, op);
}

// ---- bytes kernels (STRING / LIST<UINT8>) ------------------------------------------------------------------------------
// standard murmur3 (seed 0) of len bytes at s; four blocks per step so that their loads are in flight together
__device__ __forceinline__ uint32_t mm_row(const uint8_t* s, int32_t len)
{
  const RowWords rw(s, len);
  const int32_t nb = len >> 2;
  uint32_t h = 0, a0 = rw.word(0);
  int32_t k = 0;
  for (; k + 4 <= nb; k += 4) {
    const uint32_t a1 = rw.word(k + 1), a2 = rw.word(k + 2), a3 = rw.word(k + 3), a4 = rw.word(k + 4);
    h  = hash::mm_mix(h, rw.at(a0, a1));
    h  = hash::mm_mix(h, rw.at(a1, a2));
    h  = hash::mm_mix(h, rw.at(a2, a3));
    h  = hash::mm_mix(h, rw.at(a3, a4));
    a0 = a4;
  }
  for (; k < nb; ++k) {
    const uint32_t a1 = rw.word(k + 1);
    h  = hash::mm_mix(h, rw.at(a0, a1));
    a0 = a1;
  }
  const int tail = len & 3;
  if (tail) h = hash::mm_tail_std(h, rw.at(a0, rw.word(nb + 1)) & ((1u << (8 * tail)) - 1u));
  return hash::mm_fmix(h, static_cast<uint32_t>(len));
}

__global__ void __launch_bounds__(kIceThreads) bucket_bytes_kernel(const uint8_t* __restrict__ bytes, const int32_t* __restrict__ off,
                                                                   const uint32_t* __restrict__ mask, int64_t n, uint32_t d, uint32_t m,
                                                                   int32_t* __restrict__ out)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kIceThreads + threadIdx.x;
  if (r >= n) return;
  int32_t res = 0;
  if (!mask || ((__ldg(mask + (r >> 5)) >> (r & 31)) & 1u)) {
    const int32_t beg = __ldg(off + r);
    res = static_cast<int32_t>(mod_v1(mm_row(bytes + beg, __ldg(off + r + 1) - beg) & 0x7fffffffu, d, m));
  }
  out[r] = res;
}

// bytes before the (need)-th byte of s[0, len) that is not a continuation byte 10xxxxxx, or len when there are fewer
__device__ __forceinline__ int32_t utf8_prefix_bytes(const uint8_t* s, int32_t len, int32_t need)
{
  const RowWords rw(s, len);
  uint32_t a0 = rw.word(0);
  for (int32_t k = 0; 4 * k < len; ++k) {
    const uint32_t a1 = rw.word(k + 1);
    const uint32_t t  = (rw.at(a0, a1) & 0xc0c0c0c0u) ^ 0x80808080u;     // a byte of t is 0 iff it is a continuation byte
    uint32_t st       = (t | (t << 1)) & 0x80808080u;                     // bit 7 of each byte that starts a character
    const int32_t nb  = len - 4 * k;
    if (nb < 4) st &= (1u << (8 * nb)) - 1u;
    const int c = __popc(st);
    if (c >= need) {
      for (int i = 1; i < need; ++i) st &= st - 1u;
      return 4 * k + ((__ffs(st) - 1) >> 3);
    }
    need -= c;
    a0 = a1;
  }
  return len;
}

// sizes[r] = the output bytes of row r: 0 for a null row; min(len, width) for binary; for STRING len when len <= width
// (a row of at most width bytes has at most width characters, so its bytes are not read), else the UTF-8 prefix
__global__ void __launch_bounds__(kIceThreads) truncate_sizes_kernel(const uint8_t* __restrict__ bytes, const int32_t* __restrict__ off,
                                                                     const uint32_t* __restrict__ mask, int64_t n, int32_t width, bool utf8,
                                                                     int32_t* __restrict__ sizes)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kIceThreads + threadIdx.x;
  if (r >= n) return;
  int32_t size = 0;
  if (!mask || ((__ldg(mask + (r >> 5)) >> (r & 31)) & 1u)) {
    const int32_t beg = __ldg(off + r);
    const int32_t len = __ldg(off + r + 1) - beg;
    size = len <= width ? len : utf8 ? utf8_prefix_bytes(bytes + beg, len, width + 1) : width;
  }
  sizes[r] = size;
}

// out[out_off[r] ..) = the first out_off[r + 1] - out_off[r] bytes of input row r.  A warp owns 32 rows: each lane copies
// its own row when it is at most kLaneCopy bytes; the warp copies the longer ones together, one after the other.
__global__ void __launch_bounds__(kIceThreads) truncate_copy_kernel(const uint8_t* __restrict__ bytes, const int32_t* __restrict__ in_off,
                                                                    const int32_t* __restrict__ out_off, int64_t n, uint8_t* __restrict__ out)
{
  const int64_t r0 = (static_cast<int64_t>(blockIdx.x) * kIceThreads + threadIdx.x) & ~int64_t{31};
  if (r0 >= n) return;                                         // the whole warp leaves together
  const int lane  = threadIdx.x & 31;
  const int64_t r = r0 + lane;
  const bool live = r < n;
  int32_t src = 0, dst = 0, len = 0;
  if (live) {
    src = __ldg(in_off + r);
    dst = __ldg(out_off + r);
    len = __ldg(out_off + r + 1) - dst;
  }
  if (len <= kLaneCopy) {
    for (int32_t i = 0; i < len; ++i) out[dst + i] = __ldg(bytes + src + i);
  }
  for (uint32_t big = __ballot_sync(0xffffffffu, len > kLaneCopy); big; big &= big - 1u) {
    const int j       = __ffs(big) - 1;
    const int32_t s   = __shfl_sync(0xffffffffu, src, j);
    const int32_t d   = __shfl_sync(0xffffffffu, dst, j);
    const int32_t l   = __shfl_sync(0xffffffffu, len, j);
    for (int32_t i = lane; i < l; i += 32) out[d + i] = __ldg(bytes + s + i);
  }
}

unsigned grid_for(int64_t threads) { return static_cast<unsigned>((threads + kIceThreads - 1) / kIceThreads); }

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <class Op>
int launch_map(const srj_column& in, void* out, const Op& op, cudaStream_t stream)
{
  using In        = typename Op::In;
  using Out       = typename Op::Out;
  const int64_t n = in.size;
  const bool vec  = aligned16(in.data) && aligned16(out);
  ice_map_kernel<Op><<<grid_for((n + kIceRows - 1) / kIceRows), kIceThreads, 0, stream>>>(static_cast<const In*>(in.data), in.null_mask,
                                                                                         static_cast<Out*>(out), n, vec, op);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

int copy_mask(const srj_column& in, uint32_t* out_mask, cudaStream_t stream)
{
  if (!out_mask) return SRJ_OK;
  const size_t bytes = static_cast<size_t>((in.size + 31) / 32) * 4;
  if (in.null_mask) SRJ_CUDA_TRY(cudaMemcpyAsync(out_mask, in.null_mask, bytes, cudaMemcpyDeviceToDevice, stream));
  else SRJ_CUDA_TRY(cudaMemsetAsync(out_mask, 0xff, bytes, stream));
  return SRJ_OK;
}

// the bytes buffer of a STRING (data) or LIST<UINT8> (children[0].data) column
const uint8_t* bytes_of(const srj_column& c)
{
  return static_cast<const uint8_t*>(c.type_id == SRJ_LIST ? c.children[0].data : c.data);
}

}  // namespace

// out_mask (NULL: none) gets a copy of the input's mask, all ones when the input has none.
static int launch_iceberg_bucket(const srj_column& in, int32_t num_buckets, int32_t* out, uint32_t* out_mask, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) return SRJ_OK;
  int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  const uint32_t d = static_cast<uint32_t>(num_buckets), m = reciprocal_v1(d);
  switch (in.type_id) {
    case SRJ_INT32:
    case SRJ_TIMESTAMP_DAYS: return launch_map(in, out, BucketOp<kLong32>{d, m}, stream);
    case SRJ_INT64:
    case SRJ_TIMESTAMP_MICROSECONDS: return launch_map(in, out, BucketOp<kLong64>{d, m}, stream);
    case SRJ_DECIMAL32: return launch_map(in, out, BucketOp<kDec32>{d, m}, stream);
    case SRJ_DECIMAL64: return launch_map(in, out, BucketOp<kDec64>{d, m}, stream);
    case SRJ_DECIMAL128: return launch_map(in, out, BucketOp<kDec128>{d, m}, stream);
    default:   // STRING, LIST<UINT8>
      bucket_bytes_kernel<<<grid_for(n), kIceThreads, 0, stream>>>(bytes_of(in), in.offsets, in.null_mask, n, d, m, out);
      SRJ_CUDA_TRY(cudaGetLastError());
      return SRJ_OK;
  }
}

static int launch_iceberg_truncate_fixed(const srj_column& in, int32_t width, void* out, uint32_t* out_mask, cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  const uint32_t d32 = width < 0 ? 0u - static_cast<uint32_t>(width) : static_cast<uint32_t>(width);   // |W| <= 2^31
  const uint64_t w64 = static_cast<uint64_t>(static_cast<int64_t>(width));
  switch (in.type_id) {
    case SRJ_INT32:
    case SRJ_DECIMAL32: return launch_map(in, out, Trunc32{static_cast<uint32_t>(width), d32, reciprocal_v1(d32)}, stream);
    case SRJ_INT64:
    case SRJ_DECIMAL64: return launch_map(in, out, Trunc64{w64, d32, reciprocal_v2(d32)}, stream);
    default: return launch_map(in, out, Trunc128{w64, d32, reciprocal_v2(d32)}, stream);
  }
}

static int64_t iceberg_truncate_workspace_bytes(int64_t n) { return 4 * tmax<int64_t>(1, i32_scan_nchunks(n)); }

// STRING / LIST<UINT8>: d_offsets[0 .. n] and *h_total (reads the total back: one stream synchronisation)
static int launch_iceberg_truncate_sizes(const srj_column& in, int32_t width, int32_t* d_offsets, int64_t* h_total, void* workspace,
                                  cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(d_offsets, 0, 4, stream));
    *h_total = 0;
    return SRJ_OK;
  }
  truncate_sizes_kernel<<<grid_for(n), kIceThreads, 0, stream>>>(bytes_of(in), in.offsets, in.null_mask, n, width, in.type_id == SRJ_STRING,
                                                                  d_offsets);
  SRJ_CUDA_TRY(cudaGetLastError());
  const int rc = launch_i32_exclusive_scan(d_offsets, n, static_cast<int32_t*>(workspace), d_offsets + n, stream);
  if (rc != SRJ_OK) return rc;
  int32_t total = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(&total, d_offsets + n, 4, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  *h_total = total;
  return SRJ_OK;
}

static int launch_iceberg_truncate_bytes(const srj_column& in, const int32_t* out_offsets, uint8_t* out_bytes, uint32_t* out_mask, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) return SRJ_OK;
  int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  truncate_copy_kernel<<<grid_for(round_up64(n, 32)), kIceThreads, 0, stream>>>(bytes_of(in), in.offsets, out_offsets, n, out_bytes);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_iceberg_datetime(int32_t transform, const srj_column& in, int32_t* out, uint32_t* out_mask, cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  const bool micros = in.type_id == SRJ_TIMESTAMP_MICROSECONDS;
  switch (transform) {
    case SRJ_ICEBERG_YEARS: return micros ? launch_map(in, out, DateOp<SRJ_ICEBERG_YEARS, true>{}, stream)
                                          : launch_map(in, out, DateOp<SRJ_ICEBERG_YEARS, false>{}, stream);
    case SRJ_ICEBERG_MONTHS: return micros ? launch_map(in, out, DateOp<SRJ_ICEBERG_MONTHS, true>{}, stream)
                                           : launch_map(in, out, DateOp<SRJ_ICEBERG_MONTHS, false>{}, stream);
    case SRJ_ICEBERG_DAYS:
      if (micros) return launch_map(in, out, DateOp<SRJ_ICEBERG_DAYS, true>{}, stream);
      SRJ_CUDA_TRY(cudaMemcpyAsync(out, in.data, static_cast<size_t>(in.size) * 4, cudaMemcpyDeviceToDevice, stream));   // a copy
      return SRJ_OK;
    default: return launch_map(in, out, DateOp<SRJ_ICEBERG_HOURS, true>{}, stream);
  }
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

static bool is_binary(const srj_column* c)
{
  return c->type_id == SRJ_LIST && c->num_children >= 1 && c->children && c->children[0].type_id == SRJ_UINT8;
}

// the input's buffers for rows > 0: STRING / LIST offsets, else the data; with check_mask, an input with a mask needs an
// output mask
static int ice_check_buffers(const char* what, const srj_column* in, const uint32_t* out_mask, bool check_mask = true)
{
  if (in->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (in->size == 0) return SRJ_OK;
  const int rc = in->type_id == SRJ_STRING || in->type_id == SRJ_LIST ? check_offsets(what, "input", *in) : check_data(what, "input", *in);
  if (rc != SRJ_OK || !check_mask) return rc;
  return check_out(what, "output mask", out_mask, 1, in->null_mask != nullptr);
}

// iceberg_bucket.cu:393, 411-454
int srj_iceberg_bucket(const srj_column* input, int32_t num_buckets, int32_t* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_bucket";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (num_buckets <= 0) { set_error("%s: num_buckets must be positive", what); return SRJ_EINVAL; }
  switch (input->type_id) {
    case SRJ_INT32: case SRJ_INT64: case SRJ_DECIMAL32: case SRJ_DECIMAL64: case SRJ_DECIMAL128:
    case SRJ_TIMESTAMP_DAYS: case SRJ_TIMESTAMP_MICROSECONDS: case SRJ_STRING: break;
    case SRJ_LIST:
      if (is_binary(input)) break;
      set_error("%s: Binary type must be LIST of UINT8", what);
      return SRJ_EUNSUPPORTED;
    default: set_error("%s: Unsupported type for bucket transform: %d", what, input->type_id); return SRJ_EUNSUPPORTED;
  }
  int rc = ice_check_buffers(what, input, out_mask);
  if (rc != SRJ_OK) return rc;
  if (input->size > 0 && (rc = check_out(what, "output", out, 4)) != SRJ_OK) return rc;
  return launch_iceberg_bucket(*input, num_buckets, out, out_mask, static_cast<cudaStream_t>(stream));
}

static bool truncate_integral(int32_t t)
{
  return t == SRJ_INT32 || t == SRJ_INT64 || t == SRJ_DECIMAL32 || t == SRJ_DECIMAL64 || t == SRJ_DECIMAL128;
}

// iceberg_truncate.cu:174-175, 202-213: STRING or LIST<UINT8> with a non-nullable child, width > 0
static int truncate_bytes_check(const char* what, const srj_column* in, int32_t width)
{
  if (in->type_id != SRJ_STRING && in->type_id != SRJ_LIST) { set_error("%s: Unsupported type for truncation", what); return SRJ_EUNSUPPORTED; }
  if (width <= 0) { set_error("%s: Length must be positive", what); return SRJ_EINVAL; }
  if (in->type_id == SRJ_LIST) {
    if (!is_binary(in)) { set_error("%s: Input must be LIST(UINT8)", what); return SRJ_EUNSUPPORTED; }
    if (in->children[0].null_mask) { set_error("%s: Child column of binary column must be non-nullable", what); return SRJ_EINVAL; }
  }
  return SRJ_OK;
}

int64_t srj_iceberg_truncate_workspace_bytes(int64_t num_rows) { return iceberg_truncate_workspace_bytes(std::max<int64_t>(0, num_rows)); }

int srj_iceberg_truncate_sizes(const srj_column* input, int32_t width, int32_t* d_out_offsets, int64_t* total_bytes, void* workspace,
                               void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_truncate_sizes";
  if (!input || !d_out_offsets || !total_bytes) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  int rc = truncate_bytes_check(what, input, width);
  if (rc != SRJ_OK) return rc;
  if ((rc = ice_check_buffers(what, input, nullptr, false)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output offsets", d_out_offsets, 4)) != SRJ_OK) return rc;
  if (input->size > 0 && !workspace) { set_error("%s: the workspace is needed (srj_iceberg_truncate_workspace_bytes)", what); return SRJ_EINVAL; }
  return launch_iceberg_truncate_sizes(*input, width, d_out_offsets, total_bytes, workspace, static_cast<cudaStream_t>(stream));
}

// iceberg_truncate.cu:146-166 (integral), IcebergTruncateJni.cpp (the type switch)
int srj_iceberg_truncate(const srj_column* input, int32_t width, const srj_column* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_truncate";
  if (!input || !out) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (truncate_integral(input->type_id)) {
    if (width == 0) { set_error("%s: Width must not be zero", what); return SRJ_EINVAL; }
    int rc = ice_check_buffers(what, input, out->null_mask);
    if (rc != SRJ_OK) return rc;
    if (input->size > 0 && (rc = check_out(what, "output data", out->data, std::min(type_width(input->type_id), 8))) != SRJ_OK) return rc;
    return launch_iceberg_truncate_fixed(*input, width, out->data, out->null_mask, s);
  }
  int rc = truncate_bytes_check(what, input, width);
  if (rc != SRJ_OK) return rc;
  if ((rc = ice_check_buffers(what, input, out->null_mask)) != SRJ_OK) return rc;
  if (input->size == 0) return SRJ_OK;
  if (!out->offsets) { set_error("%s: the output needs the offsets of srj_iceberg_truncate_sizes", what); return SRJ_EINVAL; }
  if (input->type_id == SRJ_LIST && (out->num_children < 1 || !out->children)) { set_error("%s: the LIST output needs its UINT8 child", what); return SRJ_EINVAL; }
  uint8_t* bytes = static_cast<uint8_t*>(input->type_id == SRJ_LIST ? out->children[0].data : out->data);
  return launch_iceberg_truncate_bytes(*input, out->offsets, bytes, out->null_mask, s);
}

// iceberg_datetime_util.cu:137-248 and IcebergDateTimeUtil.java's type checks
int srj_iceberg_datetime(int32_t transform, const srj_column* input, int32_t* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_datetime";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (transform < SRJ_ICEBERG_YEARS || transform > SRJ_ICEBERG_HOURS) { set_error("%s: unknown transform %d", what, transform); return SRJ_EINVAL; }
  const bool days = input->type_id == SRJ_TIMESTAMP_DAYS, micros = input->type_id == SRJ_TIMESTAMP_MICROSECONDS;
  if (!micros && !(days && transform != SRJ_ICEBERG_HOURS)) {
    set_error("%s: Input column must be of type TIMESTAMP_MICROSECONDS%s (type id %d)", what, transform == SRJ_ICEBERG_HOURS ? "" : " or TIMESTAMP_DAYS",
              input->type_id);
    return SRJ_EUNSUPPORTED;
  }
  int rc = ice_check_buffers(what, input, out_mask);
  if (rc != SRJ_OK) return rc;
  if (input->size > 0 && (rc = check_out(what, "output", out, 4)) != SRJ_OK) return rc;
  return launch_iceberg_datetime(transform, *input, out, out_mask, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
