// datetime.cu -- Spark's DateTimeUtils on the device (reference datetime_rebase.cu, datetime_truncate.cu): the rebase of
// TIMESTAMP_DAYS / TIMESTAMP_MICROSECONDS values between the proleptic Gregorian and the hybrid Julian calendar, and
// trunc / date_trunc to a year, quarter, month, week, day, hour, minute, second or millisecond.
//
// Every calendar step goes through civil_date.cuh, whose dates keep the year as int16, as cuda::std::chrono::year does in
// the reference: a date outside [-32768, 32767] is rebased and truncated as the date 65536 * k years away (DESIGN 3.6j).
//
// dt_map_kernel: the rebase and the truncation to a format fixed for the call (parsed on the host, a template argument),
// map_rows.cuh's body: 4 rows per thread, 16-byte loads and stores when aligned.  dt_trunc_format_kernel: one lane per
// row of a STRING format column; the row's <= 11 bytes are read as aligned words funnel-shifted to its start, upper-cased
// a word at a time and compared with the 15 format names packed into words.  The lane writes the value, its warp the mask
// word (a ballot), its block one atomic add of the valid rows.
#include <type_traits>

#include "civil_date.cuh"
#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"
#include "map_rows.cuh"

namespace srj {

// Truncation formats, in the reference's order of families; TIMESTAMP_DAYS accepts kDtYear .. kDtWeek.
enum DtFormat : int32_t {
  kDtYear, kDtQuarter, kDtMonth, kDtWeek, kDtDay, kDtHour, kDtMinute, kDtSecond, kDtMillisecond, kDtMicrosecond, kDtInvalid
};

// ---- formats ------------------------------------------------------------------------------------------------------------
namespace {

struct FmtKey {
  int32_t len;
  uint32_t w0, w1, w2;       // the upper-case name, little-endian, zero-padded to 12 bytes
  int32_t fmt;
};

constexpr uint32_t pack4(const char* s, int32_t len, int32_t at)
{
  uint32_t w = 0;
  for (int32_t i = 3; i >= 0; --i) w = (w << 8) | (at + i < len ? static_cast<uint8_t>(s[at + i]) : 0u);
  return w;
}

#define DT_KEY(name, fmt) FmtKey{sizeof(name) - 1, pack4(name, sizeof(name) - 1, 0), pack4(name, sizeof(name) - 1, 4), pack4(name, sizeof(name) - 1, 8), fmt}

// ASCII a-z to A-Z in each byte of w; every other byte, including those >= 0x80, is kept
__host__ __device__ __forceinline__ uint32_t ascii_upper4(uint32_t w)
{
  const uint32_t t  = w & 0x7f7f7f7fu;
  const uint32_t ge = t + 0x1f1f1f1fu;                       // bit 7 set where t >= 'a' (no carry: t <= 0x7f)
  const uint32_t gt = t + 0x05050505u;                       // bit 7 set where t > 'z'
  return w ^ ((ge & ~gt & ~w & 0x80808080u) >> 2);           // 0x80 >> 2 = 0x20
}

// the format of an upper-cased name of len bytes held in w0..w2 (bytes past len zero), kDtInvalid when none
__host__ __device__ __forceinline__ int32_t parse_format_words(int32_t len, uint32_t w0, uint32_t w1, uint32_t w2)
{
  constexpr FmtKey kKeys[] = {DT_KEY("YEAR", kDtYear),     DT_KEY("YYYY", kDtYear),        DT_KEY("YY", kDtYear),
                              DT_KEY("QUARTER", kDtQuarter), DT_KEY("MONTH", kDtMonth),    DT_KEY("MM", kDtMonth),
                              DT_KEY("MON", kDtMonth),     DT_KEY("WEEK", kDtWeek),        DT_KEY("DAY", kDtDay),
                              DT_KEY("DD", kDtDay),        DT_KEY("HOUR", kDtHour),        DT_KEY("MINUTE", kDtMinute),
                              DT_KEY("SECOND", kDtSecond), DT_KEY("MILLISECOND", kDtMillisecond),
                              DT_KEY("MICROSECOND", kDtMicrosecond)};
  int32_t f = kDtInvalid;
#pragma unroll
  for (int i = 0; i < static_cast<int>(sizeof(kKeys) / sizeof(kKeys[0])); ++i)
    if (len == kKeys[i].len && w0 == kKeys[i].w0 && w1 == kKeys[i].w1 && w2 == kKeys[i].w2) f = kKeys[i].fmt;
  return f;
}

#undef DT_KEY

// TIMESTAMP_DAYS truncates only to a year, quarter, month or week
__host__ __device__ __forceinline__ bool format_fits(int32_t fmt, bool micros)
{
  return fmt != kDtInvalid && (micros || fmt <= kDtWeek);
}

}  // namespace

// the format named by len bytes at s (ASCII case-insensitive), kDtInvalid when none
static int32_t datetime_parse_format(const char* s, int32_t len)
{
  if (len < 2 || len > 11) return kDtInvalid;
  uint32_t w[3] = {0, 0, 0};
  for (int32_t i = 0; i < len; ++i) w[i >> 2] |= static_cast<uint32_t>(static_cast<uint8_t>(s[i])) << (8 * (i & 3));
  return parse_format_words(len, ascii_upper4(w[0]), ascii_upper4(w[1]), ascii_upper4(w[2]));
}

namespace {

constexpr int kDtThreads          = 256;
constexpr int32_t kGregorianStart = -141427;                       // 1582-10-15, the first day of the Gregorian calendar
constexpr int64_t kGregorianStartMicros = -12219292800000000ll;    // 1582-10-15T00:00:00Z
constexpr int32_t kJulianEndKey   = 1582 * 512 + 10 * 32 + 4;      // ymd_key(1582, 10, 4)
constexpr int32_t kGregStartKey   = 1582 * 512 + 10 * 32 + 15;     // ymd_key(1582, 10, 15)

// ---- rebase -------------------------------------------------------------------------------------------------------------
// Gregorian -> Julian of a day: its Gregorian y/m/d read as a Julian date; a date in the ten days the switch skipped
// (1582-10-05 .. 14) maps to the switch day.  kKeepLate: a date on or after 1582-10-15 is returned unchanged (the days
// path; the micros path has already returned those rows, and runs days_from_julian for any other, as the reference does).
template <bool kKeepLate>
__device__ __forceinline__ int32_t g2j_day(int32_t days)
{
  const Ymd16 ymd   = civil_from_days16(days);
  const int32_t key = ymd_key(ymd.y, ymd.m, ymd.d);
  if (key > kJulianEndKey && key < kGregStartKey) return kGregorianStart;
  if (kKeepLate && key >= kGregStartKey) return days;
  return days_from_julian(ymd.y, ymd.m, ymd.d);
}

__device__ __forceinline__ int32_t j2g_day(int32_t days)
{
  const Ymd16 ymd = julian_from_days16(days);
  return days_from_civil(ymd.y, ymd.m, ymd.d);
}

// the day reattached to the time of day, wrapping in int64 as the reference's arithmetic does
__device__ __forceinline__ int64_t at_day(int32_t days, int64_t tod)
{
  return static_cast<int64_t>(static_cast<uint64_t>(static_cast<int64_t>(days)) * static_cast<uint64_t>(kMicrosPerDay) +
                              static_cast<uint64_t>(tod));
}

template <int kDir, bool kMicros>   // kDir: SRJ_DATETIME_GREGORIAN_TO_JULIAN / JULIAN_TO_GREGORIAN
struct RebaseOp {
  using In                       = typename std::conditional<kMicros, int64_t, int32_t>::type;
  using Out                      = In;
  static constexpr bool kNullsZero = false;   // rows under nulls are computed from their bits, as in the reference
  __device__ __forceinline__ In operator()(In v) const
  {
    if constexpr (kMicros) {
      if (v >= kGregorianStartMicros) return v;
      const int64_t days = floor_div_const<kMicrosPerDay>(v);
      const int64_t tod  = v - days * kMicrosPerDay;
      const int32_t d    = static_cast<int32_t>(days);
      return at_day(kDir == SRJ_DATETIME_GREGORIAN_TO_JULIAN ? g2j_day<false>(d) : j2g_day(d), tod);
    } else {
      if (kDir == SRJ_DATETIME_GREGORIAN_TO_JULIAN) return g2j_day<true>(v);
      return v >= kGregorianStart ? v : j2g_day(v);
    }
  }
};

// ---- truncation ---------------------------------------------------------------------------------------------------------
// the first day of the year / quarter / month (fmt kDtYear .. kDtMonth) or the Monday on or before (kDtWeek) of a day
__device__ __forceinline__ int32_t trunc_day(int32_t days, int32_t fmt)
{
  if (fmt == kDtWeek) {
    // 1970-01-01 was a Thursday: (days + 3) mod 7 days since the Monday.  64-bit, so the largest days are defined too;
    // the difference wraps in int32, as the reference's does
    const int64_t since = static_cast<int64_t>(days) + 3 - 7 * floor_div_const<7>(static_cast<int64_t>(days) + 3);
    return static_cast<int32_t>(static_cast<uint32_t>(days) - static_cast<uint32_t>(since));
  }
  const Ymd16 ymd = civil_from_days16(days);
  const uint32_t m = fmt == kDtYear ? 1u : fmt == kDtQuarter ? (ymd.m - 1) / 3 * 3 + 1 : ymd.m;
  return days_from_civil(ymd.y, m, 1);
}

template <bool kMicros>
__device__ __forceinline__ typename std::conditional<kMicros, int64_t, int32_t>::type trunc_value(
  typename std::conditional<kMicros, int64_t, int32_t>::type v, int32_t fmt)
{
  if constexpr (!kMicros) {
    return trunc_day(v, fmt);
  } else {
    if (fmt == kDtMicrosecond) return v;
    const int64_t days64 = floor_div_const<kMicrosPerDay>(v);
    const int32_t days   = static_cast<int32_t>(days64);
    if (fmt <= kDtWeek) return at_day(trunc_day(days, fmt), 0);
    const int64_t tod = v - days64 * kMicrosPerDay;                   // [0, 86400e6)
    // DAY .. MILLISECOND rebuild the day from its y/m/d, so they carry the int16 year too
    const Ymd16 ymd   = civil_from_days16(days);
    const int32_t day = days_from_civil(ymd.y, ymd.m, ymd.d);
    int64_t kept;
    switch (fmt) {
      case kDtDay: kept = 0; break;
      case kDtHour: kept = tod / kMicrosPerHour * kMicrosPerHour; break;
      case kDtMinute: kept = tod / 60000000 * 60000000; break;
      case kDtSecond: kept = tod / 1000000 * 1000000; break;
      default: kept = tod / 1000 * 1000; break;                       // MILLISECOND
    }
    return at_day(day, kept);
  }
}

template <int kFmt, bool kMicros>
struct TruncOp {
  using In                       = typename std::conditional<kMicros, int64_t, int32_t>::type;
  using Out                      = In;
  static constexpr bool kNullsZero = true;    // a null row holds 0, as the reference writes for it
  __device__ __forceinline__ In operator()(In v) const { return trunc_value<kMicros>(v, kFmt); }
};

template <class Op>
__global__ void __launch_bounds__(kDtThreads) dt_map_kernel(const typename Op::In* __restrict__ in, const uint32_t* __restrict__ mask,
                                                            typename Op::Out* __restrict__ out, int64_t n, bool vec, const Op op)
{
  map_rows<kDtThreads>(in, mask, out, n, vec, op);
}

__device__ __forceinline__ bool bit_of(const uint32_t* m, int64_t i) { return !m || ((__ldg(m + (i >> 5)) >> (i & 31)) & 1u); }

// One lane per output row r.  The datetime row is r, or 0 when broadcast.  A row is valid when its datetime and its
// format are, and the format parses to one that fits the type; an invalid row holds 0.  out_mask gets one ballot word per
// warp; *valid_rows the count of valid rows.
template <bool kMicros>
__global__ void __launch_bounds__(kDtThreads) dt_trunc_format_kernel(const typename std::conditional<kMicros, int64_t, int32_t>::type* __restrict__ dt,
                                                                     const uint32_t* __restrict__ dt_mask, bool broadcast,
                                                                     const uint8_t* __restrict__ chars, const int32_t* __restrict__ off,
                                                                     const uint32_t* __restrict__ fmt_mask, int64_t n,
                                                                     typename std::conditional<kMicros, int64_t, int32_t>::type* __restrict__ out,
                                                                     uint32_t* __restrict__ out_mask, unsigned long long* __restrict__ valid_rows)
{
  using T         = typename std::conditional<kMicros, int64_t, int32_t>::type;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kDtThreads + threadIdx.x;
  bool ok         = false;
  T res           = 0;
  if (r < n) {
    const int64_t i = broadcast ? 0 : r;
    if (bit_of(dt_mask, i) && bit_of(fmt_mask, r)) {
      const int32_t beg = __ldg(off + r);
      const int32_t len = __ldg(off + r + 1) - beg;
      int32_t fmt       = kDtInvalid;
      if (len >= 2 && len <= 11) {
        const RowWords rw(chars + beg, len);
        const uint32_t a0 = rw.word(0), a1 = rw.word(1), a2 = rw.word(2), a3 = rw.word(3);
        // bytes past len are zeroed: word k keeps min(4, len - 4k) bytes (len >= 2, so word 0 keeps at least 2)
        const uint32_t m0 = len >= 4 ? ~0u : (1u << (8 * len)) - 1u;
        const uint32_t m1 = len >= 8 ? ~0u : len <= 4 ? 0u : (1u << (8 * (len - 4))) - 1u;
        const uint32_t m2 = len <= 8 ? 0u : (1u << (8 * (len - 8))) - 1u;   // len <= 11
        fmt = parse_format_words(len, ascii_upper4(rw.at(a0, a1) & m0), ascii_upper4(rw.at(a1, a2) & m1), ascii_upper4(rw.at(a2, a3) & m2));
      }
      if (format_fits(fmt, kMicros)) {
        ok  = true;
        res = trunc_value<kMicros>(ld_elem(dt + i), fmt);
      }
    }
    out[r] = res;
  }
  const uint32_t bits = __ballot_sync(0xffffffffu, ok);
  const int lane      = threadIdx.x & 31;
  if (lane == 0 && r < n) out_mask[r >> 5] = bits;          // r is a multiple of 32: the warp's rows are one mask word
  __shared__ int warp_valid[kDtThreads / 32];
  if (lane == 0) warp_valid[threadIdx.x >> 5] = __popc(bits);
  __syncthreads();
  if (threadIdx.x == 0) {
    int v = 0;
#pragma unroll
    for (int w = 0; w < kDtThreads / 32; ++w) v += warp_valid[w];
    if (v) atomicAdd(valid_rows, static_cast<unsigned long long>(v));
  }
}

unsigned grid_for(int64_t threads) { return static_cast<unsigned>((threads + kDtThreads - 1) / kDtThreads); }

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <class Op>
int launch_map(const srj_column& in, void* out, const Op& op, cudaStream_t stream)
{
  using In        = typename Op::In;
  using Out       = typename Op::Out;
  const int64_t n = in.size;
  const bool vec  = aligned16(in.data) && aligned16(out);
  dt_map_kernel<Op><<<grid_for((n + kMapRows - 1) / kMapRows), kDtThreads, 0, stream>>>(static_cast<const In*>(in.data), in.null_mask,
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

template <bool kMicros>
int launch_trunc_scalar(int32_t fmt, const srj_column& in, void* out, cudaStream_t stream)
{
  switch (fmt) {
    case kDtYear: return launch_map(in, out, TruncOp<kDtYear, kMicros>{}, stream);
    case kDtQuarter: return launch_map(in, out, TruncOp<kDtQuarter, kMicros>{}, stream);
    case kDtMonth: return launch_map(in, out, TruncOp<kDtMonth, kMicros>{}, stream);
    case kDtWeek: return launch_map(in, out, TruncOp<kDtWeek, kMicros>{}, stream);
    default: break;
  }
  if constexpr (kMicros) {
    switch (fmt) {
      case kDtDay: return launch_map(in, out, TruncOp<kDtDay, true>{}, stream);
      case kDtHour: return launch_map(in, out, TruncOp<kDtHour, true>{}, stream);
      case kDtMinute: return launch_map(in, out, TruncOp<kDtMinute, true>{}, stream);
      case kDtSecond: return launch_map(in, out, TruncOp<kDtSecond, true>{}, stream);
      case kDtMillisecond: return launch_map(in, out, TruncOp<kDtMillisecond, true>{}, stream);
      default: return launch_map(in, out, TruncOp<kDtMicrosecond, true>{}, stream);
    }
  }
  return SRJ_EINVAL;   // unreachable: the caller has checked the format fits
}

}  // namespace

// out_mask (NULL: none) gets a copy of the input's mask, all ones when the input has none
static int launch_datetime_rebase(int32_t direction, const srj_column& in, void* out, uint32_t* out_mask, cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  const int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  const bool micros = in.type_id == SRJ_TIMESTAMP_MICROSECONDS;
  if (direction == SRJ_DATETIME_GREGORIAN_TO_JULIAN)
    return micros ? launch_map(in, out, RebaseOp<SRJ_DATETIME_GREGORIAN_TO_JULIAN, true>{}, stream)
                  : launch_map(in, out, RebaseOp<SRJ_DATETIME_GREGORIAN_TO_JULIAN, false>{}, stream);
  return micros ? launch_map(in, out, RebaseOp<SRJ_DATETIME_JULIAN_TO_GREGORIAN, true>{}, stream)
                : launch_map(in, out, RebaseOp<SRJ_DATETIME_JULIAN_TO_GREGORIAN, false>{}, stream);
}

// a format that does not fit the type zeroes out and out_mask (which must then be given); otherwise as the rebase
static int launch_datetime_truncate_scalar(int32_t fmt, const srj_column& in, void* out, uint32_t* out_mask, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) return SRJ_OK;
  const bool micros = in.type_id == SRJ_TIMESTAMP_MICROSECONDS;
  if (!format_fits(fmt, micros)) {                          // all null
    SRJ_CUDA_TRY(cudaMemsetAsync(out, 0, static_cast<size_t>(n) * (micros ? 8 : 4), stream));
    SRJ_CUDA_TRY(cudaMemsetAsync(out_mask, 0, static_cast<size_t>((n + 31) / 32) * 4, stream));
    return SRJ_OK;
  }
  const int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  return micros ? launch_trunc_scalar<true>(fmt, in, out, stream) : launch_trunc_scalar<false>(fmt, in, out, stream);
}

// fmt.size rows; dt has one row (broadcast) or fmt.size.  Writes out, out_mask and *null_count (one read-back).
static int launch_datetime_truncate_column(const srj_column& dt, const srj_column& fmt, void* out, uint32_t* out_mask, int64_t* null_count,
                                    cudaStream_t stream)
{
  const int64_t n = fmt.size;
  *null_count     = 0;
  if (n == 0) return SRJ_OK;
  unsigned long long* d_valid = nullptr;
  int rc = null_counter(&d_valid);
  if (rc != SRJ_OK) return rc;
  SRJ_CUDA_TRY(cudaMemsetAsync(d_valid, 0, sizeof(*d_valid), stream));
  const bool broadcast = dt.size == 1;
  const auto* chars    = static_cast<const uint8_t*>(fmt.data);
  if (dt.type_id == SRJ_TIMESTAMP_MICROSECONDS)
    dt_trunc_format_kernel<true><<<grid_for(n), kDtThreads, 0, stream>>>(static_cast<const int64_t*>(dt.data), dt.null_mask, broadcast, chars,
                                                                         fmt.offsets, fmt.null_mask, n, static_cast<int64_t*>(out), out_mask, d_valid);
  else
    dt_trunc_format_kernel<false><<<grid_for(n), kDtThreads, 0, stream>>>(static_cast<const int32_t*>(dt.data), dt.null_mask, broadcast, chars,
                                                                          fmt.offsets, fmt.null_mask, n, static_cast<int32_t*>(out), out_mask, d_valid);
  SRJ_CUDA_TRY(cudaGetLastError());
  unsigned long long h_valid = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(&h_valid, d_valid, sizeof(h_valid), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  *null_count = n - static_cast<int64_t>(h_valid);
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

static bool is_datetime(int32_t t) { return t == SRJ_TIMESTAMP_DAYS || t == SRJ_TIMESTAMP_MICROSECONDS; }

// datetime_rebase.cu:342-372
int srj_datetime_rebase(int32_t direction, const srj_column* input, void* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "datetime_rebase";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (direction != SRJ_DATETIME_GREGORIAN_TO_JULIAN && direction != SRJ_DATETIME_JULIAN_TO_GREGORIAN) {
    set_error("%s: unknown direction %d", what, direction);
    return SRJ_EINVAL;
  }
  if (!is_datetime(input->type_id)) { set_error("%s: The input must be either day or microsecond timestamps to rebase.", what); return SRJ_EUNSUPPORTED; }
  if (input->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (input->size == 0) return SRJ_OK;
  int rc = check_data(what, "datetime", *input);
  if (rc == SRJ_OK) rc = check_out(what, "output", out, type_width(input->type_id));
  if (rc == SRJ_OK) rc = check_out_mask(what, input->null_mask, out_mask);
  if (rc != SRJ_OK) return rc;
  return launch_datetime_rebase(direction, *input, out, out_mask, static_cast<cudaStream_t>(stream));
}

// datetime_truncate.cu:327-376
int srj_datetime_truncate(const srj_column* datetime, const srj_column* format_col, const char* format, int32_t format_len, void* out,
                          uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "datetime_truncate";
  if (!datetime || !null_count || (format_col == nullptr) == (format == nullptr) || (format && format_len < 0)) {
    set_error("%s: bad argument (give exactly one of a format column and a format string, and a null count)", what);
    return SRJ_EINVAL;
  }
  if (!is_datetime(datetime->type_id)) { set_error("%s: The date/time input must be either day or microsecond timestamps.", what); return SRJ_EUNSUPPORTED; }
  if (format_col && format_col->type_id != SRJ_STRING) { set_error("%s: The format input must be of string type.", what); return SRJ_EUNSUPPORTED; }
  if (datetime->size < 0 || (format_col && format_col->size < 0)) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (format_col && datetime->size != 1 && datetime->size != format_col->size) {
    set_error("%s: The input date/time column must have exactly one row or the same number of rows as the format column.", what);
    return SRJ_EINVAL;
  }
  const int64_t rows = format_col ? format_col->size : datetime->size;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows == 0) {
    *null_count = 0;
    return SRJ_OK;
  }
  int rc = check_data(what, "datetime", *datetime);
  if (rc == SRJ_OK) rc = check_out(what, "output", out, type_width(datetime->type_id));
  if (rc != SRJ_OK) return rc;
  if (format_col) {
    if ((rc = check_offsets(what, "format", *format_col)) != SRJ_OK || (rc = check_out_mask(what, true, out_mask)) != SRJ_OK) return rc;
    return launch_datetime_truncate_column(*datetime, *format_col, out, out_mask, null_count, s);
  }
  const int32_t fmt = datetime_parse_format(format, format_len);
  const bool fits   = format_fits(fmt, datetime->type_id == SRJ_TIMESTAMP_MICROSECONDS);
  if ((rc = check_out_mask(what, !fits || datetime->null_mask, out_mask)) != SRJ_OK) return rc;
  *null_count = fits ? -1 : rows;
  return launch_datetime_truncate_scalar(fmt, *datetime, out, out_mask, s);
}

}  // extern "C"
