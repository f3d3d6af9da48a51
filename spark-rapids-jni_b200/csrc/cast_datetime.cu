// cast_datetime.cu -- CastStrings' string-to-timestamp and string-to-date parses on the device (reference
// cast_string_to_datetime.cu, after Spark 3.5's SparkDateTimeUtils.stringToTimestamp / stringToDate).
//
// parse_ts_kernel: one lane per row.  It trims bytes <= 32 and 127, runs Spark's segment state machine over
// [+-]yyyy[y][y]-m[m]-d[d][ T]h[h]:m[m]:s[s][.ffffff][zone] (or a time alone), parses the zone (Z, [+-] offsets, the
// UT / UTC / GMT prefixes, or a name looked up by binary search in the sorted STRUCT<name STRING, index INT32> map) and
// writes the six columns of the intermediate: result, UTC-less seconds, microseconds, tz type, fixed offset, tz index.
// A time alone takes its date from default_epoch_day (no zone), from now + offset (a fixed zone) or from now converted
// into the named zone with tz_eval.cuh's SRJ_ZONE_SHIFT, the code tz_multi_kernel converts with.
// parse_date_kernel: one lane per row; [+-]yyyy[yyy][-m[m][-d[d][( |T)...]]] to TIMESTAMP_DAYS; each mask word comes
// from a warp ballot and each block adds its valid rows to one counter.
//
// Bytes are read one at a time through the read-only path: neighbouring lanes read neighbouring rows, so a warp's bytes
// share a few L1 lines.  The segments live in named registers (a switch on the segment index), never in an array a lane
// indexes, so nothing spills to local memory.
#include "civil_date.cuh"
#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"
#include "tz_eval.cuh"

namespace srj {
namespace {

constexpr int kCastThreads = 256;
enum : uint8_t { kTzUnspecified = 0, kTzFixed = 1, kTzOther = 2, kTzInvalid = 3 };

__device__ __forceinline__ uint32_t byte_at(const uint8_t* p, int32_t i) { return __ldg(p + i); }
__device__ __forceinline__ bool is_trim(uint32_t c) { return c <= 32 || c == 127; }
__device__ __forceinline__ uint32_t digit(uint32_t c) { return c - '0'; }   // > 9 unless c is a digit

// a zone as parsed: for kTzOther the name is bytes [pos, end) of the row
struct Zone {
  uint32_t type;
  int32_t offset;
  int32_t pos, end;
};

__device__ __forceinline__ Zone fixed_zone(int32_t offset) { return Zone{kTzFixed, offset, 0, 0}; }
__device__ __forceinline__ Zone invalid_zone() { return Zone{kTzInvalid, 0, 0, 0}; }

// up to max_digits digits at pos: the count read, their value in *v
__device__ __forceinline__ int32_t parse_digits(const uint8_t* p, int32_t& pos, int32_t end, int32_t* v, int32_t max_digits)
{
  int32_t value = 0, digits = 0;
  while (pos < end) {
    const uint32_t d = digit(byte_at(p, pos));
    if (d > 9) break;
    value = value * 10 + static_cast<int32_t>(d);
    ++pos;
    if (++digits == max_digits) break;
  }
  *v = value;
  return digits;
}

// the offset after its sign (parse_tz_from_sign): [h]h, hh[mm[ss]], [h]h:m[m], [h]h:mm:ss; at most 18:00:00.  Spark 3.2.0
// rejects a one-digit minute after a colon.
__device__ Zone parse_offset(const uint8_t* p, int32_t& pos, int32_t end, int32_t sign, bool is_320)
{
  int32_t hour = 0, minute = 0, second = 0, m_digits = 0, s_digits = 0;
  const int32_t h_digits = parse_digits(p, pos, end, &hour, 2);
  if (h_digits == 0) return invalid_zone();
  if (pos < end) {
    if (byte_at(p, pos) == ':') {
      ++pos;
      m_digits = parse_digits(p, pos, end, &minute, 2);
      if (m_digits == 0 || (is_320 && m_digits == 1)) return invalid_zone();
      if (pos < end) {
        if (byte_at(p, pos) != ':') return invalid_zone();
        ++pos;
        s_digits = parse_digits(p, pos, end, &second, 2);
        if (s_digits != 2 || pos < end) return invalid_zone();
      }
    } else {
      if (h_digits != 2) return invalid_zone();
      m_digits = parse_digits(p, pos, end, &minute, 2);
      s_digits = parse_digits(p, pos, end, &second, 2);
      if ((m_digits != 2 && m_digits != 0) || (s_digits != 2 && s_digits != 0) || pos < end) return invalid_zone();
    }
  }
  if (hour > 18 || minute > 59 || second > 59) return invalid_zone();
  const int32_t secs = hour * 3600 + minute * 60 + second;
  if (secs > 18 * 3600) return invalid_zone();
  if (s_digits > 0 && m_digits != 2) return invalid_zone();
  return fixed_zone(sign * secs);
}

// the zone of bytes [pos, end), pos at its first byte (parse_from_tz / parse_tz and the U / G prefixes)
__device__ Zone parse_zone(const uint8_t* p, int32_t pos, int32_t end, bool is_320)
{
  while (pos < end && is_trim(byte_at(p, pos))) ++pos;
  if (pos >= end) return invalid_zone();
  const uint32_t c0 = byte_at(p, pos);
  if (end - pos == 1 && c0 == 'Z') return fixed_zone(0);
  const Zone other{kTzOther, 0, pos, end};
  const int32_t start = pos++;
  if (c0 == '+' || c0 == '-') return parse_offset(p, pos, end, c0 == '+' ? 1 : -1, is_320);
  if (c0 == 'U') {
    if (pos >= end) return invalid_zone();                                       // "U"
    if (byte_at(p, pos) != 'T') return other;                                     // e.g. US/Pacific
    if (++pos >= end) return fixed_zone(0);                                       // "UT"
    if (byte_at(p, pos) == 'C' && ++pos >= end) return fixed_zone(0);             // "UTC"
    const uint32_t s = byte_at(p, pos);                                           // UT or UTC, then a sign or a name
    if (s == '+' || s == '-') {
      ++pos;
      return parse_offset(p, pos, end, s == '+' ? 1 : -1, is_320);
    }
    return Zone{kTzOther, 0, start, end};
  }
  if (c0 == 'G') {
    if (end - pos < 2 || byte_at(p, pos) != 'M' || byte_at(p, pos + 1) != 'T') return other;   // e.g. GB
    if (end - pos == 2) return fixed_zone(0);                                                  // "GMT"
    pos += 2;
    const uint32_t s = byte_at(p, pos);
    if (s == '+' || s == '-') {
      ++pos;
      return parse_offset(p, pos, end, s == '+' ? 1 : -1, is_320);
    }
    if (s == '0' && pos + 1 == end) return fixed_zone(0);                                      // "GMT0"
    return other;
  }
  return other;
}

// is_valid_digits: the year 4 to 6 digits, the fraction any, a Spark 3.2.0 offset hour up to 2, the rest 1 or 2
__device__ __forceinline__ bool valid_digits(int32_t segment, int32_t digits)
{
  return segment == 6 || (segment == 0 && digits >= 4 && digits <= 6) || (segment == 7 && digits <= 2) ||
         (segment != 0 && segment != 6 && segment != 7 && digits > 0 && digits <= 2);
}

struct Segments {
  int32_t v[9];   // indexed only with constants: set() selects the register
  __device__ __forceinline__ void set(int32_t i, int32_t x)
  {
    switch (i) {
      case 0: v[0] = x; break;
      case 1: v[1] = x; break;
      case 2: v[2] = x; break;
      case 3: v[3] = x; break;
      case 4: v[4] = x; break;
      case 5: v[5] = x; break;
      case 6: v[6] = x; break;
      case 7: v[7] = x; break;
      case 8: v[8] = x; break;
      default: break;   // a tenth segment (Spark 3.2.0's "+hh:mm:ss" after the time) is dropped
    }
  }
};

__device__ __forceinline__ bool leap(int32_t y) { return (y % 4 == 0 && y % 100 != 0) || y % 400 == 0; }

__device__ __forceinline__ bool valid_month_day(int32_t y, int32_t m, int32_t d)
{
  if (m < 1 || m > 12 || d < 1) return false;
  const int32_t dim = m == 2 ? (leap(y) ? 29 : 28) : (m == 4 || m == 6 || m == 9 || m == 11) ? 30 : 31;
  return d <= dim;
}

struct TsParse {
  bool ok;
  bool just_time;
  Zone tz;
  int64_t seconds;
  int32_t micros;
};

// parse_timestamp_string, step for step
__device__ TsParse parse_timestamp(const uint8_t* p, int32_t len, bool is_320, bool is_400)
{
  TsParse r{false, false, Zone{kTzUnspecified, 0, 0, 0}, 0, 0};
  int32_t pos = 0, end = len;
  while (pos < end && is_trim(byte_at(p, pos))) ++pos;
  while (pos < end && is_trim(byte_at(p, end - 1))) --end;
  if (pos >= end) return r;
  const int32_t n = end - pos;
  Segments seg{{1970, 1, 1, 0, 0, 0, 0, 0, 0}};
  int32_t i = 0, j = 0, digits_frac = 0, sign = 1;
  uint32_t cur = 0;
  int32_t cur_digits = 0;
  bool has_sign = false, sign_tz_320 = false, tz_plus_320 = false;
  const uint32_t first = byte_at(p, pos);
  if (first == '-' || first == '+') {
    has_sign = true;
    sign     = first == '-' ? -1 : 1;
    j        = 1;
  }
  const bool no_leading_time = is_400 && pos > 0;   // SPARK-52351: Spark 4.0 / Databricks 14.3 reject spaces + "Thh:mm:ss"
  for (; j < n; ++j) {
    const uint32_t b = byte_at(p, pos + j);
    const uint32_t d = digit(b);
    if (d <= 9) {
      if (i == 6) ++digits_frac;
      if (i != 6 || cur_digits < 6) cur = cur * 10 + d;   // the fraction keeps 6 digits: the rest is truncated
      ++cur_digits;
      continue;
    }
    // a separator closes segment i
    if (j == 0 && b == 'T' && !no_leading_time) {
      r.just_time = true;
      i += 3;
      continue;
    }
    bool close = false;
    int32_t next = i + 1;
    if (i < 2) {
      if (b == '-') {
        close = true;
      } else if (i == 0 && b == ':' && !has_sign) {
        r.just_time = true;
        if (!valid_digits(3, cur_digits)) return r;
        seg.set(3, static_cast<int32_t>(cur));
        cur = 0, cur_digits = 0, i = 4;
        continue;
      } else {
        return r;
      }
    } else if (i == 2) {
      if (b != ' ' && b != 'T') return r;
      close = true;
    } else if (i == 3 || i == 4) {
      if (b != ':') return r;
      close = true;
    } else if (i == 5 || i == 6) {
      if (!valid_digits(i, cur_digits)) return r;
      seg.set(i, static_cast<int32_t>(cur));
      cur = 0, cur_digits = 0;
      const int32_t was = i;
      ++i;
      if (is_320 && (b == '-' || b == '+')) {
        sign_tz_320 = true;
        tz_plus_320 = b == '+';
      } else if (!(b == '.' && was == 5)) {
        r.tz = parse_zone(p, pos + j, end, is_320);
        if (r.tz.type == kTzInvalid) return r;
        j = n - 1;
      }
      if (i == 6 && b != '.') ++i;
      continue;
    } else {
      if (i < 9 && (b == ':' || b == ' ')) close = true;
      else return r;
    }
    if (close) {
      if (!valid_digits(i, cur_digits)) return r;
      seg.set(i, static_cast<int32_t>(cur));
      cur = 0, cur_digits = 0, i = next;
    }
  }
  if (!valid_digits(i, cur_digits)) return r;
  seg.set(i, static_cast<int32_t>(cur));
  for (; digits_frac < 6; ++digits_frac) seg.v[6] *= 10;
  if (sign_tz_320) {
    const int32_t h = seg.v[7], m = seg.v[8];
    if (h > 18 || m > 59 || h * 3600 + m * 60 > 18 * 3600) return r;
    r.tz = fixed_zone((tz_plus_320 ? 1 : 0) * (h * 3600 + m * 60));   // the reference multiplies by (sign == '+'): 1 or 0
  }
  const int32_t year = seg.v[0] * sign;
  if (year < -300000 || year > 300000 || !valid_month_day(year, seg.v[1], seg.v[2])) return r;
  if (seg.v[3] < 0 || seg.v[3] > 23 || seg.v[4] < 0 || seg.v[4] > 59 || seg.v[5] < 0 || seg.v[5] > 59 || seg.v[6] < 0 || seg.v[6] > 999999)
    return r;
  if (r.tz.type == kTzInvalid) return r;
  const int64_t days = days_from_civil64(year, static_cast<uint32_t>(seg.v[1]), static_cast<uint32_t>(seg.v[2]));
  r.seconds = days * kSecPerDay + seg.v[3] * 3600ll + seg.v[4] * 60ll + seg.v[5];
  r.micros  = seg.v[6];
  r.ok      = true;
  return r;
}

// the map's index of the name bytes [pos, end) of p, -1 when absent: lower_bound over names ordered by bytes
__device__ int32_t find_zone(const uint8_t* p, int32_t pos, int32_t end, const int32_t* name_off, const uint8_t* name_chars,
                             const int32_t* name_idx, int32_t names)
{
  const int32_t len = end - pos;
  int32_t lo = 0, count = names;
  int32_t cmp_at_lo = 1;
  while (count > 0) {
    const int32_t half = count >> 1, mid = lo + half;
    const int32_t b = __ldg(name_off + mid), e = __ldg(name_off + mid + 1), nl = e - b;
    int32_t c = 0;                                               // sign of name[mid] - target
    const int32_t m = nl < len ? nl : len;
    for (int32_t k = 0; k < m && c == 0; ++k) c = static_cast<int32_t>(__ldg(name_chars + b + k)) - static_cast<int32_t>(byte_at(p, pos + k));
    if (c == 0) c = nl - len;
    if (c < 0) {
      lo = mid + 1;
      count -= half + 1;
    } else {
      count     = half;
      cmp_at_lo = c;
    }
  }
  return lo < names && cmp_at_lo == 0 ? __ldg(name_idx + lo) : -1;
}

struct CastTsArgs {
  const uint8_t* chars;
  const int32_t* offsets;
  const uint32_t* mask;
  int64_t n;
  const int32_t* name_off;
  const uint8_t* name_chars;
  const int32_t* name_idx;
  int32_t names;
  TzTable utc_table;          // inst = utcInstant: the current date of a named zone is now converted from UTC
  int32_t default_tz;
  int64_t default_epoch_day;
  int64_t now;
  bool is_320, is_400;
  uint8_t* result;
  int64_t* seconds;
  int32_t* micros;
  uint8_t* tz_type;
  int32_t* tz_offset;
  int32_t* tz_index;
};

// C's truncating division of the seconds of a local date-time to its day, as the reference takes it
__device__ __forceinline__ int64_t day_start(int64_t s) { return s / kSecPerDay * kSecPerDay; }

__global__ void __launch_bounds__(kCastThreads) parse_ts_kernel(const CastTsArgs a)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kCastThreads + threadIdx.x;
  if (r >= a.n) return;
  const bool valid = !a.mask || ((__ldg(a.mask + (r >> 5)) >> (r & 31)) & 1u);
  TsParse t{false, false, Zone{kTzUnspecified, 0, 0, 0}, 0, 0};
  const uint8_t* p = nullptr;
  if (valid) {                                                   // a null row is invalid whatever its offsets span
    const int32_t b = __ldg(a.offsets + r);
    p               = a.chars + b;
    t               = parse_timestamp(p, __ldg(a.offsets + r + 1) - b, a.is_320, a.is_400);
  }
  uint8_t result = t.ok ? 0 : 1;
  uint8_t type   = static_cast<uint8_t>(t.tz.type);
  int32_t index  = -1;
  int64_t sec    = t.seconds;
  if (t.ok) {
    if (t.tz.type == kTzUnspecified) {
      type  = kTzOther;
      index = a.default_tz;
      if (t.just_time) sec += a.default_epoch_day * kSecPerDay;
    } else if (t.tz.type == kTzFixed) {
      if (t.just_time) sec += day_start(a.now + t.tz.offset);
    } else {
      index = find_zone(p, t.tz.pos, t.tz.end, a.name_off, a.name_chars, a.name_idx, a.names);
      if (index < 0) {
        result = 1;
      } else if (t.just_time) {
        bool known    = false;
        int64_t local = 0;
        SRJ_ZONE_SHIFT(false, a.utc_table, index, a.now, known, local);
        if (known) sec += day_start(local);
        else result = 1;                                         // a map index outside the table, or a malformed zone
      }
    }
  }
  a.result[r]    = result;
  a.seconds[r]   = sec;
  a.micros[r]    = t.micros;
  a.tz_type[r]   = type;
  a.tz_offset[r] = t.tz.offset;                                  // 0 unless the zone is a fixed offset
  a.tz_index[r]  = index;
}

// parse_date, step for step: *days when it parses to a valid date of a 7-digit year at most
__device__ bool parse_date(const uint8_t* p, int32_t len, int64_t* days)
{
  int32_t pos = 0, end = len;
  while (pos < end && is_trim(byte_at(p, pos))) ++pos;
  while (pos < end && is_trim(byte_at(p, end - 1))) --end;
  if (pos >= end) return false;
  const uint32_t s = byte_at(p, pos);
  const bool neg   = s == '-';
  if (s == '-' || s == '+') ++pos;
  int32_t year = 0, month = 1, day = 1;
  const int32_t yd = [&] {                                        // parse_int: fails beyond 7 digits
    int32_t v = 0, digits = 0;
    while (pos < end) {
      const uint32_t d = digit(byte_at(p, pos));
      if (d > 9) break;
      if (++digits > 7) return -1;
      v = v * 10 + static_cast<int32_t>(d);
      ++pos;
    }
    year = v;
    return digits;
  }();
  if (yd < 4) return false;
  if (neg) year = -year;
  bool ok = true;
  if (pos < end) {
    const auto part = [&](int32_t* out) {                         // "-" then 1 or 2 digits
      if (byte_at(p, pos++) != '-') return false;
      int32_t v = 0, digits = 0;
      while (pos < end) {
        const uint32_t d = digit(byte_at(p, pos));
        if (d > 9) break;
        if (++digits > 2) return false;
        v = v * 10 + static_cast<int32_t>(d);
        ++pos;
      }
      *out = v;
      return digits >= 1;
    };
    ok = part(&month);
    if (ok && pos < end) {
      ok = part(&day);
      if (ok && pos < end) {
        const uint32_t c = byte_at(p, pos);
        ok               = c == ' ' || c == 'T';                  // anything may follow the separator
      }
    }
  }
  if (!ok || year < -10000000 || year > 10000000 || !valid_month_day(year, month, day)) return false;
  *days = days_from_civil64(year, static_cast<uint32_t>(month), static_cast<uint32_t>(day));
  return *days >= INT32_MIN && *days <= INT32_MAX;
}

__global__ void __launch_bounds__(kCastThreads) parse_date_kernel(const uint8_t* __restrict__ chars, const int32_t* __restrict__ offsets,
                                                                  const uint32_t* __restrict__ mask, int64_t n, int32_t* __restrict__ out,
                                                                  uint32_t* __restrict__ out_mask, unsigned long long* __restrict__ valid_rows)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kCastThreads + threadIdx.x;
  bool ok         = false;
  int64_t days    = 0;
  if (r < n && (!mask || ((__ldg(mask + (r >> 5)) >> (r & 31)) & 1u))) {
    const int32_t b = __ldg(offsets + r);
    ok              = parse_date(chars + b, __ldg(offsets + r + 1) - b, &days);
  }
  if (r < n) out[r] = ok ? static_cast<int32_t>(days) : 0;
  const uint32_t bits = __ballot_sync(0xffffffffu, ok);
  const int lane      = threadIdx.x & 31;
  if (lane == 0 && r < n) out_mask[r >> 5] = bits;               // r is a multiple of 32: the warp's rows are one mask word
  __shared__ int warp_valid[kCastThreads / 32];
  if (lane == 0) warp_valid[threadIdx.x >> 5] = __popc(bits);
  __syncthreads();
  if (threadIdx.x == 0) {
    int v = 0;
#pragma unroll
    for (int w = 0; w < kCastThreads / 32; ++w) v += warp_valid[w];
    if (v) atomicAdd(valid_rows, static_cast<unsigned long long>(v));
  }
}

unsigned blocks_for(int64_t n) { return static_cast<unsigned>((n + kCastThreads - 1) / kCastThreads); }

}  // namespace

// name_map: STRUCT<STRING, INT32>; fixed / dst: the time zone table; default_tz inside the table.  Asynchronous.
static int launch_cast_parse_timestamps(const srj_column& in, const srj_column& name_map, const srj_column& fixed, const srj_column& dst,
                                 int32_t default_tz, int64_t default_epoch_day, int64_t now, bool is_320, bool is_400, uint8_t* result,
                                 int64_t* seconds, int32_t* micros, uint8_t* tz_type, int32_t* tz_offset, int32_t* tz_index,
                                 cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  const srj_column& names   = name_map.children[0];
  const srj_column& entries = fixed.children[0];
  const CastTsArgs a{static_cast<const uint8_t*>(in.data),
                     in.offsets,
                     in.null_mask,
                     in.size,
                     names.offsets,
                     static_cast<const uint8_t*>(names.data),
                     static_cast<const int32_t*>(name_map.children[1].data),
                     static_cast<int32_t>(name_map.size),
                     TzTable{fixed.offsets, static_cast<const int64_t*>(entries.children[0].data), static_cast<const int32_t*>(entries.children[2].data),
                             dst.offsets, static_cast<const int32_t*>(dst.children[0].data), static_cast<int32_t>(fixed.size)},
                     default_tz,
                     default_epoch_day,
                     now,
                     is_320,
                     is_400,
                     result,
                     seconds,
                     micros,
                     tz_type,
                     tz_offset,
                     tz_index};
  parse_ts_kernel<<<blocks_for(in.size), kCastThreads, 0, stream>>>(a);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// writes out, out_mask and *null_count (one read-back)
static int launch_cast_parse_dates(const srj_column& in, int32_t* out, uint32_t* out_mask, int64_t* null_count, cudaStream_t stream)
{
  const int64_t n = in.size;
  *null_count     = 0;
  if (n == 0) return SRJ_OK;
  unsigned long long* d_valid = nullptr;
  int rc = null_counter(&d_valid);
  if (rc != SRJ_OK) return rc;
  SRJ_CUDA_TRY(cudaMemsetAsync(d_valid, 0, sizeof(*d_valid), stream));
  parse_date_kernel<<<blocks_for(n), kCastThreads, 0, stream>>>(static_cast<const uint8_t*>(in.data), in.offsets, in.null_mask, n, out, out_mask,
                                                                d_valid);
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

// a STRING column: int32 offsets[rows + 1] at 4 bytes.  Its chars may be NULL only when it holds none: a column with rows
// and NULL chars has its first and last offsets read back (one stream synchronisation, on that path alone) and is
// SRJ_EINVAL when they span any byte.
static int cast_check_strings(const char* what, const char* name, const srj_column* c, cudaStream_t stream)
{
  if (!c) { set_error("%s: the %s column is null", what, name); return SRJ_EINVAL; }
  if (c->type_id != SRJ_STRING) { set_error("%s: the %s column must be STRING (type id %d)", what, name, c->type_id); return SRJ_EINVAL; }
  if (c->size < 0 || c->size > INT32_MAX) { set_error("%s: bad %s row count", what, name); return SRJ_EINVAL; }
  if (c->size > 0 && check_offsets(what, name, *c) != SRJ_OK) return SRJ_EINVAL;
  if (c->null_mask && !aligned_to(c->null_mask, 4)) { set_error("%s: the %s null mask is not 4-byte aligned", what, name); return SRJ_EINVAL; }
  if (c->size > 0 && !c->data) {
    int32_t ends[2] = {0, 0};
    SRJ_CUDA_TRY(cudaMemcpyAsync(&ends[0], c->offsets, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    SRJ_CUDA_TRY(cudaMemcpyAsync(&ends[1], c->offsets + c->size, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
    if (ends[0] != ends[1]) { set_error("%s: the %s column has no chars but its offsets span %d bytes", what, name, ends[1] - ends[0]); return SRJ_EINVAL; }
  }
  return SRJ_OK;
}

// cast_string_to_datetime.cu:870-948, 1110-1133; version.hpp:64-68
int srj_cast_parse_timestamps(const srj_column* input, const srj_column* tz_name_map, const srj_column* fixed_transitions, const srj_column* dst_rules,
                              int32_t default_tz_index, int64_t default_epoch_day, int64_t now_seconds, int32_t spark_platform, int32_t spark_major,
                              int32_t spark_minor, int32_t spark_patch, uint8_t* out_result, int64_t* out_seconds, int32_t* out_micros,
                              uint8_t* out_tz_type, int32_t* out_tz_offset, int32_t* out_tz_index, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "cast_parse_timestamps";
  int rc           = cast_check_strings(what, "input", input, static_cast<cudaStream_t>(stream));
  if (rc != SRJ_OK) return rc;
  if (!tz_name_map || tz_name_map->type_id != SRJ_STRUCT || tz_name_map->num_children < 2 || !tz_name_map->children || tz_name_map->size < 0) {
    set_error("%s: the time zone name map must be STRUCT<STRING, INT32>", what);
    return SRJ_EINVAL;
  }
  const srj_column* names = &tz_name_map->children[0];
  if ((rc = cast_check_strings(what, "time zone name", names, static_cast<cudaStream_t>(stream))) != SRJ_OK) return rc;
  if (names->size != tz_name_map->size) { set_error("%s: the time zone name map's fields have mismatched row counts", what); return SRJ_EINVAL; }
  if ((rc = tz_check_flat(what, "time zone index", &tz_name_map->children[1], SRJ_INT32, -1, tz_name_map->size)) != SRJ_OK) return rc;
  if ((rc = tz_check_table(what, fixed_transitions, dst_rules)) != SRJ_OK) return rc;
  if (default_tz_index < 0 || default_tz_index >= fixed_transitions->size) {
    set_error("%s: default time zone index %d is outside the table of %lld zones", what, default_tz_index,
              static_cast<long long>(fixed_transitions->size));
    return SRJ_EINVAL;
  }
  const int64_t n = input->size;
  if (n == 0) return SRJ_OK;
  if ((rc = check_out(what, "result output", out_result, 1)) != SRJ_OK || (rc = check_out(what, "seconds output", out_seconds, 8)) != SRJ_OK ||
      (rc = check_out(what, "microseconds output", out_micros, 4)) != SRJ_OK || (rc = check_out(what, "tz type output", out_tz_type, 1)) != SRJ_OK ||
      (rc = check_out(what, "tz offset output", out_tz_offset, 4)) != SRJ_OK || (rc = check_out(what, "tz index output", out_tz_index, 4)) != SRJ_OK)
    return rc;
  // is_vanilla_320 and is_vanilla_400_or_later || is_databricks_14_3_or_later
  const auto ge = [&](int32_t a, int32_t b, int32_t c) {
    return spark_major > a || (spark_major == a && (spark_minor > b || (spark_minor == b && spark_patch >= c)));
  };
  const bool is_320 = spark_platform == SRJ_SPARK_VANILLA && spark_major == 3 && spark_minor == 2 && spark_patch == 0;
  const bool is_400 = (spark_platform == SRJ_SPARK_VANILLA && ge(4, 0, 0)) || (spark_platform == SRJ_SPARK_DATABRICKS && ge(14, 3, 0));
  return launch_cast_parse_timestamps(*input, *tz_name_map, *fixed_transitions, *dst_rules, default_tz_index, default_epoch_day, now_seconds, is_320,
                                      is_400, out_result, out_seconds, out_micros, out_tz_type, out_tz_offset, out_tz_index,
                                      static_cast<cudaStream_t>(stream));
}

// cast_string_to_datetime.cu:1034-1106, 1135-1140
int srj_cast_parse_dates(const srj_column* input, int32_t* out, uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "cast_parse_dates";
  if (!null_count) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  int rc = cast_check_strings(what, "input", input, static_cast<cudaStream_t>(stream));
  if (rc != SRJ_OK) return rc;
  if (input->size == 0) {
    *null_count = 0;
    return SRJ_OK;
  }
  if ((rc = check_out(what, "output", out, 4)) != SRJ_OK || (rc = check_out_mask(what, true, out_mask)) != SRJ_OK) return rc;
  return launch_cast_parse_dates(*input, out, out_mask, null_count, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
