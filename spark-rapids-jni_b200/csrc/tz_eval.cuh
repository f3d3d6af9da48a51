// tz_eval.cuh -- the offset of a time zone of GpuTimeZoneDB's table at a second (reference datetime_utils.cuh:278-588):
// Java's two DST rules evaluated for a year, and the per-row search of a zone's transitions.  Shared by timezone.cu
// (tz_multi_kernel: local time to UTC) and cast_datetime.cu (the current date of a zone: UTC to local time).
#pragma once

#include <stdint.h>

#include "civil_date.cuh"

namespace srj {
namespace {   // internal to each including file, as these helpers were to timezone.cu

constexpr int64_t kSecPerDay = 86400;

struct TzRule {
  int32_t month, dom, dow, time, before, after;
};

__device__ __forceinline__ TzRule load_rule(const int32_t* p)
{
  return TzRule{__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3), __ldg(p + 4), __ldg(p + 5)};
}

// ---- date_time_utils, step for step: the int32 / uint32 / int64 widths and C's truncating % are the reference's ----------
__device__ __forceinline__ int64_t tz_epoch_day(int32_t year, int32_t month, int32_t day)
{
  const int32_t y    = year - (month <= 2);
  const int32_t era  = (y >= 0 ? y : y - 399) / 400;
  const uint32_t yoe = static_cast<uint32_t>(y - era * 400);
  const uint32_t doy = static_cast<uint32_t>((153 * (month > 2 ? month - 3 : month + 9) + 2) / 5 + day - 1);
  const uint32_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097ll + static_cast<int64_t>(doe) - 719468ll;
}

__device__ __forceinline__ int32_t tz_days_in_month(int32_t year, int32_t month)
{
  if (month == 2) return ((year % 4 == 0 && year % 100 != 0) || year % 400 == 0) ? 29 : 28;
  return (month == 4 || month == 6 || month == 9 || month == 11) ? 30 : 31;
}

// 0 = Monday; negative below day INT32_MIN - 8, as the reference's % gives
__device__ __forceinline__ int64_t tz_weekday(int64_t days) { return (days - (static_cast<int64_t>(INT32_MIN) - 8)) % 7; }

// the year of floor(s / 86400), the day count taken as an int32 as the reference's to_date takes it
__device__ __forceinline__ int32_t tz_year(int64_t s)
{
  int32_t y, m;
  civil_year_month(static_cast<int32_t>(floor_div_const<kSecPerDay>(s)), &y, &m);
  return y;
}

// the UTC second at which rule r takes effect in year
__device__ __forceinline__ int64_t rule_instant(int32_t year, const TzRule& r)
{
  int64_t days;
  if (r.dom > 0) {
    days = tz_epoch_day(year, r.month, r.dom);
    if (r.dow >= 0) days += 6 - (tz_weekday(days) + (6 - r.dow)) % 7;            // next or same weekday
  } else {
    days = tz_epoch_day(year, r.month, tz_days_in_month(year, r.month) + 1 + r.dom);
    if (r.dow >= 0) days -= (tz_weekday(days) + (7 - r.dow)) % 7;                // previous or same weekday
  }
  return days * kSecPerDay + r.time - r.before;
}

// The two thresholds of a year: before t0 the offset is r0.before, from t0 to t1 r0.after, then r1.after.  From UTC they
// are the rules' instants (get_offset_for_utc_time); to UTC their local times, the gap's later and the overlap's earlier
// wall clock, chosen by whether rule 0 is a gap (get_offset_for_local_time).
struct Thresholds {
  int64_t t0, t1;
};

template <bool kToUtc>
__device__ __forceinline__ Thresholds rule_thresholds(int32_t year, const TzRule& r0, const TzRule& r1)
{
  const int64_t u0 = rule_instant(year, r0), u1 = rule_instant(year, r1);
  if (!kToUtc) return Thresholds{u0, u1};
  const bool gap = r0.after > r0.before;
  return Thresholds{u0 + (gap ? r0.after : r0.before), u1 + (gap ? r1.before : r1.after)};
}

__device__ __forceinline__ int32_t rule_offset(int64_t s, const Thresholds& t, const TzRule& r0, const TzRule& r1)
{
  return s < t.t0 ? r0.before : s < t.t1 ? r0.after : r1.after;
}

// The whole table in global memory (small enough to stay in L2).  inst is the instant searched: each entry's
// localInstant converting to UTC, its utcInstant converting from UTC.
struct TzTable {
  const int32_t* list;     // zones + 1 offsets into the entries
  const int64_t* inst;     // localInstant or utcInstant of every entry
  const int32_t* off;      // offset of every entry
  const int32_t* rule_list;
  const int32_t* rules;
  int32_t zones;
};

// SRJ_ZONE_SHIFT(kToUtc, t, z, s, known, out): out = s - o converting to UTC, s + o from UTC (wrapping in int64), o the
// offset of zone z of table t at second s (convert_timestamp): past the last instant of a zone with rules, the rules of
// year(floor(s / 86400)); otherwise the last entry whose instant is <= s.  known = false, leaving out alone, when z is
// outside the table or the zone has no entry or other than 0 or 12 rule integers.  s is evaluated more than once.
// A statement macro rather than a function: tz_multi_kernel compiled with this code in its body before it was shared, and
// any inline function, however written, changes that kernel's register allocation and instruction order; the macro
// expands to the same code, so the kernel's SASS is unchanged (tests/test_cast_datetime_surface.py checks it).
#define SRJ_ZONE_SHIFT(kToUtc, t, z_expr, s, known, out)                                                                  \
  do {                                                                                                                    \
    const int32_t z_ = (z_expr);                                                                                          \
    known            = z_ >= 0 && z_ < (t).zones;                                                                         \
    int32_t beg_ = 0, cnt_ = 0, rb_ = 0, rc_ = 0;                                                                         \
    if (known) {                                                                                                          \
      beg_  = __ldg((t).list + z_);                                                                                       \
      cnt_  = __ldg((t).list + z_ + 1) - beg_;                                                                            \
      rb_   = __ldg((t).rule_list + z_);                                                                                  \
      rc_   = __ldg((t).rule_list + z_ + 1) - rb_;                                                                        \
      known = cnt_ >= 1 && (rc_ == 0 || rc_ == 12);                                                                       \
    }                                                                                                                     \
    if (known) {                                                                                                          \
      const int64_t* inst_ = (t).inst + beg_;                                                                             \
      int32_t o_;                                                                                                         \
      if (rc_ == 12 && (s) > __ldg(reinterpret_cast<const long long*>(inst_ + cnt_ - 1))) {                               \
        const TzRule a_ = load_rule((t).rules + rb_), b_ = load_rule((t).rules + rb_ + 6);                                \
        o_ = rule_offset((s), rule_thresholds<kToUtc>(tz_year(s), a_, b_), a_, b_);                                       \
      } else {                                                                                                            \
        int32_t base_ = 0, m_ = cnt_;                                                                                     \
        while (m_ > 1) {                                                                                                  \
          const int32_t half_ = m_ >> 1;                                                                                  \
          base_ = __ldg(reinterpret_cast<const long long*>(inst_ + base_ + half_)) <= (s) ? base_ + half_ : base_;         \
          m_ -= half_;                                                                                                    \
        }                                                                                                                 \
        o_ = __ldg((t).off + beg_ + base_);                                                                               \
      }                                                                                                                   \
      out = kToUtc ? static_cast<int64_t>(static_cast<uint64_t>(s) - static_cast<uint64_t>(static_cast<int64_t>(o_)))     \
                   : static_cast<int64_t>(static_cast<uint64_t>(s) + static_cast<uint64_t>(static_cast<int64_t>(o_)));    \
    }                                                                                                                     \
  } while (0)

}  // namespace
}  // namespace srj
