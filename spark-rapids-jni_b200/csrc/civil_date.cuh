// civil_date.cuh -- day counts from 1970-01-01 <-> year / month / day in the proleptic Gregorian and the Julian calendars,
// after H. Hinnant's "chrono-Compatible Low-Level Date Algorithms" (integer arithmetic, no table), and floor division by a
// constant.  Shared by iceberg.cu (year / month transforms) and datetime.cu (rebase, truncation).
#pragma once

#include <stdint.h>

namespace srj {

constexpr int64_t kMicrosPerDay  = 86400000000ll;
constexpr int64_t kMicrosPerHour = 3600000000ll;

template <int64_t D>
__host__ __device__ __forceinline__ int64_t floor_div_const(int64_t t)
{
  const int64_t q = t / D;                    // by a constant: multiply-high, no division subroutine
  return q - (t - q * D < 0);
}

// proleptic Gregorian year and month (1..12) of a day count from 1970-01-01 (Hinnant, civil_from_days)
__device__ __forceinline__ void civil_year_month(int32_t days, int32_t* year, int32_t* month)
{
  const int64_t z    = static_cast<int64_t>(days) + 719468;               // days from 0000-03-01
  const int64_t era  = (z >= 0 ? z : z - 146096) / 146097;
  const uint32_t doe = static_cast<uint32_t>(z - era * 146097);           // [0, 146096]
  const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);           // [0, 365], from March 1
  const uint32_t mp  = (5 * doy + 2) / 153;                               // [0, 11], March = 0
  *month             = static_cast<int32_t>(mp < 10 ? mp + 3 : mp - 9);
  *year              = static_cast<int32_t>(yoe) + static_cast<int32_t>(era) * 400 + (*month <= 2);
}

// A calendar date whose year is reduced to int16 (two's complement), as cuda::std::chrono::year stores it: Spark's
// rebase and truncation on the device go through that type, so their results carry the reduction.
struct Ymd16 {
  int32_t y;          // in [-32768, 32767]
  uint32_t m, d;      // 1..12, 1..31
};

__host__ __device__ __forceinline__ int32_t wrap16(int32_t y) { return static_cast<int16_t>(static_cast<uint16_t>(y)); }

// (y, m, d) as one ordered key: a lexicographic compare of dates is a compare of keys
__host__ __device__ __forceinline__ int32_t ymd_key(int32_t y, uint32_t m, uint32_t d) { return y * 512 + static_cast<int32_t>(m * 32 + d); }

// civil_from_days with the int16 year; z is 64-bit, so every int32 day count has a defined result
__device__ __forceinline__ Ymd16 civil_from_days16(int32_t days)
{
  const int64_t z    = static_cast<int64_t>(days) + 719468;
  const int64_t era  = (z >= 0 ? z : z - 146096) / 146097;
  const uint32_t doe = static_cast<uint32_t>(z - era * 146097);
  const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const uint32_t mp  = (5 * doy + 2) / 153;
  const uint32_t m   = mp < 10 ? mp + 3 : mp - 9;
  const uint32_t d   = doy - (153 * mp + 2) / 5 + 1;
  return Ymd16{wrap16(static_cast<int32_t>(yoe) + static_cast<int32_t>(era) * 400 + (m <= 2)), m, d};
}

// Hinnant's days_from_civil (proleptic Gregorian); |y| <= 32768 keeps every step in int32
__device__ __forceinline__ int32_t days_from_civil(int32_t y, uint32_t m, uint32_t d)
{
  y -= m <= 2;
  const int32_t era  = (y >= 0 ? y : y - 399) / 400;
  const uint32_t yoe = static_cast<uint32_t>(y - era * 400);                       // [0, 399]
  const uint32_t doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;            // [0, 365]
  const uint32_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;                      // [0, 146096]
  return era * 146097 + static_cast<int32_t>(doe) - 719468;
}

// days_from_civil with an int64 era term, for every int32 year whose y - 399 does not overflow (the reference's
// date_time_utils::to_epoch_day): string casts reach years of 6 (timestamps) and 7 (dates) digits
__device__ __forceinline__ int64_t days_from_civil64(int32_t y, uint32_t m, uint32_t d)
{
  y -= m <= 2;
  const int32_t era  = (y >= 0 ? y : y - 399) / 400;
  const uint32_t yoe = static_cast<uint32_t>(y - era * 400);                       // [0, 399]
  const uint32_t doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;            // [0, 365]
  const uint32_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;                      // [0, 146096]
  return era * 146097ll + static_cast<int64_t>(doe) - 719468ll;
}

// Hinnant's days_from_julian: the day count of a date of the Julian calendar
__device__ __forceinline__ int32_t days_from_julian(int32_t y, uint32_t m, uint32_t d)
{
  y -= m <= 2;
  const int32_t era  = (y >= 0 ? y : y - 3) / 4;
  const uint32_t yoe = static_cast<uint32_t>(y - era * 4);                         // [0, 3]
  const uint32_t doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;            // [0, 365]
  return era * 1461 + static_cast<int32_t>(yoe * 365 + doy) - 719470;
}

// Hinnant's julian_from_days, with the int16 year; days + 719470 must not overflow (callers pass days < -141427)
__device__ __forceinline__ Ymd16 julian_from_days16(int32_t days)
{
  const int32_t z    = days + 719470;
  const int32_t era  = (z >= 0 ? z : z - 1460) / 1461;
  const uint32_t doe = static_cast<uint32_t>(z - era * 1461);                      // [0, 1460]
  const uint32_t yoe = (doe - doe / 1460) / 365;                                   // [0, 3]
  const uint32_t doy = doe - 365 * yoe;                                            // [0, 365]
  const uint32_t mp  = (5 * doy + 2) / 153;
  const uint32_t m   = mp < 10 ? mp + 3 : mp - 9;
  const uint32_t d   = doy - (153 * mp + 2) / 5 + 1;
  return Ymd16{wrap16(static_cast<int32_t>(yoe) + era * 4 + (m <= 2)), m, d};
}

}  // namespace srj
