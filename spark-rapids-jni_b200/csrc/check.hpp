// check.hpp -- host-only helpers of the C-ABI entry points: the NVTX range of a call, the width of a fixed-width type
// and the argument checks the modules share.  A failing check sets the last error and returns SRJ_EINVAL.
#pragma once
#include <algorithm>

#include <nvtx3/nvToolsExt.h>

#include "common.cuh"

namespace srj {

// NVTX range of one C-ABI call (the reference wraps its entry points the same way: nvtx_ranges.hpp:24-46,
// SRJ_FUNC_RANGE); header-only NVTX v3, a no-op unless a profiler is attached.
struct ApiRange {
  explicit ApiRange(const char* name) { nvtxRangePushA(name); }
  ~ApiRange() { nvtxRangePop(); }
};
#define SRJ_API_RANGE() ::srj::ApiRange _srj_range(__func__)

// bytes of one element of a fixed-width type, 0 for any other type
inline int type_width(int32_t type_id)
{
  switch (type_id) {
    case SRJ_INT8: case SRJ_UINT8: case SRJ_BOOL8: return 1;
    case SRJ_INT16: case SRJ_UINT16: return 2;
    case SRJ_INT32: case SRJ_UINT32: case SRJ_FLOAT32: case SRJ_TIMESTAMP_DAYS: case SRJ_DURATION_DAYS: case SRJ_DECIMAL32: return 4;
    case SRJ_INT64: case SRJ_UINT64: case SRJ_FLOAT64: case SRJ_TIMESTAMP_SECONDS: case SRJ_TIMESTAMP_MILLISECONDS:
    case SRJ_TIMESTAMP_MICROSECONDS: case SRJ_TIMESTAMP_NANOSECONDS: case SRJ_DURATION_SECONDS: case SRJ_DURATION_MILLISECONDS:
    case SRJ_DURATION_MICROSECONDS: case SRJ_DURATION_NANOSECONDS: case SRJ_DECIMAL64: return 8;
    case SRJ_DECIMAL128: return 16;
    default: return 0;
  }
}

inline bool aligned_to(const void* p, int a) { return (reinterpret_cast<uintptr_t>(p) & static_cast<uintptr_t>(a - 1)) == 0; }

// every column of cols[0 .. n) has `rows` rows
inline int check_rows(const char* what, const srj_column* cols, int32_t n, int64_t rows)
{
  for (int32_t c = 0; c < n; ++c)
    if (cols[c].size != rows) {
      set_error("%s: column %d has %lld rows, expected %lld", what, c, static_cast<long long>(cols[c].size), static_cast<long long>(rows));
      return SRJ_EINVAL;
    }
  return SRJ_OK;
}

// a column with rows has its data, aligned to its element (at most 8 bytes: DECIMAL128 is loaded as two longs).  The
// column is "the <name>", or "<name> <index>" when index >= 0.
inline int check_data(const char* what, const char* name, const srj_column& c, int index = -1)
{
  const int a = std::min(type_width(c.type_id), 8);
  if (c.size <= 0 || (c.data && aligned_to(c.data, a))) return SRJ_OK;
  if (index < 0) set_error("%s: the %s data is missing or not aligned to %d bytes", what, name, a);
  else set_error("%s: %s %d has no data or data not aligned to %d bytes", what, name, index, a);
  return SRJ_EINVAL;
}

// a STRING or LIST column's offsets are present and 4-byte aligned (the callers decide whether zero rows need them).
// The column is named as for check_data.
inline int check_offsets(const char* what, const char* name, const srj_column& c, int index = -1)
{
  if (c.offsets && aligned_to(c.offsets, 4)) return SRJ_OK;
  if (index < 0) set_error("%s: the %s offsets are missing or not 4-byte aligned", what, name);
  else set_error("%s: %s %d has no offsets or offsets not 4-byte aligned", what, name, index);
  return SRJ_EINVAL;
}

// an output buffer aligned to `a` bytes, and present when `needed`
inline int check_out(const char* what, const char* name, const void* p, int a, bool needed = true)
{
  if ((p || !needed) && aligned_to(p, a)) return SRJ_OK;
  set_error("%s: the %s is missing or not aligned to %d bytes", what, name, a);
  return SRJ_EINVAL;
}

// when `needed` (the result can hold nulls, as when an input has a null mask), the output mask is present and 4-byte aligned
inline int check_out_mask(const char* what, bool needed, const uint32_t* out_mask)
{
  if (!needed || (out_mask && aligned_to(out_mask, 4))) return SRJ_OK;
  set_error("%s: the result can hold nulls but no 4-byte aligned output mask was given", what);
  return SRJ_EINVAL;
}

}  // namespace srj
