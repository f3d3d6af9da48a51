// timezone.cu -- GpuTimeZoneDB on the device (reference timezones.cu, datetime_utils.cuh:278-588): timestamps to and from
// a time zone given as Java's transition table, one zone per row for string-to-timestamp casts, and ORC's conversion
// between a writer's and a reader's java.util.TimeZone.
//
// A zone is one row of two LIST columns: entries (utcInstant, localInstant, offset) in seconds, entry 0 at INT64_MIN,
// and 0 or 12 ints holding two DST rules (month, dayOfMonthIndicator, dayOfWeek, secondsFromMidnight, offsetBefore,
// offsetAfter).  A value's seconds s are truncated toward zero; beyond the last instant of a zone with rules the offset
// comes from the rules evaluated for year(floor(s / 86400)), otherwise from the last entry whose instant is <= s.
//
// tz_convert_kernel: one zone for the call.  A grid of a few CTAs per SM; each stages the zone's instants and offsets in
// shared memory and, for a zone with rules, the two rule thresholds of every year in [kWinFirst, kWinFirst + kWinYears),
// then loops over map_rows.cuh's groups (4 rows per thread, 16-byte accesses when aligned).  A row of a year in the window
// makes two compares; any other evaluates the rules itself.
// tz_multi_kernel: one lane per row, its zone searched in the global table (small enough to stay in L2); the warp writes
// each mask word from a ballot and the block adds its valid rows to one counter.
// orc_tz_kernel: the grid-stride map again, both tables staged in shared memory when they fit.
#include "civil_date.cuh"
#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"
#include "map_rows.cuh"
#include "tz_eval.cuh"

namespace srj {
namespace {

constexpr int kTzThreads     = 256;
constexpr int32_t kStageMax  = 1024;    // entries of a zone (or of each ORC table) a CTA stages: 12 bytes each
constexpr int32_t kWinFirst  = 1900;    // the years whose rule thresholds a CTA precomputes: 1900 .. 2200
constexpr int32_t kWinYears  = 301;

// the last i in [0, n) with a[i] <= x (0 when none): upper_bound - 1 over an ascending list whose entry 0 is INT64_MIN
__device__ __forceinline__ int32_t last_le(const int64_t* a, int32_t n, int64_t x)
{
  int32_t base = 0;
  while (n > 1) {
    const int32_t half = n >> 1;
    base               = a[base + half] <= x ? base + half : base;
    n -= half;
  }
  return base;
}

// one zone's conversion of a value in units of 1 / kUnit seconds; inst / off are shared or global memory
template <int64_t kUnit, bool kToUtc>
struct TzOp {
  using In                         = int64_t;
  using Out                        = int64_t;
  static constexpr bool kNullsZero = false;   // rows under nulls are converted from their bits, as in the reference
  const int64_t* inst;
  const int32_t* off;
  int32_t entries;
  int64_t last;                               // inst[entries - 1]
  bool dst;
  TzRule r0, r1;
  const int64_t* win;                         // t0, t1 of the years of the window
  __device__ __forceinline__ int64_t operator()(int64_t v) const
  {
    const int64_t s = v / kUnit;              // duration_cast: toward zero
    int32_t o;
    if (dst && s > last) {
      const int32_t y = tz_year(s);
      const uint32_t w = static_cast<uint32_t>(y - kWinFirst);
      const Thresholds t = w < static_cast<uint32_t>(kWinYears) ? Thresholds{win[2 * w], win[2 * w + 1]} : rule_thresholds<kToUtc>(y, r0, r1);
      o = rule_offset(s, t, r0, r1);
    } else {
      o = off[last_le(inst, entries, s)];
    }
    const uint64_t d = static_cast<uint64_t>(static_cast<int64_t>(o)) * static_cast<uint64_t>(kUnit);
    return static_cast<int64_t>(kToUtc ? static_cast<uint64_t>(v) - d : static_cast<uint64_t>(v) + d);   // wraps in int64
  }
};

template <int64_t kUnit, bool kToUtc>
__global__ void __launch_bounds__(kTzThreads) tz_convert_kernel(const int64_t* __restrict__ in, int64_t* __restrict__ out, int64_t n, bool vec,
                                                                const int64_t* __restrict__ g_inst, const int32_t* __restrict__ g_off,
                                                                int32_t entries, const int32_t* __restrict__ rules)
{
  __shared__ int64_t s_inst[kStageMax];
  __shared__ int32_t s_off[kStageMax];
  __shared__ int64_t s_win[2 * kWinYears];
  const bool staged = entries <= kStageMax;
  if (staged)
    for (int32_t i = threadIdx.x; i < entries; i += kTzThreads) {
      s_inst[i] = __ldg(reinterpret_cast<const long long*>(g_inst + i));
      s_off[i]  = __ldg(g_off + i);
    }
  TzRule a{}, b{};
  if (rules) {
    a = load_rule(rules);
    b = load_rule(rules + 6);
    for (int32_t i = threadIdx.x; i < kWinYears; i += kTzThreads) {
      const Thresholds t = rule_thresholds<kToUtc>(kWinFirst + i, a, b);
      s_win[2 * i]       = t.t0;
      s_win[2 * i + 1]   = t.t1;
    }
  }
  __syncthreads();
  const TzOp<kUnit, kToUtc> op{staged ? s_inst : g_inst, staged ? s_off : g_off, entries,
                               __ldg(reinterpret_cast<const long long*>(g_inst + entries - 1)), rules != nullptr, a, b, s_win};
  const int64_t step = static_cast<int64_t>(gridDim.x) * kTzThreads * kMapRows;
  for (int64_t r = (static_cast<int64_t>(blockIdx.x) * kTzThreads + threadIdx.x) * kMapRows; r < n; r += step)
    map_rows_at(r, in, static_cast<const uint32_t*>(nullptr), out, n, vec, op);
}

// ---- one zone per row ---------------------------------------------------------------------------------------------------
// overflow_checker::get_timestamp_overflow, literally (its test at the minimum second included)
__device__ __forceinline__ bool add_micros_overflows(int64_t seconds, int32_t micros, int64_t* result)
{
  constexpr int64_t kMaxSec = INT64_MAX / 1000000;
  constexpr int64_t kMinSec = INT64_MIN / 1000000 - 1;
  *result = static_cast<int64_t>(static_cast<uint64_t>(seconds) * 1000000ull + static_cast<uint64_t>(static_cast<int64_t>(micros)));
  if (seconds > kMaxSec || seconds < kMinSec) return true;
  if (seconds > 0) return micros > INT64_MAX - seconds * 1000000;
  if (seconds == kMinSec) return micros >= 224192;
  return false;
}

__global__ void __launch_bounds__(kTzThreads) tz_multi_kernel(const int64_t* __restrict__ sec, const int32_t* __restrict__ us,
                                                              const uint8_t* __restrict__ invalid, const uint8_t* __restrict__ type,
                                                              const int32_t* __restrict__ fixed_off, const int32_t* __restrict__ idx,
                                                              const TzTable t, int64_t n, int64_t* __restrict__ out,
                                                              uint32_t* __restrict__ out_mask, unsigned long long* __restrict__ valid_rows)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kTzThreads + threadIdx.x;
  bool ok         = false;
  int64_t res     = 0;
  if (r < n && !__ldg(invalid + r)) {
    const int64_t s = __ldg(reinterpret_cast<const long long*>(sec + r));
    int64_t conv    = 0;
    bool known      = true;
    if (__ldg(type + r) == 1) {                                   // FIXED_TZ
      conv = static_cast<int64_t>(static_cast<uint64_t>(s) - static_cast<uint64_t>(static_cast<int64_t>(__ldg(fixed_off + r))));
    } else {
      SRJ_ZONE_SHIFT(true, t, __ldg(idx + r), s, known, conv);
    }
    if (known) {
      int64_t v;
      if (!add_micros_overflows(conv, __ldg(us + r), &v)) {
        ok  = true;
        res = v;
      }
    }
  }
  if (r < n) out[r] = res;
  const uint32_t bits = __ballot_sync(0xffffffffu, ok);
  const int lane      = threadIdx.x & 31;
  if (lane == 0 && r < n) out_mask[r >> 5] = bits;              // r is a multiple of 32: the warp's rows are one mask word
  __shared__ int warp_valid[kTzThreads / 32];
  if (lane == 0) warp_valid[threadIdx.x >> 5] = __popc(bits);
  __syncthreads();
  if (threadIdx.x == 0) {
    int v = 0;
#pragma unroll
    for (int w = 0; w < kTzThreads / 32; ++w) v += warp_valid[w];
    if (v) atomicAdd(valid_rows, static_cast<unsigned long long>(v));
  }
}

// ---- ORC ------------------------------------------------------------------------------------------------------------------
// get_transition_index (timezones.cu:258-289): the raw offset for an empty table, past the last transition or before the
// first; an exact match's own offset; otherwise the previous transition's
__device__ __forceinline__ int32_t orc_offset(const int64_t* t, const int32_t* o, int32_t n, int32_t raw, int64_t ms)
{
  if (n == 0) return raw;
  int32_t lo = 0, len = n;                                        // upper_bound
  while (len > 0) {
    const int32_t half = len >> 1;
    const bool right   = t[lo + half] <= ms;
    lo                 = right ? lo + half + 1 : lo;
    len                = right ? len - half - 1 : half;
  }
  if (lo == n) return raw;
  if (t[lo] == ms) return o[lo];
  return lo == 0 ? raw : o[lo - 1];
}

struct OrcOp {
  using In                         = int64_t;
  using Out                        = int64_t;
  static constexpr bool kNullsZero = false;
  const int64_t *wt, *rt;
  const int32_t *wo, *ro;
  int32_t wn, rn, wraw, rraw;
  __device__ __forceinline__ int64_t operator()(int64_t us) const
  {
    const int64_t ms  = us / 1000;                                // duration_cast: toward zero
    const int32_t w   = orc_offset(wt, wo, wn, wraw, ms);
    const int32_t r   = orc_offset(rt, ro, rn, rraw, ms);
    const int32_t r2  = orc_offset(rt, ro, rn, rraw, ms + (w - r));
    return static_cast<int64_t>(static_cast<uint64_t>(us) + static_cast<uint64_t>(static_cast<int64_t>(w - r2) * 1000));
  }
};

__global__ void __launch_bounds__(kTzThreads) orc_tz_kernel(const int64_t* __restrict__ in, int64_t* __restrict__ out, int64_t n, bool vec,
                                                            const int64_t* __restrict__ wt, const int32_t* __restrict__ wo, int32_t wn,
                                                            int32_t wraw, const int64_t* __restrict__ rt, const int32_t* __restrict__ ro,
                                                            int32_t rn, int32_t rraw)
{
  __shared__ int64_t s_t[2 * kStageMax];
  __shared__ int32_t s_o[2 * kStageMax];
  const bool staged = wn <= kStageMax && rn <= kStageMax;
  if (staged) {
    for (int32_t i = threadIdx.x; i < wn; i += kTzThreads) {
      s_t[i] = __ldg(reinterpret_cast<const long long*>(wt + i));
      s_o[i] = __ldg(wo + i);
    }
    for (int32_t i = threadIdx.x; i < rn; i += kTzThreads) {
      s_t[kStageMax + i] = __ldg(reinterpret_cast<const long long*>(rt + i));
      s_o[kStageMax + i] = __ldg(ro + i);
    }
  }
  __syncthreads();
  const OrcOp op = staged ? OrcOp{s_t, s_t + kStageMax, s_o, s_o + kStageMax, wn, rn, wraw, rraw} : OrcOp{wt, rt, wo, ro, wn, rn, wraw, rraw};
  const int64_t step = static_cast<int64_t>(gridDim.x) * kTzThreads * kMapRows;
  for (int64_t r = (static_cast<int64_t>(blockIdx.x) * kTzThreads + threadIdx.x) * kMapRows; r < n; r += step)
    map_rows_at(r, in, static_cast<const uint32_t*>(nullptr), out, n, vec, op);
}

// ---- host -----------------------------------------------------------------------------------------------------------------
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// a grid of as many CTAs as fit on the device at once, at most one per group of rows
template <class K>
int stride_grid(K kernel, int64_t n, unsigned* grid)
{
  int per_sm = 0;
  SRJ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kTzThreads, 0));
  const int64_t groups = (n + static_cast<int64_t>(kTzThreads) * kMapRows - 1) / (static_cast<int64_t>(kTzThreads) * kMapRows);
  *grid = static_cast<unsigned>(tmin<int64_t>(groups, static_cast<int64_t>(sm_count()) * (per_sm > 0 ? per_sm : 1)));
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

template <int64_t kUnit, bool kToUtc>
int launch_convert(const srj_column& in, void* out, const int64_t* inst, const int32_t* off, int32_t entries, const int32_t* rules,
                   cudaStream_t stream)
{
  unsigned grid = 0;
  const int rc  = stride_grid(tz_convert_kernel<kUnit, kToUtc>, in.size, &grid);
  if (rc != SRJ_OK) return rc;
  const bool vec = aligned16(in.data) && aligned16(out);
  tz_convert_kernel<kUnit, kToUtc><<<grid, kTzThreads, 0, stream>>>(static_cast<const int64_t*>(in.data), static_cast<int64_t*>(out), in.size,
                                                                     vec, inst, off, entries, rules);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

template <bool kToUtc>
int launch_convert_unit(const srj_column& in, void* out, const int64_t* inst, const int32_t* off, int32_t entries, const int32_t* rules,
                        cudaStream_t stream)
{
  switch (in.type_id) {
    case SRJ_TIMESTAMP_SECONDS: return launch_convert<1, kToUtc>(in, out, inst, off, entries, rules, stream);
    case SRJ_TIMESTAMP_MILLISECONDS: return launch_convert<1000, kToUtc>(in, out, inst, off, entries, rules, stream);
    case SRJ_TIMESTAMP_MICROSECONDS: return launch_convert<1000000, kToUtc>(in, out, inst, off, entries, rules, stream);
    default: return launch_convert<1000000000, kToUtc>(in, out, inst, off, entries, rules, stream);
  }
}

}  // namespace

// reads the zone's bounds back (one synchronisation), checks it has an entry and 0 or 12 rule integers, then launches
static int launch_timezone_convert(bool to_utc, const srj_column& in, const srj_column& fixed, const srj_column& dst, int32_t tz_index, void* out,
                            uint32_t* out_mask, cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  int32_t b[4] = {0, 0, 0, 0};                                    // the zone's entry and rule bounds: the one read-back
  SRJ_CUDA_TRY(cudaMemcpyAsync(b, fixed.offsets + tz_index, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaMemcpyAsync(b + 2, dst.offsets + tz_index, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  const srj_column& entries = fixed.children[0];
  const int32_t count = b[1] - b[0], rules = b[3] - b[2];
  if (b[0] < 0 || b[1] > entries.size || count < 1) {
    set_error("timezone_convert: zone %d has %d transitions (at %d) in a table of %lld; it needs at least its fixed entry", tz_index, count, b[0],
              static_cast<long long>(entries.size));
    return SRJ_EINVAL;
  }
  if (b[2] < 0 || b[3] > dst.children[0].size || (rules != 0 && rules != 12)) {
    set_error("timezone_convert: zone %d has %d DST integers; a zone has 0 or 12", tz_index, rules);
    return SRJ_EINVAL;
  }
  const int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  const int64_t* inst = static_cast<const int64_t*>(entries.children[to_utc ? 1 : 0].data) + b[0];
  const int32_t* off  = static_cast<const int32_t*>(entries.children[2].data) + b[0];
  const int32_t* rl   = rules ? static_cast<const int32_t*>(dst.children[0].data) + b[2] : nullptr;
  return to_utc ? launch_convert_unit<true>(in, out, inst, off, count, rl, stream) : launch_convert_unit<false>(in, out, inst, off, count, rl, stream);
}

// in[0..5]: seconds, micros, invalid, tz type, tz offset, tz indices.  Writes out, out_mask and *null_count (one read-back).
static int launch_timezone_convert_multi(const srj_column* in, const srj_column& fixed, const srj_column& dst, int64_t* out, uint32_t* out_mask,
                                  int64_t* null_count, cudaStream_t stream)
{
  const int64_t n = in[0].size;
  *null_count     = 0;
  if (n == 0) return SRJ_OK;
  unsigned long long* d_valid = nullptr;
  int rc = null_counter(&d_valid);
  if (rc != SRJ_OK) return rc;
  SRJ_CUDA_TRY(cudaMemsetAsync(d_valid, 0, sizeof(*d_valid), stream));
  const srj_column& entries = fixed.children[0];
  const TzTable t{fixed.offsets,  static_cast<const int64_t*>(entries.children[1].data), static_cast<const int32_t*>(entries.children[2].data),
                  dst.offsets, static_cast<const int32_t*>(dst.children[0].data), static_cast<int32_t>(fixed.size)};
  tz_multi_kernel<<<static_cast<unsigned>((n + kTzThreads - 1) / kTzThreads), kTzThreads, 0, stream>>>(
    static_cast<const int64_t*>(in[0].data), static_cast<const int32_t*>(in[1].data), static_cast<const uint8_t*>(in[2].data),
    static_cast<const uint8_t*>(in[3].data), static_cast<const int32_t*>(in[4].data), static_cast<const int32_t*>(in[5].data), t, n, out,
    out_mask, d_valid);
  SRJ_CUDA_TRY(cudaGetLastError());
  unsigned long long h_valid = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(&h_valid, d_valid, sizeof(h_valid), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  *null_count = n - static_cast<int64_t>(h_valid);
  return SRJ_OK;
}

// a table of 0 transitions is a fixed offset (its pointers may be NULL)
static int launch_orc_convert_timezones(const srj_column& in, const int64_t* wt, const int32_t* wo, int32_t wn, int32_t wraw, const int64_t* rt,
                                 const int32_t* ro, int32_t rn, int32_t rraw, void* out, uint32_t* out_mask, cudaStream_t stream)
{
  if (in.size == 0) return SRJ_OK;
  int rc = copy_mask(in, out_mask, stream);
  if (rc != SRJ_OK) return rc;
  unsigned grid = 0;
  if ((rc = stride_grid(orc_tz_kernel, in.size, &grid)) != SRJ_OK) return rc;
  const bool vec = aligned16(in.data) && aligned16(out);
  orc_tz_kernel<<<grid, kTzThreads, 0, stream>>>(static_cast<const int64_t*>(in.data), static_cast<int64_t*>(out), in.size, vec, wt, wo, wn, wraw,
                                                 rt, ro, rn, rraw);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

int tz_check_flat(const char* what, const char* name, const srj_column* c, int32_t t, int32_t t2, int64_t rows)
{
  if (!c) { set_error("%s: the %s column is null", what, name); return SRJ_EINVAL; }
  if (c->type_id != t && c->type_id != t2) { set_error("%s: the %s column has type id %d", what, name, c->type_id); return SRJ_EINVAL; }
  if (c->size != rows) { set_error("%s: the %s column has %lld rows, not %lld", what, name, static_cast<long long>(c->size), static_cast<long long>(rows)); return SRJ_EINVAL; }
  return check_data(what, name, *c);
}

// the two columns of a time zone table (GpuTimeZoneDB.loadData's layout)
int tz_check_table(const char* what, const srj_column* fixed, const srj_column* dst)
{
  if (!fixed || !dst) { set_error("%s: the time zone table is null", what); return SRJ_EINVAL; }
  if (fixed->type_id != SRJ_LIST || dst->type_id != SRJ_LIST || fixed->num_children < 1 || !fixed->children || dst->num_children < 1 || !dst->children) {
    set_error("%s: the time zone table must be LIST<STRUCT<INT64, INT64, INT32>> and LIST<INT32>", what);
    return SRJ_EINVAL;
  }
  if (fixed->size < 0 || fixed->size > INT32_MAX || dst->size != fixed->size) { set_error("%s: the time zone table's columns have mismatched row counts", what); return SRJ_EINVAL; }
  int rc = check_offsets(what, "transitions' list", *fixed);
  if (rc == SRJ_OK) rc = check_offsets(what, "DST rules' list", *dst);
  if (rc != SRJ_OK) return rc;
  const srj_column* s = &fixed->children[0];
  if (s->type_id != SRJ_STRUCT || s->num_children != 3 || !s->children) { set_error("%s: the transitions must be STRUCT<INT64, INT64, INT32>", what); return SRJ_EINVAL; }
  static const char* const names[3] = {"utcInstant", "localInstant", "offset"};
  for (int i = 0; i < 3; ++i) {
    rc = tz_check_flat(what, names[i], &s->children[i], i < 2 ? SRJ_INT64 : SRJ_INT32, -1, s->size);
    if (rc != SRJ_OK) return rc;
  }
  return tz_check_flat(what, "DST rules", &dst->children[0], SRJ_INT32, -1, dst->children[0].size);
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

static bool is_timestamp_64(int32_t t) { return t >= SRJ_TIMESTAMP_SECONDS && t <= SRJ_TIMESTAMP_NANOSECONDS; }

// an input of type t with rows > 0 needs its data and out at 8 bytes, and out_mask when it has a mask
static int tz_check_io(const char* what, const srj_column* in, const void* out, const uint32_t* out_mask)
{
  if (in->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (in->size == 0) return SRJ_OK;
  int rc = check_data(what, "input", *in);
  if (rc == SRJ_OK) rc = check_out(what, "output", out, 8);
  if (rc == SRJ_OK) rc = check_out_mask(what, in->null_mask || out_mask, out_mask);   // a mask given is written
  return rc;
}

// timezones.cu:80-111, 494-539
int srj_timezone_convert(int32_t direction, const srj_column* input, const srj_column* fixed_transitions, const srj_column* dst_rules,
                         int32_t tz_index, void* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "timezone_convert";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (direction != SRJ_TIMEZONE_TO_UTC && direction != SRJ_TIMEZONE_FROM_UTC) { set_error("%s: unknown direction %d", what, direction); return SRJ_EINVAL; }
  if (!is_timestamp_64(input->type_id)) { set_error("%s: Unsupported timestamp unit for timezone conversion (type id %d)", what, input->type_id); return SRJ_EUNSUPPORTED; }
  int rc = tz_check_table(what, fixed_transitions, dst_rules);
  if (rc != SRJ_OK) return rc;
  if (tz_index < 0 || tz_index >= fixed_transitions->size) {
    set_error("%s: time zone index %d is outside the table of %lld zones", what, tz_index, static_cast<long long>(fixed_transitions->size));
    return SRJ_EINVAL;
  }
  if ((rc = tz_check_io(what, input, out, out_mask)) != SRJ_OK) return rc;
  return launch_timezone_convert(direction == SRJ_TIMEZONE_TO_UTC, *input, *fixed_transitions, *dst_rules, tz_index, out, out_mask,
                                 static_cast<cudaStream_t>(stream));
}

// timezones.cu:186-240
int srj_timezone_convert_multi(const srj_column* seconds, const srj_column* micros, const srj_column* invalid, const srj_column* tz_type,
                               const srj_column* tz_offset, const srj_column* fixed_transitions, const srj_column* dst_rules,
                               const srj_column* tz_indices, int64_t* out, uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "timezone_convert_multi";
  if (!seconds || !null_count) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (seconds->type_id != SRJ_INT64) { set_error("%s: seconds column must be of type INT64", what); return SRJ_EUNSUPPORTED; }
  if (micros && micros->type_id != SRJ_INT32) { set_error("%s: microseconds column must be of type INT32", what); return SRJ_EUNSUPPORTED; }
  const int64_t n = seconds->size;
  if (n < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  int rc = tz_check_table(what, fixed_transitions, dst_rules);
  if (rc != SRJ_OK) return rc;
  const srj_column* cols[6] = {seconds, micros, invalid, tz_type, tz_offset, tz_indices};
  static const char* const names[6] = {"seconds", "microseconds", "invalid", "tz type", "tz offset", "tz indices"};
  static const int32_t types[6][2] = {{SRJ_INT64, -1}, {SRJ_INT32, -1}, {SRJ_BOOL8, SRJ_UINT8}, {SRJ_UINT8, -1}, {SRJ_INT32, -1}, {SRJ_INT32, -1}};
  for (int i = 0; i < 6; ++i)
    if ((rc = tz_check_flat(what, names[i], cols[i], types[i][0], types[i][1], n)) != SRJ_OK) return rc;
  if (n == 0) {
    *null_count = 0;
    return SRJ_OK;
  }
  if ((rc = check_out(what, "output", out, 8)) != SRJ_OK || (rc = check_out_mask(what, true, out_mask)) != SRJ_OK) return rc;
  const srj_column in[6] = {*seconds, *micros, *invalid, *tz_type, *tz_offset, *tz_indices};
  return launch_timezone_convert_multi(in, *fixed_transitions, *dst_rules, out, out_mask, null_count, static_cast<cudaStream_t>(stream));
}

// timezones.cu:380-486; a NULL table is a fixed offset
int srj_orc_convert_timezones(const srj_column* input, const srj_column* writer_transitions, const srj_column* writer_offsets,
                              int32_t writer_raw_offset, const srj_column* reader_transitions, const srj_column* reader_offsets,
                              int32_t reader_raw_offset, void* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "orc_convert_timezones";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (input->type_id != SRJ_TIMESTAMP_MICROSECONDS) { set_error("%s: Input column must be of type TIMESTAMP_MICROSECONDS", what); return SRJ_EUNSUPPORTED; }
  const srj_column* tr[2] = {writer_transitions, reader_transitions};
  const srj_column* of[2] = {writer_offsets, reader_offsets};
  int32_t rows[2]         = {0, 0};
  for (int i = 0; i < 2; ++i) {
    const char* side = i ? "reader" : "writer";
    if (!tr[i] && !of[i]) continue;
    if (!tr[i] || !of[i]) { set_error("%s: the %s table needs both its transitions and its offsets", what, side); return SRJ_EINVAL; }
    if (tr[i]->size < 0 || tr[i]->size > INT32_MAX) { set_error("%s: bad %s table size", what, side); return SRJ_EINVAL; }
    int rc = tz_check_flat(what, i ? "reader transitions" : "writer transitions", tr[i], SRJ_INT64, -1, tr[i]->size);
    if (rc == SRJ_OK) rc = tz_check_flat(what, i ? "reader offsets" : "writer offsets", of[i], SRJ_INT32, -1, tr[i]->size);
    if (rc != SRJ_OK) return rc;
    rows[i] = static_cast<int32_t>(tr[i]->size);
  }
  const int rc = tz_check_io(what, input, out, out_mask);
  if (rc != SRJ_OK) return rc;
  auto ptr64 = [&](int i) { return rows[i] ? static_cast<const int64_t*>(tr[i]->data) : nullptr; };
  auto ptr32 = [&](int i) { return rows[i] ? static_cast<const int32_t*>(of[i]->data) : nullptr; };
  return launch_orc_convert_timezones(*input, ptr64(0), ptr32(0), rows[0], writer_raw_offset, ptr64(1), ptr32(1), rows[1], reader_raw_offset, out,
                                      out_mask, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
