// histogram.cu -- Histogram.percentileFromHistogram and Histogram.createHistogramIfValid on the device (reference
// histogram.cu, Histogram.java): Spark's percentile(col, p [, freq]) and median(col) over cudf HISTOGRAM lists.
//
// percentile: each input row is a LIST<STRUCT<value T, count INT64>>.  Its non-null values are ordered by a 64-bit key
// that preserves T's order (signed: sign bit flipped; floats: the IEEE total order with every NaN one key above +inf,
// -0.0 before 0.0; BOOL8: != 0), their counts are summed in that order into acc, and percentage p reads the elements
// at ranks lower + 1 and higher + 1 (lower / higher = floor / ceil of (acc.last - 1) * p; the first element whose acc
// reaches the rank, or the last one when none does) and interpolates between them.  A value is recovered from its key.
//
// Rows are sorted into tiers by length in the size call (pct_classify_kernel, one appended list per tier):
//   <= kWarpCap  elements: one warp per row (pct_group_kernel<32>), 8 rows per CTA, each warp with its own 4 KB of shared
//                memory: load (nulls dropped), bitonic sort, scan, answer every percentage, write.
//   <= kCtaCap   elements: one 512-thread CTA per row (pct_group_kernel<512>), the same steps in 128 KB of shared memory.
//   >  kCtaCap   elements: a weighted radix select over the whole GPU (sel_*_kernel): per pass and target rank, a 256-bin
//                int64 histogram of the next key byte among the elements that still match the target's prefix (built
//                in shared memory, merged with global atomics), then one warp per target picks its bin.  One pass per key
//                byte (1 to 8); the 2P targets are lower + 1 and higher + 1 of each percentage, kSelGroup per group.
// No intermediate leaves the chip on the first two tiers: every element is read once.
//
// createHistogramIfValid: hc_flag_kernel flags negative and zero frequencies and counts what the output holds (read back
// once); hc_write_kernel writes values, mask, frequencies and, for lists, the offsets of the rows kept (an exclusive scan
// of the keep flags).
#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"

#include <vector>

namespace srj {
namespace {

constexpr int kWarpCap    = 256;    // elements of a row sorted by one warp (4 KB of keys and counts)
constexpr int kWarpRows   = 8;      // warps (rows in flight) per CTA of the warp tier
constexpr int kCtaThreads = 512;
constexpr int kCtaCap     = SRJ_HISTOGRAM_CTA_ELEMENTS;   // K: elements of a row sorted by one CTA (64 KB of keys + 64 KB of counts)
constexpr int kSelGroup   = 16;     // targets per radix-select group (32 KB of shared bins)
constexpr int kSelThreads = 256;
constexpr int kRowThreads = 256;

struct PctHeader {
  int32_t count[3];                 // rows appended to the warp, CTA and select tiers
  int32_t empty;                    // 1: the rows reference no element (histogram.cu:170: every row null, one per row)
};

struct PctArgs {
  const int32_t* offsets;           // rows + 1 (offsets[0] may be > 0: a sliced list column)
  const uint8_t* values;
  const uint32_t* vmask;            // NULL: no null values
  const int64_t* counts;
  const double* pct;                // device copy of the percentages
  const int32_t* pos;               // rows + 1: exclusive scan of the valid-row flags
  const int32_t* list;              // this tier's rows
  const int32_t* list_count;
  double* out;
  int32_t type, P, lists;
};

__device__ __forceinline__ bool bit_at(const uint32_t* m, int64_t i) { return (__ldg(m + (i >> 5)) >> (i & 31)) & 1u; }

__device__ __forceinline__ uint64_t to_key(const uint8_t* v, int64_t i, int type)
{
  switch (type) {
    case SRJ_INT8: return static_cast<uint8_t>(__ldg(v + i) ^ 0x80u);
    case SRJ_INT16: return static_cast<uint16_t>(__ldg(reinterpret_cast<const uint16_t*>(v) + i) ^ 0x8000u);
    case SRJ_INT32: return __ldg(reinterpret_cast<const uint32_t*>(v) + i) ^ 0x80000000u;
    case SRJ_INT64: return __ldg(reinterpret_cast<const unsigned long long*>(v) + i) ^ 0x8000000000000000ull;
    case SRJ_UINT8: return __ldg(v + i);
    case SRJ_UINT16: return __ldg(reinterpret_cast<const uint16_t*>(v) + i);
    case SRJ_UINT32: return __ldg(reinterpret_cast<const uint32_t*>(v) + i);
    case SRJ_UINT64: return __ldg(reinterpret_cast<const unsigned long long*>(v) + i);
    case SRJ_FLOAT32: {
      const uint32_t b = __ldg(reinterpret_cast<const uint32_t*>(v) + i);
      if ((b & 0x7fffffffu) > 0x7f800000u) return 0xffc00000u;                  // every NaN: the canonical one's key
      return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    }
    case SRJ_FLOAT64: {
      const uint64_t b = __ldg(reinterpret_cast<const unsigned long long*>(v) + i);
      if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return 0xfff8000000000000ull;
      return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
    }
    default: return __ldg(v + i) != 0;                                              // BOOL8
  }
}

__device__ __forceinline__ double key_value(uint64_t k, int type)
{
  switch (type) {
    case SRJ_INT8: return static_cast<int8_t>(static_cast<uint8_t>(k ^ 0x80u));
    case SRJ_INT16: return static_cast<int16_t>(static_cast<uint16_t>(k ^ 0x8000u));
    case SRJ_INT32: return static_cast<int32_t>(static_cast<uint32_t>(k ^ 0x80000000u));
    case SRJ_INT64: return static_cast<double>(static_cast<int64_t>(k ^ 0x8000000000000000ull));
    case SRJ_FLOAT32: {
      const uint32_t b = static_cast<uint32_t>(k);
      return __uint_as_float((b & 0x80000000u) ? (b ^ 0x80000000u) : ~b);
    }
    case SRJ_FLOAT64: return __longlong_as_double(static_cast<long long>((k & 0x8000000000000000ull) ? (k ^ 0x8000000000000000ull) : ~k));
    default: return static_cast<double>(k);                                         // unsigned, BOOL8
  }
}

struct Ranks {
  double position;
  int64_t lower, higher;
};

__device__ __forceinline__ Ranks ranks_of(int64_t last, double p)
{
  Ranks r;
  r.position = static_cast<double>(last - 1) * p;
  r.lower    = static_cast<int64_t>(floor(r.position));
  r.higher   = static_cast<int64_t>(ceil(r.position));
  return r;
}

// histogram.cu:79-99; the two products are rounded separately, as the reference's volatile parts are
__device__ __forceinline__ double combine(int type, const Ranks& r, uint64_t klo, uint64_t khi)
{
  const double lo = key_value(klo, type);
  if (r.higher == r.lower) return lo;
  const double hi = key_value(khi, type);
  const bool eq   = (type == SRJ_FLOAT32 || type == SRJ_FLOAT64) ? lo == hi : klo == khi;   // equality in T
  if (eq) return lo;
  return __dadd_rn(__dmul_rn(__dsub_rn(static_cast<double>(r.higher), r.position), lo),
                   __dmul_rn(__dsub_rn(r.position, static_cast<double>(r.lower)), hi));
}

template <int G>
__device__ __forceinline__ void gsync()
{
  if constexpr (G == 32) __syncwarp();
  else __syncthreads();
}

// exclusive scan of one int64 per thread over a group of G threads; tmp: 32 int64 of shared memory (G > 32 only)
template <int G>
__device__ __forceinline__ int64_t group_excl_scan(int64_t v, int64_t* tmp, int t)
{
  const int lane = t & 31;
  int64_t x      = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(~0u, x, o);
    if (lane >= o) x += y;
  }
  if constexpr (G == 32) {
    return x - v;
  } else {
    const int w = t >> 5;
    if (lane == 31) tmp[w] = x;
    __syncthreads();
    if (w == 0) {
      const int64_t s0 = lane < G / 32 ? tmp[lane] : 0;
      int64_t s        = s0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(~0u, s, o);
        if (lane >= o) s += y;
      }
      if (lane < G / 32) tmp[lane] = s - s0;
    }
    __syncthreads();
    const int64_t r = x - v + tmp[w];
    __syncthreads();
    return r;
  }
}

// bitonic order: key ascending; among equal keys a padding entry (count 0) never precedes a nonzero count
__device__ __forceinline__ bool after(uint64_t ka, int64_t ca, uint64_t kb, int64_t cb)
{
  return ka > kb || (ka == kb && ca == 0 && cb != 0);
}

// One row by a group of G threads (t = the thread's index in the group): keys / cnt hold `cap` entries.
template <int G>
__device__ void group_row(const PctArgs& a, int32_t row, uint64_t* keys, int64_t* cnt, int* s_n, int64_t* tmp, int t)
{
  const int32_t s = __ldg(a.offsets + row), e = __ldg(a.offsets + row + 1);
  const int lane  = t & 31;
  if (t == 0) *s_n = 0;
  gsync<G>();
  for (int64_t i0 = s; i0 < e; i0 += G) {                       // uniform per warp: the ballot sees every lane
    const int64_t i    = i0 + t;
    const bool v       = i < e && (!a.vmask || bit_at(a.vmask, i));
    const unsigned b   = __ballot_sync(~0u, v);
    int base           = 0;
    if (lane == 0 && b) base = atomicAdd(s_n, __popc(b));
    base = __shfl_sync(~0u, base, 0);
    if (v) {
      const int k = base + __popc(b & ((1u << lane) - 1u));
      keys[k]     = to_key(a.values, i, a.type);
      cnt[k]      = __ldg(a.counts + i);
    }
  }
  gsync<G>();
  const int nv = *s_n;                                          // >= 1: the row is valid
  int m        = 1;
  while (m < nv) m <<= 1;
  for (int k = nv + t; k < m; k += G) {
    keys[k] = ~0ull;
    cnt[k]  = 0;
  }
  gsync<G>();
  for (int k = 2; k <= m; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < (m >> 1); i += G) {
        const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1));
        const int hi = lo + j;
        const uint64_t ka = keys[lo], kb = keys[hi];
        const int64_t ca = cnt[lo], cb = cnt[hi];
        if (after(ka, ca, kb, cb) == ((lo & k) == 0)) {
          keys[lo] = kb; keys[hi] = ka;
          cnt[lo]  = cb; cnt[hi]  = ca;
        }
      }
      gsync<G>();
    }
  }
  // inclusive scan of the counts: thread t owns a contiguous chunk
  const int chunk = (nv + G - 1) / G;
  const int b0 = tmin(t * chunk, nv), b1 = tmin(b0 + chunk, nv);
  int64_t sum = 0;
  for (int k = b0; k < b1; ++k) sum += cnt[k];
  int64_t run = group_excl_scan<G>(sum, tmp, t);
  for (int k = b0; k < b1; ++k) {
    run += cnt[k];
    cnt[k] = run;
  }
  gsync<G>();
  const int64_t last = cnt[nv - 1];
  double* out        = a.out + static_cast<int64_t>(a.lists ? __ldg(a.pos + row) : row) * a.P;
  auto lower_bound   = [&](int64_t target) {
    int lo = 0, hi = nv;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cnt[mid] < target) lo = mid + 1;
      else hi = mid;
    }
    return tmin(lo, nv - 1);
  };
  for (int q = t; q < a.P; q += G) {
    const Ranks r      = ranks_of(last, __ldg(a.pct + q));
    const uint64_t klo = keys[lower_bound(r.lower + 1)];
    const uint64_t khi = r.higher == r.lower ? klo : keys[lower_bound(r.higher + 1)];
    out[q]             = combine(a.type, r, klo, khi);
  }
  gsync<G>();                                                   // the next row reuses keys / cnt / s_n
}

template <int G>
__global__ void __launch_bounds__(G == 32 ? 32 * kWarpRows : G) pct_group_kernel(const __grid_constant__ PctArgs a)
{
  constexpr int kGroups = G == 32 ? kWarpRows : 1;
  constexpr int kCap    = G == 32 ? kWarpCap : kCtaCap;
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ int64_t s_tmp[32];
  __shared__ int s_n[kGroups];
  const int grp  = G == 32 ? static_cast<int>(threadIdx.x >> 5) : 0;
  const int t    = G == 32 ? static_cast<int>(threadIdx.x & 31) : static_cast<int>(threadIdx.x);
  auto* keys     = reinterpret_cast<uint64_t*>(smem) + static_cast<int64_t>(grp) * kCap;
  auto* cnt      = reinterpret_cast<int64_t*>(smem) + static_cast<int64_t>(kGroups) * kCap + static_cast<int64_t>(grp) * kCap;
  const int32_t n = *a.list_count;
  for (int32_t it = blockIdx.x * kGroups + grp; it < n; it += gridDim.x * kGroups)
    group_row<G>(a, __ldg(a.list + it), keys, cnt, s_n + grp, s_tmp, t);
}

// one thread per row: valid flag (some non-null element, and P > 0) and the row's tier list
struct ClassifyArgs {
  const int32_t* offsets;
  const uint32_t* vmask;
  int64_t rows;
  int32_t P;
  int32_t* flag;          // rows: 1 for a valid row (scanned into positions afterwards)
  int32_t* list[3];
  PctHeader* hdr;
  int4* large;            // select tier: {row, start, end, 0}
};

__global__ void __launch_bounds__(kRowThreads) pct_classify_kernel(const __grid_constant__ ClassifyArgs a)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  const int lane  = lane_id();
  bool valid      = false;
  int tier        = 0;
  int32_t s = 0, e = 0;
  if (r < a.rows) {
    s     = __ldg(a.offsets + r);
    e     = __ldg(a.offsets + r + 1);
    valid = a.P > 0 && e > s;
    if (valid && a.vmask) {                                    // the first word holding a valid bit ends the search
      valid = false;
      for (int64_t w = s >> 5; w <= static_cast<int64_t>(e - 1) >> 5 && !valid; ++w) {
        uint32_t m = __ldg(a.vmask + w);
        if (w == (s >> 5)) m &= ~0u << (s & 31);
        if (w == (static_cast<int64_t>(e - 1) >> 5)) m &= ~0u >> (31 - ((e - 1) & 31));
        valid = m != 0;
      }
    }
    a.flag[r] = valid;
    tier      = e - s <= kWarpCap ? 0 : e - s <= kCtaCap ? 1 : 2;
    if (r == 0) a.hdr->empty = __ldg(a.offsets + a.rows) == s;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const unsigned b = __ballot_sync(~0u, valid && tier == k);
    if (!b) continue;
    int base = 0;
    if (lane == __ffs(b) - 1) base = atomicAdd(&a.hdr->count[k], __popc(b));
    base = __shfl_sync(~0u, base, __ffs(b) - 1);
    if (valid && tier == k) {
      const int at = base + __popc(b & ((1u << lane) - 1u));
      a.list[k][at] = static_cast<int32_t>(r);
      if (k == 2) a.large[at] = make_int4(static_cast<int>(r), s, e, 0);
    }
  }
}

// one thread per row: the row mask (list output, or one double per row), list offsets (pos * P), zeros under the null
// rows of the flat output (`stride` doubles per row)
__global__ void __launch_bounds__(kRowThreads) pct_rows_kernel(const int32_t* pos, int64_t rows, int32_t P, int32_t stride, int32_t lists,
                                                               double* out, uint32_t* out_mask, int32_t* out_offsets)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  const bool live = r < rows;
  const bool v    = live && pos[r + 1] > pos[r];
  const unsigned b = __ballot_sync(~0u, v);
  if (live && lane_id() == 0 && (lists || stride == 1)) out_mask[r >> 5] = b;
  if (!live) return;
  if (lists) {
    out_offsets[r] = pos[r] * P;
    if (r == rows - 1) out_offsets[rows] = pos[rows] * P;
  } else if (!v) {
    for (int q = 0; q < stride; ++q) out[r * stride + q] = 0.0;
  }
}

// flat output with stride > 1 doubles per row: one thread per output mask word, bit i set when row i / stride is valid
__global__ void __launch_bounds__(kRowThreads) pct_flat_mask_kernel(const int32_t* pos, int64_t values, int32_t stride, uint32_t* out_mask)
{
  const int64_t w = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  if (w >= (values + 31) / 32) return;
  // values <= INT32_MAX: one 32-bit division per word, then the row advances every `stride` bits
  const uint32_t e0 = static_cast<uint32_t>(32 * w);
  uint32_t r = e0 / static_cast<uint32_t>(stride), q = e0 - r * static_cast<uint32_t>(stride);
  bool v     = pos[r + 1] > pos[r];
  uint32_t m = 0;
  for (int b = 0; b < 32 && e0 + b < values; ++b) {
    if (v) m |= 1u << b;
    if (++q == static_cast<uint32_t>(stride) && e0 + b + 1 < values) {
      q = 0;
      ++r;
      v = pos[r + 1] > pos[r];
    }
  }
  out_mask[w] = m;
}

// ---- radix select (rows longer than kCtaCap) -----------------------------------------------------------------------
struct SelState {
  unsigned long long* total;     // acc.last of the row
  unsigned long long* prefix;    // [2P] key bits chosen so far
  long long* rem;                // [2P] rank still to find inside the chosen prefix
  unsigned long long* bins;      // [kSelGroup][256] weights
  uint32_t* pres;                // [kSelGroup][8] bins holding at least one element
};

__global__ void __launch_bounds__(kSelThreads) sel_total_kernel(const uint32_t* vmask, const int64_t* counts, int32_t s, int32_t e,
                                                                unsigned long long* total)
{
  int64_t sum = 0;
  for (int64_t i = s + static_cast<int64_t>(blockIdx.x) * kSelThreads + threadIdx.x; i < e; i += static_cast<int64_t>(gridDim.x) * kSelThreads)
    if (!vmask || bit_at(vmask, i)) sum += __ldg(counts + i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(~0u, sum, o);
  if (lane_id() == 0 && sum) atomicAdd(total, static_cast<unsigned long long>(sum));
}

__global__ void __launch_bounds__(kSelThreads) sel_init_kernel(const double* pct, int32_t P, SelState st)
{
  const int j = blockIdx.x * kSelThreads + threadIdx.x;
  if (j >= 2 * P) return;
  const Ranks r = ranks_of(static_cast<int64_t>(*st.total), pct[j >> 1]);
  st.prefix[j]  = 0;
  st.rem[j]     = ((j & 1) ? r.higher : r.lower) + 1;
}

// weights of key byte `shift / 8` among the elements matching each target's prefix above it; targets [j0, j0 + g)
__global__ void __launch_bounds__(kSelThreads) sel_hist_kernel(const uint8_t* values, const uint32_t* vmask, const int64_t* counts, int type,
                                                               int32_t s, int32_t e, int32_t j0, int32_t g, int32_t shift, SelState st)
{
  __shared__ unsigned long long s_bins[kSelGroup * 256];
  __shared__ uint32_t s_pres[kSelGroup * 8];
  __shared__ unsigned long long s_pref[kSelGroup];
  for (int i = threadIdx.x; i < g * 256; i += kSelThreads) s_bins[i] = 0;
  for (int i = threadIdx.x; i < g * 8; i += kSelThreads) s_pres[i] = 0;
  if (threadIdx.x < g) s_pref[threadIdx.x] = st.prefix[j0 + threadIdx.x];
  __syncthreads();
  for (int64_t i = s + static_cast<int64_t>(blockIdx.x) * kSelThreads + threadIdx.x; i < e; i += static_cast<int64_t>(gridDim.x) * kSelThreads) {
    if (vmask && !bit_at(vmask, i)) continue;
    const uint64_t k = to_key(values, i, type);
    const int64_t c  = __ldg(counts + i);
    const int d      = static_cast<int>((k >> shift) & 255u);
    for (int j = 0; j < g; ++j) {
      if (shift + 8 < 64 && ((k ^ s_pref[j]) >> (shift + 8)) != 0) continue;
      if (c) atomicAdd(&s_bins[j * 256 + d], static_cast<unsigned long long>(c));
      const uint32_t bit = 1u << (d & 31);
      if (!(s_pres[j * 8 + (d >> 5)] & bit)) atomicOr(&s_pres[j * 8 + (d >> 5)], bit);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < g * 256; i += kSelThreads)
    if (s_bins[i]) atomicAdd(&st.bins[i], s_bins[i]);
  for (int i = threadIdx.x; i < g * 8; i += kSelThreads)
    if (s_pres[i]) atomicOr(&st.pres[i], s_pres[i]);
}

// one warp per target: the first bin holding an element whose running weight reaches the rank, else the last bin
// holding one; the target's prefix takes the bin and its rank loses the weight before it.  Clears the bins it read.
__global__ void __launch_bounds__(32 * kSelGroup) sel_pick_kernel(int32_t j0, int32_t g, int32_t shift, SelState st)
{
  const int j = threadIdx.x >> 5, lane = lane_id();
  if (j >= g) return;
  unsigned long long* bins = st.bins + j * 256 + lane * 8;
  const uint32_t present   = (st.pres[j * 8 + (lane >> 2)] >> (8 * (lane & 3))) & 0xffu;
  int64_t w[8];
  int64_t sum = 0;
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    w[d] = static_cast<int64_t>(bins[d]);
    sum += w[d];
  }
  int64_t run = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(~0u, run, o);
    if (lane >= o) run += y;
  }
  run -= sum;                                                   // weight of the bins before this lane's
  const int64_t rem = st.rem[j0 + j];
  int found = -1, last = -1;
  int64_t before_found = 0, before_last = 0;
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    if ((present >> d) & 1u) {
      if (found < 0 && run + w[d] >= rem) { found = d; before_found = run; }
      last = d;
      before_last = run;
    }
    run += w[d];
  }
  const unsigned bf = __ballot_sync(~0u, found >= 0);
  const unsigned bl = __ballot_sync(~0u, last >= 0);
  const int src     = bf ? __ffs(bf) - 1 : 31 - __clz(bl);
  const int digit   = __shfl_sync(~0u, bf ? found : last, src) + 8 * src;
  const int64_t bef = __shfl_sync(~0u, bf ? before_found : before_last, src);
  if (lane == 0) {
    st.prefix[j0 + j] |= static_cast<unsigned long long>(digit) << shift;
    st.rem[j0 + j] = rem - bef;
  }
#pragma unroll
  for (int d = 0; d < 8; ++d) bins[d] = 0;
  if (lane < 8) st.pres[j * 8 + lane] = 0;
}

__global__ void __launch_bounds__(kSelThreads) sel_finish_kernel(const double* pct, int32_t P, int type, int32_t row, const int32_t* pos,
                                                                 int32_t lists, double* out, SelState st)
{
  const int q = blockIdx.x * kSelThreads + threadIdx.x;
  if (q >= P) return;
  const Ranks r = ranks_of(static_cast<int64_t>(*st.total), pct[q]);
  out[static_cast<int64_t>(lists ? pos[row] : row) * P + q] = combine(type, r, st.prefix[2 * q], st.prefix[2 * q + 1]);
}

// ---- createHistogramIfValid ------------------------------------------------------------------------------------------
struct HcHeader {
  unsigned long long kept;          // rows with frequency > 0
  unsigned long long struct_nulls;  // rows whose value is null or whose frequency is 0
  unsigned long long list_nulls;    // kept rows whose value is null
  uint32_t negative, zero;
};

__global__ void __launch_bounds__(kRowThreads) hc_flag_kernel(const int64_t* freq, const uint32_t* vmask, int64_t rows, int32_t* keep,
                                                              HcHeader* h)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  const bool live = r < rows;
  const int64_t f = live ? __ldg(freq + r) : 1;
  const bool vv   = !live || !vmask || bit_at(vmask, r);
  if (live) keep[r] = f > 0;
  const unsigned kept = __ballot_sync(~0u, live && f > 0);
  const unsigned sn   = __ballot_sync(~0u, live && (!vv || f == 0));
  const unsigned ln   = __ballot_sync(~0u, live && f > 0 && !vv);
  const unsigned neg  = __ballot_sync(~0u, f < 0);
  const unsigned zero = __ballot_sync(~0u, live && f == 0);
  if (lane_id() == 0) {
    if (kept) atomicAdd(&h->kept, static_cast<unsigned long long>(__popc(kept)));
    if (sn) atomicAdd(&h->struct_nulls, static_cast<unsigned long long>(__popc(sn)));
    if (ln) atomicAdd(&h->list_nulls, static_cast<unsigned long long>(__popc(ln)));
    if (neg) atomicOr(&h->negative, 1u);
    if (zero) atomicOr(&h->zero, 1u);
  }
}

__device__ __forceinline__ void copy_elem(const uint8_t* src, uint8_t* dst, int64_t from, int64_t to, int w)
{
  switch (w) {
    case 1: dst[to] = __ldg(src + from); break;
    case 2: reinterpret_cast<uint16_t*>(dst)[to] = __ldg(reinterpret_cast<const uint16_t*>(src) + from); break;
    case 4: reinterpret_cast<uint32_t*>(dst)[to] = __ldg(reinterpret_cast<const uint32_t*>(src) + from); break;
    case 8: reinterpret_cast<unsigned long long*>(dst)[to] = __ldg(reinterpret_cast<const unsigned long long*>(src) + from); break;
    default: {                                                  // 16 bytes as two longs (8-byte alignment only)
      const auto* s = reinterpret_cast<const unsigned long long*>(src) + 2 * from;
      auto* d       = reinterpret_cast<unsigned long long*>(dst) + 2 * to;
      d[0] = __ldg(s);
      d[1] = __ldg(s + 1);
    }
  }
}

struct HcWriteArgs {
  const uint8_t* values;
  const uint32_t* vmask;
  const int64_t* freq;
  const int32_t* pos;               // lists: exclusive scan of the keep flags, rows + 1
  const HcHeader* h;
  int64_t rows;
  int32_t width, lists;
  uint8_t* out_values;
  uint32_t* out_mask;               // lists: zeroed by the caller; NULL when no mask is written
  int64_t* out_freq;
  int32_t* out_offsets;
};

__global__ void __launch_bounds__(kRowThreads) hc_write_kernel(const __grid_constant__ HcWriteArgs a)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  const int lane  = lane_id();
  const bool live = r < a.rows;
  const int64_t f = live ? __ldg(a.freq + r) : 0;
  const bool vv   = live && (!a.vmask || bit_at(a.vmask, r));
  if (!a.lists) {                                               // histogram.cu:328-372, 403-411
    const bool ok    = vv && f != 0;
    const unsigned b = __ballot_sync(~0u, ok);
    if (!live) return;
    if (a.out_mask && lane == 0) a.out_mask[r >> 5] = b;
    copy_elem(a.values, a.out_values, r, r, a.width);
    a.out_freq[r] = (a.h->zero && !ok) ? 1 : f;
    return;
  }
  // histogram.cu:374-402: rows with frequency 0 leave the child; the child keeps the values' nulls and the frequencies
  const int32_t p  = live ? a.pos[r] : 0;
  const bool kept  = live && f > 0;
  if (kept) {
    copy_elem(a.values, a.out_values, r, p, a.width);
    a.out_freq[p] = f;
  }
  if (a.out_mask) {
    const bool set       = kept && vv;
    const unsigned word  = set ? static_cast<unsigned>(p >> 5) : 0x80000000u | lane;   // lanes setting nothing: unique
    const unsigned peers = __match_any_sync(~0u, word);
    const unsigned bits  = __reduce_or_sync(peers, set ? 1u << (p & 31) : 0u);
    if (set && lane == __ffs(peers) - 1) atomicOr(a.out_mask + word, bits);
  }
  if (!live) return;
  a.out_offsets[r] = p;
  if (r == a.rows - 1) a.out_offsets[a.rows] = p + (kept ? 1 : 0);
}

// the list child's mask words: ceil(*kept / 32) of them (kept = the scanned keep flags' total)
__global__ void __launch_bounds__(kRowThreads) hc_clear_mask_kernel(const int32_t* kept, uint32_t* out_mask)
{
  const int64_t w = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  if (w < (static_cast<int64_t>(*kept) + 31) / 32) out_mask[w] = 0;
}

// ---- workspaces --------------------------------------------------------------------------------------------------------
struct PctWs {
  PctHeader* hdr;
  double* pct;
  int32_t* pos;                     // rows + 1
  int32_t* sums;
  int32_t* list[3];
  int4* large;
  SelState sel;
};

int64_t large_capacity(int64_t rows, int64_t elements) { return tmin(rows, elements / (kCtaCap + 1)) + 1; }

int64_t pct_layout(int64_t rows, int64_t elements, int32_t P, uint8_t* base, PctWs* w)
{
  int64_t o = 0;
  auto take = [&](int64_t bytes) { uint8_t* p = base ? base + o : nullptr; o += round_up64(bytes, 256); return p; };
  const int64_t cap = large_capacity(rows, elements);
  PctWs x{};
  x.hdr        = reinterpret_cast<PctHeader*>(take(sizeof(PctHeader)));
  x.pct        = reinterpret_cast<double*>(take(8 * tmax<int64_t>(P, 1)));
  x.pos        = reinterpret_cast<int32_t*>(take(4 * (rows + 1)));
  x.sums       = reinterpret_cast<int32_t*>(take(4 * tmax<int64_t>(i32_scan_nchunks(rows), 1)));
  for (auto& l : x.list) l = reinterpret_cast<int32_t*>(take(4 * tmax<int64_t>(rows, 1)));
  x.large      = reinterpret_cast<int4*>(take(16 * cap));
  x.sel.total  = reinterpret_cast<unsigned long long*>(take(8));
  x.sel.prefix = reinterpret_cast<unsigned long long*>(take(16 * tmax<int64_t>(P, 1)));
  x.sel.rem    = reinterpret_cast<long long*>(take(16 * tmax<int64_t>(P, 1)));
  x.sel.bins   = reinterpret_cast<unsigned long long*>(take(8 * kSelGroup * 256));
  x.sel.pres   = reinterpret_cast<uint32_t*>(take(4 * kSelGroup * 8));
  if (w) *w = x;
  return o;
}

int64_t hc_layout(int64_t rows, uint8_t* base, HcHeader** h, int32_t** keep, int32_t** sums)
{
  int64_t o = 0;
  auto take = [&](int64_t bytes) { uint8_t* p = base ? base + o : nullptr; o += round_up64(bytes, 256); return p; };
  auto* hh  = reinterpret_cast<HcHeader*>(take(sizeof(HcHeader)));
  auto* kk  = reinterpret_cast<int32_t*>(take(4 * (rows + 1)));
  auto* ss  = reinterpret_cast<int32_t*>(take(4 * tmax<int64_t>(i32_scan_nchunks(rows), 1)));
  if (h) { *h = hh; *keep = kk; *sums = ss; }
  return o;
}

unsigned row_grid(int64_t rows) { return static_cast<unsigned>((rows + kRowThreads - 1) / kRowThreads); }

}  // namespace

static int launch_pct_classify(const srj_column& list, const srj_column& vals, int64_t elements, int32_t P, int32_t lists, const PctWs& w,
                               int64_t* valid_rows, int64_t* num_values, cudaStream_t stream)
{
  const int64_t rows = list.size;
  SRJ_CUDA_TRY(cudaMemsetAsync(w.hdr, 0, sizeof(PctHeader), stream));
  ClassifyArgs a{};
  a.offsets = list.offsets;
  a.vmask   = elements > 0 ? vals.null_mask : nullptr;
  a.rows    = rows;
  a.P       = P;
  a.flag    = w.pos;
  for (int k = 0; k < 3; ++k) a.list[k] = w.list[k];
  a.hdr   = w.hdr;
  a.large = w.large;
  pct_classify_kernel<<<row_grid(rows), kRowThreads, 0, stream>>>(a);
  SRJ_CUDA_TRY(cudaGetLastError());
  const int rc = launch_i32_exclusive_scan(w.pos, rows, w.sums, w.pos + rows, stream);
  if (rc != SRJ_OK) return rc;
  int32_t total = 0;
  PctHeader h{};
  SRJ_CUDA_TRY(cudaMemcpyAsync(&total, w.pos + rows, 4, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaMemcpyAsync(&h, w.hdr, sizeof(h), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  *valid_rows = total;
  *num_values = lists ? total * static_cast<int64_t>(P) : (h.empty || P == 0) ? rows : rows * P;
  return SRJ_OK;
}

static int launch_pct_fill(const srj_column& list, const srj_column& vals, const srj_column& counts, const double* h_pct, int32_t P,
                           int32_t lists, double* out, uint32_t* out_mask, int32_t* out_offsets, const PctWs& w, cudaStream_t stream)
{
  const int64_t rows = list.size;
  PctHeader h{};
  // the header and the whole select-tier list (at most one 16-byte entry per kCtaCap + 1 elements) in one read-back
  std::vector<int4> large(static_cast<size_t>(large_capacity(rows, vals.size)));
  SRJ_CUDA_TRY(cudaMemcpyAsync(&h, w.hdr, sizeof(h), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaMemcpyAsync(large.data(), w.large, 16 * large.size(), cudaMemcpyDeviceToHost, stream));
  if (P > 0) SRJ_CUDA_TRY(cudaMemcpyAsync(w.pct, h_pct, 8 * static_cast<size_t>(P), cudaMemcpyHostToDevice, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  PctArgs a{};
  a.offsets = list.offsets;
  a.values  = static_cast<const uint8_t*>(vals.data);
  a.vmask   = vals.null_mask;
  a.counts  = static_cast<const int64_t*>(counts.data);
  a.pct     = w.pct;
  a.pos     = w.pos;
  a.out     = out;
  a.type    = vals.type_id;
  a.P       = P;
  a.lists   = lists;
  const int sms = sm_count();
  if (h.count[0] > 0) {
    a.list       = w.list[0];
    a.list_count = &w.hdr->count[0];
    const size_t smem = static_cast<size_t>(kWarpRows) * kWarpCap * 16;
    const unsigned grid = static_cast<unsigned>(tmin<int64_t>((h.count[0] + kWarpRows - 1) / kWarpRows, static_cast<int64_t>(sms) * 8));
    pct_group_kernel<32><<<grid, 32 * kWarpRows, smem, stream>>>(a);
    SRJ_CUDA_TRY(cudaGetLastError());
  }
  if (h.count[1] > 0) {
    a.list       = w.list[1];
    a.list_count = &w.hdr->count[1];
    const size_t smem = static_cast<size_t>(kCtaCap) * 16;
    SRJ_CUDA_TRY(cudaFuncSetAttribute(pct_group_kernel<kCtaThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    const unsigned grid = static_cast<unsigned>(tmin<int64_t>(h.count[1], sms));
    pct_group_kernel<kCtaThreads><<<grid, kCtaThreads, smem, stream>>>(a);
    SRJ_CUDA_TRY(cudaGetLastError());
  }
  const int32_t stride = (h.empty || P == 0) ? 1 : P;
  pct_rows_kernel<<<row_grid(rows), kRowThreads, 0, stream>>>(w.pos, rows, P, stride, lists, out, out_mask, out_offsets);
  if (!lists && stride > 1) pct_flat_mask_kernel<<<row_grid((rows * stride + 31) / 32), kRowThreads, 0, stream>>>(w.pos, rows * stride, stride, out_mask);
  SRJ_CUDA_TRY(cudaGetLastError());
  if (h.count[2] == 0) return SRJ_OK;
  large.resize(static_cast<size_t>(h.count[2]));
  SRJ_CUDA_TRY(cudaMemsetAsync(w.sel.bins, 0, 8 * kSelGroup * 256, stream));
  SRJ_CUDA_TRY(cudaMemsetAsync(w.sel.pres, 0, 4 * kSelGroup * 8, stream));
  const int nbytes = type_width(vals.type_id);
  for (const int4& L : large) {
    const int32_t s = L.y, e = L.z;
    const unsigned grid = static_cast<unsigned>(tmin<int64_t>((e - s + kSelThreads * 8 - 1) / (kSelThreads * 8), static_cast<int64_t>(sms) * 4));
    SRJ_CUDA_TRY(cudaMemsetAsync(w.sel.total, 0, 8, stream));
    sel_total_kernel<<<grid, kSelThreads, 0, stream>>>(vals.null_mask, a.counts, s, e, w.sel.total);
    sel_init_kernel<<<static_cast<unsigned>((2 * P + kSelThreads - 1) / kSelThreads), kSelThreads, 0, stream>>>(w.pct, P, w.sel);
    for (int32_t j0 = 0; j0 < 2 * P; j0 += kSelGroup) {
      const int32_t g = tmin(kSelGroup, 2 * P - j0);
      for (int b = nbytes - 1; b >= 0; --b) {
        sel_hist_kernel<<<grid, kSelThreads, 0, stream>>>(a.values, vals.null_mask, a.counts, vals.type_id, s, e, j0, g, 8 * b, w.sel);
        sel_pick_kernel<<<1, 32 * kSelGroup, 0, stream>>>(j0, g, 8 * b, w.sel);
      }
    }
    sel_finish_kernel<<<static_cast<unsigned>((P + kSelThreads - 1) / kSelThreads), kSelThreads, 0, stream>>>(w.pct, P, vals.type_id, L.x, w.pos,
                                                                                                              lists, out, w.sel);
    SRJ_CUDA_TRY(cudaGetLastError());
  }
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

static bool pct_value_type(int32_t t)
{
  switch (t) {
    case SRJ_INT8: case SRJ_INT16: case SRJ_INT32: case SRJ_INT64: case SRJ_UINT8: case SRJ_UINT16: case SRJ_UINT32: case SRJ_UINT64:
    case SRJ_FLOAT32: case SRJ_FLOAT64: case SRJ_BOOL8: return true;
    default: return false;
  }
}

// histogram.cu:226-249 in its order, then the value type (histogram.cu:138-156), then this library's buffer checks.
// A null mask counts as nulls: pass NULL for a column without nulls.
static int pct_check(const char* what, const srj_column* input, int32_t P, const srj_column** vals, const srj_column** counts)
{
  if (!input || P < 0 || input->size < 0) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (input->type_id != SRJ_LIST) { set_error("%s: The input column must be of type LIST.", what); return SRJ_EINVAL; }
  if (input->num_children != 1 || !input->children) { set_error("%s: the LIST column has no child", what); return SRJ_EINVAL; }
  const srj_column& child = input->children[0];
  if (child.null_mask) { set_error("%s: Child of the input column must not have nulls.", what); return SRJ_EINVAL; }
  if (child.type_id != SRJ_STRUCT || child.num_children != 2 || !child.children) {
    set_error("%s: Child of the input column must be of STRUCT type having two children.", what);
    return SRJ_EINVAL;
  }
  const srj_column& v = child.children[0];
  const srj_column& c = child.children[1];
  if (c.null_mask) { set_error("%s: Child of the input column must have its second child containing non-null elements.", what); return SRJ_EINVAL; }
  if (c.type_id != SRJ_INT64) { set_error("%s: Child of the input column must have its second child of type INT64.", what); return SRJ_EINVAL; }
  if (input->size * static_cast<int64_t>(P) > INT32_MAX) { set_error("%s: Size of output exceeds cudf column size limit.", what); return SRJ_EOVERFLOW; }
  if (!pct_value_type(v.type_id)) { set_error("%s: Unsupported type in histogram-to-percentile evaluation.", what); return SRJ_EUNSUPPORTED; }
  if (v.size != child.size || c.size != child.size || child.size > INT32_MAX) {
    set_error("%s: the histogram values (%lld), counts (%lld) and structs (%lld) differ in size", what, static_cast<long long>(v.size),
              static_cast<long long>(c.size), static_cast<long long>(child.size));
    return SRJ_EINVAL;
  }
  int rc = SRJ_OK;
  if (input->size > 0 && (rc = check_offsets(what, "input", *input)) != SRJ_OK) return rc;
  if ((rc = check_data(what, "values", v)) != SRJ_OK) return rc;
  if ((rc = check_data(what, "counts", c)) != SRJ_OK) return rc;
  if (v.null_mask && !aligned_to(v.null_mask, 4)) { set_error("%s: the values mask is not 4-byte aligned", what); return SRJ_EINVAL; }
  *vals   = &v;
  *counts = &c;
  return SRJ_OK;
}

int64_t srj_percentile_workspace_bytes(int64_t num_rows, int64_t num_elements, int32_t num_percentages)
{
  return pct_layout(tmax<int64_t>(num_rows, 0), tmax<int64_t>(num_elements, 0), tmax(num_percentages, 0), nullptr, nullptr);
}

int srj_percentile_from_histogram_size(const srj_column* input, int32_t num_percentages, int32_t output_as_lists, int64_t* valid_rows,
                                       int64_t* num_values, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "percentile_from_histogram_size";
  const srj_column *v = nullptr, *c = nullptr;
  int rc = pct_check(what, input, num_percentages, &v, &c);
  if (rc != SRJ_OK) return rc;
  if (!valid_rows || !num_values) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *valid_rows = *num_values = 0;
  if (input->size == 0) return SRJ_OK;
  if ((rc = check_out(what, "workspace (srj_percentile_workspace_bytes)", workspace, 256)) != SRJ_OK) return rc;
  PctWs w{};
  pct_layout(input->size, v->size, num_percentages, static_cast<uint8_t*>(workspace), &w);
  return launch_pct_classify(*input, *v, v->size, num_percentages, output_as_lists != 0, w, valid_rows, num_values, static_cast<cudaStream_t>(stream));
}

int srj_percentile_from_histogram(const srj_column* input, const double* percentages, int32_t num_percentages, int32_t output_as_lists,
                                  double* out, uint32_t* out_mask, int32_t* out_offsets, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "percentile_from_histogram";
  const srj_column *v = nullptr, *c = nullptr;
  int rc = pct_check(what, input, num_percentages, &v, &c);
  if (rc != SRJ_OK) return rc;
  if (input->size == 0) return SRJ_OK;
  if (num_percentages > 0 && !percentages) { set_error("%s: the percentages are missing", what); return SRJ_EINVAL; }
  if ((rc = check_out(what, "output", out, 8, !output_as_lists)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output mask", out_mask, 4)) != SRJ_OK) return rc;
  if (output_as_lists && (rc = check_out(what, "output offsets", out_offsets, 4)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "workspace (srj_percentile_workspace_bytes)", workspace, 256)) != SRJ_OK) return rc;
  PctWs w{};
  pct_layout(input->size, v->size, num_percentages, static_cast<uint8_t*>(workspace), &w);
  return launch_pct_fill(*input, *v, *c, percentages, num_percentages, output_as_lists != 0, out, out_mask, out_offsets, w,
                         static_cast<cudaStream_t>(stream));
}

// histogram.cu:280-287 in its order, then the value type and this library's buffer checks
static int hc_check(const char* what, const srj_column* values, const srj_column* freq)
{
  if (!values || !freq) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (freq->null_mask) { set_error("%s: The input frequencies must not have nulls.", what); return SRJ_EINVAL; }
  if (freq->type_id != SRJ_INT64) { set_error("%s: The input frequencies must be of type INT64.", what); return SRJ_EINVAL; }
  if (values->size != freq->size) { set_error("%s: The input values and frequencies must have the same size.", what); return SRJ_EINVAL; }
  if (type_width(values->type_id) == 0) { set_error("%s: only fixed-width values are supported (type id %d)", what, values->type_id); return SRJ_EUNSUPPORTED; }
  if (values->size < 0 || values->size > INT32_MAX) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  int rc = SRJ_OK;
  if ((rc = check_data(what, "values", *values)) != SRJ_OK) return rc;
  if ((rc = check_data(what, "frequencies", *freq)) != SRJ_OK) return rc;
  if (values->null_mask && !aligned_to(values->null_mask, 4)) { set_error("%s: the values mask is not 4-byte aligned", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

int64_t srj_histogram_workspace_bytes(int64_t num_rows) { return hc_layout(tmax<int64_t>(num_rows, 0), nullptr, nullptr, nullptr, nullptr); }

int srj_histogram_create_size(const srj_column* values, const srj_column* frequencies, int32_t output_as_lists, int64_t* out_rows,
                              int64_t* value_nulls, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "histogram_create_size";
  int rc = hc_check(what, values, frequencies);
  if (rc != SRJ_OK) return rc;
  if (!out_rows || !value_nulls) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  *out_rows = *value_nulls = 0;
  const int64_t rows = values->size;
  if (rows == 0) return SRJ_OK;
  if ((rc = check_out(what, "workspace (srj_histogram_workspace_bytes)", workspace, 256)) != SRJ_OK) return rc;
  HcHeader* hd = nullptr;
  int32_t *keep = nullptr, *sums = nullptr;
  hc_layout(rows, static_cast<uint8_t*>(workspace), &hd, &keep, &sums);
  auto s = static_cast<cudaStream_t>(stream);
  SRJ_CUDA_TRY(cudaMemsetAsync(hd, 0, sizeof(HcHeader), s));
  hc_flag_kernel<<<row_grid(rows), kRowThreads, 0, s>>>(static_cast<const int64_t*>(frequencies->data), values->null_mask, rows, keep, hd);
  SRJ_CUDA_TRY(cudaGetLastError());
  HcHeader h{};
  SRJ_CUDA_TRY(cudaMemcpyAsync(&h, hd, sizeof(h), cudaMemcpyDeviceToHost, s));
  SRJ_CUDA_TRY(cudaStreamSynchronize(s));
  if (h.negative) { set_error("%s: The input frequencies must not contain negative values.", what); return SRJ_EINVAL; }
  *out_rows    = output_as_lists ? static_cast<int64_t>(h.kept) : rows;
  *value_nulls = static_cast<int64_t>(output_as_lists ? h.list_nulls : h.struct_nulls);
  return SRJ_OK;
}

int srj_histogram_create(const srj_column* values, const srj_column* frequencies, int32_t output_as_lists, void* out_values,
                         uint32_t* out_values_mask, int64_t* out_frequencies, int32_t* out_offsets, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "histogram_create";
  int rc = hc_check(what, values, frequencies);
  if (rc != SRJ_OK) return rc;
  const int64_t rows = values->size;
  if (rows == 0) return SRJ_OK;
  const int w = type_width(values->type_id);
  if ((rc = check_out(what, "output values", out_values, std::min(w, 8), false)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output frequencies", out_frequencies, 8, false)) != SRJ_OK) return rc;
  if ((rc = check_out_mask(what, !output_as_lists || values->null_mask, out_values_mask)) != SRJ_OK) return rc;
  if (output_as_lists && (rc = check_out(what, "output offsets", out_offsets, 4)) != SRJ_OK) return rc;
  if (!output_as_lists && (!out_values || !out_frequencies)) { set_error("%s: the outputs are missing", what); return SRJ_EINVAL; }
  if ((rc = check_out(what, "workspace (srj_histogram_workspace_bytes)", workspace, 256)) != SRJ_OK) return rc;
  HcHeader* hd = nullptr;
  int32_t *keep = nullptr, *sums = nullptr;
  hc_layout(rows, static_cast<uint8_t*>(workspace), &hd, &keep, &sums);
  auto s = static_cast<cudaStream_t>(stream);
  HcWriteArgs a{};
  a.values      = static_cast<const uint8_t*>(values->data);
  a.vmask       = values->null_mask;
  a.freq        = static_cast<const int64_t*>(frequencies->data);
  a.pos         = keep;
  a.h           = hd;
  a.rows        = rows;
  a.width       = w;
  a.lists       = output_as_lists != 0;
  a.out_values  = static_cast<uint8_t*>(out_values);
  a.out_mask    = out_values_mask;
  a.out_freq    = out_frequencies;
  a.out_offsets = out_offsets;
  if (output_as_lists) {
    if ((rc = launch_i32_exclusive_scan(keep, rows, sums, keep + rows, s)) != SRJ_OK) return rc;
    // the child's mask holds the kept rows only: clear ceil(kept / 32) words, the kept count read on the device
    if (out_values_mask && values->null_mask) hc_clear_mask_kernel<<<row_grid((rows + 31) / 32), kRowThreads, 0, s>>>(keep + rows, out_values_mask);
    else a.out_mask = nullptr;
  }
  hc_write_kernel<<<row_grid(rows), kRowThreads, 0, s>>>(a);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // extern "C"
