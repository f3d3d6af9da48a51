// join.cu -- JoinPrimitives on the device (reference join_primitives.cu): the hash inner join of two key tables and the
// helpers that turn its gather maps into left outer, full outer, semi and anti joins.
//
// Hash inner join, build on the right table and probe with the left (DESIGN 3.6k):
//   join_build_kernel    : every right row whose keys are not null (or every row, with nulls equal) is inserted into an
//                          open-addressing multimap in the caller's workspace.  A slot is one uint64: the row's 32-bit
//                          key hash above its row index; all ones is empty.  The table has a power-of-two count of
//                          32-byte buckets (4 slots, one L2 sector) at load factor <= 0.5; a key probes linearly from
//                          bucket hash & (buckets - 1), and a row claims a slot with one 64-bit CAS.
//   join_count_kernel    : one lane per left row walks the chain to the first empty slot, compares the stored hash,
//                          then the keys, and writes the row's match count; each tile of kTileRows rows writes its int64
//                          sum.  The tile sums are scanned (kudo.cu's one-CTA int64 scan) and the total read back.
//   join_retrieve_kernel : a block scan of the counts gives each row its offset within the tile; rows with matches walk
//                          their chain again and write (left, right) pairs there, so the left map is non-decreasing.
// Key equality: fixed-width values compare by their bits after canonicalisation (BOOL8 as 0 / 1; FLOAT32 / FLOAT64 with
// every NaN one NaN and -0.0 as 0.0, cudf's nan_equal_physical_equality_comparator); STRING by length, then bytes read as
// aligned words.  The hash is Murmur3 over the same canonical bits (mm_u32 / mm_u64 / mm_bytes of hash_device.cuh).
//
// Gather-map helpers: join_mark_kernel sets one bit per table row named by an in-range map entry and counts the bits it
// newly set; join_tile_count_kernel, the shared int32 scan and join_compact_kernel write the ascending set or clear rows;
// join_fill_kernel writes INT32_MIN sentinels; join_matched_rows_kernel writes BOOL8 flags.
#include <algorithm>

#include "check.hpp"
#include "common.cuh"
#include "hash_device.cuh"
#include "kernels.hpp"
#include "map_rows.cuh"

namespace srj {
namespace {

constexpr int kJoinThreads      = 256;
constexpr int kRowsPerThread    = 8;
constexpr int kTileRows         = kJoinThreads * kRowsPerThread;   // rows per count / retrieve tile
constexpr int kMaskTileRows     = kJoinThreads * 32;               // rows per compaction tile (one mask word a lane)
constexpr uint64_t kEmptySlot   = ~0ull;
constexpr uint32_t kNullKeyWord = 0x9e3779b9u;                    // mixed into the hash for a null key (nulls equal)

using hash::mm_bytes;
using hash::mm_mix;
using hash::mm_u32;
using hash::mm_u64;
using hash::norm_f32;
using hash::norm_f64;

struct JCol {
  int32_t type, width;            // width 0: STRING
  const uint8_t* data;
  const uint32_t* mask;
  const int32_t* offsets;
};
struct JKeys {
  JCol l[SRJ_MAX_JOIN_KEYS], r[SRJ_MAX_JOIN_KEYS];
  int32_t n;
};

__device__ __forceinline__ bool valid_at(const uint32_t* m, int64_t i) { return !m || ((__ldg(m + (i >> 5)) >> (i & 31)) & 1u); }

// the canonical bits of a fixed-width value (hi: the upper half of a DECIMAL128)
__device__ __forceinline__ uint64_t canon(const JCol& c, int64_t i, uint64_t& hi)
{
  hi = 0;
  switch (c.width) {
    case 1: {
      const uint64_t v = __ldg(c.data + i);
      return c.type == SRJ_BOOL8 ? uint64_t{v != 0} : v;
    }
    case 2: return __ldg(reinterpret_cast<const uint16_t*>(c.data) + i);
    case 4: {
      const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(c.data) + i);
      return c.type == SRJ_FLOAT32 ? norm_f32(v, true) : v;
    }
    case 8: {
      const uint64_t v = __ldg(reinterpret_cast<const unsigned long long*>(c.data) + i);
      return c.type == SRJ_FLOAT64 ? norm_f64(v, true) : v;
    }
    default: {
      const auto* p = reinterpret_cast<const unsigned long long*>(c.data) + 2 * i;
      hi            = __ldg(p + 1);
      return __ldg(p);
    }
  }
}

// Murmur3 of a row's keys, column by column; *has_null when a key is null
__device__ __forceinline__ uint32_t row_hash(const JCol* cols, int32_t n, int64_t r, bool* has_null)
{
  uint32_t h = 0;
  bool any   = false;
  for (int32_t c = 0; c < n; ++c) {
    const JCol& k = cols[c];
    if (!valid_at(k.mask, r)) {
      any = true;
      h   = mm_mix(h, kNullKeyWord);
    } else if (k.width == 0) {
      const int32_t b = __ldg(k.offsets + r);
      h               = mm_bytes(k.data + b, __ldg(k.offsets + r + 1) - b, h);
    } else {
      uint64_t hi;
      const uint64_t v = canon(k, r, hi);
      h                = k.width <= 4 ? mm_u32(static_cast<uint32_t>(v), h) : k.width == 8 ? mm_u64(v, h) : mm_u64(hi, mm_u64(v, h));
    }
  }
  *has_null = any;
  return h;
}

// len bytes at a and at b, compared as aligned words funnel-shifted to each start
__device__ __forceinline__ bool bytes_equal(const uint8_t* a, const uint8_t* b, int32_t len)
{
  const RowWords ra(a, len), rb(b, len);
  uint32_t a0 = ra.word(0), b0 = rb.word(0);
  for (int32_t j = 0; 4 * j < len; ++j) {
    const uint32_t a1 = ra.word(j + 1), b1 = rb.word(j + 1);
    uint32_t x        = ra.at(a0, a1) ^ rb.at(b0, b1);
    if (len - 4 * j < 4) x &= (1u << (8 * (len - 4 * j))) - 1u;
    if (x) return false;
    a0 = a1;
    b0 = b1;
  }
  return true;
}

// left row l and right row r have equal keys (both null counts as equal: only reachable with nulls equal)
__device__ __forceinline__ bool keys_equal(const JKeys& k, int64_t l, int64_t r)
{
  for (int32_t c = 0; c < k.n; ++c) {
    const JCol &a = k.l[c], &b = k.r[c];
    const bool va = valid_at(a.mask, l), vb = valid_at(b.mask, r);
    if (va != vb) return false;
    if (!va) continue;
    if (a.width == 0) {
      const int32_t ab = __ldg(a.offsets + l), bb = __ldg(b.offsets + r);
      const int32_t len = __ldg(a.offsets + l + 1) - ab;
      if (len != __ldg(b.offsets + r + 1) - bb || !bytes_equal(a.data + ab, b.data + bb, len)) return false;
    } else {
      uint64_t ah, bh;
      if (canon(a, l, ah) != canon(b, r, bh) || ah != bh) return false;
    }
  }
  return true;
}

// f(right row) for every right row whose keys equal left row l's (hash h), in chain order
template <class F>
__device__ __forceinline__ void walk_chain(const JKeys& k, int64_t l, uint32_t h, const unsigned long long* __restrict__ table, uint64_t bmask,
                                           F&& f)
{
  for (uint64_t b = h & bmask;; b = (b + 1) & bmask) {
    const auto* p             = reinterpret_cast<const ulonglong2*>(table + 4 * b);
    const ulonglong2 s01      = __ldg(p), s23 = __ldg(p + 1);
    const unsigned long long s[4] = {s01.x, s01.y, s23.x, s23.y};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (s[j] == kEmptySlot) return;
      if (static_cast<uint32_t>(s[j] >> 32) == h) {
        const int32_t r = static_cast<int32_t>(static_cast<uint32_t>(s[j]));
        if (keys_equal(k, l, r)) f(r);
      }
    }
  }
}

__global__ void __launch_bounds__(kJoinThreads) join_build_kernel(const __grid_constant__ JKeys k, int64_t n, bool nulls_equal,
                                                                  unsigned long long* __restrict__ table, uint64_t bmask)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kJoinThreads + threadIdx.x;
  if (r >= n) return;
  bool has_null;
  const uint32_t h = row_hash(k.r, k.n, r, &has_null);
  if (has_null && !nulls_equal) return;
  const unsigned long long slot = (static_cast<unsigned long long>(h) << 32) | static_cast<uint32_t>(r);
  for (uint64_t b = h & bmask;; b = (b + 1) & bmask) {
    unsigned long long* s = table + 4 * b;
#pragma unroll
    for (int j = 0; j < 4; ++j)   // a slot only goes from empty to full: a stale read costs one failed CAS
      if (s[j] == kEmptySlot && atomicCAS(s + j, kEmptySlot, slot) == kEmptySlot) return;
  }
}

template <class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* s_warp, T& total)
{
  const int lane = lane_id(), w = warp_id();
  T x            = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[w] = x;
  __syncthreads();
  if (w == 0) {
    T t = lane < kJoinThreads / 32 ? s_warp[lane] : T{0};
#pragma unroll
    for (int o = 1; o < kJoinThreads / 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    if (lane < kJoinThreads / 32) s_warp[lane] = t;
  }
  __syncthreads();
  const T ex = (w ? s_warp[w - 1] : T{0}) + x - v;
  total      = s_warp[kJoinThreads / 32 - 1];
  __syncthreads();   // s_warp is reused by the next scan
  return ex;
}

__global__ void __launch_bounds__(kJoinThreads) join_count_kernel(const __grid_constant__ JKeys k, int64_t n, bool nulls_equal,
                                                                  const unsigned long long* __restrict__ table, uint64_t bmask,
                                                                  int32_t* __restrict__ counts, long long* __restrict__ tile_sums)
{
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kTileRows + threadIdx.x;
  long long sum      = 0;
  for (int i = 0; i < kRowsPerThread; ++i) {
    const int64_t l = base + i * kJoinThreads;
    if (l >= n) break;
    bool has_null;
    const uint32_t h = row_hash(k.l, k.n, l, &has_null);
    int32_t cnt      = 0;
    if (!has_null || nulls_equal) walk_chain(k, l, h, table, bmask, [&](int32_t) { ++cnt; });
    counts[l] = cnt;
    sum += cnt;
  }
  __shared__ long long s_warp[kJoinThreads / 32];
  long long total;
  block_exclusive_scan(sum, s_warp, total);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kJoinThreads) join_retrieve_kernel(const __grid_constant__ JKeys k, int64_t n,
                                                                     const unsigned long long* __restrict__ table, uint64_t bmask,
                                                                     const int32_t* __restrict__ counts, const long long* __restrict__ tile_offsets,
                                                                     int32_t* __restrict__ left_map, int32_t* __restrict__ right_map)
{
  __shared__ long long s_warp[kJoinThreads / 32];
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kTileRows + threadIdx.x;
  long long carry    = tile_offsets[blockIdx.x];
  for (int i = 0; i < kRowsPerThread; ++i) {
    const int64_t l = base + i * kJoinThreads;
    if (l - threadIdx.x >= n) break;                           // block-uniform: the scan needs every lane
    const long long cnt = l < n ? __ldg(counts + l) : 0;
    long long total;
    long long pos = carry + block_exclusive_scan(cnt, s_warp, total);
    carry += total;
    if (cnt > 0) {
      bool has_null;
      const uint32_t h = row_hash(k.l, k.n, l, &has_null);
      walk_chain(k, l, h, table, bmask, [&](int32_t r) {
        left_map[pos]  = static_cast<int32_t>(l);
        right_map[pos] = r;
        ++pos;
      });
    }
  }
}

// ---- gather-map helpers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kJoinThreads) join_mark_kernel(const int32_t* __restrict__ map, int64_t n, int32_t rows,
                                                                 uint32_t* __restrict__ mask, unsigned long long* __restrict__ matched)
{
  unsigned long long fresh = 0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kJoinThreads + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * kJoinThreads) {
    const int32_t idx = __ldg(map + i);
    if (idx >= 0 && idx < rows) {
      const uint32_t bit = 1u << (idx & 31);
      if (!(atomicOr(mask + (idx >> 5), bit) & bit)) ++fresh;
    }
  }
  fresh = warp_sum(fresh);
  if (lane_id() == 0 && fresh) atomicAdd(matched, fresh);
}

// the bits of mask word w that select rows (set ones, or clear ones when !set), rows past the end dropped
__device__ __forceinline__ uint32_t wanted_bits(const uint32_t* mask, int64_t w, int64_t rows, bool set)
{
  uint32_t x        = __ldg(mask + w);
  x                 = set ? x : ~x;
  const int64_t rem = rows - 32 * w;
  return rem < 32 ? x & ((1u << rem) - 1u) : x;
}

__global__ void __launch_bounds__(kJoinThreads) join_tile_count_kernel(const uint32_t* __restrict__ mask, int64_t rows, bool set,
                                                                       int32_t* __restrict__ tile_counts)
{
  const int64_t w = static_cast<int64_t>(blockIdx.x) * kJoinThreads + threadIdx.x;
  const int32_t c = 32 * w < rows ? __popc(wanted_bits(mask, w, rows, set)) : 0;
  __shared__ int32_t s_warp[kJoinThreads / 32];
  int32_t total;
  block_exclusive_scan(c, s_warp, total);
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kJoinThreads) join_compact_kernel(const uint32_t* __restrict__ mask, int64_t rows, bool set,
                                                                    const int32_t* __restrict__ tile_offsets, int32_t* __restrict__ out)
{
  const int64_t w = static_cast<int64_t>(blockIdx.x) * kJoinThreads + threadIdx.x;
  uint32_t x      = 32 * w < rows ? wanted_bits(mask, w, rows, set) : 0u;
  __shared__ int32_t s_warp[kJoinThreads / 32];
  int32_t total;
  int32_t pos = __ldg(tile_offsets + blockIdx.x) + block_exclusive_scan(static_cast<int32_t>(__popc(x)), s_warp, total);
  while (x) {
    out[pos++] = static_cast<int32_t>(32 * w) + __ffs(x) - 1;
    x &= x - 1;
  }
}

// one lane per entry: a grid-stride loop here is unrolled behind a 64-bit trip-count division (a CALL)
__global__ void __launch_bounds__(kJoinThreads) join_fill_kernel(int32_t* __restrict__ out, int64_t n, int32_t value)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kJoinThreads + threadIdx.x;
  if (i < n) out[i] = value;
}

__global__ void __launch_bounds__(kJoinThreads) join_matched_rows_kernel(const int32_t* __restrict__ map, int64_t n, int32_t rows,
                                                                         uint8_t* __restrict__ out)
{
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kJoinThreads + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * kJoinThreads) {
    const int32_t idx = __ldg(map + i);
    if (idx >= 0 && idx < rows) out[idx] = 1;
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------------
unsigned blocks_for(int64_t items, int64_t per_block) { return static_cast<unsigned>((items + per_block - 1) / per_block); }

unsigned stride_grid(int64_t n) { return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(blocks_for(n, kJoinThreads), 8LL * sm_count()))); }

// buckets of the build table: a power of two with at least 2 * right_rows slots
uint64_t join_buckets(int64_t right_rows)
{
  uint64_t b = 1;
  while (4 * b < 2 * static_cast<uint64_t>(right_rows)) b <<= 1;
  return b;
}

int64_t join_tiles(int64_t left_rows) { return (left_rows + kTileRows - 1) / kTileRows; }

struct JoinWs {
  unsigned long long* table;
  long long* tile_sums;   // join_tiles + 1
  int32_t* counts;        // left rows
};

JoinWs join_ws(void* ws, int64_t left_rows, int64_t right_rows)
{
  auto* p = static_cast<uint8_t*>(ws);
  JoinWs w;
  w.table     = reinterpret_cast<unsigned long long*>(p);
  p += round_up64(static_cast<int64_t>(join_buckets(right_rows)) * 32, 256);
  w.tile_sums = reinterpret_cast<long long*>(p);
  p += round_up64((join_tiles(left_rows) + 1) * 8, 256);
  w.counts    = reinterpret_cast<int32_t*>(p);
  return w;
}

JKeys join_keys(const srj_column* left, const srj_column* right, int32_t n)
{
  JKeys k{};
  k.n = n;
  for (int32_t c = 0; c < n; ++c) {
    for (int side = 0; side < 2; ++side) {
      const srj_column& s = side ? right[c] : left[c];
      JCol& d             = side ? k.r[c] : k.l[c];
      d.type              = s.type_id;
      d.width             = s.type_id == SRJ_STRING ? 0 : type_width(s.type_id);
      d.data              = static_cast<const uint8_t*>(s.data);
      d.mask              = s.null_mask;
      d.offsets           = s.offsets;
    }
  }
  return k;
}

struct MaskWs {
  unsigned long long* matched;
  uint32_t* mask;
  int32_t* tile_counts;
  int32_t* scan_sums;
};

int64_t mask_tiles(int64_t rows) { return (rows + kMaskTileRows - 1) / kMaskTileRows; }

MaskWs mask_ws(const void* ws, int64_t rows)
{
  auto* p = static_cast<uint8_t*>(const_cast<void*>(ws));
  MaskWs m;
  m.matched     = reinterpret_cast<unsigned long long*>(p);
  p += 256;
  m.mask        = reinterpret_cast<uint32_t*>(p);
  p += round_up64((rows + 31) / 32 * 4, 256);
  m.tile_counts = reinterpret_cast<int32_t*>(p);
  p += round_up64(mask_tiles(rows) * 4, 256);
  m.scan_sums   = reinterpret_cast<int32_t*>(p);
  return m;
}

}  // namespace

static int64_t hash_join_workspace_bytes(int64_t left_rows, int64_t right_rows)
{
  return round_up64(static_cast<int64_t>(join_buckets(right_rows)) * 32, 256) + round_up64((join_tiles(left_rows) + 1) * 8, 256) +
         round_up64(left_rows * 4, 256);
}

// builds the table on the right keys, counts each left row's matches and reads the pair count back (one synchronisation)
static int launch_hash_join_size(const srj_column* left, const srj_column* right, int32_t ncols, int64_t left_rows, int64_t right_rows, bool nulls_equal,
                          int64_t* num_pairs, void* workspace, cudaStream_t stream)
{
  const JKeys k         = join_keys(left, right, ncols);
  const JoinWs w        = join_ws(workspace, left_rows, right_rows);
  const uint64_t nb     = join_buckets(right_rows);
  const int64_t ntiles  = join_tiles(left_rows);
  SRJ_CUDA_TRY(cudaMemsetAsync(w.table, 0xff, nb * 32, stream));
  join_build_kernel<<<blocks_for(right_rows, kJoinThreads), kJoinThreads, 0, stream>>>(k, right_rows, nulls_equal, w.table, nb - 1);
  SRJ_CUDA_TRY(cudaGetLastError());
  join_count_kernel<<<static_cast<unsigned>(ntiles), kJoinThreads, 0, stream>>>(k, left_rows, nulls_equal, w.table, nb - 1, w.counts, w.tile_sums);
  SRJ_CUDA_TRY(cudaGetLastError());
  int rc = launch_i64_scan_small(reinterpret_cast<int64_t*>(w.tile_sums), static_cast<int>(ntiles), stream);
  if (rc != SRJ_OK) return rc;
  long long total = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(&total, w.tile_sums + ntiles, sizeof(total), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  *num_pairs = total;
  return SRJ_OK;
}

// writes the pairs from the table and counts launch_hash_join_size left in the workspace
static int launch_hash_join(const srj_column* left, const srj_column* right, int32_t ncols, int64_t left_rows, int64_t right_rows, int32_t* left_map,
                     int32_t* right_map, void* workspace, cudaStream_t stream)
{
  const JKeys k     = join_keys(left, right, ncols);
  const JoinWs w    = join_ws(workspace, left_rows, right_rows);
  const uint64_t nb = join_buckets(right_rows);
  join_retrieve_kernel<<<static_cast<unsigned>(join_tiles(left_rows)), kJoinThreads, 0, stream>>>(k, left_rows, w.table, nb - 1, w.counts, w.tile_sums,
                                                                                                  left_map, right_map);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int64_t join_mask_workspace_bytes(int64_t rows)
{
  const int64_t tiles = mask_tiles(rows);
  return 256 + round_up64((rows + 31) / 32 * 4, 256) + round_up64(tiles * 4, 256) + round_up64(i32_scan_nchunks(tiles) * 4, 256);
}

static int launch_join_mark(const int32_t* map, int64_t n, int64_t rows, void* workspace, cudaStream_t stream)
{
  const MaskWs m = mask_ws(workspace, rows);
  SRJ_CUDA_TRY(cudaMemsetAsync(m.matched, 0, 256 + (rows + 31) / 32 * 4, stream));   // the counter, its padding and the mask
  if (n == 0 || rows == 0) return SRJ_OK;
  join_mark_kernel<<<stride_grid(n), kJoinThreads, 0, stream>>>(map, n, static_cast<int32_t>(rows), m.mask, m.matched);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int read_join_matched(const void* const* workspaces, int32_t count, int64_t* matched, cudaStream_t stream)
{
  for (int32_t i = 0; i < count; ++i)
    SRJ_CUDA_TRY(cudaMemcpyAsync(matched + i, workspaces[i], sizeof(int64_t), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  return SRJ_OK;
}

static int launch_join_compact(const void* workspace, int64_t rows, bool set, int32_t* out, cudaStream_t stream)
{
  if (rows == 0) return SRJ_OK;
  const MaskWs m      = mask_ws(workspace, rows);
  const int64_t tiles = mask_tiles(rows);
  join_tile_count_kernel<<<static_cast<unsigned>(tiles), kJoinThreads, 0, stream>>>(m.mask, rows, set, m.tile_counts);
  SRJ_CUDA_TRY(cudaGetLastError());
  const int rc = launch_i32_exclusive_scan(m.tile_counts, tiles, m.scan_sums, nullptr, stream);
  if (rc != SRJ_OK) return rc;
  join_compact_kernel<<<static_cast<unsigned>(tiles), kJoinThreads, 0, stream>>>(m.mask, rows, set, m.tile_counts, out);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_join_fill(int32_t* out, int64_t n, int32_t value, cudaStream_t stream)
{
  if (n == 0) return SRJ_OK;
  join_fill_kernel<<<blocks_for(n, kJoinThreads), kJoinThreads, 0, stream>>>(out, n, value);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_join_matched_rows(const int32_t* map, int64_t n, int64_t rows, uint8_t* out, cudaStream_t stream)
{
  if (rows == 0) return SRJ_OK;
  SRJ_CUDA_TRY(cudaMemsetAsync(out, 0, static_cast<size_t>(rows), stream));
  if (n == 0) return SRJ_OK;
  join_matched_rows_kernel<<<stride_grid(n), kJoinThreads, 0, stream>>>(map, n, static_cast<int32_t>(rows), out);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

// join_primitives.cu:212-220 and cudf's validate_hash_join_probe: key counts first, an empty side returns empty, then the
// schema.  *rows[2] receive the row counts; *empty is set when either is 0 (nothing else was checked then).
static int join_check(const char* what, const srj_column* l, int32_t nl, const srj_column* r, int32_t nr, int64_t rows[2], bool* empty)
{
  if (!l || !r || nl < 0 || nr < 0) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (nl == 0) { set_error("%s: Left keys table must have at least one column", what); return SRJ_EINVAL; }
  if (nr == 0) { set_error("%s: Right keys table must have at least one column", what); return SRJ_EINVAL; }
  for (int side = 0; side < 2; ++side) {
    const srj_column* t = side ? r : l;
    const int32_t n     = side ? nr : nl;
    rows[side]          = t[0].size;
    for (int32_t c = 0; c < n; ++c)
      if (t[c].size < 0 || t[c].size != rows[side]) { set_error("%s: the %s key columns have differing or negative row counts", what, side ? "right" : "left"); return SRJ_EINVAL; }
  }
  *empty = rows[0] == 0 || rows[1] == 0;
  if (*empty) return SRJ_OK;
  for (int side = 0; side < 2; ++side) {
    const srj_column* t = side ? r : l;
    for (int32_t c = 0; c < (side ? nr : nl); ++c)
      if (t[c].type_id != SRJ_STRING && type_width(t[c].type_id) == 0) { set_error("%s: key type %d is not supported", what, t[c].type_id); return SRJ_EUNSUPPORTED; }
  }
  if (nl != nr) { set_error("%s: Mismatch in number of columns to be joined on", what); return SRJ_EINVAL; }
  if (nl > SRJ_MAX_JOIN_KEYS) { set_error("%s: more than %d key columns", what, SRJ_MAX_JOIN_KEYS); return SRJ_EUNSUPPORTED; }
  for (int32_t c = 0; c < nl; ++c)
    if (l[c].type_id != r[c].type_id || l[c].scale != r[c].scale) { set_error("%s: Mismatch in joining column data types", what); return SRJ_EINVAL; }
  if (rows[0] > INT32_MAX || rows[1] > INT32_MAX) { set_error("%s: more than INT32_MAX rows", what); return SRJ_EINVAL; }
  for (int side = 0; side < 2; ++side) {
    const srj_column* t = side ? r : l;
    for (int32_t c = 0; c < nl; ++c) {
      const char* name = side ? "right key column" : "left key column";
      const int rc     = t[c].type_id == SRJ_STRING ? check_offsets(what, name, t[c], c) : check_data(what, name, t[c], c);
      if (rc != SRJ_OK) return rc;
      if (!aligned_to(t[c].null_mask, 4)) { set_error("%s: %s %d has a null mask not 4-byte aligned", what, name, c); return SRJ_EINVAL; }
    }
  }
  return SRJ_OK;
}

int64_t srj_hash_join_workspace_bytes(int64_t left_rows, int64_t right_rows)
{
  return hash_join_workspace_bytes(std::max<int64_t>(0, left_rows), std::max<int64_t>(0, right_rows));
}

int srj_hash_inner_join_size(const srj_column* left_keys, int32_t num_left_keys, const srj_column* right_keys, int32_t num_right_keys,
                             int32_t nulls_equal, int64_t* num_pairs, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "hash_inner_join_size";
  if (!num_pairs) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  int64_t rows[2];
  bool empty  = false;
  const int rc = join_check(what, left_keys, num_left_keys, right_keys, num_right_keys, rows, &empty);
  if (rc != SRJ_OK) return rc;
  *num_pairs = 0;
  if (empty) return SRJ_OK;
  if (!workspace) { set_error("%s: the workspace is needed (srj_hash_join_workspace_bytes)", what); return SRJ_EINVAL; }
  return launch_hash_join_size(left_keys, right_keys, num_left_keys, rows[0], rows[1], nulls_equal != 0, num_pairs, workspace,
                               static_cast<cudaStream_t>(stream));
}

int srj_hash_inner_join(const srj_column* left_keys, int32_t num_left_keys, const srj_column* right_keys, int32_t num_right_keys,
                        int32_t nulls_equal, int32_t* left_map, int32_t* right_map, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "hash_inner_join";
  int64_t rows[2];
  bool empty  = false;
  int rc = join_check(what, left_keys, num_left_keys, right_keys, num_right_keys, rows, &empty);
  if (rc != SRJ_OK || empty) return rc;
  (void)nulls_equal;   // the size call's counts already hold it
  if ((rc = check_out(what, "workspace", workspace, 1)) != SRJ_OK || (rc = check_out(what, "left map", left_map, 4)) != SRJ_OK ||
      (rc = check_out(what, "right map", right_map, 4)) != SRJ_OK)
    return rc;
  return launch_hash_join(left_keys, right_keys, num_left_keys, rows[0], rows[1], left_map, right_map, workspace, static_cast<cudaStream_t>(stream));
}

// a gather map of map_len entries (4-byte aligned; NULL only when empty) over a table of table_rows rows
static int join_check_map(const char* what, const int32_t* map, int64_t map_len, int64_t table_rows)
{
  if (map_len < 0 || table_rows < 0) { set_error("%s: Table sizes must be non-negative", what); return SRJ_EINVAL; }
  if (table_rows > INT32_MAX) { set_error("%s: more than INT32_MAX table rows", what); return SRJ_EINVAL; }
  return check_out(what, "gather map", map, 4, map_len > 0);
}

int64_t srj_join_mask_workspace_bytes(int64_t table_rows) { return join_mask_workspace_bytes(std::max<int64_t>(0, table_rows)); }

int srj_join_mark(const int32_t* map, int64_t map_len, int64_t table_rows, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_mark";
  int rc           = join_check_map(what, map, map_len, table_rows);
  if (rc != SRJ_OK || (rc = check_out(what, "workspace", workspace, 8)) != SRJ_OK) return rc;
  return launch_join_mark(map, map_len, table_rows, workspace, static_cast<cudaStream_t>(stream));
}

int srj_join_matched_counts(const void* const* workspaces, int32_t count, int64_t* matched, void* stream)
{
  SRJ_API_RANGE();
  if (count < 0 || (count > 0 && (!workspaces || !matched))) { set_error("join_matched_counts: bad argument"); return SRJ_EINVAL; }
  for (int32_t i = 0; i < count; ++i)
    if (!workspaces[i]) { set_error("join_matched_counts: workspace %d is null", i); return SRJ_EINVAL; }
  if (count == 0) return SRJ_OK;
  return read_join_matched(workspaces, count, matched, static_cast<cudaStream_t>(stream));
}

int srj_join_compact(const void* workspace, int64_t table_rows, int32_t matched, int32_t* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_compact";
  int rc           = join_check_map(what, nullptr, 0, table_rows);
  if (rc != SRJ_OK || table_rows == 0) return rc;
  if ((rc = check_out(what, "workspace", workspace, 1)) != SRJ_OK || (rc = check_out(what, "output", out, 4)) != SRJ_OK) return rc;
  return launch_join_compact(workspace, table_rows, matched != 0, out, static_cast<cudaStream_t>(stream));
}

// join_primitives.cu:358-461
int srj_join_make_outer(const int32_t* left_map, const int32_t* right_map, int64_t map_len, int64_t left_rows, int64_t right_rows,
                        const void* left_ws, int64_t left_unmatched, const void* right_ws, int64_t right_unmatched, int32_t* out_left,
                        int32_t* out_right, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_make_outer";
  int rc           = join_check_map(what, left_map, map_len, left_rows);
  if (rc != SRJ_OK || (rc = join_check_map(what, right_map, map_len, right_rows)) != SRJ_OK) return rc;
  const bool full = right_ws != nullptr;
  if (left_unmatched < 0 || left_unmatched > left_rows || (full && (right_unmatched < 0 || right_unmatched > right_rows))) {
    set_error("%s: unmatched counts outside the table sizes", what);
    return SRJ_EINVAL;
  }
  const int64_t total = map_len + left_unmatched + (full ? right_unmatched : 0);
  if (total == 0) return SRJ_OK;
  if ((rc = check_out(what, "left workspace", left_ws, 1)) != SRJ_OK || (rc = check_out(what, "left output", out_left, 4)) != SRJ_OK ||
      (rc = check_out(what, "right output", out_right, 4)) != SRJ_OK)
    return rc;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (map_len > 0) {
    SRJ_CUDA_TRY(cudaMemcpyAsync(out_left, left_map, static_cast<size_t>(map_len) * 4, cudaMemcpyDeviceToDevice, s));
    SRJ_CUDA_TRY(cudaMemcpyAsync(out_right, right_map, static_cast<size_t>(map_len) * 4, cudaMemcpyDeviceToDevice, s));
  }
  if (left_unmatched > 0) {
    if ((rc = launch_join_compact(left_ws, left_rows, false, out_left + map_len, s)) != SRJ_OK) return rc;
    if ((rc = launch_join_fill(out_right + map_len, left_unmatched, INT32_MIN, s)) != SRJ_OK) return rc;
  }
  if (full && right_unmatched > 0) {
    const int64_t at = map_len + left_unmatched;
    if ((rc = launch_join_compact(right_ws, right_rows, false, out_right + at, s)) != SRJ_OK) return rc;
    if ((rc = launch_join_fill(out_left + at, right_unmatched, INT32_MIN, s)) != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

// join_primitives.cu:549-576
int srj_join_matched_rows(const int32_t* map, int64_t map_len, int64_t table_rows, uint8_t* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_matched_rows";
  int rc           = join_check_map(what, map, map_len, table_rows);
  if (rc != SRJ_OK || table_rows == 0) return rc;
  if ((rc = check_out(what, "output", out, 1)) != SRJ_OK) return rc;
  return launch_join_matched_rows(map, map_len, table_rows, out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
