// partition.cu -- Spark HashPartitioning on the device (SURVEY §8f rank 1): partition id of every row =
// pmod(murmur3_32(seed, keys), P), then a STABLE partition of the table's rows by that id (the rows of partition p
// contiguous, in input order) with the partition offsets a shuffle writer slices at.  The reference repo holds the
// hash (hash/murmur_hash.cu, Hash.murmurHash32) and the step after (shuffle_split.hpp:60-189 takes the table plus
// exactly these split offsets); the id + partition step itself sits in the plugin (GpuHashPartitioning ->
// Table.partition): this file is that step, built on the hashes of hash.cu.
//
//   part_ids_kernel   : hash -> id in place (Spark pmod: ((h % P) + P) % P), per-tile histogram in shared memory,
//                       written partition-major ([P][ntiles]) so that one exclusive scan over the whole matrix yields,
//                       for every (partition, tile), where that tile's rows of that partition start.
//   i32 scan          : three-step exclusive scan of the matrix.
//   part_rank_kernel  : tile = one CTA; warp w owns a contiguous run of the tile's rows.  Per-warp counts of every
//                       partition (match.any: one leader per distinct id in a 32-row chunk, no atomics), a prefix over
//                       the warps, then the warp walks its rows again in order: destination = running count of
//                       (warp, id) + rank of the row among its chunk's rows of the same id.  Writes both maps:
//                       scatter_map[src] = dest (coalesced) and gather_map[dest] = src.
//   partition_scatter_*: fixed-width data moves src-ordered (coalesced reads, writes land in runs: the rows a tile sends
//                       to one partition are contiguous); validity bits and string lengths move dest-ordered through
//                       gather_map (a mask is n / 8 bytes: L2-resident); chars: a warp per 32 destination rows, lane = byte.
#include <algorithm>

#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"

namespace srj {

constexpr int kPartThreads = 1024;
constexpr int kPartMaxP    = 1 << 14;  // partitions (shared memory of the rank kernel: (warps + 1) x P ints)

__device__ __forceinline__ int32_t spark_pmod(int32_t h, int32_t P)
{
  const int32_t r = h % P;  // Spark Pmod: r < 0 ? (r + n) % n : r
  return r < 0 ? (r + P) % P : r;
}

// ---- ids + histogram -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPartThreads) part_ids_kernel(int32_t* __restrict__ ids, int64_t n, int32_t P, int32_t tile_rows,
                                                              int32_t ntiles, int32_t* __restrict__ hist)
{
  extern __shared__ int32_t s_hist[];
  for (int p = threadIdx.x; p < P; p += kPartThreads) s_hist[p] = 0;
  __syncthreads();
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * tile_rows;
  const int64_t r1 = tmin<int64_t>(n, r0 + tile_rows);
  for (int64_t r = r0 + threadIdx.x; r < r1; r += kPartThreads) {
    const int32_t id = spark_pmod(ids[r], P);
    ids[r]           = id;
    atomicAdd(&s_hist[id], 1);
  }
  __syncthreads();
  for (int p = threadIdx.x; p < P; p += kPartThreads) hist[static_cast<int64_t>(p) * ntiles + blockIdx.x] = s_hist[p];
}

// ---- exclusive scan of int32 (three steps: chunk sums, scan of the sums by one CTA, apply) -----------------------------
constexpr int kScanThreads = 256;
constexpr int kScanPer     = 16;  // elements per thread
constexpr int kScanChunk   = kScanThreads * kScanPer;

__device__ __forceinline__ int32_t block_exclusive_scan(int32_t v, int32_t* s_warp, int32_t& total)
{
  const int lane = lane_id(), w = warp_id();
  int32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[w] = x;
  __syncthreads();
  if (w == 0) {
    int32_t t = lane < kScanThreads / 32 ? s_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    s_warp[lane] = t;  // inclusive over the warps (entries past the last warp repeat the total)
  }
  __syncthreads();
  total              = s_warp[kScanThreads / 32 - 1];
  const int32_t base = w > 0 ? s_warp[w - 1] : 0;
  __syncthreads();
  return base + x - v;
}

__global__ void __launch_bounds__(kScanThreads) i32_chunk_sums_kernel(const int32_t* __restrict__ v, int64_t n, int32_t* __restrict__ sums)
{
  __shared__ int32_t s_warp[32];
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kScanChunk;
  int32_t acc = 0;
#pragma unroll
  for (int k = 0; k < kScanPer; ++k) {
    const int64_t i = base + k * kScanThreads + threadIdx.x;
    if (i < n) acc += v[i];
  }
  int32_t total;
  block_exclusive_scan(acc, s_warp, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) i32_scan_sums_kernel(int32_t* sums, int32_t nchunks)
{
  __shared__ int32_t s_warp[32];
  int32_t carry = 0;
  for (int32_t b = 0; b < nchunks; b += kScanThreads) {
    const int32_t i = b + threadIdx.x;
    const int32_t v = i < nchunks ? sums[i] : 0;
    int32_t total;
    const int32_t ex = block_exclusive_scan(v, s_warp, total);
    if (i < nchunks) sums[i] = carry + ex;
    carry += total;
  }
}

// exclusive scan in place; element i of `tail` (when given) receives the grand total
__global__ void __launch_bounds__(kScanThreads) i32_scan_apply_kernel(int32_t* __restrict__ v, int64_t n, const int32_t* __restrict__ sums,
                                                                     int32_t* __restrict__ tail)
{
  __shared__ int32_t s_warp[32];
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kScanChunk + static_cast<int64_t>(threadIdx.x) * kScanPer;
  int32_t x[kScanPer];
  int32_t acc = 0;
#pragma unroll
  for (int k = 0; k < kScanPer; ++k) {
    x[k] = base + k < n ? v[base + k] : 0;
    acc += x[k];
  }
  int32_t total;
  int32_t run = sums[blockIdx.x] + block_exclusive_scan(acc, s_warp, total);
#pragma unroll
  for (int k = 0; k < kScanPer; ++k) {
    if (base + k < n) v[base + k] = run;
    run += x[k];
  }
  if (tail && blockIdx.x == gridDim.x - 1 && threadIdx.x == kScanThreads - 1) *tail = run;
}

int64_t i32_scan_nchunks(int64_t n) { return (n + kScanChunk - 1) / kScanChunk; }

int launch_i32_exclusive_scan(int32_t* v, int64_t n, int32_t* sums /* nchunks ints */, int32_t* tail, cudaStream_t stream)
{
  if (n <= 0) return SRJ_OK;
  const int64_t nchunks = i32_scan_nchunks(n);
  i32_chunk_sums_kernel<<<static_cast<unsigned>(nchunks), kScanThreads, 0, stream>>>(v, n, sums);
  i32_scan_sums_kernel<<<1, kScanThreads, 0, stream>>>(sums, static_cast<int32_t>(nchunks));
  i32_scan_apply_kernel<<<static_cast<unsigned>(nchunks), kScanThreads, 0, stream>>>(v, n, sums, tail);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// ---- stable ranks ------------------------------------------------------------------------------------------------------
struct RankParams {
  const int32_t* ids;
  const int32_t* base;  // scanned histogram [P][ntiles]
  int64_t n;
  int32_t P, tile_rows, ntiles, nwarps;
  int32_t* scatter_map;  // [n] or NULL
  int32_t* gather_map;   // [n] or NULL
  int32_t* local_pos;    // [n]: rank of the row among its tile's rows ordered by destination (the tile kernel's staging order)
  int32_t* part_offsets; // [P + 1]
};

__global__ void __launch_bounds__(kPartThreads) part_rank_kernel(const __grid_constant__ RankParams p)
{
  extern __shared__ int32_t s_cnt[];  // [nwarps][P], then s_delta[P]
  __shared__ int32_t s_scan[32];
  const int W = p.nwarps, P = p.P;
  int32_t* s_delta = s_cnt + W * P;     // (rows of the tile in the partitions before p) - (where the tile's rows of p start)
  const int lane = lane_id(), w = warp_id();
  for (int i = threadIdx.x; i < W * P; i += blockDim.x) s_cnt[i] = 0;
  if (blockIdx.x == 0)
    for (int q = threadIdx.x; q <= P; q += blockDim.x)
      p.part_offsets[q] = q < P ? p.base[static_cast<int64_t>(q) * p.ntiles] : static_cast<int32_t>(p.n);
  __syncthreads();
  const int64_t t0  = static_cast<int64_t>(blockIdx.x) * p.tile_rows;
  const int rows_t  = static_cast<int>(tmin<int64_t>(p.tile_rows, p.n - t0));
  const int per_w   = ((p.tile_rows / W) + 31) & ~31;  // rows of a warp: whole 32-row chunks
  const int b0      = tmin(rows_t, w * per_w), b1 = tmin(rows_t, b0 + per_w);
  int32_t* cnt      = s_cnt + w * P;
  // A: this warp's rows per partition
  if (w < W)
    for (int c = b0; c < b1; c += 32) {
      const bool on    = c + lane < b1;
      const int32_t id = on ? p.ids[t0 + c + lane] : -1;
      const unsigned m = __match_any_sync(0xffffffffu, id);
      if (on && (m & ((1u << lane) - 1)) == 0) cnt[id] += __popc(m);  // one leader per distinct id of the chunk
      __syncwarp();
    }
  __syncthreads();
  // B: where (warp, partition) starts: the tile's base of the partition + the counts of the warps before; and the
  // exclusive prefix of the tile's own counts over the partitions (the tile-local order of its rows)
  {
    int32_t carry = 0;
    for (int q0 = 0; q0 < P; q0 += blockDim.x) {   // blockDim.x partitions per round
      const int q = q0 + threadIdx.x;
      int32_t tile_cnt = 0, b = 0;
      if (q < P) {
        b           = p.base[static_cast<int64_t>(q) * p.ntiles + blockIdx.x];
        int32_t run = b;
        for (int k = 0; k < W; ++k) {
          const int32_t c  = s_cnt[k * P + q];
          s_cnt[k * P + q] = run;
          run += c;
        }
        tile_cnt = run - b;
      }
      // block-wide exclusive scan of tile_cnt
      int32_t x = tile_cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) s_scan[w] = x;
      __syncthreads();
      if (w == 0) {
        int32_t t = s_scan[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int32_t y = __shfl_up_sync(0xffffffffu, t, o);
          if (lane >= o) t += y;
        }
        s_scan[lane] = t;
      }
      __syncthreads();
      const int32_t before = carry + (w > 0 ? s_scan[w - 1] : 0) + x - tile_cnt;
      if (q < P) s_delta[q] = before - b;
      carry += s_scan[31];
      __syncthreads();
    }
  }
  __syncthreads();
  // C: destinations, in row order
  if (w < W)
    for (int c = b0; c < b1; c += 32) {
      const bool on    = c + lane < b1;
      const int32_t id = on ? p.ids[t0 + c + lane] : -1;
      const unsigned m = __match_any_sync(0xffffffffu, id);
      if (on) {
        const int32_t dest = cnt[id] + __popc(m & ((1u << lane) - 1));
        const int64_t src  = t0 + c + lane;
        if (p.scatter_map) p.scatter_map[src] = dest;
        if (p.gather_map) p.gather_map[dest] = static_cast<int32_t>(src);
        if (p.local_pos) p.local_pos[src] = static_cast<int32_t>(t0) + dest + s_delta[id];
      }
      __syncwarp();
      if (on && (m & ((1u << lane) - 1)) == 0) cnt[id] += __popc(m);
      __syncwarp();
    }
}

// tile of a partitioning job: large enough that the histogram matrix stays small (P x ntiles ints)
static int32_t part_tile_rows(int32_t P)
{
  int32_t t = 4096;
  while (t < 8 * P) t <<= 1;
  return t;
}

// workspace: [local_pos: n ints | histogram matrix + scan partials (later: the string scans' partials)]
static int64_t partition_workspace_bytes(int64_t num_rows, int32_t P)
{
  if (num_rows <= 0 || P <= 0) return 256;
  const int64_t ntiles = (num_rows + part_tile_rows(P) - 1) / part_tile_rows(P);
  const int64_t hist   = static_cast<int64_t>(P) * ntiles;
  const int64_t tail   = std::max(hist + i32_scan_nchunks(hist), i32_scan_nchunks(num_rows + 1)) + 64;
  return ((num_rows + tail) * 4 + 255) & ~int64_t{255};
}

static int launch_partition_plan(int32_t* d_ids /* in: hashes, out: partition ids */, int64_t num_rows, int32_t P, int32_t* d_part_offsets,
                          int32_t* d_scatter_map, int32_t* d_gather_map, void* workspace, cudaStream_t stream)
{
  if (P <= 0 || P > kPartMaxP || num_rows < 0 || num_rows > INT32_MAX) return SRJ_EINVAL;
  if (num_rows == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(d_part_offsets, 0, (static_cast<size_t>(P) + 1) * 4, stream));
    return SRJ_OK;
  }
  const int32_t tile   = part_tile_rows(P);
  const int32_t ntiles = static_cast<int32_t>((num_rows + tile - 1) / tile);
  const int64_t hist_n = static_cast<int64_t>(P) * ntiles;
  int32_t* local_pos   = static_cast<int32_t*>(workspace);
  int32_t* hist        = local_pos + num_rows;
  int32_t* sums        = hist + hist_n;
  SRJ_CUDA_TRY(cudaFuncSetAttribute(part_ids_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPartMaxP * 4));
  part_ids_kernel<<<ntiles, kPartThreads, static_cast<size_t>(P) * 4, stream>>>(d_ids, num_rows, P, tile, ntiles, hist);
  const int rc = launch_i32_exclusive_scan(hist, hist_n, sums, nullptr, stream);
  if (rc != SRJ_OK) return rc;
  RankParams rp{};
  rp.ids          = d_ids;
  rp.base         = hist;
  rp.n            = num_rows;
  rp.P            = P;
  rp.tile_rows    = tile;
  rp.ntiles       = ntiles;
  rp.nwarps       = static_cast<int32_t>(std::max<int64_t>(1, std::min<int64_t>(kPartThreads / 32, (200 * 1024) / (static_cast<int64_t>(P) * 4) - 1)));
  rp.scatter_map  = d_scatter_map;
  rp.gather_map   = d_gather_map;
  rp.local_pos    = local_pos;
  rp.part_offsets = d_part_offsets;
  const size_t smem = (static_cast<size_t>(rp.nwarps) + 1) * P * 4;
  SRJ_CUDA_TRY(cudaFuncSetAttribute(part_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  part_rank_kernel<<<ntiles, kPartThreads, smem, stream>>>(rp);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// ---- moving the columns ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) scatter_fixed_kernel(const T* __restrict__ in, T* __restrict__ out, const int32_t* __restrict__ smap, int64_t n)
{
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x; r < n; r += static_cast<int64_t>(gridDim.x) * 256) out[smap[r]] = in[r];
}

// dest-ordered: validity bit of every destination row (one word per warp iteration)
__global__ void __launch_bounds__(256) gather_mask_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, const int32_t* __restrict__ gmap,
                                                         int64_t n, unsigned long long* __restrict__ null_count)
{
  const int lane = lane_id();
  int nulls      = 0;
  for (int64_t d0 = (static_cast<int64_t>(blockIdx.x) * 8 + warp_id()) * 32; d0 < n; d0 += static_cast<int64_t>(gridDim.x) * 256) {
    const int64_t d = d0 + lane;
    bool bit        = false;
    if (d < n) {
      const int32_t s = gmap[d];
      bit             = (in[s >> 5] >> (s & 31)) & 1u;
      nulls += !bit;
    }
    const unsigned word = __ballot_sync(0xffffffffu, bit);
    if (lane == 0) out[d0 >> 5] = word;
  }
  if (null_count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nulls += __shfl_down_sync(0xffffffffu, nulls, o);
    if (lane == 0 && nulls) atomicAdd(null_count, static_cast<unsigned long long>(nulls));
  }
}

// dest-ordered: out_offsets[d + 1] = length of the destination row's string (scanned afterwards); out_offsets[0] = 0
__global__ void __launch_bounds__(256) gather_lengths_kernel(const int32_t* __restrict__ in_off, int32_t* __restrict__ out_off,
                                                            const int32_t* __restrict__ gmap, int64_t n)
{
  for (int64_t d = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x; d < n; d += static_cast<int64_t>(gridDim.x) * 256) {
    const int32_t s = gmap[d];
    out_off[d]      = in_off[s + 1] - in_off[s];  // exclusive scan in place turns element d into the start of string d
  }
}

// chars: a warp per 32 destination rows; lane = destination byte, its row by a shuffle search over the 32 starts
__global__ void __launch_bounds__(256) gather_chars_kernel(const uint8_t* __restrict__ in_chars, const int32_t* __restrict__ in_off,
                                                          uint8_t* __restrict__ out_chars, const int32_t* __restrict__ out_off,
                                                          const int32_t* __restrict__ gmap, int64_t n)
{
  const int lane = lane_id();
  for (int64_t d0 = (static_cast<int64_t>(blockIdx.x) * 8 + warp_id()) * 32; d0 < n; d0 += static_cast<int64_t>(gridDim.x) * 256) {
    const int last   = static_cast<int>(tmin<int64_t>(32, n - d0)) - 1;
    const int64_t d  = tmin<int64_t>(d0 + lane, n - 1);
    const int32_t ob = out_off[d0];
    const int32_t pe = out_off[d] - ob;              // where this lane's string starts among the tile's bytes
    const int32_t so = in_off[gmap[d]];              // ... and where it comes from
    const int32_t T  = out_off[d0 + last + 1] - ob;  // bytes of the 32 strings
    for (int32_t q = lane; q < ((T + 31) & ~31); q += 32) {
      int j = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const int cand  = j + step;
        const int32_t v = __shfl_sync(0xffffffffu, pe, cand & 31);
        if (cand <= last && v <= q) j = cand;
      }
      const int32_t pj = __shfl_sync(0xffffffffu, pe, j);
      const int32_t sj = __shfl_sync(0xffffffffu, so, j);
      if (q < T) out_chars[ob + q] = in_chars[sj + (q - pj)];
    }
  }
}

// ---- moving the columns, tile by tile ------------------------------------------------------------------------------------
// One CTA per tile of the plan.  The tile's rows are staged in shared memory in destination order (local_pos), so that
// consecutive threads then write consecutive destinations: the rows a tile sends to one partition leave as one run
// instead of one 4-byte transaction per row.  The destination of every staged position is kept in shared memory for
// the whole column loop; validity bits travel the same way and reach the output words through one atomicOr per
// (warp, word).
constexpr int kMoveCols = 48;  // columns per launch (descriptor table in the kernel parameters)
struct MoveParams {
  const int32_t* smap;
  const int32_t* local_pos;
  int64_t n;
  int32_t tile_rows, ncols;
  unsigned long long* null_counts;  // [ncols of the launch] or NULL
  const void* in[kMoveCols];
  void* out[kMoveCols];
  const uint32_t* in_mask[kMoveCols];
  uint32_t* out_mask[kMoveCols];    // zeroed by the caller
  uint8_t width[kMoveCols];         // 0: no data (STRING: mask only)
};

template <typename T>
__device__ __forceinline__ void move_stage(const T* __restrict__ in, T* s_val, int64_t t0, int rows_t, const int32_t* lp, int rpt)
{
  for (int k = 0; k < rpt; ++k) {
    const int i = k * kPartThreads + threadIdx.x;
    if (i < rows_t) s_val[lp[k]] = in[t0 + i];
  }
}
template <typename T>
__device__ __forceinline__ void move_write(T* __restrict__ out, const T* s_val, const int32_t* s_dest, int rows_t, int rpt)
{
  for (int k = 0; k < rpt; ++k) {
    const int i = k * kPartThreads + threadIdx.x;
    if (i < rows_t) out[s_dest[i]] = s_val[i];
  }
}

constexpr int kMoveMaxRpt = 8;    // tile_rows <= 8 x 1024
constexpr int kMoveGroupB = 16;   // bytes per row staged between two CTA barriers: columns move in groups of <= 16 bytes

__global__ void __launch_bounds__(kPartThreads) partition_move_tile_kernel(const __grid_constant__ MoveParams p)
{
  extern __shared__ __align__(16) uint8_t s_raw[];
  __shared__ int s_nulls[kMoveGroupB];
  int32_t* s_dest = reinterpret_cast<int32_t*>(s_raw);                     // [tile_rows]
  uint8_t* s_val  = s_raw + static_cast<size_t>(p.tile_rows) * 4;         // [tile_rows] x 16 bytes
  const int64_t t0 = static_cast<int64_t>(blockIdx.x) * p.tile_rows;
  const int rows_t = static_cast<int>(tmin<int64_t>(p.tile_rows, p.n - t0));
  const int rpt    = p.tile_rows / kPartThreads;
  const int lane   = lane_id();
  int32_t lp[kMoveMaxRpt];
#pragma unroll
  for (int k = 0; k < kMoveMaxRpt; ++k) {
    lp[k]       = 0;
    const int i = k * kPartThreads + threadIdx.x;
    if (k < rpt && i < rows_t) {
      lp[k]         = p.local_pos[t0 + i] - static_cast<int32_t>(t0);   // (see part_rank_kernel: rank inside the tile)
      s_dest[lp[k]] = p.smap[t0 + i];
    }
  }
  __syncthreads();
  // ---- data: groups of columns whose widths add up to <= 16 bytes share one stage / write round ----
  for (int c0 = 0; c0 < p.ncols;) {
    int c1 = c0, acc = 0;
    while (c1 < p.ncols && acc + p.width[c1] <= kMoveGroupB) acc += p.width[c1++];
    for (int pass = 0; pass < 2; ++pass) {
      int at = 0;
      for (int c = c0; c < c1; ++c) {
        const int W = p.width[c];
        uint8_t* area = s_val + static_cast<size_t>(at) * p.tile_rows;   // every area starts 16-byte aligned: tile_rows is a multiple of 1024
        at += W;
        switch (W) {
          case 1: pass == 0 ? move_stage(static_cast<const uint8_t*>(p.in[c]), area, t0, rows_t, lp, rpt) : move_write(static_cast<uint8_t*>(p.out[c]), area, s_dest, rows_t, rpt); break;
          case 2: pass == 0 ? move_stage(static_cast<const uint16_t*>(p.in[c]), reinterpret_cast<uint16_t*>(area), t0, rows_t, lp, rpt) : move_write(static_cast<uint16_t*>(p.out[c]), reinterpret_cast<uint16_t*>(area), s_dest, rows_t, rpt); break;
          case 4: pass == 0 ? move_stage(static_cast<const uint32_t*>(p.in[c]), reinterpret_cast<uint32_t*>(area), t0, rows_t, lp, rpt) : move_write(static_cast<uint32_t*>(p.out[c]), reinterpret_cast<uint32_t*>(area), s_dest, rows_t, rpt); break;
          case 8: pass == 0 ? move_stage(static_cast<const uint2*>(p.in[c]), reinterpret_cast<uint2*>(area), t0, rows_t, lp, rpt) : move_write(static_cast<uint2*>(p.out[c]), reinterpret_cast<uint2*>(area), s_dest, rows_t, rpt); break;
          case 16: pass == 0 ? move_stage(static_cast<const uint4*>(p.in[c]), reinterpret_cast<uint4*>(area), t0, rows_t, lp, rpt) : move_write(static_cast<uint4*>(p.out[c]), reinterpret_cast<uint4*>(area), s_dest, rows_t, rpt); break;
          default: break;
        }
      }
      __syncthreads();
    }
    c0 = c1 > c0 ? c1 : c0 + 1;
  }
  // ---- null masks: up to 16 columns' validity bits per round, one byte per (row, column) ----
  for (int c0 = 0; c0 < p.ncols; c0 += kMoveGroupB) {
    const int c1 = tmin(p.ncols, c0 + kMoveGroupB);
    bool any = false;
    for (int c = c0; c < c1; ++c) any |= p.in_mask[c] && p.out_mask[c];
    if (!any) continue;   // CTA-uniform
    if (threadIdx.x < kMoveGroupB) s_nulls[threadIdx.x] = 0;
    for (int k = 0; k < rpt; ++k) {
      const int i = k * kPartThreads + threadIdx.x;
      if (i < rows_t)
        for (int c = c0; c < c1; ++c) {
          const uint32_t* im = p.in_mask[c];
          if (im && p.out_mask[c]) s_val[static_cast<size_t>(c - c0) * p.tile_rows + lp[k]] = static_cast<uint8_t>((im[(t0 + i) >> 5] >> ((t0 + i) & 31)) & 1u);
        }
    }
    __syncthreads();
    for (int k = 0; k < rpt; ++k) {
      const int i     = k * kPartThreads + threadIdx.x;
      const bool on   = i < rows_t;
      const int32_t d = on ? s_dest[i] : -2;
      // lanes whose destinations are consecutive and fall into one output word form a segment; its head ORs the
      // segment's bits into that word with one atomic
      const int32_t dprev  = __shfl_up_sync(0xffffffffu, d, 1);
      const bool head      = on && (lane == 0 || d != dprev + 1 || (d & 31) == 0);
      const unsigned heads = __ballot_sync(0xffffffffu, head || !on);
      const unsigned later = lane < 31 ? heads >> (lane + 1) : 0u;
      const int seg_len    = later ? __ffs(later) : 32 - lane;   // lanes up to the next head (or the end of the warp)
      const unsigned seg   = (seg_len >= 32 ? 0xffffffffu : ((1u << seg_len) - 1u)) << lane;
      for (int c = c0; c < c1; ++c) {
        uint32_t* om = p.out_mask[c];
        if (!p.in_mask[c] || !om) continue;
        const uint32_t b     = on ? s_val[static_cast<size_t>(c - c0) * p.tile_rows + i] : 0u;
        const unsigned valid = __ballot_sync(0xffffffffu, b != 0);
        if (head) {
          const uint32_t wd = ((valid & seg) >> lane) << (d & 31);
          if (wd) atomicOr(om + (d >> 5), wd);
        }
        if (p.null_counts) {   // per CTA in shared memory first: one global atomic per (tile, column)
          const int nulls = __popc(__ballot_sync(0xffffffffu, on) & ~valid);
          if (lane == 0 && nulls) atomicAdd(&s_nulls[c - c0], nulls);
        }
      }
    }
    __syncthreads();
    if (p.null_counts && threadIdx.x < c1 - c0 && s_nulls[threadIdx.x]) atomicAdd(p.null_counts + c0 + threadIdx.x, static_cast<unsigned long long>(s_nulls[threadIdx.x]));
    __syncthreads();
  }
}

// local_pos as written by part_rank_kernel is an ABSOLUTE position (tile start + rank inside the tile); every column
// (data of fixed-width columns, null masks of all) of `in` moves to `out`.  Returns SRJ_EUNSUPPORTED when the plan's
// tiles do not fit the staging buffers (more than 1024 partitions): the caller then uses the per-row kernels.
static int launch_partition_move_tiles(const srj_column* in, const srj_column* out, const int* elem_size, int32_t ncols, int64_t n, int32_t P,
                                const int32_t* d_scatter_map, const void* workspace, unsigned long long* d_null_counts, cudaStream_t stream)
{
  const int32_t tile = part_tile_rows(P);
  if (tile > kMoveMaxRpt * kPartThreads) return SRJ_EUNSUPPORTED;
  if (n == 0 || ncols == 0) return SRJ_OK;
  const int32_t ntiles = static_cast<int32_t>((n + tile - 1) / tile);
  const size_t smem    = static_cast<size_t>(tile) * 20;
  SRJ_CUDA_TRY(cudaFuncSetAttribute(partition_move_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMoveMaxRpt * kPartThreads * 20));
  for (int32_t c0 = 0; c0 < ncols; c0 += kMoveCols) {
    MoveParams mp{};
    mp.smap        = d_scatter_map;
    mp.local_pos   = static_cast<const int32_t*>(workspace);
    mp.n           = n;
    mp.tile_rows   = tile;
    mp.ncols       = std::min(kMoveCols, ncols - c0);
    mp.null_counts = d_null_counts ? d_null_counts + c0 : nullptr;
    for (int k = 0; k < mp.ncols; ++k) {
      const srj_column& a = in[c0 + k];
      const srj_column& b = out[c0 + k];
      mp.width[k]    = static_cast<uint8_t>(elem_size[c0 + k]);
      mp.in[k]       = a.data;
      mp.out[k]      = b.data;
      mp.in_mask[k]  = a.null_mask;
      mp.out_mask[k] = a.null_mask ? b.null_mask : nullptr;
      if (a.null_mask && b.null_mask) SRJ_CUDA_TRY(cudaMemsetAsync(b.null_mask, 0, static_cast<size_t>((n + 31) / 32) * 4, stream));
    }
    partition_move_tile_kernel<<<ntiles, kPartThreads, smem, stream>>>(mp);
  }
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static unsigned grid_for(int64_t n, int per_block)
{
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + per_block - 1) / per_block, int64_t{sm_count()} * 16)));
}

static int launch_partition_scatter_fixed(const void* in, void* out, int elem_size, const int32_t* d_scatter_map, int64_t n, cudaStream_t stream)
{
  if (n == 0) return SRJ_OK;
  const unsigned g = grid_for(n, 256);
  switch (elem_size) {
    case 1: scatter_fixed_kernel<uint8_t><<<g, 256, 0, stream>>>(static_cast<const uint8_t*>(in), static_cast<uint8_t*>(out), d_scatter_map, n); break;
    case 2: scatter_fixed_kernel<uint16_t><<<g, 256, 0, stream>>>(static_cast<const uint16_t*>(in), static_cast<uint16_t*>(out), d_scatter_map, n); break;
    case 4: scatter_fixed_kernel<uint32_t><<<g, 256, 0, stream>>>(static_cast<const uint32_t*>(in), static_cast<uint32_t*>(out), d_scatter_map, n); break;
    case 8: scatter_fixed_kernel<uint2><<<g, 256, 0, stream>>>(static_cast<const uint2*>(in), static_cast<uint2*>(out), d_scatter_map, n); break;
    case 16: scatter_fixed_kernel<uint4><<<g, 256, 0, stream>>>(static_cast<const uint4*>(in), static_cast<uint4*>(out), d_scatter_map, n); break;
    default: return SRJ_EUNSUPPORTED;
  }
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_partition_gather_mask(const uint32_t* in, uint32_t* out, const int32_t* d_gather_map, int64_t n, unsigned long long* d_null_count,
                                 cudaStream_t stream)
{
  if (n == 0) return SRJ_OK;
  gather_mask_kernel<<<grid_for(n, 256), 256, 0, stream>>>(in, out, d_gather_map, n, d_null_count);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// out_off[0 .. n] <- offsets of the partitioned column; *d_total (device int32, = out_off[n]) the chars it needs
static int launch_partition_string_offsets(const int32_t* in_off, int32_t* out_off, const int32_t* d_gather_map, int64_t n, void* scan_ws,
                                    cudaStream_t stream)
{
  if (n == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(out_off, 0, 4, stream));
    return SRJ_OK;
  }
  gather_lengths_kernel<<<grid_for(n, 256), 256, 0, stream>>>(in_off, out_off, d_gather_map, n);
  // exclusive scan of the n lengths in place; the grand total lands in out_off[n]
  return launch_i32_exclusive_scan(out_off, n, static_cast<int32_t*>(scan_ws), out_off + n, stream);
}

static int launch_partition_gather_chars(const uint8_t* in_chars, const int32_t* in_off, uint8_t* out_chars, const int32_t* out_off,
                                  const int32_t* d_gather_map, int64_t n, cudaStream_t stream)
{
  if (n == 0) return SRJ_OK;
  gather_chars_kernel<<<grid_for(n, 256), 256, 0, stream>>>(in_chars, in_off, out_chars, out_off, d_gather_map, n);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

int64_t srj_partition_workspace_bytes(int64_t num_rows, int32_t num_partitions)
{
  return partition_workspace_bytes(num_rows, num_partitions);
}

int srj_partition_plan(int32_t* d_partition_ids, int64_t num_rows, int32_t num_partitions, int32_t* d_partition_offsets,
                       int32_t* d_scatter_map, int32_t* d_gather_map, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  if (num_rows < 0 || num_partitions <= 0 || !d_partition_offsets || (num_rows > 0 && (!d_partition_ids || !workspace))) {
    set_error("partition_plan: bad argument");
    return SRJ_EINVAL;
  }
  if (num_rows > INT32_MAX || num_partitions > (1 << 14)) {
    set_error("partition_plan: %lld rows / %d partitions exceed the int32 row index / 16384 partitions", static_cast<long long>(num_rows), num_partitions);
    return SRJ_EUNSUPPORTED;
  }
  return launch_partition_plan(d_partition_ids, num_rows, num_partitions, d_partition_offsets, d_scatter_map, d_gather_map, workspace,
                               static_cast<cudaStream_t>(stream));
}

int srj_hash_partition(const srj_column* keys, int32_t num_keys, int64_t num_rows, uint32_t seed, int32_t num_partitions,
                       int32_t* d_partition_ids, int32_t* d_partition_offsets, int32_t* d_scatter_map, int32_t* d_gather_map,
                       void* workspace, void* stream)
{
  SRJ_API_RANGE();
  if (num_keys <= 0 || !keys) { set_error("hash_partition: no key columns"); return SRJ_EINVAL; }
  if (num_rows > 0 && !d_partition_ids) { set_error("hash_partition: bad argument"); return SRJ_EINVAL; }
  // the partition count is checked before the keys are hashed: a refused call launches nothing
  if (num_partitions <= 0) { set_error("hash_partition: %d partitions", num_partitions); return SRJ_EINVAL; }
  if (num_partitions > (1 << 14)) { set_error("hash_partition: %d partitions exceed 16384 partitions", num_partitions); return SRJ_EUNSUPPORTED; }
  // the hashes go where the ids will be: part_ids_kernel turns them into ids in place
  int rc = hash_columns(SRJ_HASH_MURMUR3_32, keys, num_keys, num_rows, seed, d_partition_ids, static_cast<cudaStream_t>(stream));
  if (rc != SRJ_OK) return rc;
  return srj_partition_plan(d_partition_ids, num_rows, num_partitions, d_partition_offsets, d_scatter_map, d_gather_map, workspace, stream);
}

int srj_partition_columns(const srj_column* in, const srj_column* out, int32_t num_columns, int64_t num_rows, int32_t num_partitions,
                          const int32_t* d_scatter_map, const int32_t* d_gather_map, int64_t* d_null_counts, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (num_columns < 0 || num_rows < 0 || num_partitions <= 0 || (num_columns > 0 && (!in || !out))) { set_error("partition_columns: bad argument"); return SRJ_EINVAL; }
  if (num_rows > 0 && (!d_scatter_map || !d_gather_map || !workspace)) { set_error("partition_columns: the maps and the plan's workspace are needed"); return SRJ_EINVAL; }
  if (d_null_counts && num_columns > 0) SRJ_CUDA_TRY(cudaMemsetAsync(d_null_counts, 0, sizeof(int64_t) * num_columns, st));
  std::vector<int> esz(static_cast<size_t>(num_columns), 0);
  for (int32_t c = 0; c < num_columns; ++c) {
    const srj_column& a = in[c];
    const srj_column& b = out[c];
    if (a.type_id != b.type_id || a.size != num_rows || b.size != num_rows) { set_error("partition_columns: column %d: type / size mismatch", c); return SRJ_EINVAL; }
    if (a.type_id == SRJ_STRING) {
      if (!a.offsets || !b.offsets) { set_error("partition_columns: STRING column %d needs offsets", c); return SRJ_EINVAL; }
    } else {
      esz[c] = type_width(a.type_id);
      if (esz[c] <= 0) { set_error("partition_columns: column %d: unsupported type %d", c, a.type_id); return SRJ_EUNSUPPORTED; }
      if (num_rows > 0 && (!a.data || !b.data)) { set_error("partition_columns: column %d: NULL data", c); return SRJ_EINVAL; }
    }
    if (a.null_mask && !b.null_mask) { set_error("partition_columns: column %d has a null mask but its output has none", c); return SRJ_EINVAL; }
    if (!a.null_mask && b.null_mask && num_rows > 0) SRJ_CUDA_TRY(cudaMemsetAsync(b.null_mask, 0xff, static_cast<size_t>((num_rows + 31) / 32) * 4, st));
  }
  // fixed-width data and every null mask: tile by tile, staged in destination order (plans of <= 1024 partitions) ...
  int rc = launch_partition_move_tiles(in, out, esz.data(), num_columns, num_rows, num_partitions, d_scatter_map, workspace,
                                       reinterpret_cast<unsigned long long*>(d_null_counts), st);
  if (rc == SRJ_EUNSUPPORTED) {
    // ... or row by row
    rc = SRJ_OK;
    for (int32_t c = 0; c < num_columns && rc == SRJ_OK && num_rows > 0; ++c) {
      if (esz[c] > 0) rc = launch_partition_scatter_fixed(in[c].data, out[c].data, esz[c], d_scatter_map, num_rows, st);
      if (rc == SRJ_OK && in[c].null_mask)
        rc = launch_partition_gather_mask(in[c].null_mask, out[c].null_mask, d_gather_map, num_rows,
                                          d_null_counts ? reinterpret_cast<unsigned long long*>(d_null_counts + c) : nullptr, st);
    }
  }
  if (rc != SRJ_OK) return rc;
  // STRING columns: the output offsets (lengths through the gather map, then a scan; partials behind the plan's tile order)
  for (int32_t c = 0; c < num_columns; ++c) {
    if (in[c].type_id != SRJ_STRING) continue;
    if (num_rows == 0) {
      SRJ_CUDA_TRY(cudaMemsetAsync(out[c].offsets, 0, 4, st));   // an empty STRING column still has its offsets[0] = 0
      continue;
    }
    rc = launch_partition_string_offsets(in[c].offsets, out[c].offsets, d_gather_map, num_rows, static_cast<int32_t*>(workspace) + num_rows, st);
    if (rc != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

int srj_partition_strings(const srj_column* in, const srj_column* out, int32_t num_columns, int64_t num_rows, const int32_t* d_gather_map,
                          void* stream)
{
  SRJ_API_RANGE();
  if (num_columns < 0 || num_rows < 0 || (num_columns > 0 && (!in || !out))) { set_error("partition_strings: bad argument"); return SRJ_EINVAL; }
  for (int32_t c = 0; c < num_columns; ++c) {
    if (in[c].type_id != SRJ_STRING || num_rows == 0) continue;
    if (!out[c].offsets || !in[c].offsets) { set_error("partition_strings: column %d: NULL offsets", c); return SRJ_EINVAL; }
    const int rc = launch_partition_gather_chars(static_cast<const uint8_t*>(in[c].data), in[c].offsets, static_cast<uint8_t*>(out[c].data),
                                                 out[c].offsets, d_gather_map, num_rows, static_cast<cudaStream_t>(stream));
    if (rc != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

}  // extern "C"
