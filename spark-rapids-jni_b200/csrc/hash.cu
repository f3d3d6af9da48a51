// hash.cu -- standalone Spark row hashes over columns (reference: hash/xxhash64.cu:550-579,
// hash/murmur_hash.cu:191-221, hash/hive_hash.cu:474-500; the reference runs
// thrust::tabulate with a per-row type_dispatcher over a table_device_view).
//
// Here the column descriptors travel as a __grid_constant__ kernel parameter (no
// table_device_view allocation / H2D copy); tables wider than kHashColsPerLaunch are hashed in
// column chunks chained through the output column (the accumulator IS the next chunk's seed, which
// is exactly the Spark chaining rule), so there is no hidden allocation at any width.
#include <algorithm>
#include <cstdlib>
#include <type_traits>
#include "check.hpp"
#include "common.cuh"
#include "hash_device.cuh"
#include "kernels.hpp"
#include "movers.cuh"

namespace srj {

constexpr int kHashColsPerLaunch = 48;
constexpr int kHashThreads       = 256;

struct HashCol {
  const uint8_t* data;
  const uint32_t* mask;
  const int32_t* offsets;
  int16_t type;
  int16_t kind;  // 0 = generic dispatch, 1 = plain 4-byte value, 2 = plain 8-byte value (hashed as raw bits)
  int32_t size;  // bytes per element (0 for STRING)
};

struct HashParams {
  HashCol cols[kHashColsPerLaunch];
  int32_t ncols;
  int32_t kind;
  int32_t first;  // 1: accumulator starts from the seed; 0: from out[r] (a previous column chunk)
  int32_t pad;
  int64_t seed;
  int64_t n;
  void* out;
};

__device__ __forceinline__ bool row_valid(const uint32_t* m, int64_t r)
{
  return !m || ((__ldg(m + (r >> 5)) >> (r & 31)) & 1u);
}

__device__ __forceinline__ void load_fixed(const HashCol& c, int64_t r, uint64_t& v, uint64_t& v2)
{
  v2 = 0;
  switch (c.size) {
    case 1: v = __ldg(c.data + r); break;
    case 2: v = __ldg(reinterpret_cast<const uint16_t*>(c.data) + r); break;
    case 4: v = __ldg(reinterpret_cast<const uint32_t*>(c.data) + r); break;
    case 8: v = __ldg(reinterpret_cast<const unsigned long long*>(c.data) + r); break;
    default: {
      const ulonglong2 q = __ldg(reinterpret_cast<const ulonglong2*>(c.data) + r);
      v                  = q.x;
      v2                 = q.y;
    }
  }
}

// Each thread hashes kRowsPerThread rows (strided by the block size, so every load stays coalesced): the
// per-column dispatch is paid once per kRowsPerThread rows, the dependent multiply chains of the rows
// overlap (ILP), and the NEXT column's values and mask words are fetched (unconditionally: fixed-width
// reads never depend on validity) while the current column is hashed -- the memory-level parallelism a
// one-row-per-thread loop (thrust::tabulate in the reference) lacks.
constexpr int kRowsPerThread = 4;

struct Fetched {
  uint64_t v[kRowsPerThread];
  uint64_t v2[kRowsPerThread];
  bool ok[kRowsPerThread];
};

__device__ __forceinline__ void fetch_column(const HashCol& col, const int64_t (&r)[kRowsPerThread],
                                             const bool (&live)[kRowsPerThread], Fetched& f)
{
  if (col.type == SRJ_STRING) {  // strings are read where they are hashed
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) f.ok[j] = live[j] && row_valid(col.mask, r[j]);
    return;
  }
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    f.v[j] = f.v2[j] = 0;
    if (live[j]) {
      if (col.kind == 1) f.v[j] = __ldg(reinterpret_cast<const uint32_t*>(col.data) + r[j]);
      else if (col.kind == 2) f.v[j] = __ldg(reinterpret_cast<const unsigned long long*>(col.data) + r[j]);
      else load_fixed(col, r[j], f.v[j], f.v2[j]);
    }
    f.ok[j] = live[j] && row_valid(col.mask, r[j]);
  }
}

// Each thread makes one pass (load 4 rows of every key column, hash, store), so the kernel lives on occupancy:
// 4 resident CTAs (64 registers) for the multiply-heavy xxhash64 / murmur3, 5 (48 registers) for hive, rather than
// the unbounded 80-register build.
template <int KIND>
__global__ void __launch_bounds__(kHashThreads, KIND == SRJ_HASH_HIVE ? 5 : 4) row_hash_kernel(const __grid_constant__ HashParams p)
{
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * (kHashThreads * kRowsPerThread) + threadIdx.x;
  int64_t r[kRowsPerThread];
  bool live[kRowsPerThread];
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    r[j]    = r0 + static_cast<int64_t>(j) * kHashThreads;
    live[j] = r[j] < p.n;
  }
  if (!live[0]) return;
  using acc_t = typename std::conditional<KIND == SRJ_HASH_XXHASH64, uint64_t, uint32_t>::type;
  acc_t h[kRowsPerThread];
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    if (p.first || !live[j]) h[j] = KIND == SRJ_HASH_HIVE ? acc_t{0} : static_cast<acc_t>(p.seed);
    else h[j] = reinterpret_cast<const acc_t*>(p.out)[r[j]];
  }
  Fetched cur, nxt;
  fetch_column(p.cols[0], r, live, cur);
  for (int c = 0; c < p.ncols; ++c) {
    const HashCol col = p.cols[c];
    if (c + 1 < p.ncols) fetch_column(p.cols[c + 1], r, live, nxt);  // in flight while this column is hashed
    if (col.type == SRJ_STRING) {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) {
        if constexpr (KIND == SRJ_HASH_HIVE) {
          uint32_t x = 0;  // null -> 0 (hive_hash.cu:201-203)
          if (cur.ok[j]) {
            const int32_t o0 = __ldg(col.offsets + r[j]), o1 = __ldg(col.offsets + r[j] + 1);
            x                = static_cast<uint32_t>(hash::hive_bytes(col.data + o0, o1 - o0));
          }
          if (live[j]) h[j] = 31u * h[j] + x;
        } else {
          if (!cur.ok[j]) continue;  // null keeps the accumulator (xxhash64.cu:352-353, murmur_hash.cu:111-117)
          const int32_t o0 = __ldg(col.offsets + r[j]), o1 = __ldg(col.offsets + r[j] + 1);
          if constexpr (KIND == SRJ_HASH_XXHASH64) h[j] = hash::xx_bytes(col.data + o0, o1 - o0, h[j]);
          else h[j] = hash::mm_bytes(col.data + o0, o1 - o0, h[j]);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) {
        if constexpr (KIND == SRJ_HASH_XXHASH64) {
          if (cur.ok[j]) {
            if (col.kind == 1) h[j] = hash::xx_u32(static_cast<uint32_t>(cur.v[j]), h[j]);
            else if (col.kind == 2) h[j] = hash::xx_u64(cur.v[j], h[j]);
            else h[j] = hash::xx_fixed(col.type, cur.v[j], cur.v2[j], h[j]);
          }
        } else if constexpr (KIND == SRJ_HASH_MURMUR3_32) {
          if (cur.ok[j]) {
            if (col.kind == 1) h[j] = hash::mm_u32(static_cast<uint32_t>(cur.v[j]), h[j]);
            else if (col.kind == 2) h[j] = hash::mm_u64(cur.v[j], h[j]);
            else h[j] = hash::mm_fixed(col.type, cur.v[j], cur.v2[j], h[j]);
          }
        } else {
          uint32_t x = 0;
          if (cur.ok[j]) {
            if (col.kind == 1) x = static_cast<uint32_t>(cur.v[j]);                      // INT32 / DATE (hive_hash.cu:97-133)
            else if (col.kind == 2) x = static_cast<uint32_t>((cur.v[j] >> 32) ^ cur.v[j]);  // INT64 (hive_hash.cu:44-47)
            else x = static_cast<uint32_t>(hash::hive_fixed(col.type, cur.v[j]));
          }
          if (live[j]) h[j] = 31u * h[j] + x;  // hive_hash.cu:179-191
        }
      }
    }
    cur = nxt;
  }
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j)
    if (live[j]) reinterpret_cast<acc_t*>(p.out)[r[j]] = h[j];
}


// Every key column is a plain 4- or 8-byte value hashed as stored (32/64-bit integers, dates, timestamps,
// durations, DECIMAL64): no type dispatch, no 16-byte lane, no string branch -- fewer registers and ~25 % fewer
// instructions per row than the general kernel above.  Same structure: 4 rows per thread, next column in flight.
template <int KIND>
__global__ void __launch_bounds__(kHashThreads, KIND == SRJ_HASH_HIVE ? 5 : 4) row_hash_plain_kernel(const __grid_constant__ HashParams p)
{
  // grid-stride over row blocks: a resident CTA keeps going (no relaunch gap between blocks)
  const int64_t nblk = (p.n + kHashThreads * kRowsPerThread - 1) / (kHashThreads * kRowsPerThread);
  for (int64_t blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
  const int64_t r0 = blk * (kHashThreads * kRowsPerThread) + threadIdx.x;
  int64_t r[kRowsPerThread];
  bool live[kRowsPerThread];
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    r[j]    = r0 + static_cast<int64_t>(j) * kHashThreads;
    live[j] = r[j] < p.n;
  }
  if (!live[0]) continue;
  using acc_t = typename std::conditional<KIND == SRJ_HASH_XXHASH64, uint64_t, uint32_t>::type;
  acc_t h[kRowsPerThread];
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    if (p.first || !live[j]) h[j] = KIND == SRJ_HASH_HIVE ? acc_t{0} : static_cast<acc_t>(p.seed);
    else h[j] = reinterpret_cast<const acc_t*>(p.out)[r[j]];
  }
  uint64_t cv[kRowsPerThread], nv[kRowsPerThread];
  bool cok[kRowsPerThread], nok[kRowsPerThread];
  auto fetch = [&](const HashCol& col, uint64_t (&v)[kRowsPerThread], bool (&ok)[kRowsPerThread]) {
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      v[j] = 0;
      if (live[j]) {
        if (col.kind == 1) v[j] = __ldg(reinterpret_cast<const uint32_t*>(col.data) + r[j]);
        else v[j] = __ldg(reinterpret_cast<const unsigned long long*>(col.data) + r[j]);
      }
      ok[j] = live[j] && row_valid(col.mask, r[j]);
    }
  };
  fetch(p.cols[0], cv, cok);
  for (int c = 0; c < p.ncols; ++c) {
    const bool four = p.cols[c].kind == 1;
    if (c + 1 < p.ncols) fetch(p.cols[c + 1], nv, nok);  // in flight while this column is hashed
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      if constexpr (KIND == SRJ_HASH_XXHASH64) {
        const uint64_t t = four ? hash::xx_u32(static_cast<uint32_t>(cv[j]), h[j]) : hash::xx_u64(cv[j], h[j]);
        h[j]             = cok[j] ? t : h[j];  // a null keeps the accumulator (xxhash64.cu:352-353)
      } else if constexpr (KIND == SRJ_HASH_MURMUR3_32) {
        const uint32_t t = four ? hash::mm_u32(static_cast<uint32_t>(cv[j]), h[j]) : hash::mm_u64(cv[j], h[j]);
        h[j]             = cok[j] ? t : h[j];  // murmur_hash.cu:111-117
      } else {
        const uint32_t x = four ? static_cast<uint32_t>(cv[j]) : static_cast<uint32_t>((cv[j] >> 32) ^ cv[j]);
        h[j]             = 31u * h[j] + (cok[j] ? x : 0u);  // hive_hash.cu:179-203 (null -> 0)
      }
    }
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      cv[j]  = nv[j];
      cok[j] = nok[j];
    }
  }
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j)
    if (live[j]) reinterpret_cast<acc_t*>(p.out)[r[j]] = h[j];
  }
}

// --------------------------------------------------------------------------------------------------
// Streaming row hash for fixed-width keys (the shuffle-partitioning case: a few 4/8-byte key columns, 10^8 rows).
// The kernels above issue their global loads from the hashing threads, so every row block waits a DRAM round trip
// before its multiply chains can start (long-scoreboard stalls dominate).  Here the
// loads are decoupled from the arithmetic, the way the conversion kernels do it:
//   producer warp : per chunk of kHsRows rows, one TMA bulk copy per key column (a contiguous, 16-byte aligned piece
//                   of the column) and per mask into a ring of shared-memory stages guarded by full/empty mbarriers;
//   consumer warps: lane = row, four rows per lane (four independent multiply chains), values read from shared
//                   memory (conflict-free: consecutive lanes, consecutive elements), chained across the key columns
//                   with the Spark rules, one coalesced store of the hash per row group.
// --------------------------------------------------------------------------------------------------
constexpr int kHsRows    = 2048;  // rows per chunk
constexpr int kHsWarps   = 16;    // consumer warps: 4 row groups of a chunk each
constexpr int kHsMaxCols = 16;    // key columns per launch
constexpr int kHsMaxStages = 6;
constexpr int kHsThreads = (kHsWarps + 1) * 32;

struct HsParams {
  HashCol cols[kHsMaxCols];
  int32_t col_off[kHsMaxCols];   // byte offset of the column's values inside a stage
  int32_t mask_off[kHsMaxCols];  // byte offset of its 64 mask words, or -1 (no mask: all valid)
  int32_t ncols, first, stage_bytes, nstages;
  int64_t seed;
  int64_t nchunks;
  void* out;
};

// One key column of a chunk for this lane's four rows (values at base + 32 j SIZE in the stage, mask words at mwa + 4 j).
template <int KIND, int SIZE, bool PLAIN, class acc_t>
__device__ __forceinline__ void hs_column(acc_t (&h)[4], uint32_t base, uint32_t mwa, int lane, int type)
{
  uint32_t mw[4];
  uint64_t v[4], v2[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    mw[j] = mwa ? lds_u32(mwa + 4 * j) : 0xffffffffu;
    const Reg<SIZE> q = lds_elem<SIZE>(base + 32 * j * SIZE);
    v[j]  = q.v[0];
    v2[j] = 0;
    if constexpr (SIZE >= 8) v[j] |= static_cast<uint64_t>(q.v[1]) << 32;
    if constexpr (SIZE == 16) v2[j] = static_cast<uint64_t>(q.v[2]) | (static_cast<uint64_t>(q.v[3]) << 32);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const bool ok = (mw[j] >> lane) & 1u;
    if constexpr (KIND == SRJ_HASH_XXHASH64) {
      uint64_t t;
      if constexpr (PLAIN && SIZE == 4) t = hash::xx_u32(static_cast<uint32_t>(v[j]), h[j]);
      else if constexpr (PLAIN) t = hash::xx_u64(v[j], h[j]);
      else t = hash::xx_fixed(type, v[j], v2[j], h[j]);
      h[j] = ok ? t : h[j];   // a null keeps the accumulator (xxhash64.cu:352-353)
    } else if constexpr (KIND == SRJ_HASH_MURMUR3_32) {
      uint32_t t;
      if constexpr (PLAIN && SIZE == 4) t = hash::mm_u32(static_cast<uint32_t>(v[j]), h[j]);
      else if constexpr (PLAIN) t = hash::mm_u64(v[j], h[j]);
      else t = hash::mm_fixed(type, v[j], v2[j], h[j]);
      h[j] = ok ? t : h[j];   // murmur_hash.cu:111-117
    } else {
      uint32_t x;
      if constexpr (PLAIN && SIZE == 4) x = static_cast<uint32_t>(v[j]);
      else if constexpr (PLAIN) x = static_cast<uint32_t>((v[j] >> 32) ^ v[j]);
      else x = static_cast<uint32_t>(hash::hive_fixed(type, v[j]));
      h[j] = 31u * h[j] + (ok ? x : 0u);   // hive_hash.cu:179-203 (null -> 0)
    }
  }
}

template <int KIND>
__global__ void __launch_bounds__(kHsThreads, 1) row_hash_stream_kernel(const __grid_constant__ HsParams p)
{
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full  = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(p.nstages) * p.stage_bytes);
  uint64_t* empty = full + kHsMaxStages;
  const int NS    = p.nstages;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kHsWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int lane = lane_id();
  if (warp_id() == 0) {
    // =================================== producer ===================================
    uint32_t tx = 0;
    for (int c = 0; c < p.ncols; ++c) tx += static_cast<uint32_t>(kHsRows) * p.cols[c].size + (p.mask_off[c] >= 0 ? 256u : 0u);
    int it = 0;
    for (int64_t ch = blockIdx.x; ch < p.nchunks; ch += gridDim.x, ++it) {
      const int s        = it % NS;
      const uint32_t par = ((it / NS) & 1) ^ 1;
      if (lane == 0) {
        mbar_wait(&empty[s], par);
        mbar_arrive_expect_tx(&full[s], tx);
      }
      __syncwarp();
      uint8_t* st = smem + static_cast<size_t>(s) * p.stage_bytes;
      if (lane < p.ncols) {   // one lane per key column: its values, then its mask words
        const HashCol& col = p.cols[lane];
        tma_load_1d(st + p.col_off[lane], col.data + ch * kHsRows * col.size, static_cast<uint32_t>(kHsRows) * col.size, &full[s]);
        if (p.mask_off[lane] >= 0) tma_load_1d(st + p.mask_off[lane], col.mask + ch * (kHsRows / 32), 256u, &full[s]);
      }
    }
  } else {
    // =================================== consumers ===================================
    using acc_t  = typename std::conditional<KIND == SRJ_HASH_XXHASH64, uint64_t, uint32_t>::type;
    const int w  = warp_id() - 1;
    int it       = 0;
    for (int64_t ch = blockIdx.x; ch < p.nchunks; ch += gridDim.x, ++it) {
      const int s        = it % NS;
      const uint32_t par = (it / NS) & 1;
      mbar_wait(&full[s], par);
      const uint32_t st_s = smem_u32(smem + static_cast<size_t>(s) * p.stage_bytes);
      const int64_t r0    = ch * kHsRows + (w * 4) * 32 + lane;   // this lane's rows: r0 + 32 j
      acc_t h[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (p.first) h[j] = KIND == SRJ_HASH_HIVE ? acc_t{0} : static_cast<acc_t>(p.seed);
        else h[j] = reinterpret_cast<const acc_t*>(p.out)[r0 + 32 * j];
      }
      for (int c = 0; c < p.ncols; ++c) {
        // the column's element size and hash flavour are warp-uniform: dispatch once per column, not per value
        const int size = p.cols[c].size, type = p.cols[c].type;
        const uint32_t base = st_s + static_cast<uint32_t>(p.col_off[c]) + static_cast<uint32_t>((w * 128 + lane) * size);
        const uint32_t mwa  = p.mask_off[c] >= 0 ? st_s + static_cast<uint32_t>(p.mask_off[c]) + static_cast<uint32_t>(w * 16) : 0u;
        if (p.cols[c].kind == 1) hs_column<KIND, 4, true>(h, base, mwa, lane, type);
        else if (p.cols[c].kind == 2) hs_column<KIND, 8, true>(h, base, mwa, lane, type);
        else if (size == 4) hs_column<KIND, 4, false>(h, base, mwa, lane, type);
        else if (size == 8) hs_column<KIND, 8, false>(h, base, mwa, lane, type);
        else if (size == 16) hs_column<KIND, 16, false>(h, base, mwa, lane, type);
        else if (size == 2) hs_column<KIND, 2, false>(h, base, mwa, lane, type);
        else hs_column<KIND, 1, false>(h, base, mwa, lane, type);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);   // the stage is free once its values are in registers
#pragma unroll
      for (int j = 0; j < 4; ++j) reinterpret_cast<acc_t*>(p.out)[r0 + 32 * j] = h[j];
    }
  }
}

// Runs the streaming kernel over the whole chunks of the table when it applies; *done = rows it covered.
static int launch_hash_stream(int kind, const HashParams& hp, int64_t num_rows, cudaStream_t stream, int64_t* done)
{
  *done = 0;
  if (hp.ncols > kHsMaxCols || num_rows < 4 * kHsRows) return SRJ_OK;
  HsParams p{};
  int off = 0;
  for (int c = 0; c < hp.ncols; ++c) {
    const HashCol& col = hp.cols[c];
    if (col.size == 0) return SRJ_OK;                                              // STRING key: not staged
    if (reinterpret_cast<uintptr_t>(col.data) & 15) return SRJ_OK;                 // TMA needs 16-byte aligned pieces
    if (col.mask && (reinterpret_cast<uintptr_t>(col.mask) & 15)) return SRJ_OK;
    p.cols[c]    = col;
    p.col_off[c] = off;
    off += kHsRows * col.size;
    p.mask_off[c] = col.mask ? off : -1;
    if (col.mask) off += 256;
  }
  p.ncols       = hp.ncols;
  p.first       = hp.first;
  p.seed        = hp.seed;
  p.out         = hp.out;
  p.stage_bytes = (off + 127) & ~127;
  p.nstages     = std::min<int>(kHsMaxStages, (200 * 1024) / p.stage_bytes);
  if (p.nstages < 2) return SRJ_OK;
  p.nchunks = num_rows / kHsRows;
  int dev = 0, nsm = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(nsm, p.nchunks));
  const size_t smem   = static_cast<size_t>(p.nstages) * p.stage_bytes + 2 * kHsMaxStages * 8;
  auto go = [&](auto kern) -> int {
    SRJ_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    kern<<<grid, kHsThreads, smem, stream>>>(p);
    return SRJ_OK;
  };
  int rc;
  if (kind == SRJ_HASH_XXHASH64) rc = go(row_hash_stream_kernel<SRJ_HASH_XXHASH64>);
  else if (kind == SRJ_HASH_MURMUR3_32) rc = go(row_hash_stream_kernel<SRJ_HASH_MURMUR3_32>);
  else rc = go(row_hash_stream_kernel<SRJ_HASH_HIVE>);
  if (rc != SRJ_OK) return rc;
  *done = p.nchunks * kHsRows;
  return SRJ_OK;
}

int launch_hash(int kind, const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t seed, void* out,
                cudaStream_t stream)
{
  if (num_columns == 0 || num_rows == 0) return SRJ_OK;  // xxhash64.cu:564
  for (int c = 0; c < num_columns; ++c) {
    const int32_t t = cols[c].type_id;
    const bool ok   = (t == SRJ_STRING) || type_width(t) > 0;
    if (!ok) { set_error("hash: column %d has unsupported type id %d (nested/dictionary types are not on this path)", c, t); return SRJ_EUNSUPPORTED; }
    if (kind == SRJ_HASH_HIVE && !hash::hive_supported(t)) { set_error("hive_hash: column %d has unsupported type id %d (hive_hash.cu:63-66)", c, t); return SRJ_EUNSUPPORTED; }
    if (cols[c].size != num_rows) { set_error("hash: column %d has %lld rows, expected %lld", c, (long long)cols[c].size, (long long)num_rows); return SRJ_EINVAL; }
  }
  const int64_t per_block = static_cast<int64_t>(kHashThreads) * kRowsPerThread;
  for (int c0 = 0; c0 < num_columns; c0 += kHashColsPerLaunch) {
    HashParams p{};
    p.ncols = std::min(kHashColsPerLaunch, num_columns - c0);
    p.kind  = kind;
    p.first = c0 == 0;
    p.seed  = seed;
    p.n     = num_rows;
    p.out   = out;
    for (int i = 0; i < p.ncols; ++i) {
      const srj_column& c = cols[c0 + i];
      const int32_t t     = c.type_id;
      int kind2           = 0;
      if (kind == SRJ_HASH_HIVE) {
        if (t == SRJ_INT32 || t == SRJ_TIMESTAMP_DAYS) kind2 = 1;
        else if (t == SRJ_INT64) kind2 = 2;
      } else {
        if (t == SRJ_INT32 || t == SRJ_UINT32 || t == SRJ_TIMESTAMP_DAYS || t == SRJ_DURATION_DAYS) kind2 = 1;
        else if (type_width(t) == 8 && t != SRJ_FLOAT64) kind2 = 2;  // ints, timestamps, durations, DECIMAL64: raw 8 bytes
      }
      p.cols[i] = HashCol{static_cast<const uint8_t*>(c.data), c.null_mask, c.offsets, static_cast<int16_t>(t),
                          static_cast<int16_t>(kind2), type_width(t)};
    }
    // whole chunks of fixed-width keys: the streaming kernel; the kernels below take what is left (tail rows, STRING keys)
    {
      int64_t done = 0;
      const int rcs = launch_hash_stream(kind, p, num_rows, stream, &done);
      if (rcs != SRJ_OK) return rcs;
      if (done == num_rows) continue;
      if (done > 0) {   // done is a multiple of 2048 rows: element, mask-word and output pointers simply advance
        for (int i = 0; i < p.ncols; ++i) {
          p.cols[i].data += done * p.cols[i].size;
          if (p.cols[i].mask) p.cols[i].mask += done / 32;
        }
        p.n   = num_rows - done;
        p.out = static_cast<uint8_t*>(out) + done * (kind == SRJ_HASH_XXHASH64 ? 8 : 4);
      }
    }
    const unsigned grid = static_cast<unsigned>((p.n + per_block - 1) / per_block);
    bool plain = true;
    for (int i = 0; i < p.ncols; ++i) plain = plain && p.cols[i].kind != 0;
    if (plain) {
      // persistent launch: as many CTAs as stay resident (the kernel strides over the row blocks)
      int dev = 0, nsm = 0;
      SRJ_CUDA_TRY(cudaGetDevice(&dev));
      SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
      // grid = resident CTAs per SM (occupancy) x rounds: the multiply-heavy kernels take 4 rounds rather than one CTA
      // per row block, hive -- pure streaming -- exactly one; a grid that is not a multiple of the resident count
      // leaves a straggler CTA per SM.
      static int occ_cache[4] = {0, 0, 0, 0};  // per hash kind; the same for every sm_90a device (benign race)
      int occ = occ_cache[kind & 3];
      if (occ == 0) {
        if (kind == SRJ_HASH_XXHASH64)
          SRJ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, row_hash_plain_kernel<SRJ_HASH_XXHASH64>, kHashThreads, 0));
        else if (kind == SRJ_HASH_MURMUR3_32)
          SRJ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, row_hash_plain_kernel<SRJ_HASH_MURMUR3_32>, kHashThreads, 0));
        else
          SRJ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, row_hash_plain_kernel<SRJ_HASH_HIVE>, kHashThreads, 0));
        occ_cache[kind & 3] = occ = std::max(1, occ);
      }
      const int waves      = occ * (kind == SRJ_HASH_HIVE ? 1 : 4);  // CTAs per SM
      const unsigned pgrid = std::min<unsigned>(grid, static_cast<unsigned>(nsm * waves));
      if (kind == SRJ_HASH_XXHASH64)
        row_hash_plain_kernel<SRJ_HASH_XXHASH64><<<pgrid, kHashThreads, 0, stream>>>(p);
      else if (kind == SRJ_HASH_MURMUR3_32)
        row_hash_plain_kernel<SRJ_HASH_MURMUR3_32><<<pgrid, kHashThreads, 0, stream>>>(p);
      else
        row_hash_plain_kernel<SRJ_HASH_HIVE><<<pgrid, kHashThreads, 0, stream>>>(p);
    } else if (kind == SRJ_HASH_XXHASH64)
      row_hash_kernel<SRJ_HASH_XXHASH64><<<grid, kHashThreads, 0, stream>>>(p);
    else if (kind == SRJ_HASH_MURMUR3_32)
      row_hash_kernel<SRJ_HASH_MURMUR3_32><<<grid, kHashThreads, 0, stream>>>(p);
    else
      row_hash_kernel<SRJ_HASH_HIVE><<<grid, kHashThreads, 0, stream>>>(p);
  }
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj
