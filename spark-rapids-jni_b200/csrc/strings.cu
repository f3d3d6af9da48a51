// strings.cu -- STRING-column stages of convert_from_rows:
//   (1) lengths -> offsets: batched (all STRING columns in one launch) three-step scan replacing the
//       per-column thrust::exclusive_scan + .element() sync loop of the reference (RC:2375-2395);
//   (2) chars gather: replaces copy_strings_from_rows (RC:1110-1150).
#include <algorithm>
#include <cstdlib>
#include "common.cuh"
#include "kernels.hpp"
#include "movers.cuh"
#include "plan.hpp"

namespace srj {

constexpr int kScanThreads = 256;
constexpr int kScanIter    = kScanThreads * 4;  // elements per block iteration
constexpr int kScanChunk   = kScanIter * 4;     // elements per CTA

__device__ __forceinline__ int64_t block_sum(int64_t v, int64_t* s_warp)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if (lane_id() == 0) s_warp[warp_id()] = v;
  __syncthreads();
  int64_t t = 0;
  if (threadIdx.x < kScanThreads / 32) t = s_warp[threadIdx.x];
  if (warp_id() == 0) {
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if (lane_id() == 0) s_warp[0] = t;
  }
  __syncthreads();
  t = s_warp[0];
  __syncthreads();
  return t;
}

// Element i of the scan input for a column: 0 for i == 0, else the uint32 length stored at offs[i].
__global__ void __launch_bounds__(kScanThreads) scan_partials_kernel(int32_t* const* offsets, int64_t n1 /* n + 1 */,
                                                                      int nchunks, int64_t* partials)
{
  __shared__ int64_t s_warp[kScanThreads / 32];
  const int c         = blockIdx.y;
  const int k         = blockIdx.x;
  const int32_t* offs = offsets[c];
  const int64_t beg   = static_cast<int64_t>(k) * kScanChunk;
  const int64_t end   = tmin(n1, beg + kScanChunk);
  int64_t acc         = 0;
  for (int64_t i = beg + threadIdx.x; i < end; i += kScanThreads)
    if (i > 0) acc += static_cast<uint32_t>(offs[i]);
  acc = block_sum(acc, s_warp);
  if (threadIdx.x == 0) partials[static_cast<int64_t>(c) * nchunks + k] = acc;
}

// exclusive scan of each column's chunk sums, in place; writes the column total
__global__ void __launch_bounds__(kScanThreads) scan_chunks_kernel(int64_t* partials, int nchunks,
                                                                    const int32_t* string_cols, int64_t* char_totals,
                                                                    unsigned long long* status)
{
  __shared__ int64_t s_warp[kScanThreads / 32];
  __shared__ int64_t s_carry;
  const int c  = blockIdx.x;
  int64_t* p   = partials + static_cast<int64_t>(c) * nchunks;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < nchunks; base += kScanThreads) {
    const int i     = base + threadIdx.x;
    const int64_t v = i < nchunks ? p[i] : 0;
    // block inclusive scan
    int64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane_id() >= o) x += y;
    }
    if (lane_id() == 31) s_warp[warp_id()] = x;
    __syncthreads();
    int64_t wpre = 0;
    for (int w = 0; w < warp_id(); ++w) wpre += s_warp[w];
    const int64_t carry = s_carry;
    if (i < nchunks) p[i] = carry + wpre + x - v;  // exclusive
    __syncthreads();
    if (threadIdx.x == kScanThreads - 1) s_carry = carry + wpre + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int64_t total = s_carry;
    if (char_totals) char_totals[string_cols[c]] = total;
    if (total > INT32_MAX && status) atomicOr(status, 2ull);  // cudf strings offsets are int32: bit 1 of the status word
  }
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(int32_t* const* offsets, int64_t n1, int nchunks,
                                                                   const int64_t* partials)
{
  __shared__ int64_t s_warp[kScanThreads / 32];
  __shared__ int64_t s_carry;
  const int c   = blockIdx.y;
  const int k   = blockIdx.x;
  int32_t* offs = offsets[c];
  if (threadIdx.x == 0) s_carry = partials[static_cast<int64_t>(c) * nchunks + k];
  __syncthreads();
  const int64_t beg = static_cast<int64_t>(k) * kScanChunk;
  const int64_t end = tmin(n1, beg + kScanChunk);
  for (int64_t base = beg; base < end; base += kScanIter) {
    const int64_t i0 = base + threadIdx.x * 4;
    int64_t v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t i = i0 + j;
      v[j]            = (i < end && i > 0) ? static_cast<int64_t>(static_cast<uint32_t>(offs[i])) : 0;
    }
    const int64_t tsum = v[0] + v[1] + v[2] + v[3];
    int64_t x          = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane_id() >= o) x += y;
    }
    if (lane_id() == 31) s_warp[warp_id()] = x;
    __syncthreads();
    int64_t wpre = 0;
    for (int w = 0; w < warp_id(); ++w) wpre += s_warp[w];
    const int64_t carry = s_carry;
    int64_t run         = carry + wpre + x - tsum;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      run += v[j];
      const int64_t i = i0 + j;
      if (i < end) offs[i] = static_cast<int32_t>(run);
    }
    __syncthreads();
    if (threadIdx.x == kScanThreads - 1) s_carry = run;
    __syncthreads();
  }
}

int64_t string_scan_partials_bytes(int nstr, int64_t num_rows)
{
  const int64_t nchunks = (num_rows + 1 + kScanChunk - 1) / kScanChunk;
  return static_cast<int64_t>(nstr) * nchunks * 8;
}

int launch_string_offsets_scan(int32_t* const* d_offsets, const int32_t* d_string_cols, int nstr, int64_t num_rows,
                               int64_t* d_char_totals, int64_t* d_status, void* d_partials, cudaStream_t stream)
{
  if (nstr == 0) return SRJ_OK;
  const int64_t n1  = num_rows + 1;
  const int nchunks = static_cast<int>((n1 + kScanChunk - 1) / kScanChunk);
  auto* partials    = static_cast<int64_t*>(d_partials);
  dim3 grid(nchunks, nstr);
  scan_partials_kernel<<<grid, kScanThreads, 0, stream>>>(d_offsets, n1, nchunks, partials);
  scan_chunks_kernel<<<nstr, kScanThreads, 0, stream>>>(partials, nchunks, d_string_cols, d_char_totals,
                                                        reinterpret_cast<unsigned long long*>(d_status));
  scan_apply_kernel<<<grid, kScanThreads, 0, stream>>>(d_offsets, n1, nchunks, partials);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// --------------------------------------------------------------------------------------------------
// chars gather, GENERIC path (follows the stored pair offsets, RC:1143): a warp owns (32-row tile, STRING column); lane = row reads the (offset,len)
// pair from the row, then the warp copies the tile's chars for that column -- a contiguous
// destination range -- with lane = destination byte, locating the source row by a shuffle search.
// Destination stores are fully coalesced; source reads stay inside 2-3 sectors per instruction.
// --------------------------------------------------------------------------------------------------

// ---- shared-memory helpers of the chars gathers (32-bit shared-space addresses) ----------------------------------
// A warp's staging line holds the T chars of one (32-row tile, column) at the byte positions [a, a + T), a = the
// destination's offset inside its 16-byte granule.  Flush: whole 16-byte chunks with one ld.shared.v4 /
// st.global.v4 per lane; the bytes of the two partial chunks at the ends (their neighbours belong to other tiles /
// warps) one per lane: lanes 0-15 the head chunk, lanes 16-31 the tail chunk.
__device__ __forceinline__ void flush_staging_line(uint32_t stg_s, uint8_t* D, int a, int T, int lane)
{
  uint8_t* Dal      = D - a;  // 16-byte aligned
  const int aT      = a + T;
  const int c_first = (a + 15) >> 4;  // first whole chunk
  const int c_end   = aT >> 4;        // one past the last whole chunk
  {
    const int c = c_first + lane;     // T <= 1024: at most three rounds, nearly always one
    if (c < c_end) {
      uint32_t v0, v1, v2, v3;
      asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "r"(stg_s + 16 * c));
      asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(Dal + 16 * c), "r"(v0), "r"(v1), "r"(v2), "r"(v3));
    }
  }
  if (c_end - c_first > 32) {  // warp-uniform
    for (int c = c_first + 32 + lane; c < c_end; c += 32) {
      uint32_t v0, v1, v2, v3;
      asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "r"(stg_s + 16 * c));
      asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(Dal + 16 * c), "r"(v0), "r"(v1), "r"(v2), "r"(v3));
    }
  }
  // partial chunks, one byte per lane: lanes 0-15 the head chunk [a, min(16, aT)) when a > 0; lanes 16-31 the tail
  // chunk [16 c_end, aT) unless it is the head chunk
  const int hl    = lane & 15;
  const bool tail = lane >= 16;
  const int pos   = (tail ? 16 * c_end : 0) + hl;
  const int lo    = tail ? 0 : a;
  const int hi    = tail ? aT : tmin(16, aT);
  const bool en   = tail ? (a == 0 || c_end > 0) : (a > 0);
  if (en && pos >= lo && pos < hi) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(stg_s + pos));
    asm volatile("st.global.u8 [%0], %1;" ::"l"(Dal + pos), "r"(v));
  }
}

// lane's string = L bytes at GLOBAL address S -> staging byte ds (shared address).  Aligned 32-bit source words
// (only words that overlap the string are read), funnel shift to the staging alignment, st.shared.u32 for whole
// words; the <= 3 edge bytes at each end come straight from the source.  maxL (<= 32) is the warp's longest string.
__device__ __forceinline__ void copy_global_to_staging(uint64_t S, uint32_t ds, int L, int maxL)
{
  const int dsh      = static_cast<int>(ds & 3u);
  const int ssh      = static_cast<int>(S & 3u);
  const int dlt      = ssh - dsh;
  const int pre      = ssh + (dlt < 0 ? 4 : 0);
  const uint64_t sp  = S - pre;
  const int sh       = (dlt & 3) * 8;
  const int end      = dsh + L;
  const int kfull1   = end >> 2;
  const uint32_t w0s = ds - dsh;
  const int lim      = L > 0 ? L + pre : 0;
  const int Kmax     = (maxL + 6) >> 2;
  const int nh       = dsh ? tmin(L, 4 - dsh) : 0;
  const int nt       = (kfull1 > 0 || !dsh) ? (end & 3) : 0;
  const uint8_t* Sb  = reinterpret_cast<const uint8_t*>(S);
  uint32_t hb[3], tb[3];
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    hb[t] = tb[t] = 0;
    if (t < nh) hb[t] = __ldg(Sb + t);
    if (t < nt) tb[t] = __ldg(Sb + (L - nt) + t);
  }
  uint32_t w[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    w[k]            = 0;
    const bool need = k == 0 ? (lim > 0 && pre < 4) : (4 * k < lim);
    if (need) w[k] = __ldg(reinterpret_cast<const uint32_t*>(sp + 4 * k));
  }
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    if (t < nh) sts_u8(ds + t, hb[t]);
    if (t < nt) sts_u8(ds + (L - nt) + t, tb[t]);
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    if (k < Kmax) {
      const uint32_t y = __funnelshift_r(w[k], w[k + 1], sh);
      const bool full  = k == 0 ? (dsh == 0 && kfull1 > 0) : (k < kfull1);
      if (full) sts_u32(w0s + 4 * k, y);
    }
  }
}

constexpr int kStrWarps = 8;
constexpr int kStrLine  = 16 + 1024 + 32;  // per-warp staging line

// The gather itself: warp `wlin` of `wtot` takes the tasks wlin, wlin + wtot, ...; stg_s = the warp's staging line.
__device__ __forceinline__ void generic_gather(const uint8_t* __restrict__ rows, const int32_t* __restrict__ row_offsets,
                                               int64_t row_stride, int64_t num_rows, int nstr,
                                               const int32_t* __restrict__ string_start, int32_t* const* offsets,
                                               uint8_t* const* chars, int64_t ntiles, const uint32_t* bases, int64_t wlin,
                                               int64_t wtot, uint32_t stg_s)
{
  // bases != NULL (wide tables between the two phases): offsets[s][r + 1] holds the inclusive sum inside row r's 32-row
  // group and bases[s][group] the chars of the column before the group; the finished offsets are written here.
  const int lane = lane_id();
  // one task = (32-row tile, STRING column); tasks are dealt to the warps of the whole grid, so every warp is busy
  // whatever the number of STRING columns (tables with 1-3 strings are the common case)
  const int64_t ntasks = ntiles * nstr;
  for (int64_t task = wlin; task < ntasks; task += wtot) {
    const int64_t tile = task / nstr;
    const int s        = static_cast<int>(task - tile * nstr);
    const int64_t r    = tile * 32 + lane;
    const bool active  = r < num_rows;
    const int64_t rsta = active ? (row_offsets ? static_cast<int64_t>(row_offsets[r]) : r * row_stride) : 0;
    {
      uint32_t so = 0, len = 0;
      int32_t v = 0;
      if (active) {
        const uint8_t* pp = rows + rsta + string_start[s];
        if ((reinterpret_cast<uintptr_t>(pp) & 3) == 0) {
          so  = *reinterpret_cast<const uint32_t*>(pp);
          len = *reinterpret_cast<const uint32_t*>(pp + 4);
        } else {
          so  = pp[0] | (pp[1] << 8) | (pp[2] << 16) | (static_cast<uint32_t>(pp[3]) << 24);
          len = pp[4] | (pp[5] << 8) | (pp[6] << 16) | (static_cast<uint32_t>(pp[7]) << 24);
        }
        v = offsets[s][r + 1];
      }
      const int last       = static_cast<int>(tmin<int64_t>(31, num_rows - 1 - tile * 32));
      const int32_t dbase  = bases ? static_cast<int32_t>(bases[static_cast<int64_t>(s) * ntiles + tile]) : offsets[s][tile * 32];
      int32_t x            = v;
      if (!bases) x -= dbase;
      x                    = active ? x : 0;
      const int32_t up     = __shfl_up_sync(0xffffffffu, x, 1);
      const uint32_t pe    = static_cast<uint32_t>(lane ? up : 0);  // exclusive prefix inside the tile
      const uint32_t total = static_cast<uint32_t>(__shfl_sync(0xffffffffu, x, last));
      if (bases) {
        if (active) offsets[s][r + 1] = dbase + x;
        if (r == 0) offsets[s][0] = 0;
      }
      const int64_t srcoff = rsta + so;
      uint8_t* dst         = chars[s] + dbase;
      const int maxL       = __reduce_max_sync(0xffffffffu, active ? static_cast<int>(tmin<uint32_t>(len, 1u << 20)) : 0);
      if (total == 0) continue;
      if (maxL <= 32 && total <= 1024) {
        // short strings (the common case): lane = row copies its string into the warp's staging line, laid out
        // like the destination, and the line leaves with 16-byte stores
        const int a = static_cast<int>(reinterpret_cast<uintptr_t>(dst) & 15);
        copy_global_to_staging(reinterpret_cast<uint64_t>(rows) + static_cast<uint64_t>(srcoff), stg_s + static_cast<uint32_t>(a) + pe,
                               active ? static_cast<int>(len) : 0, maxL);
        __syncwarp();
        flush_staging_line(stg_s, dst, a, static_cast<int>(total), lane);
        __syncwarp();
        continue;
      }
      const uint32_t bound = (total + 31u) & ~31u;  // all lanes take part in the shuffles
      for (uint32_t p = lane; p < bound; p += 32) {
        int j = 0;
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
          const int cand   = j + step;
          const uint32_t v = __shfl_sync(0xffffffffu, pe, cand & 31);
          if (cand <= last && v <= p) j = cand;
        }
        const uint32_t pj  = __shfl_sync(0xffffffffu, pe, j);
        const int64_t sj   = __shfl_sync(0xffffffffu, srcoff, j);
        if (p < total) dst[p] = rows[sj + (p - pj)];
      }
    }
  }
}


__global__ void __launch_bounds__(kStrWarps * 32) strings_from_rows_kernel(
  const uint8_t* __restrict__ rows, const int32_t* __restrict__ row_offsets, int64_t row_stride, int64_t num_rows,
  int nstr, const int32_t* __restrict__ string_start, int32_t* const* __restrict__ offsets,
  uint8_t* const* __restrict__ chars, int64_t ntiles, const uint32_t* bases)
{
  __shared__ __align__(16) uint8_t s_line[kStrWarps * kStrLine];
  generic_gather(rows, row_offsets, row_stride, num_rows, nstr, string_start, offsets, chars, ntiles, bases,
                 static_cast<int64_t>(blockIdx.x) * kStrWarps + warp_id(), static_cast<int64_t>(gridDim.x) * kStrWarps,
                 smem_u32(s_line + warp_id() * kStrLine));
}

// --------------------------------------------------------------------------------------------------
// chars gather, FAST path (canonical rows: a row's chars follow its fixed section in column order, which is
// what convert_to_rows writes and what phase 1 verified).
//
// A tile is one 32-row group.  The CTA keeps kSwNG tiles in flight, each owned by a group of `wpt` consumer
// warps; warp i of a group gathers the STRING columns [i * cpw, (i + 1) * cpw) of its tile.
//
//   producer warps: lane = row; one TMA bulk copy per row of JUST the row's variable section
//                   [offsets[r] + size_per_row, offsets[r + 1]) into a ring of 2 * kSwNG stages (two per
//                   group), so the fixed section -- 79 % of a C3 row -- is never read by this phase.  A copy costs
//                   its issuing warp ~70 cycles, one lane at a time, so kSwProducers warps share the rows of a tile:
//                   producer q issues the copies of the rows whose lane index is congruent to q and arrives on the
//                   stage's full barrier with the bytes of its own copies.  Each one scans the tile's row offsets
//                   itself (so they agree on the slots and on `direct`), and loads those of its NEXT tile while the
//                   current tile's copies are issued;
//   consumer warps: lane = row.  The warp reads its columns' offsets entries of the tile (one coalesced 128-byte
//                   load per column; those of the group's next tile are loaded before it waits for the current
//                   one, so that round trip overlaps the current tile's work), turns them into lengths, and the warps
//                   of the group exchange their
//                   per-row byte sums through shared memory (one named barrier per tile) to find where in the
//                   row's variable section their first column starts.  Per column the lane's string moves as
//                   aligned 32-bit words from the row image, funnel-shifted to the destination's byte
//                   alignment, into a per-warp staging line laid out like the destination, which leaves with
//                   aligned 16-byte st.global (the chars of consecutive rows of a column are contiguous).
//   offsets       : for wide tables (from_rows_wide.cu) phase 1 left group-local inclusive sums in the offsets arrays
//                   and the chars before each 32-row group in the workspace; the absolute offsets are written here,
//                   on the way (one coalesced store per column and tile).
// --------------------------------------------------------------------------------------------------
constexpr int kSwNG     = 3;   // tiles in flight per CTA (groups of consumer warps)
constexpr int kSwMaxWpt = 8;   // consumer warps per tile
constexpr int kSwMaxCpw = 8;   // STRING columns per warp (held in registers)
constexpr int kSwStages = 2 * kSwNG;
constexpr int kSwFront  = 16;  // slack before a stage's payload (word reads may start up to 7 bytes early)
constexpr int kSwBack   = 48;  // slack after it (word reads may run up to 44 bytes past a string)
constexpr int kSwLine   = 16 + 1024 + 32;  // per-warp staging line
constexpr int kSwProducers  = 4;           // producer warps, one per scheduler (a power of two)
constexpr int kSwMaxThreads = (kSwProducers + kSwNG * kSwMaxWpt) * 32;
static_assert((kSwProducers & (kSwProducers - 1)) == 0 && kSwProducers <= 32, "kSwProducers: a power of two");

struct SwHdr {
  int32_t rows;    // 0 = end
  int32_t direct;  // 1 = variable sections not staged (tile larger than a stage): read them from global memory
};

struct SwParams {
  const uint8_t* rows;
  const int32_t* row_offsets;
  int64_t rows_bytes;
  int64_t num_rows;
  int32_t nstr, size_per_row, wpt, cpw, stage_bytes, fixed_row_size;
  const uint32_t* bases;  // non-NULL: offsets hold group-local inclusive sums, bases[nstr][ntiles] the chars before each group
  const int32_t* string_start;  // [nstr] row byte offset of each pair (generic gather only)
  const int64_t* status;
  // per-call pointer tables, as kernel parameters (no staging copy): the fast gather takes <= 64 STRING columns
  int32_t* offsets[kSwMaxWpt * kSwMaxCpw];
  uint8_t* chars[kSwMaxWpt * kSwMaxCpw];
};

__device__ __forceinline__ int32_t ldg_s32(const int32_t* p)
{
  int32_t v;
  asm volatile("ld.global.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

// lane = destination byte, source row by a shuffle search (long strings, tiles that were not staged)
__device__ __noinline__ void gather_bytes_slow(uint8_t* D, uint32_t T, uint32_t pe, uint64_t src, int last, int lane)
{
  const uint32_t bound = (T + 31u) & ~31u;  // all lanes take part in the shuffles
  for (uint32_t q = lane; q < bound; q += 32) {
    int j = 0;
#pragma unroll
    for (int step = 16; step > 0; step >>= 1) {
      const int cand   = j + step;
      const uint32_t v = __shfl_sync(0xffffffffu, pe, cand & 31);
      if (cand <= last && v <= q) j = cand;
    }
    const uint32_t pj = __shfl_sync(0xffffffffu, pe, j);
    const uint64_t sj = __shfl_sync(0xffffffffu, src, j);
    if (q < T) D[q] = *reinterpret_cast<const uint8_t*>(sj + (q - pj));
  }
}

__global__ void __launch_bounds__(kSwMaxThreads, 1) strings_wide_kernel(const __grid_constant__ SwParams p)
{
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int NS     = kSwStages;
  const int stage_span = kSwFront + p.stage_bytes + kSwBack;  // multiple of 16
  const int wpt        = p.wpt;
  uint8_t* payload0    = smem;
  int32_t* rowsm0      = reinterpret_cast<int32_t*>(smem + static_cast<size_t>(NS) * stage_span);  // [NS][32]
  SwHdr* hdr0          = reinterpret_cast<SwHdr*>(rowsm0 + NS * 32);
  uint64_t* full       = reinterpret_cast<uint64_t*>(hdr0 + NS);
  uint64_t* empty      = full + NS;
  int32_t** s_offs     = reinterpret_cast<int32_t**>(empty + NS);
  uint8_t** s_chars    = reinterpret_cast<uint8_t**>(s_offs + p.nstr);
  int32_t* blk0        = reinterpret_cast<int32_t*>(s_chars + p.nstr);  // [2][kSwNG][kSwMaxWpt][32]
  uint8_t* stg0        = reinterpret_cast<uint8_t*>(blk0 + 2 * kSwNG * kSwMaxWpt * 32);
  stg0                 = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(stg0) + 15) & ~uintptr_t{15});

  const int tid  = threadIdx.x;
  const int lane = lane_id();
  for (int i = tid; i < p.nstr; i += blockDim.x) {
    s_offs[i]  = p.offsets[i];
    s_chars[i] = p.chars[i];
  }
  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], kSwProducers);
      mbar_init(&empty[s], wpt);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (p.status && (*p.status & 1)) {
    // phase 1 saw rows that do not use the canonical layout: follow the stored pair offsets (RC:1143) with the generic
    // gather, every consumer warp of the grid taking (tile, column) tasks with its own staging line
    if (warp_id() < kSwProducers) return;
    const int ncons = (blockDim.x >> 5) - kSwProducers;
    const int cw    = warp_id() - kSwProducers;
    generic_gather(p.rows, p.row_offsets, p.fixed_row_size, p.num_rows, p.nstr, p.string_start, s_offs, s_chars,
                   (p.num_rows + 31) >> 5, p.bases, static_cast<int64_t>(blockIdx.x) * ncons + cw,
                   static_cast<int64_t>(gridDim.x) * ncons, smem_u32(stg0 + static_cast<size_t>(cw) * kSwLine));
    return;
  }

  const uintptr_t b_lo = reinterpret_cast<uintptr_t>(p.rows);
  const uintptr_t b_hi = b_lo + static_cast<uintptr_t>(p.rows_bytes);
  const int64_t ntiles = (p.num_rows + 31) >> 5;

  if (warp_id() < kSwProducers) {
    // =================================== producers ===================================
    const int q     = warp_id();
    const bool mine = (lane & (kSwProducers - 1)) == q;  // the rows whose copies this warp issues
    uint32_t n0 = 0, n1 = 0;                             // row offsets [r, r + 1] of the lane's row of the next tile
    auto load_offsets = [&](int64_t T) {
      n0 = n1 = 0;
      const int64_t r = (T << 5) + lane;
      if (T < ntiles && r < p.num_rows) {
        n0 = static_cast<uint32_t>(p.row_offsets[r]);
        n1 = static_cast<uint32_t>(p.row_offsets[r + 1]);
      }
    };
    load_offsets(blockIdx.x);
    int it = 0;
    for (int64_t T = blockIdx.x;; T += gridDim.x, ++it) {
      const int s        = it % NS;
      const uint32_t par = ((it / NS) & 1) ^ 1;
      SwHdr* h           = hdr0 + s;
      if (T >= ntiles) {
        // one end marker per group of consumer warps
        if (lane == 0) {
          mbar_wait(&empty[s], par);
          if (q == 0) h->rows = 0;
          mbar_arrive(&full[s]);
        }
        if (T >= ntiles + static_cast<int64_t>(kSwNG - 1) * gridDim.x) break;
        continue;
      }
      const int64_t o0 = n0, o1 = n1;
      load_offsets(T + gridDim.x);  // in flight while this tile's copies are issued
      if (lane == 0) mbar_wait(&empty[s], par);
      __syncwarp();
      const int64_t r0 = T << 5;
      const int rows   = static_cast<int>(tmin<int64_t>(32, p.num_rows - r0));
      uint8_t* pay     = payload0 + static_cast<size_t>(s) * stage_span + kSwFront;
      int32_t* rowsm   = rowsm0 + s * 32;
      int64_t gs = o0 + p.size_per_row, ge = o1;
      if (ge < gs) ge = gs;
      const uintptr_t a_lo = b_lo + static_cast<uintptr_t>(gs);
      const uintptr_t a_hi = b_lo + static_cast<uintptr_t>(ge);
      const uintptr_t fl   = a_lo & ~uintptr_t{15};
      uintptr_t t_lo       = fl < b_lo ? fl + 16 : fl;
      uintptr_t t_hi       = (a_hi + 15) & ~uintptr_t{15};
      if (t_hi > b_hi) t_hi = a_hi & ~uintptr_t{15};
      if (t_hi < t_lo) t_hi = t_lo;
      if (lane >= rows || a_hi == a_lo) t_hi = t_lo;
      const int32_t span =
        (lane < rows) ? static_cast<int32_t>(tmin<uintptr_t>(((a_hi + 15) & ~uintptr_t{15}) - fl, 1u << 30)) : 0;
      int32_t x = span;  // inclusive scan of the window spans -> slot of each row
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      const int32_t slot = x - span;
      const bool over    = lane < rows && (x > p.stage_bytes || span >= (1 << 30));
      const bool direct  = __any_sync(0xffffffffu, over);
      uint32_t tx        = 0;
      if (!direct && lane < rows && mine) {
        tx          = static_cast<uint32_t>(t_hi - t_lo);
        rowsm[lane] = slot + static_cast<int32_t>(a_lo - fl);
        // bytes of [a_lo, a_hi) outside the TMA window [t_lo, t_hi) (only at the ends of the buffer): by hand
        const uintptr_t h_end = tmin(tmax(t_lo, a_lo), a_hi);
        for (uintptr_t a = a_lo; a < h_end; ++a) pay[slot + (a - fl)] = *reinterpret_cast<const uint8_t*>(a);
        for (uintptr_t a = tmax(tmin(t_hi, a_hi), h_end); a < a_hi; ++a) pay[slot + (a - fl)] = *reinterpret_cast<const uint8_t*>(a);
      }
      uint32_t total = tx;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
      if (lane == 0 && q == 0) {
        h->rows   = rows;
        h->direct = direct ? 1 : 0;
      }
      __syncwarp();
      if (lane == 0) {
        // release: header / rowsm / hand copies visible.  A producer none of whose rows carries bytes (null or empty
        // strings, a short last tile) arrives without a transaction count.
        if (total) mbar_arrive_expect_tx(&full[s], total);
        else mbar_arrive(&full[s]);
      }
      __syncwarp();
      if (tx) tma_load_1d(pay + slot + (t_lo - fl), reinterpret_cast<const void*>(t_lo), tx, &full[s]);
    }
  } else {
    // =================================== consumers ===================================
    const int cw         = warp_id() - kSwProducers;
    const int gi         = cw / wpt;        // tile group
    const int wi         = cw - gi * wpt;   // warp inside the group
    const int c0         = wi * p.cpw;
    const int ncol       = tmax(0, tmin(p.nstr, c0 + p.cpw) - c0);
    const uint32_t stg_s = smem_u32(stg0 + static_cast<size_t>(cw) * kSwLine);
    const bool semi      = p.bases != nullptr;  // offsets hold group-local sums: finish them here
    // this warp's columns at the group's iteration it_ (tile blockIdx.x + it_ * gridDim.x): b = the chars of column
    // c0 + lane before the tile, vv[j] = the offsets entry of column c0 + j after the lane's row
    auto load_cols = [&](int it_, int32_t& b, int32_t (&vv)[kSwMaxCpw]) {
      const int64_t T = blockIdx.x + static_cast<int64_t>(it_) * gridDim.x;
      const int64_t r = T << 5;
      b               = 0;
#pragma unroll
      for (int j = 0; j < kSwMaxCpw; ++j) vv[j] = 0;
      if (T >= ntiles) return;
      if (lane < ncol) b = semi ? static_cast<int32_t>(p.bases[static_cast<int64_t>(c0 + lane) * ntiles + T]) : ldg_s32(s_offs[c0 + lane] + r);
      const bool act = r + lane < p.num_rows;
#pragma unroll
      for (int j = 0; j < kSwMaxCpw; ++j)
        if (j < ncol && act) vv[j] = ldg_s32(s_offs[c0 + j] + r + 1 + lane);
    };
    int32_t base_l, v[kSwMaxCpw];  // this tile's, loaded one tile ahead
    load_cols(gi, base_l, v);
    for (int it = gi, k = 0;; it += kSwNG, ++k) {
      const int s        = it % NS;
      const uint32_t par = (it / NS) & 1;
      int32_t nbase, nv[kSwMaxCpw];
      load_cols(it + kSwNG, nbase, nv);  // the group's next tile: in flight during the wait and this tile's work
      mbar_wait(&full[s], par);
      const SwHdr h = hdr0[s];
      if (h.rows == 0) break;
      const int64_t r0    = (blockIdx.x + static_cast<int64_t>(it) * gridDim.x) << 5;
      const int rows      = h.rows;
      const int last      = rows - 1;
      const bool active   = lane < rows;
      const bool direct   = h.direct != 0;
      const uint32_t pay_s = smem_u32(payload0 + static_cast<size_t>(s) * stage_span + kSwFront);
      // ---- this warp's columns: offsets entries of the tile -> lengths ------------------------------------
      int32_t inc[kSwMaxCpw], len[kSwMaxCpw];
      int32_t mysum = 0;
#pragma unroll
      for (int j = 0; j < kSwMaxCpw; ++j) {
        const int32_t bj = __shfl_sync(0xffffffffu, base_l, j);
        int32_t x        = v[j];
        if (!semi) x -= bj;  // finished offsets are absolute; otherwise they are sums inside the group already
        x                = active ? x : 0;
        const int32_t up = __shfl_up_sync(0xffffffffu, x, 1);
        inc[j]           = x;
        len[j]           = active ? tmax(x - (lane ? up : 0), 0) : 0;
        mysum += (j < ncol) ? len[j] : 0;
      }
      // ---- where this warp's first column starts inside the row's variable section --------------------------
      int32_t* blk = blk0 + (((k & 1) * kSwNG + gi) * kSwMaxWpt) * 32;
      blk[wi * 32 + lane] = mysum;
      named_bar_sync(1 + gi, wpt * 32);
      int32_t run = 0;
      for (int w2 = 0; w2 < wi; ++w2) run += blk[w2 * 32 + lane];
      uint32_t var_s   = 0;   // staged: shared address of the lane's variable section
      uint64_t var_g   = 0;   // direct: its global address
      if (!direct) {
        var_s = pay_s + static_cast<uint32_t>(active ? rowsm0[s * 32 + lane] : 0);
      } else {
        var_g = reinterpret_cast<uint64_t>(p.rows) +
                (active ? static_cast<uint64_t>(static_cast<uint32_t>(p.row_offsets[r0 + lane])) + p.size_per_row : 0);
      }
#pragma unroll
      for (int j = 0; j < kSwMaxCpw; ++j) {
        if (j < ncol) {  // warp-uniform
          const int32_t L  = len[j];
          const int32_t pe = inc[j] - L;
          const int32_t T  = __shfl_sync(0xffffffffu, inc[j], last);
          const int32_t bj = __shfl_sync(0xffffffffu, base_l, j);
          const int32_t rb = run;
          run += L;
          if (semi) {  // finish the offsets: one coalesced 128-byte store per column
            if (active) asm volatile("st.global.s32 [%0], %1;" ::"l"(s_offs[c0 + j] + r0 + 1 + lane), "r"(bj + inc[j]));
            if (r0 == 0 && lane == 0) asm volatile("st.global.s32 [%0], %1;" ::"l"(s_offs[c0 + j]), "r"(0));
          }
          if (T > 0) {
            uint8_t* D     = s_chars[c0 + j] + bj;
            const int maxL = __reduce_max_sync(0xffffffffu, L);
            if (!direct && maxL <= 32 && T <= 1024) {
              const int a = static_cast<int>(reinterpret_cast<uintptr_t>(D) & 15);
              copy_shared_to_staging(var_s + static_cast<uint32_t>(rb), stg_s + static_cast<uint32_t>(a + pe), L);
              __syncwarp();
              flush_staging_line(stg_s, D, a, T, lane);
              __syncwarp();
            } else {
              const uint64_t src = direct ? var_g + static_cast<uint64_t>(rb)
                                          : reinterpret_cast<uint64_t>(payload0 + static_cast<size_t>(s) * stage_span + kSwFront) +
                                              static_cast<uint64_t>(active ? rowsm0[s * 32 + lane] : 0) + static_cast<uint64_t>(rb);
              gather_bytes_slow(D, static_cast<uint32_t>(T), static_cast<uint32_t>(pe), src, last, lane);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      base_l = nbase;
#pragma unroll
      for (int j = 0; j < kSwMaxCpw; ++j) v[j] = nv[j];
    }
  }
}

static size_t strings_wide_smem_bytes(int nstr, int stage_bytes, int wpt)
{
  size_t b = static_cast<size_t>(kSwStages) * (kSwFront + stage_bytes + kSwBack);
  b += static_cast<size_t>(kSwStages) * 32 * 4 + static_cast<size_t>(kSwStages) * sizeof(SwHdr) + 2 * kSwStages * 8;
  b += static_cast<size_t>(nstr) * 16;
  b += static_cast<size_t>(2) * kSwNG * kSwMaxWpt * 32 * 4 + 16;
  b += static_cast<size_t>(kSwNG) * wpt * kSwLine;
  return (b + 127) & ~size_t{127};
}

// Can the fast gather serve this schema?  (Host-side, per plan: phase 1 and phase 2 must agree on the offsets
// protocol.)
static bool strings_wide_eligible(const srj_plan* plan)
{
  const int nstr = plan->num_string_columns;
  return nstr >= 8 && nstr <= kSwMaxWpt * kSwMaxCpw;
}

// the fast gather needs phase 1's status word (it tells canonical rows from the rest)
bool strings_fast_path(const srj_plan* plan, const int64_t* d_status) { return d_status != nullptr && strings_wide_eligible(plan); }

// cols: the caller's columns (host array).  The fast gather gets its pointer tables as kernel parameters; schemas it
// does not serve upload them through the plan's ring (d_tab: [offsets nstr][chars nstr], already in flight).
int launch_strings_from_rows(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets, int64_t rows_bytes,
                             int64_t num_rows, const srj_column* cols, void* const* d_tab, const int64_t* d_status,
                             const uint32_t* d_bases, cudaStream_t stream)
{
  const int nstr = plan->num_string_columns;
  if (nstr == 0 || num_rows == 0) return SRJ_OK;
  int dev = 0, nsm = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  // The fast gather splits the STRING columns of a 32-row tile over the warps of a group: it needs a few columns to
  // fill them.  Tables with few STRING columns take the task-parallel generic kernel (which follows the stored
  // offsets, so it serves canonical and non-canonical rows alike).
  if (strings_fast_path(plan, d_status)) {
    SwParams p{};
    p.rows           = rows;
    p.row_offsets    = row_offsets;
    p.rows_bytes     = rows_bytes;
    p.num_rows       = num_rows;
    p.nstr           = nstr;
    p.size_per_row   = plan->size_per_row;
    p.fixed_row_size = plan->fixed_row_size;
    p.string_start   = plan->d_string_start;
    p.wpt            = std::min(kSwMaxWpt, (nstr + 3) / 4);          // >= 4 columns per warp when there are few
    p.cpw            = (nstr + p.wpt - 1) / p.wpt;
    p.bases          = d_bases;
    p.status         = d_status;
    for (int s = 0; s < nstr; ++s) {
      p.offsets[s] = cols[plan->string_columns[s]].offsets;
      p.chars[s]   = static_cast<uint8_t*>(cols[plan->string_columns[s]].data);
    }
    // stage = the variable sections of 32 average rows + 25 %, within what shared memory leaves
    const size_t fixed_smem = strings_wide_smem_bytes(nstr, 0, p.wpt);
    const int64_t cap       = (static_cast<int64_t>(232448 - fixed_smem) / kSwStages) & ~int64_t{15};
    const int64_t avg_var   = std::max<int64_t>(0, rows_bytes / num_rows - plan->size_per_row) + 16;
    int64_t stage           = (avg_var * 32 * 5 / 4 + 1023) & ~int64_t{1023};
    stage                   = std::max<int64_t>(4096, std::min(stage, cap));
    p.stage_bytes           = static_cast<int32_t>(stage);
    const int64_t ntiles    = (num_rows + 31) / 32;
    const int64_t grid      = std::min<int64_t>(nsm, ntiles);
    const size_t smem       = strings_wide_smem_bytes(nstr, p.stage_bytes, p.wpt);
    SRJ_CUDA_TRY(cudaFuncSetAttribute(strings_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    strings_wide_kernel<<<static_cast<unsigned>(grid), (kSwProducers + kSwNG * p.wpt) * 32, smem, stream>>>(p);
    SRJ_CUDA_TRY(cudaGetLastError());
    return SRJ_OK;
  }
  // generic kernel: follows the stored pair offsets
  const int64_t ntiles = (num_rows + 31) / 32;
  const int64_t grid   = std::min<int64_t>(ntiles, static_cast<int64_t>(nsm) * 8);
  strings_from_rows_kernel<<<static_cast<unsigned>(grid), kStrWarps * 32, 0, stream>>>(
    rows, row_offsets, plan->fixed_row_size, num_rows, nstr, plan->d_string_start, reinterpret_cast<int32_t* const*>(d_tab),
    reinterpret_cast<uint8_t* const*>(d_tab + nstr), ntiles, d_bases);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj
