// to_rows_var.cu -- columns -> JCUDF rows for tables with STRING columns
// (reference: copy_to_rows + copy_validity_to_rows + copy_strings_to_rows, RC:574-861).
//
// Two kernels, both lane = row (every global read is a contiguous piece of a column -- values, offsets, chars of
// consecutive rows -- and every shared-memory write lands in the lane's own row image):
//
// to_rows3_kernel (wide rows, >= ~3 KB: the C3 shape).  One CTA of 24 warps per SM owning a ~150-200 KB row-image
// buffer.  A tile = as many rows (<= 32) as fit.  Per tile:
//   1. geometry from the LIST offsets (already written by batch_offsets_kernel), every warp redundantly;
//   2. string block sums: warp b sums the lengths of its block of STRING columns per row and stages the tile's
//      chars of those columns -- one contiguous global range per column -- into the column's shared-memory slot
//      with 16-byte cp.async (no registers, no scoreboard);
//   3. wait for the previous TMA store to have read the buffer, zero it (padding bytes are 0), scan the block sums;
//   4. independent work items writing disjoint bytes, dealt to the warps once per launch by a
//      longest-processing-time rule (no atomics in the tile loop):
//        string block : (offset, len) pairs + chars.  Chars of <= 32 bytes move as aligned 32-bit words from the
//                       staging slot (or from global when a slice did not fit its slot), funnel-shifted to the
//                       destination alignment, st.shared.u32 for whole words, the <= 3 edge bytes at each end
//                       straight from the source; longer strings take a warp-cooperative byte copy;
//        fixed batch  : 8 columns of one width class with cp.async (4/8/16 B; LDG/STS for 1/2 B);
//        validity     : lane = column loads the mask word(s) covering the tile, the 32x32 bit butterfly turns them
//                       into 4 validity bytes per row;
//   5. the finished tile -- ONE contiguous byte range of the output -- leaves with a single 1-D TMA bulk store.
//
// to_rows_w_kernel (narrow rows, <= ~600 B: the common Spark shape): see the comment above the kernel.
//
// A tile whose rows do not fit raises *fail_flag; the generic kernel (to_rows.cu) launched right behind redoes
// the batch when it sees the flag.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "kernels.hpp"
#include "plan.hpp"

namespace srj {

constexpr int kT3MaxBlocks = 48;    // string blocks per row
constexpr int kT3MaxItems  = 1024;
constexpr int kHoist       = 2;     // STRING columns of a block whose offsets are fetched together (4 spills)

struct ToRows3Params {
  const void* const* col_data;
  const uint32_t* const* masks;
  const int32_t* const* str_offsets;
  const uint8_t* const* str_chars;
  int64_t row_start, row_count;
  const int32_t* out_offsets;  // batch-relative LIST offsets, already written
  uint8_t* out_data;
  int32_t ncols, nstr, nfixed;
  int32_t validity_offset, size_per_row;
  int32_t stage_bytes;   // multiple of 16
  int32_t super_rows;    // rows dealt to a CTA at a time (multiple of 8)
  int32_t sb;            // STRING columns per block
  int32_t nblocks;
  int32_t slot_bytes;    // chars staging bytes per STRING column (multiple of 16), 0 = no staging
  int32_t nitems;        // work items per tile (string blocks + fixed batches + validity groups)
  int32_t class_begin[kNumClasses + 1];
  const Entry* entries;
  const int32_t* string_start;
  int32_t* fail_flag;
};

enum : int { kItemString = 5, kItemValidity = 6 };
__host__ __device__ inline int32_t t3_item(int kind, int begin, int count) { return kind | (begin << 3) | (count << 20); }

__device__ __forceinline__ uint32_t t3_transpose32(uint32_t r, int lane)
{
  uint32_t m = 0x0000FFFFu;
#pragma unroll
  for (int j = 16; j > 0; j >>= 1) {
    const uint32_t other = __shfl_xor_sync(0xffffffffu, r, j);
    if ((lane & j) == 0) {
      const uint32_t t = ((r >> j) ^ other) & m;
      r ^= t << j;
    } else {
      const uint32_t t = ((other >> j) ^ r) & m;
      r ^= t;
    }
    m ^= m << (j >> 1);
  }
  return r;
}

__device__ __forceinline__ void t3_sts_u8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ void t3_sts_u16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ void t3_sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ void t3_sts_v2(uint32_t a, uint32_t x, uint32_t y) { asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y)); }

// U columns of element size W (>= 4) straight from the column into the lane's row image with cp.async (LDGSTS):
// no register staging and no scoreboard wait -- the warp only issues; completion is collected once per tile
// (cp.async.wait_all before the TMA store).  16-byte fields go as two 8-byte copies (rows are 8-byte aligned only).
template <int W, int U>
__device__ __forceinline__ void t3_fixed_async(const uint8_t* const* s_ent_ptr, const int32_t* s_ent_start, int begin, int count,
                                               int64_t abs_row, bool act, uint32_t row_s)
{
  static_assert(W >= 4, "cp.async moves 4, 8 or 16 bytes");
#pragma unroll
  for (int j = 0; j < U; ++j) {
    if (j < count && act) {
      const uint8_t* src = s_ent_ptr[begin + j] + abs_row * W;
      const uint32_t a   = row_s + static_cast<uint32_t>(s_ent_start[begin + j]);
      if constexpr (W == 4) asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(a), "l"(src) : "memory");
      else if constexpr (W == 8) asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(a), "l"(src) : "memory");
      else {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(a), "l"(src) : "memory");
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(a + 8), "l"(src + 8) : "memory");
      }
    }
  }
}

// U columns of element size W: loads first (independent), then the stores into the lane's row image
template <int W, int U>
__device__ __forceinline__ void t3_fixed(const uint8_t* const* s_ent_ptr, const int32_t* s_ent_start, int begin, int count,
                                         int64_t abs_row, bool act, uint32_t row_s)
{
  constexpr int NW = W >= 4 ? W / 4 : 1;
  uint32_t v[U][NW];
#pragma unroll
  for (int j = 0; j < U; ++j) {
    if (j < count && act) {
      const uint8_t* src = s_ent_ptr[begin + j] + abs_row * W;
      if constexpr (W == 1) v[j][0] = __ldcs(src);
      else if constexpr (W == 2) v[j][0] = __ldcs(reinterpret_cast<const uint16_t*>(src));
      else if constexpr (W == 4) v[j][0] = __ldcs(reinterpret_cast<const uint32_t*>(src));
      else if constexpr (W == 8) { const uint2 t = __ldcs(reinterpret_cast<const uint2*>(src)); v[j][0] = t.x; v[j][1] = t.y; }
      else { const uint4 t = __ldcs(reinterpret_cast<const uint4*>(src)); v[j][0] = t.x; v[j][1] = t.y; v[j][2] = t.z; v[j][3] = t.w; }
    }
  }
#pragma unroll
  for (int j = 0; j < U; ++j) {
    if (j < count && act) {
      const uint32_t a = row_s + static_cast<uint32_t>(s_ent_start[begin + j]);
      if constexpr (W == 1) t3_sts_u8(a, v[j][0]);
      else if constexpr (W == 2) t3_sts_u16(a, v[j][0]);
      else if constexpr (W == 4) t3_sts_u32(a, v[j][0]);
      else if constexpr (W == 8) t3_sts_v2(a, v[j][0], v[j][1]);
      else { t3_sts_v2(a, v[j][0], v[j][1]); t3_sts_v2(a + 8, v[j][2], v[j][3]); }  // rows are 8-byte aligned only
    }
  }
}

// source-space loads of the chars copy: global (read-only path) or shared (the staging slots)
template <bool SMEM>
__device__ __forceinline__ uint32_t t3_ld_u32(uint64_t a)
{
  uint32_t v;
  if constexpr (SMEM) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(static_cast<uint32_t>(a)));
  else v = __ldg(reinterpret_cast<const uint32_t*>(a));
  return v;
}
template <bool SMEM>
__device__ __forceinline__ uint32_t t3_ld_u8(uint64_t a)
{
  uint32_t v;
  if constexpr (SMEM) asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(static_cast<uint32_t>(a)));
  else v = __ldg(reinterpret_cast<const uint8_t*>(a));
  return v;
}

// chars of one STRING column for the tile: lane's string = L bytes at source address S (global, or shared when
// the tile's chars were staged) -> shared address D
template <bool SMEM>
__device__ __forceinline__ void t3_copy_chars(uint64_t S, uint32_t D, int L, int rows, int lane)
{
  const int maxL = __reduce_max_sync(0xffffffffu, L);
  if (maxL == 0) return;
  if (maxL <= 32) {
    // dst words k = 0.. start at the aligned address D - dsh; dst word k = source bytes [4k - dsh, 4k - dsh + 4) of
    // the string = funnel(w[k], w[k+1]) of the aligned source words w[k] at sp + 4k, sp = S - pre.
    const int dsh      = static_cast<int>(D & 3u);
    const int ssh      = static_cast<int>(S & 3u);
    const int dlt      = ssh - dsh;
    const int pre      = ssh + (dlt < 0 ? 4 : 0);  // string byte 0 is byte `pre` of the source word stream
    const uint64_t sp  = S - pre;
    const int sh       = (dlt & 3) * 8;
    const int end      = dsh + L;            // one past the last dst byte, relative to dst word 0
    const int kfull1   = end >> 2;           // full dst words: [dsh ? 1 : 0, kfull1)
    const uint32_t w0s = D - dsh;
    const int lim      = L > 0 ? L + pre : 0;  // source word k overlaps the string iff 4k < lim (and k > 0 or pre < 4)
    const int Kmax     = (maxL + 6) >> 2;    // warp-uniform bound on kfull1 (<= 9)
    // edge bytes straight from the source (independent of the word pipeline): the first nh bytes when the
    // destination starts inside a word, the last nt bytes when it ends inside one
    const int nh = dsh ? tmin(L, 4 - dsh) : 0;
    const int nt = (kfull1 > 0 || !dsh) ? (end & 3) : 0;
    const uint64_t St = S + (L - nt);
    uint32_t hb[3], tb[3];
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      hb[t] = tb[t] = 0;
      if (t < nh) hb[t] = t3_ld_u8<SMEM>(S + t);
      if (t < nt) tb[t] = t3_ld_u8<SMEM>(St + t);
    }
    uint32_t w[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      w[k] = 0;
      // only words that overlap [S, S+L): an aligned word that holds one valid byte is inside the buffer's page
      const bool need = k == 0 ? (lim > 0 && pre < 4) : (4 * k < lim);
      if (need) w[k] = t3_ld_u32<SMEM>(sp + 4 * k);
    }
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      if (t < nh) t3_sts_u8(D + t, hb[t]);
      if (t < nt) t3_sts_u8(D + (L - nt) + t, tb[t]);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      if (k < Kmax) {
        const uint32_t y = __funnelshift_r(w[k], w[k + 1], sh);
        const bool full  = k == 0 ? (dsh == 0 && kfull1 > 0) : (k < kfull1);
        if (full) t3_sts_u32(w0s + 4 * k, y);
      }
    }
  } else {
    // long strings: the warp copies one row's string at a time, lane = byte
    for (int i = 0; i < rows; ++i) {
      const uint64_t Si = __shfl_sync(0xffffffffu, static_cast<unsigned long long>(S), i);
      const uint32_t Di = __shfl_sync(0xffffffffu, D, i);
      const int Li      = __shfl_sync(0xffffffffu, L, i);
      for (int j = lane; j < Li; j += 32) t3_sts_u8(Di + j, t3_ld_u8<SMEM>(Si + j));
    }
  }
}

template <int kT3Warps, int kCtasPerSm>
__global__ void __launch_bounds__(kT3Warps * 32, kCtasPerSm) to_rows3_kernel(const __grid_constant__ ToRows3Params p)
{
  constexpr int kT3Threads = kT3Warps * 32;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* image = smem;  // stage_bytes + 32
  uint8_t* stg   = smem + p.stage_bytes + 32;  // nstr * slot_bytes: the tile's chars, one 16-byte aligned slice per column
  uint8_t* q     = stg + static_cast<size_t>(p.nstr) * p.slot_bytes;
  const uint8_t** s_ent_ptr = reinterpret_cast<const uint8_t**>(q);  q += sizeof(void*) * p.nfixed;
  const uint32_t** s_mask   = reinterpret_cast<const uint32_t**>(q); q += sizeof(void*) * p.ncols;
  const int32_t** s_soff    = reinterpret_cast<const int32_t**>(q);  q += sizeof(void*) * p.nstr;
  const uint8_t** s_chars   = reinterpret_cast<const uint8_t**>(q);  q += sizeof(void*) * p.nstr;
  int32_t* s_ent_start      = reinterpret_cast<int32_t*>(q);         q += 4 * p.nfixed;
  int32_t* s_sstart         = reinterpret_cast<int32_t*>(q);         q += 4 * p.nstr;
  int32_t* s_bsum           = reinterpret_cast<int32_t*>(q);         q += 4 * 32 * p.nblocks;
  int32_t* s_delta          = reinterpret_cast<int32_t*>(q);         q += 4 * p.nstr;     // staged address of chars offset 0
  int32_t* s_items          = reinterpret_cast<int32_t*>(q);         q += 4 * p.nitems;   // build order
  int32_t* s_list           = reinterpret_cast<int32_t*>(q);         q += 4 * p.nitems;   // grouped by owning warp
  uint8_t* s_owner          = q;
  __shared__ int s_nitems;
  __shared__ int s_direct[2];  // per tile parity: 1 = some column's slice did not fit its slot, read the chars from global
  __shared__ int s_wbeg[kT3Warps + 1];

  const int tid  = threadIdx.x;
  const int lane = lane_id();
  const int w    = warp_id();
  for (int i = tid; i < p.nfixed; i += kT3Threads) {
    const Entry e  = p.entries[i];
    s_ent_ptr[i]   = static_cast<const uint8_t*>(p.col_data[e.column]);
    s_ent_start[i] = e.start;
  }
  for (int i = tid; i < p.ncols; i += kT3Threads) s_mask[i] = p.masks[i];
  for (int i = tid; i < p.nstr; i += kT3Threads) {
    s_soff[i]   = p.str_offsets[i];
    s_chars[i]  = p.str_chars[i];
    s_sstart[i] = p.string_start[i];
  }
  if (tid == 0) {
    int n = 0;
    for (int b = 0; b < p.nblocks; ++b) s_items[n++] = t3_item(kItemString, b, 0);
    for (int k = kNumClasses - 1; k >= 0; --k)
    {
      const int U = 8;
      for (int e = p.class_begin[k]; e < p.class_begin[k + 1]; e += U) s_items[n++] = t3_item(k, e, tmin(U, p.class_begin[k + 1] - e));
    }
    for (int g = 0; g * 32 < p.ncols; ++g) s_items[n++] = t3_item(kItemValidity, g, 0);
    s_nitems    = n;
    s_direct[0] = 0;
    s_direct[1] = 0;
  }
  __syncthreads();
  // static schedule: items (heaviest first) go to the least-loaded warp; every warp then walks its own list
  // (no atomics in the tile loop).  Costs are in units of ~one dependent memory round trip.
  if (w == 0) {
    const int n = s_nitems;
    int load    = lane < kT3Warps ? 0 : (1 << 25);
    for (int i = 0; i < n; ++i) {
      const int32_t item = s_items[i];
      const int kind = item & 7, begin = (item >> 3) & 0x1ffff, count = item >> 20;
      const int cost = kind == kItemString ? 10 * tmin(p.sb, p.nstr - begin * p.sb) : kind == kItemValidity ? 6 : (kind >= 2 ? 3 : 4 + count);
      const int sel  = static_cast<int>(__reduce_min_sync(0xffffffffu, static_cast<unsigned>((load << 5) | lane)) & 31u);
      if (lane == sel) load += cost;
      if (lane == 0) s_owner[i] = static_cast<uint8_t>(sel);
    }
    __syncwarp();
    if (lane == 0) {
      int pos = 0;
      for (int ww = 0; ww < kT3Warps; ++ww) {
        s_wbeg[ww] = pos;
        for (int i = 0; i < n; ++i)
          if (s_owner[i] == ww) s_list[pos++] = s_items[i];
      }
      s_wbeg[kT3Warps] = pos;
    }
  }
  __syncthreads();
  const int my_beg = s_wbeg[w], my_end_item = s_wbeg[w + 1];
  const uint32_t image_s = smem_u32(image);
  const uint32_t stg_s   = smem_u32(stg);
  int tile_par           = 0;

  const uintptr_t out_g  = reinterpret_cast<uintptr_t>(p.out_data);
  const int nvb          = (p.ncols + 7) >> 3;

  const int64_t nsuper = (p.row_count + p.super_rows - 1) / p.super_rows;
  for (int64_t st = blockIdx.x; st < nsuper; st += gridDim.x) {
    int64_t r          = st * p.super_rows;
    const int64_t rend = tmin<int64_t>(p.row_count, r + p.super_rows);
    while (r < rend) {
      const int rem      = static_cast<int>(tmin<int64_t>(32, rend - r));
      const int64_t abs0 = p.row_start + r;
      // ---- 1. geometry: every warp reads the tile's LIST offsets itself (no header hand-off).  Fetching the next
      // tile's offsets a tile ahead was measured slower (the early loads pin a scoreboard the tile's other
      // memory operations then wait on) ----------------------------------------------------------------------------
      int32_t oa = 0, ob = 0;
      if (lane < rem) {
        oa = p.out_offsets[r + lane];
        ob = p.out_offsets[r + lane + 1];
      }
      // ---- 2. string block sums + staging of the tile's chars ---------------------------------------------
      bool direct = p.slot_bytes == 0;
      for (int b = w; b < p.nblocks; b += kT3Warps) {
        const int s0 = b * p.sb, s1 = tmin(p.nstr, s0 + p.sb);
        int32_t sum = 0;
        for (int sA = s0; sA < s1; sA += 4) {
          int32_t o0[4], o1[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            o0[j] = o1[j] = 0;
            if (sA + j < s1 && lane < rem) {
              const int32_t* so = s_soff[sA + j] + abs0 + lane;
              o0[j]             = __ldg(so);
              o1[j]             = __ldg(so + 1);
            }
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (sA + j < s1) {  // warp-uniform
              const int sj = sA + j;
              sum += o1[j] - o0[j];
              if (p.slot_bytes > 0) {
                // stage the column's chars for rows [abs0, abs0 + rem): ONE contiguous global range, copied by
                // 16-byte cp.async (no registers, no scoreboard) into the column's slot; only granules that hold
                // at least one valid byte are read
                const int32_t first = __shfl_sync(0xffffffffu, o0[j], 0);
                const int32_t last  = __shfl_sync(0xffffffffu, o1[j], rem - 1);
                if (last > first) {
                  const uintptr_t cb = reinterpret_cast<uintptr_t>(s_chars[sj]);
                  const uintptr_t g0 = (cb + static_cast<uint32_t>(first)) & ~uintptr_t{15};
                  const uintptr_t g1 = (cb + static_cast<uint32_t>(last) + 15) & ~uintptr_t{15};
                  const int64_t span = static_cast<int64_t>(g1 - g0);
                  if (span > p.slot_bytes) {
                    direct = true;
                  } else {
                    const uint32_t slot_s = stg_s + static_cast<uint32_t>(sj) * static_cast<uint32_t>(p.slot_bytes);
                    for (int c = lane * 16; c < static_cast<int>(span); c += 512)
                      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot_s + c), "l"(g0 + c) : "memory");
                    if (lane == 0) s_delta[sj] = static_cast<int32_t>(slot_s) - static_cast<int32_t>(static_cast<int64_t>(g0) - static_cast<int64_t>(cb));
                  }
                }
              }
            }
          }
        }
        s_bsum[b * 32 + lane] = sum;
      }
      if (direct && lane == 0) s_direct[tile_par] = 1;
      const int64_t lo      = static_cast<uint32_t>(__shfl_sync(0xffffffffu, oa, 0));
      const int skew        = static_cast<int>((out_g + lo) & 15);
      const int my_off      = static_cast<int>(static_cast<uint32_t>(oa) - static_cast<uint32_t>(lo)) + skew;
      const int my_end      = static_cast<int>(static_cast<uint32_t>(ob) - static_cast<uint32_t>(lo)) + skew;
      const bool fits       = lane < rem && my_end <= p.stage_bytes;
      int rows              = __popc(__ballot_sync(0xffffffffu, fits));
      if (rows < rem) rows &= ~7;
      if (rows == 0) {  // cannot hold 8 rows: the generic kernel redoes the batch
        if (tid == 0) { atomicExch(p.fail_flag, 1); tma_store_wait_all<0>(); }
        return;
      }
      const int hi_rel = __shfl_sync(0xffffffffu, my_end, rows - 1);
      const bool act   = lane < rows;
      const uint32_t row_s = image_s + static_cast<uint32_t>(my_off);
      // ---- 3. buffer free -> zero fill -----------------------------------------------------------------
      if (tid == 0) { tma_store_wait_read<0>(); s_direct[tile_par ^ 1] = 0; }
      __syncthreads();
      if (w == kT3Warps - 1) {  // block sums -> exclusive prefix per row (published by the barrier below)
        int32_t acc = p.size_per_row;  // RC:838: chars start right behind the fixed section
        for (int b = 0; b < p.nblocks; ++b) {
          const int32_t v       = s_bsum[b * 32 + lane];
          s_bsum[b * 32 + lane] = acc;
          acc += v;
        }
      }
      {
        const uint32_t ze = image_s + static_cast<uint32_t>(hi_rel);
#pragma unroll 4
        for (uint32_t a = image_s + 16u * tid; a < ze; a += 16u * kT3Threads)
          asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0u));
      }
      asm volatile("cp.async.wait_all;" ::: "memory");  // this thread's slice of the chars staging has landed
      __syncthreads();
      const bool tile_direct = s_direct[tile_par] != 0;
      // ---- 4. this warp's items ----------------------------------------------------------------------------
      for (int qi = my_beg; qi < my_end_item; ++qi) {
        const int32_t item = s_list[qi];
        const int kind = item & 7, begin = (item >> 3) & 0x1ffff, count = item >> 20;
        if (kind == kItemString) {
          const int s0 = begin * p.sb, s1 = tmin(p.nstr, s0 + p.sb);
          int32_t run = s_bsum[begin * 32 + lane];
          for (int sA = s0; sA < s1; sA += kHoist) {
            int32_t o0[kHoist], Ls[kHoist];
#pragma unroll
            for (int j = 0; j < kHoist; ++j) {  // the offsets of kHoist columns first (L1 / L2 hits: step 2 touched them)
              o0[j] = Ls[j] = 0;
              if (sA + j < s1 && act) {
                const int32_t* so = s_soff[sA + j] + abs0 + lane;
                o0[j]             = __ldg(so);
                Ls[j]             = tmax(__ldg(so + 1) - o0[j], 0);
              }
            }
#pragma unroll
            for (int j = 0; j < kHoist; ++j) {
              if (sA + j < s1) {
                const int s = sA + j;
                if (act) {
                  const uint32_t pa = row_s + static_cast<uint32_t>(s_sstart[s]);
                  t3_sts_u32(pa, static_cast<uint32_t>(run));        // RC:848
                  t3_sts_u32(pa + 4, static_cast<uint32_t>(Ls[j]));  // RC:849
                }
                if (tile_direct)
                  t3_copy_chars<false>(reinterpret_cast<uintptr_t>(s_chars[s]) + static_cast<uint32_t>(o0[j]), row_s + static_cast<uint32_t>(run), Ls[j], rows, lane);
                else
                  t3_copy_chars<true>(static_cast<uint32_t>(s_delta[s] + o0[j]), row_s + static_cast<uint32_t>(run), Ls[j], rows, lane);
                run += Ls[j];
              }
            }
          }
        } else if (kind == kItemValidity) {
          const int c      = begin * 32 + lane;
          uint32_t bits    = 0;
          if (c < p.ncols) {
            const uint32_t* m = s_mask[c];
            if (m == nullptr) {
              bits = 0xffffffffu;
            } else {
              const int64_t wi  = abs0 >> 5;
              const int shb     = static_cast<int>(abs0 & 31);
              const uint32_t w0 = __ldg(m + wi);
              uint32_t w1       = 0;
              if (shb != 0 && ((abs0 + rows - 1) >> 5) > wi) w1 = __ldg(m + wi + 1);
              bits = __funnelshift_r(w0, w1, shb);
            }
          }
          const uint32_t t = t3_transpose32(bits, lane);  // lane = row: bit j = column begin*32 + j
          if (act) {
            const uint32_t a = row_s + static_cast<uint32_t>(p.validity_offset + begin * 4);
            const int nb     = tmin(4, nvb - begin * 4);
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (k < nb) t3_sts_u8(a + k, t >> (8 * k));
          }
        } else {
          const int64_t ar = abs0 + lane;
          switch (kind) {
            case 4: t3_fixed_async<16, 8>(s_ent_ptr, s_ent_start, begin, count, ar, act, row_s); break;
            case 3: t3_fixed_async<8, 8>(s_ent_ptr, s_ent_start, begin, count, ar, act, row_s); break;
            case 2: t3_fixed_async<4, 8>(s_ent_ptr, s_ent_start, begin, count, ar, act, row_s); break;
            case 1: t3_fixed<2, 8>(s_ent_ptr, s_ent_start, begin, count, ar, act, row_s); break;
            default: t3_fixed<1, 8>(s_ent_ptr, s_ent_start, begin, count, ar, act, row_s); break;
          }
        }
      }
      asm volatile("cp.async.wait_all;" ::: "memory");  // this thread's cp.async copies have landed
      fence_proxy_async();  // generic-proxy smem writes -> visible to the TMA store
      __syncthreads();
      // ---- 5. write out ------------------------------------------------------------------------------------
      if (tid == 0) {
        const uintptr_t g_lo = out_g + lo;
        const uintptr_t g_hi = g_lo + (hi_rel - skew);
        const uintptr_t fl   = g_lo - skew;  // global address of image byte 0
        const uintptr_t t_lo = (g_lo + 15) & ~uintptr_t{15};
        const uintptr_t t_hi = g_hi & ~uintptr_t{15};
        uintptr_t h_end      = tmin(t_lo, g_hi);
        uintptr_t t_beg      = tmax(t_hi, h_end);
        if (t_hi > t_lo) {
          tma_store_1d(reinterpret_cast<void*>(t_lo), image + (t_lo - fl), static_cast<uint32_t>(t_hi - t_lo));
        } else {
          h_end = g_hi;
          t_beg = g_hi;
        }
        tma_store_commit();
        for (uintptr_t a = g_lo; a < h_end; a += 8)
          *reinterpret_cast<uint2*>(a) = *reinterpret_cast<const uint2*>(image + (a - fl));
        for (uintptr_t a = t_beg; a < g_hi; a += 8)
          *reinterpret_cast<uint2*>(a) = *reinterpret_cast<const uint2*>(image + (a - fl));
      }
      r += rows;
      tile_par ^= 1;
    }
  }
  if (tid == 0) tma_store_wait_all<0>();
}


// ==================================================================================================
// Narrow rows with STRING columns (a few hundred bytes per row -- the common Spark shape): every warp owns a private
// row-image buffer and converts 32-row tiles on its own: no CTA barrier anywhere in the tile loop.
//   lane = row: LIST offsets -> geometry; zero the image; fixed-width fields by cp.async (4/8/16 B) or LDG/STS
//   (1/2 B); validity by the 32x32 bit butterfly; per STRING column the (offset, len) pair and the chars (aligned
//   32-bit words from global, funnel-shifted, see t3_copy_chars); then the warp flushes its image -- ONE contiguous
//   byte range of the output -- with 16-byte coalesced stores.
// A tile whose rows do not fit the warp's buffer raises *fail_flag (generic kernel redoes the batch).
// ==================================================================================================
constexpr int kTwWarps = 24;

struct ToRowsWParams {
  const void* const* col_data;
  const uint32_t* const* masks;
  const int32_t* const* str_offsets;
  const uint8_t* const* str_chars;
  int64_t row_start, row_count;
  const int32_t* out_offsets;
  uint8_t* out_data;
  int32_t ncols, nstr, nfixed;
  int32_t validity_offset, size_per_row;
  int32_t wbuf_bytes;  // per-warp image bytes (multiple of 16)
  int32_t class_begin[kNumClasses + 1];
  const Entry* entries;
  const int32_t* string_start;
  int32_t* fail_flag;
};

__global__ void __launch_bounds__(kTwWarps * 32, 1) to_rows_w_kernel(const __grid_constant__ ToRowsWParams p)
{
  constexpr int kThreads = kTwWarps * 32;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* q = smem + static_cast<size_t>(kTwWarps) * (p.wbuf_bytes + 32);
  const uint8_t** s_ent_ptr = reinterpret_cast<const uint8_t**>(q);  q += sizeof(void*) * p.nfixed;
  const uint32_t** s_mask   = reinterpret_cast<const uint32_t**>(q); q += sizeof(void*) * p.ncols;
  const int32_t** s_soff    = reinterpret_cast<const int32_t**>(q);  q += sizeof(void*) * p.nstr;
  const uint8_t** s_chars   = reinterpret_cast<const uint8_t**>(q);  q += sizeof(void*) * p.nstr;
  int32_t* s_ent_start      = reinterpret_cast<int32_t*>(q);         q += 4 * p.nfixed;
  int32_t* s_sstart         = reinterpret_cast<int32_t*>(q);

  const int tid  = threadIdx.x;
  const int lane = lane_id();
  const int w    = warp_id();
  for (int i = tid; i < p.nfixed; i += kThreads) {
    const Entry e  = p.entries[i];
    s_ent_ptr[i]   = static_cast<const uint8_t*>(p.col_data[e.column]);
    s_ent_start[i] = e.start;
  }
  for (int i = tid; i < p.ncols; i += kThreads) s_mask[i] = p.masks[i];
  for (int i = tid; i < p.nstr; i += kThreads) {
    s_soff[i]   = p.str_offsets[i];
    s_chars[i]  = p.str_chars[i];
    s_sstart[i] = p.string_start[i];
  }
  __syncthreads();
  uint8_t* image         = smem + static_cast<size_t>(w) * (p.wbuf_bytes + 32);
  const uint32_t image_s = smem_u32(image);
  const uintptr_t out_g  = reinterpret_cast<uintptr_t>(p.out_data);
  const int nvb          = (p.ncols + 7) >> 3;
  const int ngv          = (p.ncols + 31) >> 5;

  // 32-row groups are dealt to the warps of the grid; a group takes one or more tiles (rows that fit the buffer)
  const int64_t ngroups = (p.row_count + 31) >> 5;
  const int64_t gstep   = static_cast<int64_t>(gridDim.x) * kTwWarps;
  for (int64_t grp = static_cast<int64_t>(blockIdx.x) * kTwWarps + w; grp < ngroups; grp += gstep) {
    int64_t r          = grp * 32;
    const int64_t rend = tmin<int64_t>(p.row_count, r + 32);
    while (r < rend) {
      const int rem      = static_cast<int>(rend - r);
      const int64_t abs0 = p.row_start + r;
      int32_t oa = 0, ob = 0;
      if (lane < rem) {
        oa = p.out_offsets[r + lane];
        ob = p.out_offsets[r + lane + 1];
      }
      // the offsets of the first STRING columns are fetched with the geometry: their latency hides behind the zero
      // fill, the cp.async issue and the validity transpose instead of heading the chars chain
      constexpr int kPre = 4;
      int32_t po0[kPre], pL[kPre];
#pragma unroll
      for (int j = 0; j < kPre; ++j) {
        po0[j] = pL[j] = 0;
        if (j < p.nstr && lane < rem) {
          const int32_t* so = s_soff[j] + abs0 + lane;
          po0[j]            = __ldg(so);
          pL[j]             = __ldg(so + 1);
        }
      }
      const int64_t lo = static_cast<uint32_t>(__shfl_sync(0xffffffffu, oa, 0));
      const int skew   = static_cast<int>((out_g + lo) & 15);
      const int my_off = static_cast<int>(static_cast<uint32_t>(oa) - static_cast<uint32_t>(lo)) + skew;
      const int my_end = static_cast<int>(static_cast<uint32_t>(ob) - static_cast<uint32_t>(lo)) + skew;
      const bool fits  = lane < rem && my_end <= p.wbuf_bytes;
      int rows         = __popc(__ballot_sync(0xffffffffu, fits));
      if (rows == 0) {  // a row larger than the warp's buffer: the generic kernel redoes the batch
        if (lane == 0) atomicExch(p.fail_flag, 1);
        return;
      }
      const int hi_rel     = __shfl_sync(0xffffffffu, my_end, rows - 1);
      const bool act       = lane < rows;
      const uint32_t row_s = image_s + static_cast<uint32_t>(my_off);
      // ---- zero fill (padding bytes are 0) ------------------------------------------------------------
      for (uint32_t a = image_s + 16u * lane; a < image_s + static_cast<uint32_t>(hi_rel); a += 512u)
        asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0u));
      __syncwarp();
      // ---- fixed-width fields -------------------------------------------------------------------------
      const int64_t ar = abs0 + lane;
      for (int e = p.class_begin[4]; e < p.class_begin[5]; e += 8) t3_fixed_async<16, 8>(s_ent_ptr, s_ent_start, e, tmin(8, p.class_begin[5] - e), ar, act, row_s);
      for (int e = p.class_begin[3]; e < p.class_begin[4]; e += 8) t3_fixed_async<8, 8>(s_ent_ptr, s_ent_start, e, tmin(8, p.class_begin[4] - e), ar, act, row_s);
      for (int e = p.class_begin[2]; e < p.class_begin[3]; e += 8) t3_fixed_async<4, 8>(s_ent_ptr, s_ent_start, e, tmin(8, p.class_begin[3] - e), ar, act, row_s);
      for (int e = p.class_begin[1]; e < p.class_begin[2]; e += 4) t3_fixed<2, 4>(s_ent_ptr, s_ent_start, e, tmin(4, p.class_begin[2] - e), ar, act, row_s);
      for (int e = p.class_begin[0]; e < p.class_begin[1]; e += 4) t3_fixed<1, 4>(s_ent_ptr, s_ent_start, e, tmin(4, p.class_begin[1] - e), ar, act, row_s);
      // ---- validity -----------------------------------------------------------------------------------
      for (int g = 0; g < ngv; ++g) {
        const int c   = g * 32 + lane;
        uint32_t bits = 0;
        if (c < p.ncols) {
          const uint32_t* m = s_mask[c];
          if (m == nullptr) {
            bits = 0xffffffffu;
          } else {
            const int64_t wi  = abs0 >> 5;
            const int shb     = static_cast<int>(abs0 & 31);
            const uint32_t w0 = __ldg(m + wi);
            uint32_t w1       = 0;
            if (shb != 0 && ((abs0 + rows - 1) >> 5) > wi) w1 = __ldg(m + wi + 1);
            bits = __funnelshift_r(w0, w1, shb);
          }
        }
        const uint32_t t = t3_transpose32(bits, lane);  // lane = row: bit j = column g*32 + j
        if (act) {
          const uint32_t a = row_s + static_cast<uint32_t>(p.validity_offset + g * 4);
          const int nb     = tmin(4, nvb - g * 4);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < nb) t3_sts_u8(a + k, t >> (8 * k));
        }
      }
      // ---- strings: pairs + chars (RC:838-858) ---------------------------------------------------------
      int32_t run = p.size_per_row;
#pragma unroll
      for (int j = 0; j < kPre; ++j) {
        if (j < p.nstr) {
          const int32_t o0 = po0[j];
          const int32_t L  = act ? tmax(pL[j] - o0, 0) : 0;
          if (act) {
            const uint32_t pa = row_s + static_cast<uint32_t>(s_sstart[j]);
            t3_sts_u32(pa, static_cast<uint32_t>(run));
            t3_sts_u32(pa + 4, static_cast<uint32_t>(L));
          }
          t3_copy_chars<false>(reinterpret_cast<uintptr_t>(s_chars[j]) + static_cast<uint32_t>(o0), row_s + static_cast<uint32_t>(run), L, rows, lane);
          run += L;
        }
      }
      for (int s = kPre; s < p.nstr; ++s) {
        int32_t o0 = 0, L = 0;
        if (act) {
          const int32_t* so = s_soff[s] + abs0 + lane;
          o0                = __ldg(so);
          L                 = tmax(__ldg(so + 1) - o0, 0);
          const uint32_t pa = row_s + static_cast<uint32_t>(s_sstart[s]);
          t3_sts_u32(pa, static_cast<uint32_t>(run));
          t3_sts_u32(pa + 4, static_cast<uint32_t>(L));
        }
        t3_copy_chars<false>(reinterpret_cast<uintptr_t>(s_chars[s]) + static_cast<uint32_t>(o0), row_s + static_cast<uint32_t>(run), L, rows, lane);
        run += L;
      }
      asm volatile("cp.async.wait_all;" ::: "memory");
      __syncwarp();
      // ---- flush: the image is one contiguous byte range of the output ------------------------------------
      {
        const uintptr_t g_lo = out_g + lo;
        const uintptr_t g_hi = g_lo + (hi_rel - skew);
        const uintptr_t fl   = g_lo - skew;  // global address of image byte 0 (16-byte aligned)
        const uintptr_t t_lo = (g_lo + 15) & ~uintptr_t{15};
        const uintptr_t t_hi = tmax(g_hi & ~uintptr_t{15}, t_lo);
        for (uintptr_t a = t_lo + 16u * lane; a < t_hi; a += 512) {
          uint32_t v0, v1, v2, v3;
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "r"(image_s + static_cast<uint32_t>(a - fl)));
          asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(a), "r"(v0), "r"(v1), "r"(v2), "r"(v3));
        }
        // rows are 8-byte aligned: at most one 8-byte piece before the first and after the last 16-byte chunk
        if (lane == 0 && g_lo < tmin(t_lo, g_hi)) *reinterpret_cast<uint2*>(g_lo) = *reinterpret_cast<const uint2*>(image + (g_lo - fl));
        if (lane == 1 && t_hi < g_hi && t_hi >= t_lo && g_hi > t_lo) *reinterpret_cast<uint2*>(t_hi) = *reinterpret_cast<const uint2*>(image + (t_hi - fl));
      }
      __syncwarp();  // the image is reused by the next tile
      r += rows;
    }
  }
}

static int launch_to_rows_warp(const srj_plan* plan, const void* const* d_col_data, const uint32_t* const* d_masks,
                               const int32_t* const* d_str_offsets, const uint8_t* const* d_str_chars, int64_t row_start,
                               int64_t row_count, const int32_t* out_offsets, uint8_t* out_data, int64_t avg_row,
                               int32_t* d_fail_flag, cudaStream_t stream, int* launched)
{
  const int nstr = plan->num_string_columns;
  ToRowsWParams p{};
  p.nfixed = static_cast<int32_t>(plan->tr_entries.size());
  p.ncols  = plan->num_columns;
  p.nstr   = nstr;
  const size_t tables = sizeof(void*) * (static_cast<size_t>(p.nfixed) + p.ncols + 2 * static_cast<size_t>(nstr)) +
                        4 * (static_cast<size_t>(p.nfixed) + nstr) + 128;
  const int64_t budget = 232448 - 1024 - 64 - static_cast<int64_t>(tables);
  const int64_t wbuf   = (budget / kTwWarps - 32) / 16 * 16;
  // want >= 16 rows per tile on average (half the lanes busy), and at least one maximal fixed section
  if (wbuf < 1024 || wbuf < plan->fixed_row_size + 64 || avg_row * 16 > wbuf) return SRJ_OK;
  p.col_data        = d_col_data;
  p.masks           = d_masks;
  p.str_offsets     = d_str_offsets;
  p.str_chars       = d_str_chars;
  p.row_start       = row_start;
  p.row_count       = row_count;
  p.out_offsets     = out_offsets;
  p.out_data        = out_data;
  p.validity_offset = plan->validity_offset;
  p.size_per_row    = plan->size_per_row;
  p.wbuf_bytes      = static_cast<int32_t>(wbuf);
  for (int k = 0; k <= kNumClasses; ++k) p.class_begin[k] = plan->tr_class_begin[k];
  p.entries      = plan->d_tr_entries;
  p.string_start = plan->d_string_start;
  p.fail_flag    = d_fail_flag;
  int dev = 0, nsm = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  const int64_t ngroups = (row_count + 31) / 32;
  const int64_t grid    = std::min<int64_t>(nsm, (ngroups + kTwWarps - 1) / kTwWarps);
  const size_t smem     = static_cast<size_t>(kTwWarps) * (wbuf + 32) + tables;
  SRJ_CUDA_TRY(cudaMemsetAsync(d_fail_flag, 0, sizeof(int32_t), stream));
  SRJ_CUDA_TRY(cudaFuncSetAttribute(to_rows_w_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448 - 1024));
  to_rows_w_kernel<<<static_cast<unsigned>(grid), kTwWarps * 32, smem, stream>>>(p);
  SRJ_CUDA_TRY(cudaGetLastError());
  *launched = 1;
  return SRJ_OK;
}

// Returns SRJ_OK and sets *launched when the kernel was launched (the caller then launches the generic kernel
// guarded by d_fail_flag); *launched = 0 means the table is not eligible.
int launch_to_rows_var(const srj_plan* plan, const void* const* d_col_data, const uint32_t* const* d_masks,
                       const int32_t* const* d_str_offsets, const uint8_t* const* d_str_chars, int64_t row_start,
                       int64_t row_count, const int32_t* out_offsets, uint8_t* out_data, int64_t out_bytes,
                       int32_t* d_fail_flag, cudaStream_t stream, const void* const* h_col_data, int* launched)
{
  *launched = 0;
  const int nstr = plan->num_string_columns;
  if (nstr == 0 || row_count == 0 || !d_fail_flag || !h_col_data) return SRJ_OK;
  if ((reinterpret_cast<uintptr_t>(out_data) & 7) != 0) return SRJ_OK;
  for (const Entry& e : plan->tr_entries)
    if (reinterpret_cast<uintptr_t>(h_col_data[e.column]) & static_cast<uintptr_t>(plan->col_size[e.column] - 1)) return SRJ_OK;

  // narrow rows: warp-private tiles (to_rows_w_kernel); wide rows: CTA tiles (to_rows3_kernel) below
  const int64_t avg_row = std::max<int64_t>(plan->fixed_row_size, out_bytes / row_count);
  const int rc = launch_to_rows_warp(plan, d_col_data, d_masks, d_str_offsets, d_str_chars, row_start, row_count, out_offsets,
                                     out_data, avg_row, d_fail_flag, stream, launched);
  if (rc != SRJ_OK || *launched) return rc;
  ToRows3Params p{};
  p.nfixed  = static_cast<int32_t>(plan->tr_entries.size());
  p.ncols   = plan->num_columns;
  p.nstr    = nstr;
  p.sb      = std::max(4, (nstr + kT3MaxBlocks - 1) / kT3MaxBlocks);
  p.nblocks = (nstr + p.sb - 1) / p.sb;
  int nitems = p.nblocks + (p.ncols + 31) / 32;
  for (int k = 0; k < kNumClasses; ++k) {
    const int U = 8;
    nitems += (plan->tr_class_begin[k + 1] - plan->tr_class_begin[k] + U - 1) / U;
  }
  if (nitems > kT3MaxItems) return SRJ_OK;
  p.nitems = nitems;
  const size_t tables = sizeof(void*) * (static_cast<size_t>(p.nfixed) + p.ncols + 2 * static_cast<size_t>(nstr)) +
                        4 * (static_cast<size_t>(p.nfixed) + nstr + 32 * static_cast<size_t>(p.nblocks) + nstr + 2 * static_cast<size_t>(nitems)) +
                        ((static_cast<size_t>(nitems) + 15) & ~size_t{15}) + 32 + 128;
  const int64_t budget = 232448 - 1024 - 64;
  // chars staging: a quarter of the budget at most, 1 KB per STRING column at most
  int64_t slot = std::min<int64_t>((budget - static_cast<int64_t>(tables)) / 4, 1024ll * nstr) / nstr / 16 * 16;
  if (slot < 128) slot = 0;
  p.slot_bytes         = static_cast<int32_t>(slot);
  int64_t stage        = (budget - static_cast<int64_t>(tables) - slot * nstr) / 16 * 16;
  if (stage < 32 * 1024 || stage < 8ll * (plan->fixed_row_size + 64)) return SRJ_OK;
  const int fit        = static_cast<int>(std::min<int64_t>(32, stage / avg_row / 8 * 8));
  if (fit < 8 || stage / avg_row >= 64) return SRJ_OK;  // narrow rows: multi-group tiles of the generic kernel

  p.col_data        = d_col_data;
  p.masks           = d_masks;
  p.str_offsets     = d_str_offsets;
  p.str_chars       = d_str_chars;
  p.row_start       = row_start;
  p.row_count       = row_count;
  p.out_offsets     = out_offsets;
  p.out_data        = out_data;
  p.validity_offset = plan->validity_offset;
  p.size_per_row    = plan->size_per_row;
  p.stage_bytes     = static_cast<int32_t>(stage);
  p.super_rows      = fit * 2;
  for (int k = 0; k <= kNumClasses; ++k) p.class_begin[k] = plan->tr_class_begin[k];
  p.entries      = plan->d_tr_entries;
  p.string_start = plan->d_string_start;
  p.fail_flag    = d_fail_flag;

  int dev = 0, nsm = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  const int64_t nsuper = (row_count + p.super_rows - 1) / p.super_rows;
  const int64_t grid   = std::min<int64_t>(nsm, nsuper);
  const size_t smem    = static_cast<size_t>(stage) + 32 + static_cast<size_t>(slot) * nstr + tables;
  SRJ_CUDA_TRY(cudaMemsetAsync(d_fail_flag, 0, sizeof(int32_t), stream));
  SRJ_CUDA_TRY(cudaFuncSetAttribute(to_rows3_kernel<24, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448 - 1024));
  to_rows3_kernel<24, 1><<<static_cast<unsigned>(grid), 24 * 32, smem, stream>>>(p);
  SRJ_CUDA_TRY(cudaGetLastError());
  *launched = 1;
  return SRJ_OK;
}

}  // namespace srj
