// to_rows.cu -- columns -> JCUDF rows (reference: convert_to_rows, RC:1762-2055).
//
// One kernel per output batch fuses copy_to_rows + copy_validity_to_rows + copy_strings_to_rows
// (RC:574-688, 706-798, 816-861) and the batch's row-offset column:
//   - a CTA owns a contiguous row range and assembles a tile of rows -- ONE contiguous byte range
//     of the output -- in shared memory: zero fill (padding bytes are defined as 0), coalesced
//     column reads (lane = row) scattered into the row images, validity bytes gathered from the
//     column masks, (offset,len) pairs by a warp scan across the STRING columns of a row, chars
//     appended in column order;
//   - the finished tile leaves with a single 1-D TMA bulk store (cp.async.bulk.global.shared::cta),
//     double-buffered so the store of tile k overlaps the assembly of tile k+1.
// Rows too large for a stage, or unaligned output buffers, take the SAFE path: the same assembly
// code writing global memory directly, byte-wise.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "kernels.hpp"
#include "plan.hpp"

namespace srj {

constexpr int kTrThreads = 256;
constexpr int kTrWarps   = kTrThreads / 32;
constexpr int kTrSlack   = 32;

struct ToRowsParams {
  const void* const* col_data;        // [ncols] fixed-width values (STRING: unused)
  const uint32_t* const* masks;       // [ncols], entries may be NULL
  const int32_t* const* str_offsets;  // [nstr]
  const uint8_t* const* str_chars;    // [nstr]
  const uint64_t* cum;                // inclusive cumulative row sizes over the table, or NULL (fixed)
  int64_t row_start;
  int64_t row_count;
  int32_t* out_offsets;
  uint8_t* out_data;
  int64_t out_bytes;
  int64_t rows_per_cta;
  int32_t ncols, nstr;
  int32_t validity_offset, size_per_row, row_stride;
  int32_t tile_rows, rpl, stage_bytes;
  int32_t nentries;
  int32_t class_begin[kNumClasses + 1];
  const Entry* entries;
  const int32_t* string_cols;
  const int32_t* string_start;
  int32_t max_str_entries;  // capacity of the per-tile string tables (rows * nstr)
  int32_t nbuf;             // 1: single stage buffer (more CTAs per SM), 2: double buffered
  int64_t offset_bias;      // added to the values written to out_offsets (tail launches of a batch)
  const int32_t* run_if;    // non-NULL: the launch is a fallback that only runs when *run_if != 0
};

struct TrHdr {
  int64_t r;        // first batch-relative row of the tile
  int64_t lo, hi;   // batch-relative output byte range
  int32_t rows;
  int32_t safe;
  int32_t skew;     // stage byte of output byte `lo`
  int32_t pad;
};

template <int W, bool SAFE>
__device__ __forceinline__ void put_elem(uint8_t* dst, const uint8_t* src)
{
  if constexpr (W == 1) {
    *dst = __ldg(src);
  } else if constexpr (W == 2) {
    const uint16_t v = __ldg(reinterpret_cast<const uint16_t*>(src));
    if constexpr (SAFE) { dst[0] = v & 0xff; dst[1] = v >> 8; } else { *reinterpret_cast<uint16_t*>(dst) = v; }
  } else if constexpr (W == 4) {
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(src));
    if constexpr (SAFE) {
#pragma unroll
      for (int i = 0; i < 4; ++i) dst[i] = static_cast<uint8_t>(v >> (8 * i));
    } else {
      *reinterpret_cast<uint32_t*>(dst) = v;
    }
  } else if constexpr (W == 8) {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(src));
    if constexpr (SAFE) {
#pragma unroll
      for (int i = 0; i < 4; ++i) { dst[i] = static_cast<uint8_t>(v.x >> (8 * i)); dst[4 + i] = static_cast<uint8_t>(v.y >> (8 * i)); }
    } else {
      *reinterpret_cast<uint2*>(dst) = v;
    }
  } else {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src));
    if constexpr (SAFE) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        dst[i]      = static_cast<uint8_t>(v.x >> (8 * i));
        dst[4 + i]  = static_cast<uint8_t>(v.y >> (8 * i));
        dst[8 + i]  = static_cast<uint8_t>(v.z >> (8 * i));
        dst[12 + i] = static_cast<uint8_t>(v.w >> (8 * i));
      }
    } else {
      // rows are 8-byte aligned only: two 8-byte stores
      *reinterpret_cast<uint2*>(dst)     = make_uint2(v.x, v.y);
      *reinterpret_cast<uint2*>(dst + 8) = make_uint2(v.z, v.w);
    }
  }
}

struct TrTables {
  const int32_t* ent_start;
  const int32_t* ent_col;
  const uint8_t* const* col_data;
  const uint8_t* const* mask_bytes;
  int32_t* str_src;  // [rows * nstr]
  int32_t* str_len;
  int32_t* str_dst;
};

// Assemble rows [r, r+rows) of the batch into `base` (+ row offsets).  All threads of the CTA.
template <bool SAFE>
__device__ __forceinline__ void assemble_tile(const ToRowsParams& p, const TrTables& t, uint8_t* base,
                                              const int32_t* s_off, int64_t stride, int64_t r, int rows,
                                              uint8_t* zero_base, int64_t zero_bytes)
{
  const int tid  = threadIdx.x;
  const int lane = lane_id();
  const int w    = warp_id();
  auto rowptr    = [&](int i) -> uint8_t* {
    return s_off ? base + static_cast<uint32_t>(s_off[i]) : base + static_cast<int64_t>(i) * stride;
  };
  const int64_t abs0 = p.row_start + r;  // table row of tile row 0

  // ---- zero fill (padding bytes are 0) ------------------------------------------------------------
  if constexpr (SAFE) {
    for (int64_t i = tid; i < zero_bytes; i += kTrThreads) zero_base[i] = 0;
  } else {
    uint4* z        = reinterpret_cast<uint4*>(zero_base);  // stage start: 16-byte aligned
    const int64_t n = (zero_bytes + 15) >> 4;
    for (int64_t i = tid; i < n; i += kTrThreads) z[i] = make_uint4(0, 0, 0, 0);
  }
  __syncthreads();

  // ---- fixed-width fields: coalesced column reads, scatter into the row images -----------------
  const int rpl     = p.rpl;
  const int cpi     = 32 / rpl;
  const int sub     = lane / rpl;
  const int lr      = lane - sub * rpl;
  const int ngroups = (rows + rpl - 1) / rpl;
  auto run_class    = [&](auto wtag, int k) {
    constexpr int W  = decltype(wtag)::value;
    const int nb     = p.class_begin[k];
    const int ne     = p.class_begin[k + 1];
    const int nslots = (ne - nb + cpi - 1) / cpi;
    const int total  = nslots * ngroups;
    for (int item = w; item < total; item += kTrWarps) {
      const int g    = item / nslots;
      const int slot = item - g * nslots;
      const int e    = nb + slot * cpi + sub;
      const int row  = g * rpl + lr;
      if (e < ne && row < rows) {
        const uint8_t* src = t.col_data[t.ent_col[e]] + (abs0 + row) * W;
        put_elem<W, SAFE>(rowptr(row) + t.ent_start[e], src);
      }
    }
  };
  run_class(std::integral_constant<int, 16>{}, 4);
  run_class(std::integral_constant<int, 8>{}, 3);
  run_class(std::integral_constant<int, 4>{}, 2);
  run_class(std::integral_constant<int, 2>{}, 1);
  run_class(std::integral_constant<int, 1>{}, 0);

  // ---- validity: column mask bits -> row validity bytes (bit c%8 of byte c/8, RC:764-773) -------
  const int nvb    = (p.ncols + 7) >> 3;
  const int ng32   = (rows + 31) >> 5;
  const int vitems = nvb * ng32;
  for (int item = w; item < vitems; item += kTrWarps) {
    const int g   = item / nvb;
    const int b   = item - g * nvb;
    const int row = g * 32 + lane;
    if (row < rows) {
      const int64_t ra = abs0 + row;
      uint32_t byte    = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int c = b * 8 + k;
        if (c < p.ncols) {
          const uint8_t* mb = t.mask_bytes[c];
          const uint32_t v  = mb ? ((__ldg(mb + (ra >> 3)) >> (ra & 7)) & 1u) : 1u;
          byte |= v << k;
        }
      }
      rowptr(row)[p.validity_offset + b] = static_cast<uint8_t>(byte);
    }
  }

  // ---- strings -------------------------------------------------------------------------------------
  if (p.nstr > 0) {
    const int nstr = p.nstr;
    const int nent = rows * nstr;
    // The per-tile string tables are laid out [string column][row] (index = s * rows + row): consecutive threads
    // touch consecutive words in every step.
    // S1: (src offset, len) of every (row, string column); threads run over rows => coalesced offsets
    for (int idx = tid; idx < nent; idx += kTrThreads) {
      const int s           = idx / rows;
      const int row         = idx - s * rows;
      const int32_t* so     = p.str_offsets[s] + abs0 + row;
      const int32_t o0      = __ldg(so);
      const int32_t o1      = __ldg(so + 1);
      t.str_src[idx]        = o0;
      t.str_len[idx]        = o1 - o0;
    }
    __syncthreads();
    // S2: thread per row: running offset across the row's string columns (RC:838-858), pairs into the row image.
    // (A warp per row with a 32-lane scan cost 66 warp instructions per ROW whatever the number of columns.)
    for (int row = tid; row < rows; row += kTrThreads) {
      uint32_t run = static_cast<uint32_t>(p.size_per_row);  // RC:838
      uint8_t* rp  = rowptr(row);
      for (int s = 0; s < nstr; ++s) {
        const int e        = s * rows + row;
        const uint32_t len = static_cast<uint32_t>(t.str_len[e]);
        t.str_dst[e]       = static_cast<int32_t>(run);
        uint8_t* pp        = rp + p.string_start[s];
        if constexpr (SAFE) {
#pragma unroll
          for (int i = 0; i < 4; ++i) { pp[i] = static_cast<uint8_t>(run >> (8 * i)); pp[4 + i] = static_cast<uint8_t>(len >> (8 * i)); }
        } else {
          reinterpret_cast<uint32_t*>(pp)[0] = run;  // RC:848
          reinterpret_cast<uint32_t*>(pp)[1] = len;  // RC:849
        }
        run += len;
      }
    }
    __syncthreads();
    // S3: chars.  Thread per (row, string): adjacent threads read adjacent strings of one column.
    for (int idx = tid; idx < nent; idx += kTrThreads) {
      const int s        = idx / rows;
      const int row      = idx - s * rows;
      const int32_t len  = t.str_len[idx];
      const uint8_t* src = p.str_chars[s] + t.str_src[idx];
      uint8_t* dst       = rowptr(row) + static_cast<uint32_t>(t.str_dst[idx]);
      for (int32_t i = 0; i < len; ++i) dst[i] = __ldg(src + i);
    }
  }
}

// SAFE tiles are rare: out of line, so their byte-wise code does not take registers from the fast path
__device__ __noinline__ void assemble_tile_safe(const ToRowsParams& p, const TrTables& t, uint8_t* base, const int32_t* s_off,
                                                int64_t stride, int64_t r, int rows, uint8_t* zero_base, int64_t zero_bytes)
{
  assemble_tile<true>(p, t, base, s_off, stride, r, rows, zero_base, zero_bytes);
}

__global__ void __launch_bounds__(kTrThreads, 4) to_rows_kernel(const __grid_constant__ ToRowsParams p)
{
  extern __shared__ __align__(128) uint8_t smem[];
  if (p.run_if != nullptr && *p.run_if == 0) return;  // the fast kernel ahead of this launch handled the batch
  const int stage_span = p.stage_bytes + kTrSlack;
  uint8_t* stage0      = smem;
  int32_t* s_off       = reinterpret_cast<int32_t*>(smem + static_cast<size_t>(p.nbuf) * stage_span);
  const int soff_span  = (p.tile_rows + 4) & ~3;
  TrHdr* hdr           = reinterpret_cast<TrHdr*>(s_off + soff_span);
  int32_t* s_ent_start = reinterpret_cast<int32_t*>(hdr + 1);
  int32_t* s_ent_col   = s_ent_start + p.nentries;
  const uint8_t** s_col_data   = reinterpret_cast<const uint8_t**>(s_ent_col + p.nentries + ((2 * p.nentries) & 1));
  const uint8_t** s_mask_bytes = s_col_data + p.ncols;
  int32_t* s_str_src           = reinterpret_cast<int32_t*>(s_mask_bytes + p.ncols);
  int32_t* s_str_len           = s_str_src + p.max_str_entries;
  int32_t* s_str_dst           = s_str_len + p.max_str_entries;

  const int tid  = threadIdx.x;
  const int lane = lane_id();
  for (int i = tid; i < p.nentries; i += kTrThreads) {
    s_ent_start[i] = p.entries[i].start;
    s_ent_col[i]   = p.entries[i].column;
  }
  for (int i = tid; i < p.ncols; i += kTrThreads) {
    s_col_data[i]   = static_cast<const uint8_t*>(p.col_data[i]);
    s_mask_bytes[i] = reinterpret_cast<const uint8_t*>(p.masks[i]);
  }
  __syncthreads();
  TrTables t{s_ent_start, s_ent_col, s_col_data, s_mask_bytes, s_str_src, s_str_len, s_str_dst};

  const int64_t c0   = static_cast<int64_t>(blockIdx.x) * p.rows_per_cta;
  const int64_t c1   = tmin(p.row_count, c0 + p.rows_per_cta);
  const bool fixed   = p.cum == nullptr;
  const bool base_ok = (reinterpret_cast<uintptr_t>(p.out_data) & 7) == 0;
  const uint64_t cum0 = (!fixed && p.row_start > 0) ? p.cum[p.row_start - 1] : 0;
  auto row_off = [&](int64_t i) -> int64_t {  // batch-relative byte offset of batch row i (i <= row_count)
    if (fixed) return i * p.row_stride;
    const int64_t a = p.row_start + i;
    return a == 0 ? 0 : static_cast<int64_t>(p.cum[a - 1] - cum0);
  };

  int64_t r = c0;
  for (int it = 0; r < c1; ++it) {
    uint8_t* stage = stage0 + static_cast<size_t>(p.nbuf == 2 ? (it & 1) : 0) * stage_span;
    // ---- A: tile geometry (warp 0) -------------------------------------------------------------
    if (tid == 0) {  // the store that last used this stage has drained
      if (p.nbuf == 2) tma_store_wait_read<1>();
      else tma_store_wait_read<0>();
    }
    if (warp_id() == 0) {
      int rows        = static_cast<int>(tmin<int64_t>(p.tile_rows, c1 - r));
      const int64_t lo = fixed ? row_off(r) : static_cast<int64_t>(p.out_offsets[r]);
      const int64_t base = lo - static_cast<int64_t>((reinterpret_cast<uintptr_t>(p.out_data) + lo) & 15);
      bool safe       = !base_ok;
      int64_t hi;
      if (fixed) {
        hi = lo + static_cast<int64_t>(rows) * p.row_stride;
        if (hi - lo > p.stage_bytes) safe = true;
        for (int i = lane; i < rows; i += 32) p.out_offsets[r + i] = static_cast<int32_t>(p.offset_bias + lo + static_cast<int64_t>(i) * p.row_stride);
      } else {
        // row offsets were written by batch_offsets_kernel: one coalesced read gives the whole tile geometry
        int fit = 0;
        for (int i0 = 0; i0 <= rows; i0 += 32) {
          const int i = i0 + lane;
          int64_t o   = 0;
          if (i <= rows) {
            o        = p.out_offsets[r + i];
            s_off[i] = static_cast<int32_t>(o - base);
          }
          const bool ok = (i >= 1) && (i <= rows) && (round_up64(o - base, 16) <= p.stage_bytes + 16);
          fit += __popc(__ballot_sync(0xffffffffu, ok));
        }
        if (fit < rows) fit &= ~7;
        if (p.max_str_entries < rows * p.nstr) fit = 0;
        __syncwarp();
        if (fit == 0 || safe) {
          safe = true;
          rows = tmin(rows, 8);
          while (rows > 1 && rows * p.nstr > p.max_str_entries) --rows;
          hi = static_cast<int64_t>(s_off[rows]) + base;
          __syncwarp();
          for (int i = lane; i <= rows; i += 32) s_off[i] = static_cast<int32_t>(s_off[i] + base - lo);
        } else {
          rows = fit;
          hi   = static_cast<int64_t>(s_off[rows]) + base;
        }
      }
      if (fixed && r + rows == p.row_count && lane == 0) p.out_offsets[p.row_count] = static_cast<int32_t>(p.offset_bias + hi);
      if (lane == 0) {
        hdr->r    = r;
        hdr->lo   = lo;
        hdr->hi   = hi;
        hdr->rows = rows;
        hdr->safe = safe ? 1 : 0;
        hdr->skew = static_cast<int32_t>(lo - base);
      }
    }
    __syncthreads();
    const TrHdr h = *hdr;
    // ---- B/C: assemble -------------------------------------------------------------------------
    if (!h.safe) {
      const int64_t zb = h.skew + (h.hi - h.lo);
      if (fixed)
        assemble_tile<false>(p, t, stage + h.skew, nullptr, p.row_stride, h.r, h.rows, stage, zb);
      else
        assemble_tile<false>(p, t, stage, s_off, 0, h.r, h.rows, stage, zb);
      fence_proxy_async();  // generic-proxy smem writes -> visible to the TMA store
      __syncthreads();
      // ---- D: write out ------------------------------------------------------------------------
      if (tid == 0) {
        const uintptr_t g_lo = reinterpret_cast<uintptr_t>(p.out_data) + h.lo;
        const uintptr_t g_hi = reinterpret_cast<uintptr_t>(p.out_data) + h.hi;
        const uintptr_t fl   = g_lo - h.skew;  // global address of stage byte 0
        const uintptr_t t_lo = (g_lo + 15) & ~uintptr_t{15};
        const uintptr_t t_hi = g_hi & ~uintptr_t{15};
        uintptr_t h_end      = tmin(t_lo, g_hi);
        uintptr_t t_beg      = tmax(t_hi, h_end);
        if (t_hi > t_lo) {
          tma_store_1d(reinterpret_cast<void*>(t_lo), stage + (t_lo - fl), static_cast<uint32_t>(t_hi - t_lo));
        } else {
          h_end = g_hi;
          t_beg = g_hi;
        }
        tma_store_commit();
        for (uintptr_t a = g_lo; a < h_end; a += 8)
          *reinterpret_cast<uint2*>(a) = *reinterpret_cast<const uint2*>(stage + (a - fl));
        for (uintptr_t a = t_beg; a < g_hi; a += 8)
          *reinterpret_cast<uint2*>(a) = *reinterpret_cast<const uint2*>(stage + (a - fl));
      }
    } else {
      if (fixed)
        assemble_tile_safe(p, t, p.out_data + h.lo, nullptr, p.row_stride, h.r, h.rows, p.out_data + h.lo, h.hi - h.lo);
      else
        assemble_tile_safe(p, t, p.out_data + h.lo, s_off, 0, h.r, h.rows, p.out_data + h.lo, h.hi - h.lo);
      __syncthreads();
    }
    r += h.rows;
  }
  if (tid == 0) tma_store_wait_read<0>();
}


// ==================================================================================================
// to_rows, fixed-width tables, full tiles: TMA in, TMA out.
//
//   producer warp : per tile of R rows, one TMA bulk load per column (lane = column) of the R values
//                   -- a contiguous, 16-byte aligned piece of the column -- into a staging ring;
//   consumer warps: lane = row.  unit = (column, 4 row groups): conflict-free LDS of 32 consecutive
//                   values from the staging piece, STS into the row images at the column's byte
//                   offset; column mask words (fetched with plain loads at the top of the tile so
//                   their latency hides behind the transpose) are bit-transposed by the 32x32
//                   butterfly into per-row validity bytes; the LIST offsets are written on the way;
//   one thread    : the finished row images -- ONE contiguous byte range of the output -- leave with
//                   a single 1-D TMA bulk store; images are double buffered.
// Padding bytes are zeroed once per CTA (the layout is static: no tile ever writes them again).
// Tails (< R rows), strings, unaligned buffers and very wide rows go to to_rows_kernel above.
// ==================================================================================================
constexpr int kT2Consumers = 11;
constexpr int kT2Threads   = (kT2Consumers + 1) * 32;
constexpr int kT2MaxStages = 3;
constexpr int kT2Super     = 4;  // consecutive tiles a CTA takes before the round-robin moves on (longer contiguous
                                 // pieces per column and per CTA: see the from_rows super-tiles)
__device__ __forceinline__ int64_t t2_first_tile() { return static_cast<int64_t>(blockIdx.x) * kT2Super; }
__device__ __forceinline__ int64_t t2_next_tile(int64_t tile)
{
  return ((tile + 1) % kT2Super) ? tile + 1 : tile + 1 + static_cast<int64_t>(gridDim.x - 1) * kT2Super;
}

struct ToRows2Params {
  const void* const* col_data;
  const uint32_t* const* masks;
  int64_t row_start;   // table row of the batch start
  int64_t num_tiles;   // full tiles to convert
  int32_t* out_offsets;
  uint8_t* out_data;
  int64_t offset_bias;
  int32_t write_last;  // 1: this launch covers the whole batch, also write out_offsets[row_count]
  int32_t ncols, nentries;
  int32_t validity_offset, row_stride;
  int32_t R;           // rows per tile (multiple of 32)
  int32_t nstages;
  int32_t data_bytes;  // sum of the column element sizes (bytes of staging per row)
  int32_t class_begin[kNumClasses + 1];
  int32_t cs, gpu;
  int32_t cls_units[kNumClasses];
  int32_t cls_ubase[kNumClasses];
  int32_t v_ubase;
  const Entry* entries;
  const int32_t* chunk_off;  // [nentries] byte offset of the entry's piece in a staging stage, per row unit (multiply by R)
};

__device__ __forceinline__ uint32_t transpose32_t(uint32_t r, int lane)
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

template <int W>
__device__ __forceinline__ void t2_class(const ToRows2Params& p, const int32_t* s_start, const int32_t* s_coff,
                                         uint32_t stage_s, uint32_t image_s, int ustart, int k, int lane)
{
  constexpr int B = W >= 16 ? 2 : 4;
  const int nb     = p.class_begin[k];
  const int total  = p.cls_units[k];
  const int gpu    = p.gpu;
  const int chmask = (1 << p.cs) - 1;
  for (int u = ustart; u < total; u += kT2Consumers) {
    const int e      = nb + (u >> p.cs);
    const int gc     = u & chmask;
    const int row    = gc * gpu * 32 + lane;
    uint32_t src     = stage_s + static_cast<uint32_t>(s_coff[e]) * p.R + row * W;
    uint32_t dst     = image_s + row * p.row_stride + s_start[e];
    const uint32_t dstep = 32u * p.row_stride;
    for (int gi = 0; gi < gpu; gi += B) {  // host guarantees gpu % 4 == 0
      uint32_t v[B][4];
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const uint32_t a = src + j * 32 * W;
        if constexpr (W == 1) asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v[j][0]) : "r"(a));
        else if constexpr (W == 2) asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v[j][0]) : "r"(a));
        else if constexpr (W == 4) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v[j][0]) : "r"(a));
        else if constexpr (W == 8) asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v[j][0]), "=r"(v[j][1]) : "r"(a));
        else asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[j][0]), "=r"(v[j][1]), "=r"(v[j][2]), "=r"(v[j][3]) : "r"(a));
      }
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const uint32_t a = dst + j * dstep;
        if constexpr (W == 1) asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v[j][0]));
        else if constexpr (W == 2) asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "r"(v[j][0]));
        else if constexpr (W == 4) asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v[j][0]));
        else if constexpr (W == 8) asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(v[j][0]), "r"(v[j][1]));
        else {  // rows are 8-byte aligned only
          asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(v[j][0]), "r"(v[j][1]));
          asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a + 8), "r"(v[j][2]), "r"(v[j][3]));
        }
      }
      src += B * 32 * W;
      dst += B * dstep;
    }
  }
}

__global__ void __launch_bounds__(kT2Threads, 1) to_rows2_kernel(const __grid_constant__ ToRows2Params p)
{
  extern __shared__ __align__(128) uint8_t smem[];
  const int NS           = p.nstages;
  const int stage_bytes  = p.R * p.data_bytes;             // multiple of 32
  const int image_bytes  = p.R * p.row_stride;             // multiple of 256
  uint8_t* stage0        = smem;
  uint8_t* image0        = smem + static_cast<size_t>(NS) * stage_bytes;
  uint64_t* full         = reinterpret_cast<uint64_t*>(image0 + 2 * static_cast<size_t>(image_bytes));
  uint64_t* empty        = full + kT2MaxStages;
  int32_t* s_start       = reinterpret_cast<int32_t*>(empty + kT2MaxStages);
  int32_t* s_coff        = s_start + p.nentries;
  const uint8_t** s_col  = reinterpret_cast<const uint8_t**>(s_coff + p.nentries + ((2 * p.nentries) & 1));
  const uint32_t** s_msk = reinterpret_cast<const uint32_t**>(s_col + p.nentries);
  int32_t* s_w           = reinterpret_cast<int32_t*>(s_msk + p.ncols);  // [nentries] element size

  const int tid  = threadIdx.x;
  const int lane = lane_id();
  for (int i = tid; i < p.nentries; i += kT2Threads) {
    s_start[i] = p.entries[i].start;
    s_coff[i]  = p.chunk_off[i];
    s_col[i]   = static_cast<const uint8_t*>(p.col_data[p.entries[i].column]);
    int w      = 1;
    for (int k = 0; k < kNumClasses; ++k)
      if (i >= p.class_begin[k] && i < p.class_begin[k + 1]) w = 1 << k;
    s_w[i] = w;
  }
  for (int i = tid; i < p.ncols; i += kT2Threads) s_msk[i] = p.masks[i];
  // zero both row images once: padding bytes are never written again
  {
    uint4* z        = reinterpret_cast<uint4*>(image0);
    const int n16   = (2 * image_bytes) >> 4;
    for (int i = tid; i < n16; i += kT2Threads) z[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();  // every thread orders its own zero fill before the later TMA stores
  }
  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kT2Consumers);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp_id() == 0) {
    // =================================== producer ===================================
    int it = 0;
    for (int64_t tile = t2_first_tile(); tile < p.num_tiles; tile = t2_next_tile(tile), ++it) {
      const int s        = it % NS;
      const uint32_t par = ((it / NS) & 1) ^ 1;
      if (lane == 0) {
        mbar_wait(&empty[s], par);
        mbar_arrive_expect_tx(&full[s], static_cast<uint32_t>(stage_bytes));
      }
      __syncwarp();
      uint8_t* st        = stage0 + static_cast<size_t>(s) * stage_bytes;
      const int64_t arow = p.row_start + tile * p.R;
      for (int e = lane; e < p.nentries; e += 32) {
        const int w = s_w[e];
        tma_load_1d(st + static_cast<size_t>(s_coff[e]) * p.R, s_col[e] + arow * w, static_cast<uint32_t>(p.R * w), &full[s]);
      }
    }
  } else {
    // =================================== consumers ===================================
    const int cw = warp_id() - 1;
    int ustart[kNumClasses];
#pragma unroll
    for (int k = 0; k < kNumClasses; ++k) ustart[k] = (cw + kT2Consumers - (p.cls_ubase[k] % kT2Consumers)) % kT2Consumers;
    const int vstart = (cw + kT2Consumers - (p.v_ubase % kT2Consumers)) % kT2Consumers;
    const int nq     = (p.ncols + 31) >> 5;
    const int nvb    = (p.ncols + 7) >> 3;
    const int ng32   = p.R >> 5;
    const int vitems = nq * ng32;
    int it = 0;
    for (int64_t tile = t2_first_tile(); tile < p.num_tiles; tile = t2_next_tile(tile), ++it) {
      const int s        = it % NS;
      const uint32_t par = (it / NS) & 1;
      const int b        = it & 1;
      const int64_t r0   = tile * p.R;             // batch-relative row
      const int64_t arow = p.row_start + r0;       // table row
      // mask words for this warp's validity items: issued now, consumed after the transpose
      uint32_t mw[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {  // static indices: the loads stay in flight until the words are used
        const int item = vstart + k * kT2Consumers;
        mw[k]          = 0;
        if (item < vitems) {
          const int g = nq == 1 ? item : item / nq;
          const int q = nq == 1 ? 0 : item - g * nq;
          const int c = q * 32 + lane;
          if (c < p.ncols) {
            const uint32_t* mp = s_msk[c];
            mw[k]              = mp ? __ldg(mp + ((arow >> 5) + g)) : 0xffffffffu;
          }
        }
      }
      mbar_wait(&full[s], par);
      const uint32_t stage_s = smem_u32(stage0 + static_cast<size_t>(s) * stage_bytes);
      const uint32_t image_s = smem_u32(image0 + static_cast<size_t>(b) * image_bytes);
      t2_class<16>(p, s_start, s_coff, stage_s, image_s, ustart[4], 4, lane);
      t2_class<8>(p, s_start, s_coff, stage_s, image_s, ustart[3], 3, lane);
      t2_class<4>(p, s_start, s_coff, stage_s, image_s, ustart[2], 2, lane);
      t2_class<2>(p, s_start, s_coff, stage_s, image_s, ustart[1], 1, lane);
      t2_class<1>(p, s_start, s_coff, stage_s, image_s, ustart[0], 0, lane);
      // validity
      {
        int k = 0;
        for (int item = vstart; item < vitems; item += kT2Consumers, ++k) {
          const int g = nq == 1 ? item : item / nq;
          const int q = nq == 1 ? 0 : item - g * nq;
          uint32_t w;
          if (k < 4) {
            w = k == 0 ? mw[0] : k == 1 ? mw[1] : k == 2 ? mw[2] : mw[3];
          } else {
            const int c = q * 32 + lane;
            w           = 0;
            if (c < p.ncols) {
              const uint32_t* mp = s_msk[c];
              w                  = mp ? __ldg(mp + ((arow >> 5) + g)) : 0xffffffffu;
            }
          }
          const uint32_t bits = transpose32_t(w, lane);   // lane = row g*32+lane, bit = column 32q + bit
          const uint32_t a    = image_s + (g * 32 + lane) * p.row_stride + p.validity_offset + 4 * q;
          const int nbv       = tmin(4, nvb - 4 * q);
          if (nbv == 4 && ((p.validity_offset & 3) == 0)) {
            asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(bits));
          } else {
            for (int i = 0; i < nbv; ++i) asm volatile("st.shared.u8 [%0], %1;" ::"r"(a + i), "r"(bits >> (8 * i)));
          }
        }
      }
      // LIST offsets of the tile's rows
      for (int i = cw * 32 + lane; i < p.R; i += kT2Consumers * 32)
        p.out_offsets[r0 + i] = static_cast<int32_t>(p.offset_bias + (r0 + i) * p.row_stride);
      if (p.write_last && tile == p.num_tiles - 1 && cw == 0 && lane == 0)
        p.out_offsets[r0 + p.R] = static_cast<int32_t>(p.offset_bias + (r0 + p.R) * p.row_stride);
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      named_bar_sync(1, kT2Consumers * 32);  // every consumer has finished writing image b
      if (cw == 0 && lane == 0) {
        tma_store_1d(p.out_data + r0 * p.row_stride, image0 + static_cast<size_t>(b) * image_bytes,
                     static_cast<uint32_t>(image_bytes));
        tma_store_commit();
        tma_store_wait_read<1>();  // the store of the previous tile (other image) has drained
      }
      named_bar_sync(2, kT2Consumers * 32);  // the other image is free for the next tile
    }
    if (cw == 0 && lane == 0) tma_store_wait_read<0>();
  }
}

// ---- row sizes: round_up(size_per_row + sum(len), 8), inclusive scan (RC:201-257, 1490-1491) -------
// v1: per-row sizes by a simple kernel, then the same three-step scan structure (uint64).
constexpr int kRsThreads = 256;
constexpr int kRsChunk   = 4096;

__global__ void __launch_bounds__(kRsThreads) row_sizes_kernel(const int32_t* const* str_offsets, int nstr,
                                                                int32_t size_per_row, int64_t n, uint64_t* sizes)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kRsThreads + threadIdx.x;
  if (i >= n) return;
  uint64_t s = 0;
  for (int c = 0; c < nstr; ++c) {
    const int32_t* o = str_offsets[c] + i;
    s += static_cast<uint64_t>(static_cast<uint32_t>(__ldg(o + 1) - __ldg(o)));
  }
  sizes[i] = (static_cast<uint64_t>(size_per_row) + s + 7) & ~uint64_t{7};
}

__global__ void __launch_bounds__(kRsThreads) u64_partials_kernel(const uint64_t* v, int64_t n, uint64_t* partials)
{
  __shared__ uint64_t s_w[kRsThreads / 32];
  const int64_t beg = static_cast<int64_t>(blockIdx.x) * kRsChunk;
  const int64_t end = tmin(n, beg + kRsChunk);
  uint64_t acc      = 0;
  for (int64_t i = beg + threadIdx.x; i < end; i += kRsThreads) acc += v[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if (lane_id() == 0) s_w[warp_id()] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t t = 0;
    for (int i = 0; i < kRsThreads / 32; ++i) t += s_w[i];
    partials[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kRsThreads) u64_scan_chunks_kernel(uint64_t* partials, int nchunks)
{
  __shared__ uint64_t s_w[kRsThreads / 32];
  __shared__ uint64_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < nchunks; base += kRsThreads) {
    const int i      = base + threadIdx.x;
    const uint64_t v = i < nchunks ? partials[i] : 0;
    uint64_t x       = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane_id() >= o) x += y;
    }
    if (lane_id() == 31) s_w[warp_id()] = x;
    __syncthreads();
    uint64_t wpre = 0;
    for (int w = 0; w < warp_id(); ++w) wpre += s_w[w];
    const uint64_t carry = s_carry;
    if (i < nchunks) partials[i] = carry + wpre + x - v;
    __syncthreads();
    if (threadIdx.x == kRsThreads - 1) s_carry = carry + wpre + x;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kRsThreads) u64_scan_apply_kernel(uint64_t* v, int64_t n, const uint64_t* partials)
{
  __shared__ uint64_t s_w[kRsThreads / 32];
  __shared__ uint64_t s_carry;
  if (threadIdx.x == 0) s_carry = partials[blockIdx.x];
  __syncthreads();
  const int64_t beg = static_cast<int64_t>(blockIdx.x) * kRsChunk;
  const int64_t end = tmin(n, beg + kRsChunk);
  for (int64_t base = beg; base < end; base += kRsThreads) {
    const int64_t i  = base + threadIdx.x;
    const uint64_t a = i < end ? v[i] : 0;
    uint64_t x       = a;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane_id() >= o) x += y;
    }
    if (lane_id() == 31) s_w[warp_id()] = x;
    __syncthreads();
    uint64_t wpre = 0;
    for (int w = 0; w < warp_id(); ++w) wpre += s_w[w];
    const uint64_t carry = s_carry;
    if (i < end) v[i] = carry + wpre + x;
    __syncthreads();
    if (threadIdx.x == kRsThreads - 1) s_carry = carry + wpre + x;
    __syncthreads();
  }
}

// batch-relative LIST offsets of a batch: offsets[i] = cum[row_start + i - 1] - cum[row_start - 1]
__global__ void __launch_bounds__(kRsThreads) batch_offsets_kernel(const uint64_t* __restrict__ cum, int64_t row_start,
                                                                    int64_t row_count, int32_t* __restrict__ offsets)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kRsThreads + threadIdx.x;
  if (i > row_count) return;
  const uint64_t c0 = row_start > 0 ? cum[row_start - 1] : 0;
  const int64_t a   = row_start + i;
  offsets[i]        = static_cast<int32_t>(a == 0 ? 0 : cum[a - 1] - c0);
}

// d_cum_sizes: uint64[num_rows] followed by uint64[nchunks] scratch (see srj_to_rows_workspace_bytes)
int launch_row_sizes(const srj_plan* plan, const int32_t* const* d_str_offsets, int64_t num_rows,
                     uint64_t* d_cum_sizes, cudaStream_t stream)
{
  if (num_rows == 0) return SRJ_OK;
  const int nchunks  = static_cast<int>((num_rows + kRsChunk - 1) / kRsChunk);
  uint64_t* partials = d_cum_sizes + num_rows;
  row_sizes_kernel<<<static_cast<unsigned>((num_rows + kRsThreads - 1) / kRsThreads), kRsThreads, 0, stream>>>(
    d_str_offsets, plan->num_string_columns, plan->size_per_row, num_rows, d_cum_sizes);
  u64_partials_kernel<<<nchunks, kRsThreads, 0, stream>>>(d_cum_sizes, num_rows, partials);
  u64_scan_chunks_kernel<<<1, kRsThreads, 0, stream>>>(partials, nchunks);
  u64_scan_apply_kernel<<<nchunks, kRsThreads, 0, stream>>>(d_cum_sizes, num_rows, partials);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// build_batches (RC:1466-1557) on the device: one thread walks the inclusive cumulative row sizes and cuts a new batch
// wherever the bytes would pass INT32_MAX, on a 32-row boundary (a binary search per batch); the host reads the result
// with ONE copy (the reference does a thrust::lower_bound + D2H per batch, RC:1500-1544).
// out[0] = number of batches (or -1: a single row exceeds 2 GiB, -2: more than max_batches), then {row_start, row_count,
// num_bytes} triples.
__global__ void batch_cut_kernel(const uint64_t* __restrict__ cum, int64_t n, int32_t max_batches, int64_t* __restrict__ out)
{
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const uint64_t MAXB = INT32_MAX;  // MAX_BATCH_SIZE, RC:65
  const uint64_t total = cum[n - 1];
  int64_t last = 0, nb = 0;
  uint64_t cum_last = 0;  // cum[last - 1]
  while (last < n) {
    int64_t row_end;
    if (total - cum_last < MAXB) {
      row_end = n;  // everything left fits one batch
    } else {
      // first i with cum[i] - cum[last] >= MAXB (the reference's lower_bound ignores the first row of the batch; the
      // guard below covers the overshoot that can cause)
      const uint64_t cl = cum[last];
      int64_t lo = last, hi = n;
      while (lo < hi) {
        const int64_t mid = lo + (hi - lo) / 2;
        if (cum[mid] - cl < MAXB) lo = mid + 1; else hi = mid;
      }
      const int64_t bs = lo - last;
      row_end          = (lo == n) ? last + bs : last + bs / 32 * 32;
    }
    uint64_t cend = 0;
    for (;;) {
      if (row_end <= last) { out[0] = -1; return; }
      cend = cum[row_end - 1];
      if (cend - cum_last <= MAXB) break;
      const int64_t m = row_end - last;
      row_end -= (m % 32) ? (m % 32) : 32;
    }
    if (nb >= max_batches) { out[0] = -2; return; }
    out[1 + 3 * nb] = last;
    out[2 + 3 * nb] = row_end - last;
    out[3 + 3 * nb] = static_cast<int64_t>(cend - cum_last);
    ++nb;
    last     = row_end;
    cum_last = cend;
  }
  out[0] = nb;
}

int launch_batch_cut(const uint64_t* d_cum, int64_t num_rows, int32_t max_batches, int64_t* d_out, cudaStream_t stream)
{
  batch_cut_kernel<<<1, 32, 0, stream>>>(d_cum, num_rows, max_batches, d_out);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static size_t to_rows_smem_bytes(const srj_plan* plan, int tile_rows, int stage_bytes, int max_str_entries, int nbuf)
{
  const int nent = static_cast<int>(plan->tr_entries.size());
  size_t b       = static_cast<size_t>(nbuf) * static_cast<size_t>(stage_bytes + kTrSlack);
  b += static_cast<size_t>((tile_rows + 4) & ~3) * 4;
  b += sizeof(TrHdr);
  b += static_cast<size_t>(2 * nent + ((2 * nent) & 1)) * 4;
  b += static_cast<size_t>(plan->num_columns) * 16;
  b += static_cast<size_t>(max_str_entries) * 12;
  return (b + 127) & ~size_t{127};
}

static int launch_to_rows_generic(const srj_plan* plan, const void* const* d_col_data, const uint32_t* const* d_masks,
                                  const int32_t* const* d_str_offsets, const uint8_t* const* d_str_chars,
                                  int64_t row_start, int64_t row_count, const uint64_t* d_cum_sizes,
                                  int32_t* out_offsets, uint8_t* out_data, int64_t out_bytes, int64_t offset_bias,
                                  cudaStream_t stream, const int32_t* run_if = nullptr, bool write_offsets = true);

// static unit schedule shared by the two directions (see from_rows.cu)
static void t2_schedule(ToRows2Params& p)
{
  const int ngroups = p.R / 32;
  int slots         = 0;
  for (int k = 0; k < kNumClasses; ++k) slots += p.class_begin[k + 1] - p.class_begin[k];
  int cs = 0;
  while ((slots << cs) < 96 && (ngroups % (8 << cs)) == 0) ++cs;
  p.cs  = cs;
  p.gpu = (ngroups + (1 << cs) - 1) >> cs;
  int ub = 0;
  for (int k = kNumClasses - 1; k >= 0; --k) {
    p.cls_ubase[k] = ub;
    p.cls_units[k] = (p.class_begin[k + 1] - p.class_begin[k]) << cs;
    ub += p.cls_units[k];
  }
  p.v_ubase = ub;
}

int launch_to_rows(const srj_plan* plan, const void* const* d_col_data, const uint32_t* const* d_masks,
                   const int32_t* const* d_str_offsets, const uint8_t* const* d_str_chars, int64_t row_start,
                   int64_t row_count, const uint64_t* d_cum_sizes, int32_t* out_offsets, uint8_t* out_data,
                   int64_t out_bytes, cudaStream_t stream, const void* const* h_col_data, int32_t* d_fail_flag)
{
  if (row_count == 0) return SRJ_OK;
  // ---- wide variable-width rows: to_rows3_kernel (to_rows_var.cu), generic kernel behind it as the fallback ----
  if (plan->num_string_columns > 0 && d_cum_sizes != nullptr) {
    batch_offsets_kernel<<<static_cast<unsigned>((row_count + 1 + kRsThreads - 1) / kRsThreads), kRsThreads, 0, stream>>>(
      d_cum_sizes, row_start, row_count, out_offsets);
    int launched = 0;
    const int rc = launch_to_rows_var(plan, d_col_data, d_masks, d_str_offsets, d_str_chars, row_start, row_count, out_offsets,
                                      out_data, out_bytes, d_fail_flag, stream, h_col_data, &launched);
    if (rc != SRJ_OK) return rc;
    return launch_to_rows_generic(plan, d_col_data, d_masks, d_str_offsets, d_str_chars, row_start, row_count, d_cum_sizes,
                                  out_offsets, out_data, out_bytes, 0, stream, launched ? d_fail_flag : nullptr, false);
  }
  // ---- fast kernel: fixed-width tables, full tiles, 16-byte aligned buffers ------------------------
  const int S = plan->fixed_row_size;
  int D       = 0;
  for (int sz : plan->col_size) D += sz;
  bool fast = plan->num_string_columns == 0 && plan->d_tr_chunk_off != nullptr;
  int R = 0, NS = 3;
  if (fast) {
    // smem: NS staging stages of R*D bytes + 2 row images of R*S bytes (+ tables)
    const int tables = static_cast<int>(plan->tr_entries.size()) * 28 + plan->num_columns * 8 + 1024;
    const int budget = 225 * 1024 - tables;
    R                = budget / (NS * D + 2 * S) / 128 * 128;
    if (R < 128) { NS = 2; R = budget / (NS * D + 2 * S) / 32 * 32; }
    if (R > 512) R = 512;
    if (R >= 128) R = R / 128 * 128;
    fast = R >= 128 && row_count >= R && (reinterpret_cast<uintptr_t>(out_data) & 15) == 0 && (row_start % 32) == 0;
    if (fast && h_col_data)
      for (int c = 0; c < plan->num_columns && fast; ++c) fast = (reinterpret_cast<uintptr_t>(h_col_data[c]) & 15) == 0;
    else
      fast = false;
  }
  int64_t done = 0;
  if (fast) {
    ToRows2Params p{};
    p.col_data        = d_col_data;
    p.masks           = d_masks;
    p.row_start       = row_start;
    p.num_tiles       = row_count / R;
    p.out_offsets     = out_offsets;
    p.out_data        = out_data;
    p.offset_bias     = 0;
    p.write_last      = (row_count % R) == 0;
    p.ncols           = plan->num_columns;
    p.nentries        = static_cast<int32_t>(plan->tr_entries.size());
    p.validity_offset = plan->validity_offset;
    p.row_stride      = S;
    p.R               = R;
    p.nstages         = NS;
    p.data_bytes      = D;
    for (int k = 0; k <= kNumClasses; ++k) p.class_begin[k] = plan->tr_class_begin[k];
    p.entries   = plan->d_tr_entries;
    p.chunk_off = plan->d_tr_chunk_off;
    t2_schedule(p);
    int dev = 0, nsm = 0;
    SRJ_CUDA_TRY(cudaGetDevice(&dev));
    SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
    const int64_t grid = std::min<int64_t>(nsm, (p.num_tiles + kT2Super - 1) / kT2Super);
    size_t smem        = static_cast<size_t>(NS) * R * D + 2 * static_cast<size_t>(R) * S + 2 * kT2MaxStages * 8;
    smem += static_cast<size_t>(p.nentries) * (4 + 4 + 8 + 4) + 8 + static_cast<size_t>(p.ncols) * 8 + 64;
    smem = (smem + 127) & ~size_t{127};
    SRJ_CUDA_TRY(cudaFuncSetAttribute(to_rows2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    to_rows2_kernel<<<static_cast<unsigned>(grid), kT2Threads, smem, stream>>>(p);
    SRJ_CUDA_TRY(cudaGetLastError());
    done = p.num_tiles * R;
    if (done == row_count) return SRJ_OK;
  }
  // ---- generic kernel: everything else, and the tail rows of a fast launch ---------------------------
  return launch_to_rows_generic(plan, d_col_data, d_masks, d_str_offsets, d_str_chars, row_start + done, row_count - done,
                                d_cum_sizes, out_offsets + done, out_data + done * S * (plan->num_string_columns == 0 ? 1 : 0),
                                out_bytes, done * S, stream);
}

static int launch_to_rows_generic(const srj_plan* plan, const void* const* d_col_data, const uint32_t* const* d_masks,
                                  const int32_t* const* d_str_offsets, const uint8_t* const* d_str_chars,
                                  int64_t row_start, int64_t row_count, const uint64_t* d_cum_sizes,
                                  int32_t* out_offsets, uint8_t* out_data, int64_t out_bytes, int64_t offset_bias,
                                  cudaStream_t stream, const int32_t* run_if, bool write_offsets)
{
  if (row_count == 0) return SRJ_OK;
  ToRowsParams p{};
  p.run_if          = run_if;
  p.col_data        = d_col_data;
  p.masks           = d_masks;
  p.str_offsets     = d_str_offsets;
  p.str_chars       = d_str_chars;
  p.cum             = d_cum_sizes;
  p.row_start       = row_start;
  p.row_count       = row_count;
  p.out_offsets     = out_offsets;
  p.out_data        = out_data;
  p.out_bytes       = out_bytes;
  p.ncols           = plan->num_columns;
  p.nstr            = plan->num_string_columns;
  p.validity_offset = plan->validity_offset;
  p.size_per_row    = plan->size_per_row;
  p.row_stride      = plan->fixed_row_size;
  p.nentries        = static_cast<int32_t>(plan->tr_entries.size());
  for (int k = 0; k <= kNumClasses; ++k) p.class_begin[k] = plan->tr_class_begin[k];
  p.entries      = plan->d_tr_entries;
  p.string_cols  = plan->d_string_cols;
  p.string_start = plan->d_string_start;
  p.offset_bias  = offset_bias;

  // generic-kernel tiling.  The kernel is bound by the latency of its (synchronous) global reads, so it wants
  // many resident CTAs rather than deep buffering: variable-width tables use ONE 40 KB stage per CTA
  // (4-5 CTAs per SM); fixed-width tails keep two 48 KB stages.
  const bool var        = plan->num_string_columns > 0;
  int stage_bytes       = (var ? 44 : 48) * 1024;
  int nbuf              = var ? 1 : 2;
  int tile_rows         = (stage_bytes / plan->fixed_row_size) / 32 * 32;
  if (tile_rows > 512) tile_rows = 512;
  if (tile_rows < 32) tile_rows = (stage_bytes / plan->fixed_row_size) >= 16 ? 16 : 8;
  int max_str = 0;
  if (p.nstr > 0) {
    // cap the per-tile string tables at 2048 (row, string) entries
    while (tile_rows > 8 && tile_rows * p.nstr > 2048) tile_rows = tile_rows > 32 ? tile_rows - 32 : tile_rows / 2;
    max_str = std::min(tile_rows * p.nstr, 2048);
    if (max_str < p.nstr) max_str = p.nstr;  // at least one row (SAFE path walks row by row)
    if (max_str > 8192) return (set_error("to_rows: more than 8192 STRING columns is not supported"), SRJ_EUNSUPPORTED);
  }
  p.nbuf            = nbuf;
  if (d_cum_sizes && write_offsets)
    batch_offsets_kernel<<<static_cast<unsigned>((row_count + 1 + kRsThreads - 1) / kRsThreads), kRsThreads, 0, stream>>>(
      d_cum_sizes, row_start, row_count, out_offsets);
  p.tile_rows       = tile_rows;
  p.rpl             = tile_rows >= 32 ? 32 : tile_rows;
  p.stage_bytes     = stage_bytes;
  p.max_str_entries = max_str;

  int dev = 0, nsm = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  const int64_t T      = tile_rows;
  const int64_t ntiles = (row_count + T - 1) / T;
  size_t smem          = to_rows_smem_bytes(plan, tile_rows, stage_bytes, max_str, nbuf);
  // very wide schemas: the per-schema tables (entry starts, column pointers) come on top of the stages -- give up the
  // second stage, then stage height, before giving up
  while (smem > 232448 && (p.nbuf > 1 || p.stage_bytes > 16 * 1024)) {
    if (p.nbuf > 1) p.nbuf = nbuf = 1;
    else {
      p.stage_bytes = stage_bytes = stage_bytes / 2;
      tile_rows     = std::max(8, std::min(tile_rows, (stage_bytes / plan->fixed_row_size) / 8 * 8));
      p.tile_rows   = tile_rows;
      p.rpl         = tile_rows >= 32 ? 32 : tile_rows;
      if (p.nstr > 0) p.max_str_entries = max_str = std::max(p.nstr, std::min(tile_rows * p.nstr, 2048));
    }
    smem = to_rows_smem_bytes(plan, tile_rows, stage_bytes, max_str, nbuf);
  }
  if (smem > 232448) {
    set_error("to_rows: schema too wide for the kernel's shared-memory tables (%d columns need %zu bytes)", plan->num_columns, smem);
    return SRJ_EUNSUPPORTED;
  }
  const int per_sm     = std::max<int>(1, std::min<int>(8, static_cast<int>((228 * 1024) / (smem + 1024))));
  int64_t grid         = std::min<int64_t>(static_cast<int64_t>(nsm) * per_sm, ntiles);
  const int64_t per    = (ntiles + grid - 1) / grid;
  p.rows_per_cta       = per * T;
  grid                 = (row_count + p.rows_per_cta - 1) / p.rows_per_cta;
  SRJ_CUDA_TRY(cudaFuncSetAttribute(to_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
  to_rows_kernel<<<static_cast<unsigned>(grid), kTrThreads, smem, stream>>>(p);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj
