// from_rows.cu -- JCUDF rows -> columns (reference: convert_from_rows, RC:2149-2441).
//
// One persistent, warp-specialised kernel replaces copy_from_rows + copy_validity_from_rows +
// fixup_null_counts (RC:879-969, 987-1094, 2130-2136):
//
//   producer warp : walks the CTA's contiguous row range tile by tile; each tile is ONE contiguous
//                   byte range of the row buffer, moved global->shared by a single 1-D TMA bulk copy
//                   (cp.async.bulk ... mbarrier::complete_tx) into a multi-stage ring, so ~2 stages
//                   (>=100 KB) per SM are always in flight with no registers or LSU slots spent.
//   consumer warps: lane = row.  A work unit is (field, chunk of row groups): a few shared-memory
//                   reads of one field of 32 consecutive rows, batched for ILP, then coalesced
//                   st.global stores into the column; validity bytes are bit-transposed with
//                   __ballot_sync into the column masks; null counts are popc'd on the way.
//
// The unit -> (field, chunk) map is a shift/mask of host-computed constants; full tiles of
// fixed-stride tables run a predicate-free instantiation.  Rows whose tile cannot be staged (row
// larger than a stage, unaligned buffers) take the SAFE path: same code, reading global memory
// byte-wise.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "kernels.hpp"
#include "movers.cuh"
#include "plan.hpp"

namespace srj {

constexpr int kMaxStages  = 4;
constexpr int kStageSlack = 32;  // skew (<=8) + tail

struct StageHdr {
  int64_t r0;     // first table row of the tile
  int32_t rows;   // 0 = end of this CTA's range
  int32_t safe;   // 1 = not staged: read rows from global memory byte-wise
  int32_t skew;   // payload byte offset of global byte `gbase` (fixed-stride tiles)
  int32_t pad;
  int64_t gbase;  // global byte offset (from p.rows) that payload[skew] corresponds to
};

struct FromRowsParams {
  const uint8_t* rows;
  const int32_t* row_offsets;  // NULL => fixed stride
  int64_t rows_bytes;
  int64_t num_rows;
  int64_t super_rows;  // rows per super-tile; super-tiles are dealt round-robin to the CTAs
  int32_t ncols;
  int32_t validity_offset;
  int32_t row_stride;
  int32_t tile_rows;
  int32_t rpl;  // rows per item: 8, 16 or 32
  int32_t stage_bytes;
  int32_t nstages;
  int32_t nentries;
  int32_t class_begin[kNumClasses + 1];
  // static work schedule (host-computed): a unit = (entry slot, chunk of `gpu` row groups)
  int32_t cs;                      // log2(chunks per slot)
  int32_t gpu;                     // row groups per unit
  int32_t cls_units[kNumClasses];  // units of each width class  (= slots << cs)
  int32_t cls_ubase[kNumClasses];  // units before this class (balances warps across classes)
  int32_t v_ubase;                 // units before the validity items
  const Entry* entries;
  void* const* ent_dst;             // [nentries] column base pointers (STRING: offsets + 1)
  uint32_t* const* masks;           // [ncols]
  unsigned long long* null_counts;  // [ncols] or NULL
  // canonical-layout check of the STRING pairs (variable-width tables)
  int32_t nstr;
  int32_t size_per_row;
  const int32_t* string_start;   // [nstr] row byte offset of each (offset, len) pair
  unsigned long long* status;    // bit 0 <- 1 when a row's pair.offset differs from the canonical position
};

template <bool SAFE>
__device__ __forceinline__ uint64_t load_key(const uint8_t* p, int sz)
{
  if constexpr (SAFE) {
    uint64_t v = 0;
    for (int i = 0; i < sz; ++i) v |= static_cast<uint64_t>(p[i]) << (8 * i);
    return v;
  } else {
    switch (sz) {
      case 1: return *p;
      case 2: return *reinterpret_cast<const uint16_t*>(p);
      case 4: return *reinterpret_cast<const uint32_t*>(p);
      default: {
        const uint2 a = *reinterpret_cast<const uint2*>(p);
        return static_cast<uint64_t>(a.x) | (static_cast<uint64_t>(a.y) << 32);
      }
    }
  }
}

// Shared-memory resident copies of the schedule (filled once per CTA).
struct SmemTables {
  const int32_t* ent_start;  // [nentries]
  uint8_t* const* ent_dst;   // [nentries]
  uint32_t* const* masks;    // [ncols]
  int32_t* nulls;            // [ncols] or NULL
  const int32_t* string_start;  // [nstr]
};

// Per-consumer-warp schedule constants, computed once per CTA.
struct WarpSched {
  int ustart[kNumClasses];  // first unit of each width class for this warp
  int vstart;               // first validity item for this warp
  int vdq, vdg;             // NCW = vdg * nq + vdq  (validity item stepping without a division)
  int sub, lr;              // lane -> (entry within slot, row within group)
};

// Where the rows of a tile are: base + s_off[i] (VAR) or base + i * stride.
struct TileView {
  const uint8_t* base;
  const int32_t* s_off;
  uint32_t stride;
  int64_t r0;
  int rows;
  const uint8_t* lane_row;  // single-row-group tiles: this lane's row (NULL if lane >= rows)
};

template <bool VAR>
__device__ __forceinline__ const uint8_t* row_ptr(const TileView& tv, int i)
{
  if constexpr (VAR) return tv.base + static_cast<uint32_t>(tv.s_off[i]);
  else return tv.base + static_cast<uint32_t>(i) * tv.stride;
}

// ---- fixed-width fields of one width class -----------------------------------------------------------
// PRED=false: full tile of a fixed-stride table -- no row predicates at all.
template <int W, int NCW, int RPL, bool VAR, bool PRED, bool SAFE, bool ONEG>
__device__ __forceinline__ void transpose_class(const FromRowsParams& p, const SmemTables& t, const WarpSched& ws,
                                                const TileView& tv, int k)
{
  constexpr int CPI = 32 / RPL;
  constexpr int B   = W >= 16 ? 2 : 4;  // loads in flight per lane before the stores
  const int nb      = p.class_begin[k];
  const int ne      = p.class_begin[k + 1];
  const int total   = p.cls_units[k];
  const int gpu     = p.gpu;
  const int chmask  = (1 << p.cs) - 1;
  if constexpr (VAR && !SAFE && ONEG) {
    {
      // wide rows: one row group per tile; the lane's row address is hoisted per tile and four units are
      // in flight per warp (table reads, then field reads, then stores) to hide the shared-memory latency
      const int64_t roff = (tv.r0 + ws.lr) * W;
      constexpr int U    = 2;
      for (int u = ws.ustart[k]; u < total; u += U * NCW) {
        Reg<W> v[U];
        uint8_t* dst[U];
        bool ok[U];
        int32_t start[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int uj = u + j * NCW;
          const int e  = nb + (uj >> p.cs) * CPI + ws.sub;
          ok[j]        = uj < total && e < ne && tv.lane_row != nullptr;
          if (ok[j]) {
            start[j] = t.ent_start[e];
            dst[j]   = t.ent_dst[e] + roff;
          }
        }
#pragma unroll
        for (int j = 0; j < U; ++j)
          if (ok[j]) v[j] = ld_elem<W, false>(tv.lane_row + start[j]);
#pragma unroll
        for (int j = 0; j < U; ++j)
          if (ok[j]) st_elem<W>(dst[j], v[j]);
      }
      return;
    }
  }
  for (int u = ws.ustart[k]; u < total; u += NCW) {
    const int slot = u >> p.cs;
    const int gc   = u & chmask;
    const int e    = nb + slot * CPI + ws.sub;
    if (CPI > 1 && e >= ne) continue;
    const int32_t start = t.ent_start[e];
    int row             = gc * gpu * RPL + ws.lr;
    uint8_t* dst        = t.ent_dst[e] + (tv.r0 + row) * W;
    if constexpr (!VAR && !PRED) {
      const uint8_t* src     = tv.base + static_cast<uint32_t>(row) * tv.stride + start;
      const uint32_t gstride = RPL * tv.stride;
      for (int gi = 0; gi < gpu; gi += B) {  // host guarantees gpu % B == 0 for this instantiation
        Reg<W> v[B];
#pragma unroll
        for (int j = 0; j < B; ++j) v[j] = ld_elem<W, false>(src + j * gstride);
#pragma unroll
        for (int j = 0; j < B; ++j) st_elem<W>(dst + j * RPL * W, v[j]);
        src += B * gstride;
        dst += B * RPL * W;
      }
    } else {
      for (int gi = 0; gi < gpu; gi += B) {
        Reg<W> v[B];
        bool ok[B];
#pragma unroll
        for (int j = 0; j < B; ++j) {
          const int rj = row + j * RPL;
          ok[j]        = (gi + j < gpu) && (rj < tv.rows);
          if (ok[j]) v[j] = ld_elem<W, SAFE>(row_ptr<VAR>(tv, rj) + start);
        }
#pragma unroll
        for (int j = 0; j < B; ++j)
          if (ok[j]) st_elem<W>(dst + j * RPL * W, v[j]);
        row += B * RPL;
        dst += B * RPL * W;
      }
    }
  }
}

template <int NCW, bool VAR, bool PRED, bool SAFE>
__device__ __forceinline__ void validity_tile(const FromRowsParams& p, const SmemTables& t, const WarpSched& ws,
                                              const TileView& tv)
{
  const int lane   = lane_id();
  const int nvb    = (p.ncols + 7) >> 3;
  const int nq     = (p.ncols + 31) >> 5;  // groups of 32 columns
  const int ng32   = (tv.rows + 31) >> 5;
  const int vitems = nq * ng32;
  if (ws.vstart >= vitems) return;
  int g = 0, q = ws.vstart;
  if (ng32 > 1) {  // one division per tile; then incremental
    g = ws.vstart / nq;
    q = ws.vstart - g * nq;
  }
  for (int item = ws.vstart; item < vitems; item += NCW) {
    const int row = g * 32 + lane;
    uint32_t r    = 0;
    if (!PRED || row < tv.rows) {
      const uint8_t* vp = row_ptr<VAR>(tv, row) + p.validity_offset + 4 * q;
      const int nbv     = tmin(4, nvb - 4 * q);
      if (!SAFE && nbv == 4 && ((p.validity_offset & 3) == 0)) {
        r = *reinterpret_cast<const uint32_t*>(vp);  // rows are 8-byte aligned
      } else {
        for (int i = 0; i < nbv; ++i) r |= static_cast<uint32_t>(vp[i]) << (8 * i);
      }
    }
    const uint32_t mine = transpose32(r, lane);  // lane = column 32q + lane, bit = row
    const int col       = q * 32 + lane;
    if (col < p.ncols) {
      const int64_t rg = tv.r0 + g * 32;  // multiple of 8 (of 32 when !PRED)
      uint8_t* mp      = reinterpret_cast<uint8_t*>(t.masks[col]) + (rg >> 3);
      if constexpr (!PRED) {
        const int nnull = __popc(~mine);
        if (nnull && t.nulls) atomicAdd(&t.nulls[col], nnull);
        asm volatile("st.global.u32 [%0], %1;" ::"l"(mp), "r"(mine));
      } else {
        const int nact       = tmin(32, tv.rows - g * 32);
        const uint32_t amask = nact == 32 ? 0xffffffffu : ((1u << nact) - 1u);
        const int nnull      = __popc(~mine & amask);
        if (nnull && t.nulls) atomicAdd(&t.nulls[col], nnull);
        const bool tbl_end = (rg + nact) == p.num_rows;
        int nbytes         = (nact + 7) >> 3;
        // the table's last mask word is written whole so its tail bits are 0 (RC:1081-1090)
        if (tbl_end) nbytes = static_cast<int>(round_up64((rg >> 3) + nbytes, 4) - (rg >> 3));
        const uint32_t w = mine & amask;
        if (nbytes == 4 && ((rg & 31) == 0)) {
          asm volatile("st.global.u32 [%0], %1;" ::"l"(mp), "r"(w));
        } else {
          for (int i = 0; i < nbytes; ++i) mp[i] = static_cast<uint8_t>(static_cast<uint64_t>(w) >> (8 * i));
        }
      }
    }
    if (nq == 1) {
      g += NCW;
    } else {
      q += ws.vdq;
      g += ws.vdg;
      if (q >= nq) {
        q -= nq;
        ++g;
      }
    }
  }
}

// Variable-width tables: does every row place its strings where convert_to_rows would (chars of the
// STRING columns back to back, in column order, from byte size_per_row -- RC:838-858)?  Phase 2's fast
// path relies on it; a mismatch only flips a status bit that routes phase 2 to the generic gather.
// A row is canonical iff the first pair starts at size_per_row and every pair starts where its left neighbour
// ends: a purely local test.  lane = row; the (row group, block of STRING columns) items are dealt to the consumer
// warps, each lane walking its block's pairs once -- ~5 instructions per string, the same cost for 1 or 64 columns.
template <int NCW, bool SAFE>
__device__ __noinline__ void canonical_check_tile(const uint8_t* base, const int32_t* s_off, int rows, int cw,
                                                  const int32_t* s_string_start, int nstr, int size_per_row,
                                                  unsigned long long* status)
{
  TileView tv;
  tv.base  = base;
  tv.s_off = s_off;
  const int lane    = lane_id();
  const int ngroups = (rows + 31) >> 5;
  const int nblk    = tmin(nstr, NCW);
  const int nitems  = ngroups * nblk;
  bool bad          = false;
  for (int item = cw; item < nitems; item += NCW) {
    const int g   = item / nblk;
    const int b   = item - g * nblk;
    const int s0  = (b * nstr) / nblk, s1 = ((b + 1) * nstr) / nblk;
    const int row = g * 32 + lane;
    if (row < rows) {
      const uint8_t* rp = row_ptr<true>(tv, row);
      uint32_t expect   = static_cast<uint32_t>(size_per_row);
      if (s0 > 0) {
        const uint8_t* pp = rp + s_string_start[s0 - 1];
        expect            = static_cast<uint32_t>(load_key<SAFE>(pp, 4)) + static_cast<uint32_t>(load_key<SAFE>(pp + 4, 4));
      }
      for (int s = s0; s < s1; ++s) {
        const uint8_t* pp = rp + s_string_start[s];
        const uint32_t so = static_cast<uint32_t>(load_key<SAFE>(pp, 4));
        const uint32_t ln = static_cast<uint32_t>(load_key<SAFE>(pp + 4, 4));
        bad |= so != expect;
        expect = so + ln;
      }
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, 1ull);
}

template <int NCW, int RPL, bool VAR, bool PRED, bool SAFE, bool ONEG>
__device__ __forceinline__ void process_tile(const FromRowsParams& p, const SmemTables& t, const WarpSched& ws,
                                             const TileView& tv, int cw)
{
  transpose_class<16, NCW, RPL, VAR, PRED, SAFE, ONEG>(p, t, ws, tv, 4);
  transpose_class<8, NCW, RPL, VAR, PRED, SAFE, ONEG>(p, t, ws, tv, 3);
  transpose_class<4, NCW, RPL, VAR, PRED, SAFE, ONEG>(p, t, ws, tv, 2);
  transpose_class<2, NCW, RPL, VAR, PRED, SAFE, ONEG>(p, t, ws, tv, 1);
  transpose_class<1, NCW, RPL, VAR, PRED, SAFE, ONEG>(p, t, ws, tv, 0);
  validity_tile<NCW, VAR, PRED, SAFE>(p, t, ws, tv);
  if constexpr (VAR) {
    if (p.status && p.nstr > 0)
      canonical_check_tile<NCW, SAFE>(tv.base, tv.s_off, tv.rows, cw, t.string_start, p.nstr, p.size_per_row, p.status);
  }
}

// SAFE / partial tiles are kept out of line so they do not inflate the fast path's registers
template <int NCW, int RPL, bool VAR, bool SAFE, bool ONEG>
__device__ __noinline__ void process_tile_slow(const FromRowsParams& p, const SmemTables& t, const WarpSched& ws,
                                               const TileView& tv, int cw)
{
  process_tile<NCW, RPL, VAR, true, SAFE, ONEG>(p, t, ws, tv, cw);
}

// The producer warp's loop lives in its own (out-of-line) function so that its long-lived 64-bit state does
// not compete with the consumers' transpose loop for registers.  Everything it needs travels by value.
struct ProducerArgs {
  const uint8_t* rows;
  const int32_t* row_offsets;
  int64_t rows_bytes, num_rows, super_rows;
  int32_t row_stride, tile_rows, stage_bytes, nstages, stage_span, soff_span;
  uint8_t* payload0;
  int32_t* soff0;
  StageHdr* hdr0;
  uint64_t* full;
  uint64_t* empty;
  int32_t* s_next_off;
};

template <bool VAR>
__device__ __noinline__ void producer_loop(const ProducerArgs p)
{
  const int lane       = lane_id();
  const int NS         = p.nstages;
  const int stage_span = p.stage_span;
  const int soff_span  = p.soff_span;
  uint8_t* payload0    = p.payload0;
  int32_t* soff0       = p.soff0;
  StageHdr* hdr0       = p.hdr0;
  uint64_t* full       = p.full;
  uint64_t* empty      = p.empty;
  int32_t* s_next_off  = p.s_next_off;
  const bool base_ok   = (reinterpret_cast<uintptr_t>(p.rows) & 7) == 0;
  {
    // Super-tiles (a few tiles of consecutive rows) are dealt round-robin to the CTAs, so at any moment
    // the whole grid streams through one contiguous window of the row buffer and of every column --
    // the access pattern of a plain copy kernel -- instead of one far-apart range per SM.
    int64_t sup = blockIdx.x;
    int64_t r   = sup * p.super_rows;
    int64_t c1  = tmin(p.num_rows, r + p.super_rows);

    // Geometry of the tile starting at row `r` (computed one tile AHEAD, while the previous TMA load is
    // in flight, so the global reads of the LIST offsets never sit on the critical path).
    int g_rows  = 0;
    bool g_safe = false, g_end = false;
    int64_t g_lo = 0, g_hi = 0;
    auto next_geometry = [&]() {
      if (r >= c1) {  // next super-tile of this CTA
        sup += gridDim.x;
        r  = sup * p.super_rows;
        c1 = tmin(p.num_rows, r + p.super_rows);
      }
      g_end = r >= p.num_rows;
      if (g_end) return;
      int rows  = static_cast<int>(tmin<int64_t>(p.tile_rows, c1 - r));
      bool safe = !base_ok;
      if constexpr (!VAR) {
        g_lo = r * p.row_stride;
        g_hi = (r + rows) * static_cast<int64_t>(p.row_stride);
        if (g_hi - g_lo > p.stage_bytes) safe = true;
      } else {
        // load off[r .. r+rows] (coalesced) and pick the largest multiple-of-8 row count that fits.  All the loads
        // are issued before the first use: one memory round trip per tile, not one per 32 rows (a 512-row tile of
        // a narrow table spends several times longer here than its consumers need).
        constexpr int kMaxChunks = 17;  // tile_rows <= 512 -> rows + 1 <= 513 offsets
        rows = tmin(rows, 512);
        int32_t ov[kMaxChunks];
#pragma unroll
        for (int k = 0; k < kMaxChunks; ++k) {
          const int i = k * 32 + lane;
          ov[k]       = (i <= rows) ? p.row_offsets[r + i] : 0;
        }
        const int64_t a0   = static_cast<uint32_t>(__shfl_sync(0xffffffffu, ov[0], 0));
        const int64_t base = a0 - static_cast<int64_t>((reinterpret_cast<uintptr_t>(p.rows) + a0) & 15);
        int fit            = 0;
        bool misaligned    = (a0 & 7) != 0;
#pragma unroll
        for (int k = 0; k < kMaxChunks; ++k) {
          if (k * 32 <= rows) {  // warp-uniform
            const int i     = k * 32 + lane;
            const int64_t o = static_cast<uint32_t>(ov[k]);
            if (i <= rows) {
              s_next_off[i] = static_cast<int32_t>(o - base);
              if (i < rows && (o & 7)) misaligned = true;
            }
            const bool ok = (i >= 1) && (i <= rows) && (round_up64(o - base, 16) <= p.stage_bytes + 16);
            fit += __popc(__ballot_sync(0xffffffffu, ok));
          }
        }
        misaligned = __any_sync(0xffffffffu, misaligned);
        if (fit < rows) fit &= ~7;
        if (fit == 0 || misaligned || safe) {
          // a row does not fit a stage (or rows are not 8-aligned): SAFE tile of <= 8 rows
          safe = true;
          rows = tmin(rows, 8);
          __syncwarp();
          for (int i = lane; i <= rows; i += 32) s_next_off[i] = p.row_offsets[r + i];  // absolute offsets
        } else {
          rows = fit;
        }
        g_lo = a0;
        __syncwarp();
        g_hi = safe ? static_cast<int64_t>(s_next_off[rows]) : base + s_next_off[rows];
      }
      g_rows = rows;
      g_safe = safe;
      __syncwarp();
    };
    next_geometry();

    int it = 0;
    for (;; ++it) {
      const int s        = it % NS;
      const uint32_t par = ((it / NS) & 1) ^ 1;
      if (lane == 0) mbar_wait(&empty[s], par);  // first pass over the ring returns immediately
      __syncwarp();
      uint8_t* pay  = payload0 + static_cast<size_t>(s) * stage_span;
      int32_t* soff = soff0 + static_cast<size_t>(s) * soff_span;
      StageHdr* h   = hdr0 + s;
      if (g_end) {
        if (lane == 0) {
          h->rows = 0;
          mbar_arrive(&full[s]);
        }
        break;
      }
      const int rows    = g_rows;
      const bool safe   = g_safe;
      const int64_t glo = g_lo, ghi = g_hi;
      if constexpr (VAR) {
        for (int i = lane; i <= rows; i += 32) soff[i] = s_next_off[i];
      }
      uint32_t tx    = 0;
      int32_t skew   = 0;
      uintptr_t t_lo = 0, fl = 0;
      if (!safe) {
        // 16-byte aligned TMA window inside [rows, rows + rows_bytes); <16-byte head/tail remainders
        // (8-byte units) are copied by hand
        const uintptr_t a_lo = reinterpret_cast<uintptr_t>(p.rows) + glo;
        const uintptr_t a_hi = reinterpret_cast<uintptr_t>(p.rows) + ghi;
        const uintptr_t b_lo = reinterpret_cast<uintptr_t>(p.rows);
        const uintptr_t b_hi = b_lo + p.rows_bytes;
        fl                   = a_lo & ~uintptr_t{15};
        skew                 = static_cast<int32_t>(a_lo - fl);  // payload[skew] == global byte glo
        t_lo                 = fl;
        if (t_lo < b_lo) t_lo = fl + 16;  // cannot read before the buffer
        uintptr_t t_hi = (a_hi + 15) & ~uintptr_t{15};
        if (t_hi > b_hi) t_hi = a_hi & ~uintptr_t{15};  // cannot read past the buffer
        if (t_hi > t_lo) tx = static_cast<uint32_t>(t_hi - t_lo);
        uintptr_t h_end = tmin(tmax(t_lo, a_lo), a_hi);  // head  [a_lo, h_end)
        if (tx == 0) h_end = a_hi;                        // tiny tile: all by hand
        const uintptr_t t_beg = tmax(tmin(t_hi, a_hi), h_end);  // tail  [t_beg, a_hi)
        if (lane == 0) {
          for (uintptr_t a = a_lo; a < h_end; a += 8)
            *reinterpret_cast<uint2*>(pay + (a - fl)) = *reinterpret_cast<const uint2*>(a);
          for (uintptr_t a = t_beg; a < a_hi; a += 8)
            *reinterpret_cast<uint2*>(pay + (a - fl)) = *reinterpret_cast<const uint2*>(a);
        }
      }
      if (lane == 0) {
        h->r0    = r;
        h->rows  = rows;
        h->safe  = safe ? 1 : 0;
        h->skew  = skew;
        h->gbase = glo;
      }
      __syncwarp();
      if (lane == 0) {
        if (tx) {
          mbar_arrive_expect_tx(&full[s], tx);  // release: header / offsets / hand copies are visible
          tma_load_1d(pay + (t_lo - fl), reinterpret_cast<const void*>(t_lo), tx, &full[s]);
        } else {
          mbar_arrive(&full[s]);
        }
      }
      r += rows;
      next_geometry();  // overlaps with the load just issued
    }
  }
}

template <int NCW, int RPL, bool VAR, bool ONEG>
__global__ void __launch_bounds__((NCW + 1) * 32, 1) from_rows_kernel(const __grid_constant__ FromRowsParams p)
{
  constexpr int kThreads = (NCW + 1) * 32;
  extern __shared__ __align__(128) uint8_t smem[];
  const int NS         = p.nstages;
  const int stage_span = p.stage_bytes + kStageSlack;
  uint8_t* payload0    = smem;
  int32_t* soff0       = reinterpret_cast<int32_t*>(smem + static_cast<size_t>(NS) * stage_span);
  const int soff_span  = (p.tile_rows + 4) & ~3;  // ints per stage (tile_rows + 1, padded)
  StageHdr* hdr0       = reinterpret_cast<StageHdr*>(soff0 + static_cast<size_t>(NS) * soff_span);
  uint64_t* full       = reinterpret_cast<uint64_t*>(hdr0 + NS);
  uint64_t* empty      = full + kMaxStages;
  int32_t* s_ent_start = reinterpret_cast<int32_t*>(empty + kMaxStages);
  uint8_t** s_ent_dst  = reinterpret_cast<uint8_t**>(s_ent_start + ((p.nentries + 1) & ~1));
  uint32_t** s_masks   = reinterpret_cast<uint32_t**>(s_ent_dst + p.nentries);
  int32_t* s_nulls     = reinterpret_cast<int32_t*>(s_masks + p.ncols);
  int32_t* s_next_off  = s_nulls + ((p.ncols + 3) & ~3);  // producer scratch: offsets of the NEXT tile
  int32_t* s_str_start = s_next_off + ((p.tile_rows + 4) & ~3);

  const int tid = threadIdx.x;
  for (int i = tid; i < p.nentries; i += kThreads) {
    s_ent_start[i] = p.entries[i].start;
    s_ent_dst[i]   = static_cast<uint8_t*>(p.ent_dst[i]);
  }
  for (int i = tid; i < p.ncols; i += kThreads) {
    s_masks[i] = p.masks[i];
    s_nulls[i] = 0;
  }
  for (int i = tid; i < p.nstr; i += kThreads) s_str_start[i] = p.string_start[i];
  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NCW);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int lane = lane_id();
  // the staged fast path needs 8-byte aligned rows
  const bool base_ok = (reinterpret_cast<uintptr_t>(p.rows) & 7) == 0;

  if (warp_id() == 0) {
    // =================================== producer ===================================
    ProducerArgs pa;
    pa.rows        = p.rows;
    pa.row_offsets = p.row_offsets;
    pa.rows_bytes  = p.rows_bytes;
    pa.num_rows    = p.num_rows;
    pa.super_rows  = p.super_rows;
    pa.row_stride  = p.row_stride;
    pa.tile_rows   = p.tile_rows;
    pa.stage_bytes = p.stage_bytes;
    pa.nstages     = NS;
    pa.stage_span  = stage_span;
    pa.soff_span   = soff_span;
    pa.payload0    = payload0;
    pa.soff0       = soff0;
    pa.hdr0        = hdr0;
    pa.full        = full;
    pa.empty       = empty;
    pa.s_next_off  = s_next_off;
    producer_loop<VAR>(pa);
  } else {
    // =================================== consumers ===================================
    const int cw = warp_id() - 1;
    SmemTables t{s_ent_start, s_ent_dst, s_masks, p.null_counts ? s_nulls : nullptr, s_str_start};
    WarpSched ws;
#pragma unroll
    for (int k = 0; k < kNumClasses; ++k) ws.ustart[k] = (cw + NCW - (p.cls_ubase[k] % NCW)) % NCW;
    ws.vstart = (cw + NCW - (p.v_ubase % NCW)) % NCW;
    {
      const int nq = (p.ncols + 31) >> 5;
      ws.vdg       = NCW / nq;
      ws.vdq       = NCW - ws.vdg * nq;
    }
    ws.sub    = lane / RPL;
    ws.lr     = lane - ws.sub * RPL;
    for (int it = 0;; ++it) {
      const int s        = it % NS;
      const uint32_t par = (it / NS) & 1;
      mbar_wait(&full[s], par);
      const StageHdr h = hdr0[s];
      if (h.rows == 0) break;
      const uint8_t* pay  = payload0 + static_cast<size_t>(s) * stage_span;
      const int32_t* soff = soff0 + static_cast<size_t>(s) * soff_span;
      TileView tv;
      tv.s_off  = soff;
      tv.stride = static_cast<uint32_t>(p.row_stride);
      tv.r0     = h.r0;
      tv.rows   = h.rows;
      tv.lane_row = nullptr;
      if (!h.safe) {
        tv.base = VAR ? pay : pay + h.skew;
        if (VAR && ONEG && ws.lr < h.rows) tv.lane_row = pay + static_cast<uint32_t>(soff[ws.lr]);
        if (!VAR && h.rows == p.tile_rows && (p.gpu & 3) == 0)
          process_tile<NCW, RPL, VAR, false, false, false>(p, t, ws, tv, cw);
        else if (VAR)
          process_tile<NCW, RPL, VAR, true, false, ONEG>(p, t, ws, tv, cw);  // var-width tiles are always predicated
        else
          process_tile_slow<NCW, RPL, VAR, false, false>(p, t, ws, tv, cw);
      } else {
        tv.base = VAR ? p.rows : p.rows + h.gbase;
        process_tile_slow<NCW, RPL, VAR, true, false>(p, t, ws, tv, cw);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
  }
  __syncthreads();
  if (p.null_counts) {
    for (int i = tid; i < p.ncols; i += kThreads)
      if (s_nulls[i]) atomicAdd(&p.null_counts[i], static_cast<unsigned long long>(s_nulls[i]));
  }
}

// ---- host launcher -------------------------------------------------------------------------------
size_t from_rows_smem_bytes(const Tiling& tl, int nentries, int ncols, int nstr)
{
  size_t b = static_cast<size_t>(tl.num_stages) * (tl.stage_bytes + kStageSlack);
  b += static_cast<size_t>(tl.num_stages) * ((tl.tile_rows + 4) & ~3) * 4;
  b += static_cast<size_t>(tl.num_stages) * sizeof(StageHdr);
  b += 2 * kMaxStages * 8;
  b += static_cast<size_t>((nentries + 1) & ~1) * 4;
  b += static_cast<size_t>(nentries) * 8 + static_cast<size_t>(ncols) * 8 + static_cast<size_t>((ncols + 3) & ~3) * 4;
  b += static_cast<size_t>((tl.tile_rows + 4) & ~3) * 4;
  b += static_cast<size_t>(nstr + 4) * 4;
  return (b + 127) & ~size_t{127};
}

template <int NCW>
static int launch_variant(const FromRowsParams& p, unsigned grid, size_t smem, cudaStream_t stream)
{
  auto go = [&](auto kern) -> int {
    SRJ_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    kern<<<grid, (NCW + 1) * 32, smem, stream>>>(p);
    return SRJ_OK;
  };
  const bool var  = p.row_offsets != nullptr;
  const bool oneg = var && p.gpu == 1;  // one row group per tile (wide rows): hoisted row address, 4 units in flight
  switch (p.rpl) {
    case 32:
      if (!var) return go(from_rows_kernel<NCW, 32, false, false>);
      return oneg ? go(from_rows_kernel<NCW, 32, true, true>) : go(from_rows_kernel<NCW, 32, true, false>);
    case 16:
      if (!var) return go(from_rows_kernel<NCW, 16, false, false>);
      return oneg ? go(from_rows_kernel<NCW, 16, true, true>) : go(from_rows_kernel<NCW, 16, true, false>);
    default:
      if (!var) return go(from_rows_kernel<NCW, 8, false, false>);
      return oneg ? go(from_rows_kernel<NCW, 8, true, true>) : go(from_rows_kernel<NCW, 8, true, false>);
  }
}

int launch_from_rows(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets, int64_t rows_bytes,
                     int64_t num_rows, void* const* d_ent_dst, uint32_t* const* d_masks, int64_t* d_null_counts,
                     int64_t* d_status, cudaStream_t stream)
{
  if (num_rows == 0) return SRJ_OK;
  FromRowsParams p{};
  p.rows            = rows;
  p.row_offsets     = row_offsets;
  p.rows_bytes      = rows_bytes;
  p.num_rows        = num_rows;
  p.ncols           = plan->num_columns;
  p.validity_offset = plan->validity_offset;
  p.row_stride      = plan->fixed_row_size;
  p.tile_rows       = plan->tiling.tile_rows;
  p.rpl             = plan->tiling.rows_per_item;
  p.stage_bytes     = plan->tiling.stage_bytes;
  p.nstages         = plan->tiling.num_stages;
  p.nentries        = static_cast<int32_t>(plan->fr_entries.size());
  for (int k = 0; k <= kNumClasses; ++k) p.class_begin[k] = plan->fr_class_begin[k];
  {
    // static schedule: split each slot's row groups into 2^cs chunks until there are enough units to
    // balance the consumer warps; the predicate-free instantiation needs gpu % 4 == 0
    const int cpi     = 32 / p.rpl;
    const int ngroups = (p.tile_rows + p.rpl - 1) / p.rpl;
    int slots         = 0;
    for (int k = 0; k < kNumClasses; ++k) slots += (p.class_begin[k + 1] - p.class_begin[k] + cpi - 1) / cpi;
    int cs = 0;
    while ((slots << cs) < 96 && (ngroups % (8 << cs)) == 0) ++cs;  // keeps gpu a multiple of 4
    p.cs  = cs;
    p.gpu = (ngroups + (1 << cs) - 1) >> cs;
    int ub = 0;
    for (int k = kNumClasses - 1; k >= 0; --k) {  // kernel runs the classes 16,8,4,2,1
      p.cls_ubase[k] = ub;
      p.cls_units[k] = ((p.class_begin[k + 1] - p.class_begin[k] + cpi - 1) / cpi) << cs;
      ub += p.cls_units[k];
    }
    p.v_ubase = ub;
  }
  p.entries     = plan->d_fr_entries;
  p.ent_dst     = d_ent_dst;
  p.masks       = d_masks;
  p.null_counts  = reinterpret_cast<unsigned long long*>(d_null_counts);
  p.nstr         = plan->num_string_columns;
  p.size_per_row = plan->size_per_row;
  p.string_start = plan->d_string_start;
  p.status       = reinterpret_cast<unsigned long long*>(d_status);
  int dev = 0, nsm = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  // super-tile = a multiple of the tile height (=> of 32 or 8|16: mask-byte aligned).  Fixed-stride
  // tables: two tiles (faster than one, flat beyond).  Variable-width tables cut tiles adaptively inside a
  // super-tile of >= 4 tiles so the last, shorter tile of a super-tile is amortised.
  p.super_rows      = static_cast<int64_t>(p.tile_rows) * (row_offsets ? 8 : 2);
  const int64_t ns  = (num_rows + p.super_rows - 1) / p.super_rows;
  const int64_t grid = std::min<int64_t>(nsm, ns);
  const size_t smem = from_rows_smem_bytes(plan->tiling, p.nentries, p.ncols, plan->num_string_columns);
  // 11 consumer warps: 384 threads x 168 registers fills the register file with no spills (15 warps cap
  // the kernel at 128 registers and spill inside the transpose loop)
  const int rc = launch_variant<11>(p, static_cast<unsigned>(grid), smem, stream);
  if (rc != SRJ_OK) return rc;
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj
