// from_rows_wide.cu -- JCUDF rows -> columns for WIDE variable-width tables (reference: convert_from_rows,
// RC:2149-2441; kernels copy_from_rows RC:879-969, copy_validity_from_rows RC:987-1094, the per-column
// exclusive_scan loop RC:2375-2395 and fixup_null_counts RC:2130-2136).
//
// A wide row (config C3: 3096 B of fixed-width fields + validity, then ~820 B of chars) is larger than any
// useful tile of whole rows, and phase 1 needs only its fixed section.  So the fixed section is cut into
// byte-range SLABS (host-planned, ~1 KB each) and a tile is R rows (a multiple of 32) x one slab:
//
//   producer warp : lane = row; one TMA bulk copy per (row, slab) from  rows + offsets[r] + slab.begin  into
//                   that row's slot of the stage (pitch = odd multiple of 16 B, so consecutive rows start in
//                   different banks).  The chars of the row are never read here: phase 1 moves
//                   fixed + validity bytes only, the variable section is read once, by phase 2.
//   consumer warps: lane = row.  A unit = one field of the slab for all G = R/32 row groups: one 16-byte
//                   descriptor read, G shared-memory loads, G coalesced st.global (32 lanes x W contiguous
//                   bytes each); two units in flight per warp.
//   strings       : the (offset, len) pair of a STRING column is one more field.  The lengths of a 32-row
//                   group are scanned across the warp right there: offsets[r + 1] receives the inclusive
//                   sum INSIDE the group and the group total goes to a small side array, so the only scan
//                   left is over one value per 32 rows (wide_group_scan_kernel).  The same unit checks that
//                   the pair sits where convert_to_rows would have put it (pair.offset == previous
//                   pair.offset + previous len; the slab was extended backwards to hold that previous pair).
//   validity      : 32x32 bit transpose by shuffles (movers.cuh), null counts popc'd into shared counters.
//
// Tiles start on multiples of R rows, so mask words are always written whole and every 32-row group of the
// offsets protocol is owned by exactly one warp.  Rows that are not 8-byte aligned take the SAFE path of the
// same kernel (global memory, byte-wise).
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "kernels.hpp"
#include "movers.cuh"
#include "plan.hpp"

namespace srj {

constexpr int kWMaxStages = 4;
constexpr int kWMaxGrid   = 256;  // CTAs (one per SM)
constexpr int kWMaxG      = 4;
constexpr int kWSlack     = 32;

struct WHdr {
  int64_t r0;
  int32_t rows;  // 0 = end of this CTA's work
  int32_t slab;
  int32_t safe;
  int32_t pad[3];
};
static_assert(sizeof(WHdr) == 32, "WHdr is 32 bytes");

struct __align__(16) WDesc {
  uint8_t* dst;  // column data, or (int32*)offsets + 1 for a STRING column
  int32_t rel;   // field start relative to the slab's begin
  int32_t sidx;  // STRING: index among the string columns
};

struct WideParams {
  const uint8_t* rows;
  const int32_t* row_offsets;
  int64_t rows_bytes;
  int64_t num_rows;
  int64_t ngroups;  // ceil(num_rows / 32)
  int32_t ncols, nstr, size_per_row, validity_offset;
  int32_t R, G, pitch, nstages, nslabs, nent;
  const WideEntry* entries;
  const WideSlab* slabs;
  const int32_t* string_start;  // [nstr]
  int32_t want_nulls;           // null counts requested
  uint32_t* agg;                // scratch [nstr][ngroups]: chars of each 32-row group
  int32_t* null_part;           // scratch [grid][ncols]: per-CTA null counts (reduced by the scan kernel: no memset, no atomics)
  int32_t* bad_part;            // scratch [grid]: per-CTA "non-canonical row seen" flags
  uint32_t* sync_words;         // scratch [2]: {ticket, overflow} of the scan kernel, zeroed here by CTA 0
};

// Per-call pointer tables travel as kernel parameters (no staging copy, no allocation): the column count of a wide
// plan is capped so that they fit comfortably in the 32 KB parameter space.
constexpr int kWMaxCols = 448;
struct WidePtrTab {
  void* col[kWMaxCols];       // column data, STRING: offsets
  uint32_t* mask[kWMaxCols];
};
struct WideScanTab {
  int32_t* offs[kWMaxCols];   // [nstr] offsets of the STRING columns
  int32_t scol[kWMaxCols];    // [nstr] their schema column
};

__device__ __forceinline__ WDesc lds_desc(uint32_t a)
{
  uint32_t x, y, z, w;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(a));
  WDesc d;
  d.dst  = reinterpret_cast<uint8_t*>(static_cast<uint64_t>(x) | (static_cast<uint64_t>(y) << 32));
  d.rel  = static_cast<int32_t>(z);
  d.sidx = static_cast<int32_t>(w);
  return d;
}

struct WTables {
  uint32_t desc;  // shared-space address of the descriptor table
  const int16_t* first;  // [nslabs][6][NCW] first unit of (slab, class) for each consumer warp
  const WideSlab* slabs;
  const int32_t* str_start;
  uint32_t* const* masks;
  int32_t* nulls;
};

__device__ __forceinline__ uint32_t ld_bytes32(const uint8_t* p)
{
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) |
         (static_cast<uint32_t>(p[3]) << 24);
}

template <int W>
__device__ __forceinline__ Reg<W> ld_bytes(const uint8_t* src)
{
  Reg<W> r;
#pragma unroll
  for (int i = 0; i < (W + 3) / 4; ++i) r.v[i] = 0;
#pragma unroll
  for (int i = 0; i < W; ++i) r.v[i / 4] |= static_cast<uint32_t>(src[i]) << (8 * (i & 3));
  return r;
}

// first unit >= cb of this slab whose position in the slab's list is congruent to w (mod NCW): the units of a slab are
// dealt round-robin to the consumer warps across the width classes.  Tabulated once per CTA (s_first).
__device__ __forceinline__ int first_unit_of(int cb, int cb0, int w, int ncw)
{
  return cb + (w + ncw - (cb - cb0) % ncw) % ncw;
}

// ---- full tiles: G row groups, rows staged, no predicates ------------------------------------------------
template <int W, int G, int NCW>
__device__ __forceinline__ void units_full(uint32_t desc, int u0, int ue, const uint32_t (&ra)[G], int64_t rowoff)
{
  for (int u = u0; u < ue; u += 2 * NCW) {
    const bool has1 = u + NCW < ue;
    const WDesc d0  = lds_desc(desc + 16u * u);
    const WDesc d1  = lds_desc(desc + 16u * (has1 ? u + NCW : u));
    Reg<W> a[G], b[G];
#pragma unroll
    for (int g = 0; g < G; ++g) a[g] = lds_elem<W>(ra[g] + d0.rel);
#pragma unroll
    for (int g = 0; g < G; ++g) b[g] = lds_elem<W>(ra[g] + d1.rel);
    uint8_t* p0 = d0.dst + rowoff * W;
#pragma unroll
    for (int g = 0; g < G; ++g) st_elem<W>(p0 + g * 32 * W, a[g]);
    if (has1) {
      uint8_t* p1 = d1.dst + rowoff * W;
#pragma unroll
      for (int g = 0; g < G; ++g) st_elem<W>(p1 + g * 32 * W, b[g]);
    }
  }
}

__device__ __forceinline__ uint32_t warp_inclusive_scan(uint32_t x, int lane)
{
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x;
}

template <int G, int NCW>
__device__ __forceinline__ bool strings_full(const WideParams& p, const WTables& t, const WideSlab& sl, int u0,
                                             const uint32_t (&ra)[G], int64_t rowoff, int64_t group0, int lane)
{
  bool bad = false;
  for (int u = u0; u < sl.cb[6]; u += NCW) {
    const WDesc d  = lds_desc(t.desc + 16u * u);
    const int prel = d.sidx > 0 ? t.str_start[d.sidx - 1] - sl.begin : -1;
    uint32_t so[G], ln[G], ex[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      so[g] = lds_u32(ra[g] + d.rel);
      ln[g] = lds_u32(ra[g] + d.rel + 4);
      ex[g] = static_cast<uint32_t>(p.size_per_row);
      if (prel >= 0) ex[g] = lds_u32(ra[g] + prel) + lds_u32(ra[g] + prel + 4);
    }
    uint32_t* dst = reinterpret_cast<uint32_t*>(d.dst) + rowoff;
    uint32_t* ag  = p.agg + static_cast<int64_t>(d.sidx) * p.ngroups + group0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      bad |= so[g] != ex[g];
      const uint32_t inc = warp_inclusive_scan(ln[g], lane);
      asm volatile("st.global.u32 [%0], %1;" ::"l"(dst + g * 32), "r"(inc));
      if (lane == 31) ag[g] = inc;
    }
  }
  return bad;
}

// validity bytes of this slab's rows -> column mask words (+ null counts); rows < 32 * Gt only at the table end
template <int NCW, bool SAFE>
__device__ __forceinline__ void validity_tile(const WideParams& p, const WTables& t, int vrel, int w, const uint32_t* ra,
                                              const uint8_t* const* rp, int64_t r0, int rows, int lane)
{
  const int nvb   = (p.ncols + 7) >> 3;
  const int nq    = (p.ncols + 31) >> 5;
  const int Gt    = (rows + 31) >> 5;
  const int items = nq * Gt;
  for (int item = w; item < items; item += NCW) {
    const int g   = item / nq;
    const int q   = item - g * nq;
    const int row = g * 32 + lane;
    uint32_t r    = 0;
    if (row < rows) {
      const int nbv = tmin(4, nvb - 4 * q);
      if constexpr (SAFE) {
        const uint8_t* vp = rp[g] + vrel + 4 * q;
        for (int i = 0; i < nbv; ++i) r |= static_cast<uint32_t>(vp[i]) << (8 * i);
      } else {
        const uint32_t va = ra[g] + vrel + 4 * q;
        if (nbv == 4 && (vrel & 3) == 0) {
          r = lds_u32(va);
        } else {
          for (int i = 0; i < nbv; ++i) r |= lds_u8(va + i) << (8 * i);
        }
      }
    }
    const uint32_t mine = transpose32(r, lane);  // lane = column 32q + lane, bit = row of the group
    const int col       = q * 32 + lane;
    if (col < p.ncols) {
      const int nact       = tmin(32, rows - g * 32);
      const uint32_t amask = nact == 32 ? 0xffffffffu : ((1u << nact) - 1u);
      const int nnull      = __popc(~mine & amask);
      if (nnull && t.nulls) atomicAdd(&t.nulls[col], nnull);
      // groups start on multiples of 32 rows: the word is written whole, tail bits of the table's last word are 0
      asm volatile("st.global.u32 [%0], %1;" ::"l"(t.masks[col] + (r0 >> 5) + g), "r"(mine & amask));
    }
  }
}

// ---- partial tiles (the table's last rows) and SAFE tiles (unaligned rows: global memory, byte-wise) ----------
template <int W, int NCW, bool SAFE>
__device__ __forceinline__ void units_slow(uint32_t desc, int u0, int ue, const uint32_t* ra,
                                           const uint8_t* const* rp, int64_t rowoff, int rows, int lane)
{
  const int Gt = (rows + 31) >> 5;
  for (int u = u0; u < ue; u += NCW) {
    const WDesc d = lds_desc(desc + 16u * u);
    uint8_t* p0   = d.dst + rowoff * W;
    for (int g = 0; g < Gt; ++g) {
      if (g * 32 + lane < rows) {
        Reg<W> v;
        if constexpr (SAFE) v = ld_bytes<W>(rp[g] + d.rel);
        else v = lds_elem<W>(ra[g] + d.rel);
        st_elem<W>(p0 + g * 32 * W, v);
      }
    }
  }
}

template <int NCW, bool SAFE>
__device__ __forceinline__ bool strings_slow(const WideParams& p, const WTables& t, const WideSlab& sl, int u0,
                                             const uint32_t* ra, const uint8_t* const* rp, int64_t rowoff, int64_t group0,
                                             int rows, int lane)
{
  bool bad     = false;
  const int Gt = (rows + 31) >> 5;
  for (int u = u0; u < sl.cb[6]; u += NCW) {
    const WDesc d  = lds_desc(t.desc + 16u * u);
    const int prel = d.sidx > 0 ? t.str_start[d.sidx - 1] - sl.begin : -1;
    uint32_t* dst  = reinterpret_cast<uint32_t*>(d.dst) + rowoff;
    uint32_t* ag   = p.agg + static_cast<int64_t>(d.sidx) * p.ngroups + group0;
    for (int g = 0; g < Gt; ++g) {
      const bool active = g * 32 + lane < rows;
      uint32_t so = 0, ln = 0, ex = static_cast<uint32_t>(p.size_per_row);
      if (active) {
        if constexpr (SAFE) {
          so = ld_bytes32(rp[g] + d.rel);
          ln = ld_bytes32(rp[g] + d.rel + 4);
          if (prel >= 0) ex = ld_bytes32(rp[g] + prel) + ld_bytes32(rp[g] + prel + 4);
        } else {
          so = lds_u32(ra[g] + d.rel);
          ln = lds_u32(ra[g] + d.rel + 4);
          if (prel >= 0) ex = lds_u32(ra[g] + prel) + lds_u32(ra[g] + prel + 4);
        }
        bad |= so != ex;
      }
      const uint32_t inc = warp_inclusive_scan(ln, lane);
      if (active) asm volatile("st.global.u32 [%0], %1;" ::"l"(dst + g * 32), "r"(inc));
      if (lane == 31) ag[g] = inc;
    }
  }
  return bad;
}

template <int NCW, bool SAFE>
__device__ __noinline__ bool tile_slow(const WideParams& p, const WTables& t, int slab, int w, uint32_t pay_s,
                                       const int32_t* rpos, int64_t r0, int rows, int lane)
{
  const WideSlab sl = t.slabs[slab];
  uint32_t ra[kWMaxG];
  const uint8_t* rp[kWMaxG];
#pragma unroll
  for (int g = 0; g < kWMaxG; ++g) {
    const int row = g * 32 + lane;
    ra[g]         = 0;
    rp[g]         = nullptr;
    if (row < rows) {
      if constexpr (SAFE) rp[g] = p.rows + static_cast<uint32_t>(rpos[row]) + sl.begin;
      else ra[g] = pay_s + static_cast<uint32_t>(rpos[row]);
    }
  }
  const int64_t rowoff = r0 + lane;
  const int16_t* fu    = t.first + (slab * 6) * NCW + w;
  units_slow<16, NCW, SAFE>(t.desc, fu[0 * NCW], sl.cb[1], ra, rp, rowoff, rows, lane);
  units_slow<8, NCW, SAFE>(t.desc, fu[1 * NCW], sl.cb[2], ra, rp, rowoff, rows, lane);
  units_slow<4, NCW, SAFE>(t.desc, fu[2 * NCW], sl.cb[3], ra, rp, rowoff, rows, lane);
  units_slow<2, NCW, SAFE>(t.desc, fu[3 * NCW], sl.cb[4], ra, rp, rowoff, rows, lane);
  units_slow<1, NCW, SAFE>(t.desc, fu[4 * NCW], sl.cb[5], ra, rp, rowoff, rows, lane);
  const bool bad = strings_slow<NCW, SAFE>(p, t, sl, fu[5 * NCW], ra, rp, rowoff, r0 >> 5, rows, lane);
  if (slab == p.nslabs - 1) validity_tile<NCW, SAFE>(p, t, p.validity_offset - sl.begin, w, ra, rp, r0, rows, lane);
  return bad;
}

template <int G, int NCW>
__device__ __forceinline__ bool tile_full(const WideParams& p, const WTables& t, int slab, int w, uint32_t pay_s,
                                          const int32_t* rpos, int64_t r0, int lane)
{
  const WideSlab sl = t.slabs[slab];
  uint32_t ra[G];
#pragma unroll
  for (int g = 0; g < G; ++g) ra[g] = pay_s + static_cast<uint32_t>(rpos[g * 32 + lane]);
  const int64_t rowoff = r0 + lane;
  const int16_t* fu    = t.first + (slab * 6) * NCW + w;
  units_full<16, G, NCW>(t.desc, fu[0 * NCW], sl.cb[1], ra, rowoff);
  units_full<8, G, NCW>(t.desc, fu[1 * NCW], sl.cb[2], ra, rowoff);
  units_full<4, G, NCW>(t.desc, fu[2 * NCW], sl.cb[3], ra, rowoff);
  units_full<2, G, NCW>(t.desc, fu[3 * NCW], sl.cb[4], ra, rowoff);
  units_full<1, G, NCW>(t.desc, fu[4 * NCW], sl.cb[5], ra, rowoff);
  const bool bad = strings_full<G, NCW>(p, t, sl, fu[5 * NCW], ra, rowoff, r0 >> 5, lane);
  if (slab == p.nslabs - 1) validity_tile<NCW, false>(p, t, p.validity_offset - sl.begin, w, ra, nullptr, r0, G * 32, lane);
  return bad;
}

// ---- producers ------------------------------------------------------------------------------------------
// One TMA bulk copy per (row, slab) costs its issuing warp ~70 cycles (five R2UR moves + UBLKCP per lane, one lane
// at a time), so kWProducers warps -- one per scheduler -- share the rows of a tile: producer q issues the copies
// of the rows whose lane index is congruent to q.  Each arrives on the stage's full barrier with the bytes of its
// own copies.  All of them read the row offsets of the tile (of the NEXT tile, one tile ahead), so they agree on
// whether the tile is staged or SAFE.
constexpr int kWProducers = 4;

struct WProducerArgs {
  const uint8_t* rows;
  const int32_t* row_offsets;
  int64_t rows_bytes, num_rows;
  int32_t R, G, pitch, nstages, nslabs, stage_span;
  uint8_t* payload0;
  int32_t* rpos0;
  WHdr* hdr0;
  uint64_t* full;
  uint64_t* empty;
  const WideSlab* slabs;  // shared-memory copy
};

__device__ __noinline__ void wide_producer(const WProducerArgs p, const int q)
{
  const int lane       = lane_id();
  const int NS         = p.nstages;
  const uintptr_t b_lo = reinterpret_cast<uintptr_t>(p.rows);
  const uintptr_t b_hi = b_lo + static_cast<uintptr_t>(p.rows_bytes);
  const bool base_ok   = (b_lo & 7) == 0;
  const int64_t ntiles = (p.num_rows + p.R - 1) / p.R;
  const bool mine      = (lane & (kWProducers - 1)) == q;
  int it               = 0;
  auto acquire         = [&](int it_) {
    const int s        = it_ % NS;
    const uint32_t par = ((it_ / NS) & 1) ^ 1;
    if (lane == 0) mbar_wait(&p.empty[s], par);  // the first pass over the ring returns immediately
    __syncwarp();
    return s;
  };
  auto load_offsets = [&](int64_t T, int64_t (&off)[kWMaxG]) {
    const int64_t r0 = T * p.R;
#pragma unroll
    for (int k = 0; k < kWMaxG; ++k) {
      const int64_t r = r0 + k * 32 + lane;
      off[k]          = (k < p.G && T < ntiles && r < p.num_rows) ? static_cast<int64_t>(static_cast<uint32_t>(p.row_offsets[r])) : 0;
    }
  };
  int64_t nxt[kWMaxG];
  load_offsets(blockIdx.x, nxt);
  for (int64_t T = blockIdx.x; T < ntiles; T += gridDim.x) {
    const int64_t r0 = T * p.R;
    const int rows   = static_cast<int>(tmin<int64_t>(p.R, p.num_rows - r0));
    int64_t off[kWMaxG];
    bool mis = !base_ok;
#pragma unroll
    for (int k = 0; k < kWMaxG; ++k) {
      off[k] = nxt[k];
      if (off[k] & 7) mis = true;  // rows past the tile's end carry 0
    }
    mis = __any_sync(0xffffffffu, mis);
    load_offsets(T + gridDim.x, nxt);  // in flight while this tile's copies are issued
    for (int sb = 0; sb < p.nslabs; ++sb, ++it) {
      const int s    = acquire(it);
      uint8_t* pay   = p.payload0 + static_cast<size_t>(s) * p.stage_span;
      int32_t* rpos  = p.rpos0 + static_cast<size_t>(s) * p.R;
      const int sbeg = p.slabs[sb].begin, send = p.slabs[sb].end;
      uint32_t tx    = 0;
#pragma unroll
      for (int k = 0; k < kWMaxG; ++k) {
        const int j = k * 32 + lane;
        if (k < p.G && j < rows && mine) {
          if (mis) {
            rpos[j] = static_cast<int32_t>(off[k]);  // absolute row offset: the consumers read global memory
          } else {
            const uintptr_t a_lo = b_lo + static_cast<uintptr_t>(off[k]) + sbeg;
            const uintptr_t a_hi = b_lo + static_cast<uintptr_t>(off[k]) + send;
            const uintptr_t fl   = a_lo & ~uintptr_t{15};
            uintptr_t t_lo       = fl < b_lo ? fl + 16 : fl;               // cannot read before the buffer
            uintptr_t t_hi       = (a_hi + 15) & ~uintptr_t{15};
            if (t_hi > b_hi) t_hi = a_hi & ~uintptr_t{15};                  // nor past it
            if (t_hi < t_lo) t_hi = t_lo;
            uint8_t* slot = pay + static_cast<size_t>(j) * p.pitch;        // slot byte x <-> global byte fl + x
            rpos[j]       = j * p.pitch + static_cast<int32_t>(a_lo - fl);
            // the < 16-byte pieces of [a_lo, a_hi) outside the TMA window (only at the ends of the buffer): 8-byte units
            const uintptr_t h_end = tmin(tmax(t_lo, a_lo), a_hi);
            for (uintptr_t a = a_lo; a < h_end; a += 8)
              *reinterpret_cast<uint2*>(slot + (a - fl)) = *reinterpret_cast<const uint2*>(a);
            for (uintptr_t a = tmax(tmin(t_hi, a_hi), h_end); a < a_hi; a += 8)
              *reinterpret_cast<uint2*>(slot + (a - fl)) = *reinterpret_cast<const uint2*>(a);
            tx += static_cast<uint32_t>(t_hi - t_lo);
          }
        }
      }
      uint32_t total = tx;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
      if (lane == 0 && q == 0) {
        WHdr* h = p.hdr0 + s;
        h->r0   = r0;
        h->rows = rows;
        h->slab = sb;
        h->safe = mis ? 1 : 0;
      }
      __syncwarp();
      if (lane == 0) {
        if (total) mbar_arrive_expect_tx(&p.full[s], total);  // release: header / row positions / hand copies visible
        else mbar_arrive(&p.full[s]);
      }
      __syncwarp();
      if (!mis) {
#pragma unroll
        for (int k = 0; k < kWMaxG; ++k) {
          const int j = k * 32 + lane;
          if (k < p.G && j < rows && mine) {
            const uintptr_t a_lo = b_lo + static_cast<uintptr_t>(off[k]) + sbeg;
            const uintptr_t a_hi = b_lo + static_cast<uintptr_t>(off[k]) + send;
            const uintptr_t fl   = a_lo & ~uintptr_t{15};
            uintptr_t t_lo       = fl < b_lo ? fl + 16 : fl;
            uintptr_t t_hi       = (a_hi + 15) & ~uintptr_t{15};
            if (t_hi > b_hi) t_hi = a_hi & ~uintptr_t{15};
            if (t_hi > t_lo)
              tma_load_1d(pay + static_cast<size_t>(j) * p.pitch + (t_lo - fl), reinterpret_cast<const void*>(t_lo),
                          static_cast<uint32_t>(t_hi - t_lo), &p.full[s]);
          }
        }
      }
    }
  }
  const int s = acquire(it);
  if (lane == 0) {
    if (q == 0) p.hdr0[s].rows = 0;
    mbar_arrive(&p.full[s]);
  }
}

// ---- the kernel ----------------------------------------------------------------------------------------
template <int NCW, int G>
__global__ void __launch_bounds__((NCW + kWProducers) * 32, 1) from_rows_wide_kernel(const __grid_constant__ WideParams p,
                                                                                            const __grid_constant__ WidePtrTab tab)
{
  constexpr int kThreads = (NCW + kWProducers) * 32;
  extern __shared__ __align__(128) uint8_t smem[];
  const int NS         = p.nstages;
  const int stage_span = p.R * p.pitch + kWSlack;  // multiple of 16
  uint8_t* payload0    = smem;
  WDesc* s_desc        = reinterpret_cast<WDesc*>(smem + static_cast<size_t>(NS) * stage_span);
  WHdr* hdr0           = reinterpret_cast<WHdr*>(s_desc + p.nent);
  uint64_t* full       = reinterpret_cast<uint64_t*>(hdr0 + NS);
  uint64_t* empty      = full + kWMaxStages;
  uint32_t** s_masks   = reinterpret_cast<uint32_t**>(empty + kWMaxStages);
  WideSlab* s_slabs    = reinterpret_cast<WideSlab*>(s_masks + p.ncols);
  int32_t* rpos0       = reinterpret_cast<int32_t*>(s_slabs + p.nslabs);
  int32_t* s_nulls     = rpos0 + static_cast<size_t>(NS) * p.R;
  int32_t* s_str_start = s_nulls + p.ncols;
  int16_t* s_first     = reinterpret_cast<int16_t*>(s_str_start + p.nstr);  // [nslabs][6][NCW]
  int* s_bad_p         = reinterpret_cast<int*>((reinterpret_cast<uintptr_t>(s_first + p.nslabs * 6 * NCW) + 3) & ~uintptr_t{3});

  const int tid = threadIdx.x;
  for (int i = tid; i < p.nslabs; i += kThreads) s_slabs[i] = p.slabs[i];
  for (int i = tid; i < p.nslabs * 6 * NCW; i += kThreads) {
    const int sb = i / (6 * NCW), k = (i / NCW) % 6, w = i % NCW;
    s_first[i]   = static_cast<int16_t>(first_unit_of(p.slabs[sb].cb[k], p.slabs[sb].cb[0], w, NCW));
  }
  for (int i = tid; i < p.nent; i += kThreads) {
    const WideEntry e = p.entries[i];
    WDesc d;
    d.dst     = static_cast<uint8_t*>(tab.col[e.column]) + (e.sidx >= 0 ? 4 : 0);  // lengths land at offsets[1..n]
    d.rel     = e.start - p.slabs[e.slab].begin;
    d.sidx    = e.sidx;
    s_desc[i] = d;
  }
  for (int i = tid; i < p.ncols; i += kThreads) {
    s_masks[i] = tab.mask[i];
    s_nulls[i] = 0;
  }
  if (tid == 0) {
    *s_bad_p = 0;
    if (blockIdx.x == 0) {  // nothing else touches these words while this kernel runs; the scan kernel (next in the stream) uses them
      p.sync_words[0] = 0;
      p.sync_words[1] = 0;
    }
  }
  for (int i = tid; i < p.nstr; i += kThreads) s_str_start[i] = p.string_start[i];
  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], kWProducers);
      mbar_init(&empty[s], NCW);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int lane = lane_id();
  if (warp_id() < kWProducers) {
    WProducerArgs pa;
    pa.rows        = p.rows;
    pa.row_offsets = p.row_offsets;
    pa.rows_bytes  = p.rows_bytes;
    pa.num_rows    = p.num_rows;
    pa.R           = p.R;
    pa.G           = G;
    pa.pitch       = p.pitch;
    pa.nstages     = NS;
    pa.nslabs      = p.nslabs;
    pa.stage_span  = stage_span;
    pa.payload0    = payload0;
    pa.rpos0       = rpos0;
    pa.hdr0        = hdr0;
    pa.full        = full;
    pa.empty       = empty;
    pa.slabs       = s_slabs;
    wide_producer(pa, warp_id());
  } else {
    const int w = warp_id() - kWProducers;
    const WTables t{smem_u32(s_desc), s_first, s_slabs, s_str_start, s_masks, p.want_nulls ? s_nulls : nullptr};
    bool bad = false;
    for (int it = 0;; ++it) {
      const int s        = it % NS;
      const uint32_t par = (it / NS) & 1;
      mbar_wait(&full[s], par);
      const WHdr h = hdr0[s];
      if (h.rows == 0) break;
      const uint32_t pay_s = smem_u32(payload0 + static_cast<size_t>(s) * stage_span);
      const int32_t* rpos  = rpos0 + static_cast<size_t>(s) * p.R;
      if (h.safe) bad |= tile_slow<NCW, true>(p, t, h.slab, w, pay_s, rpos, h.r0, h.rows, lane);
      else if (h.rows == G * 32) bad |= tile_full<G, NCW>(p, t, h.slab, w, pay_s, rpos, h.r0, lane);
      else bad |= tile_slow<NCW, false>(p, t, h.slab, w, pay_s, rpos, h.r0, h.rows, lane);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) *s_bad_p = 1;
  }
  __syncthreads();
  if (p.want_nulls)
    for (int i = tid; i < p.ncols; i += kThreads) p.null_part[static_cast<size_t>(blockIdx.x) * p.ncols + i] = s_nulls[i];
  if (tid == 0) p.bad_part[blockIdx.x] = *s_bad_p;
}

// ---- scan over the 32-row group totals ----------------------------------------------------------------
// base[c][g] <- chars of column c before 32-row group g (exclusive scan of the group totals), in the caller's
// workspace.  The offsets arrays keep the inclusive sums inside each group that from_rows_wide_kernel wrote; phase 2
// (strings.cu) adds the group base while it gathers.
constexpr int kGsThreads = 256;
constexpr int kGsPer     = 16;                    // groups per thread
constexpr int kGsChunk   = kGsThreads * kGsPer;   // groups per CTA

struct WideScanParams {
  const uint32_t* agg;
  uint32_t* base;                   // [nstr][ngroups] chars of the column before each 32-row group
  int64_t ngroups, num_rows;
  int64_t* char_totals;             // [ncols + 1] or NULL (entry ncols = status word)
  int64_t* null_counts;             // [ncols] or NULL
  const int32_t* null_part;         // [parts][ncols]
  const int32_t* bad_part;          // [parts]
  uint32_t* sync_words;             // {ticket, overflow}
  int32_t parts, ncols, nstr;
  uint64_t str_bits[kWMaxCols / 64];   // bit c set: schema column c is a STRING column
};

__global__ void __launch_bounds__(kGsThreads) wide_group_scan_kernel(const __grid_constant__ WideScanParams q,
                                                                      const __grid_constant__ WideScanTab tab)
{
  __shared__ int64_t s_warp[kGsThreads / 32];
  __shared__ int64_t s_pre;
  __shared__ unsigned s_ticket;
  const uint32_t* agg      = q.agg;
  const int64_t ngroups    = q.ngroups;
  int64_t* char_totals     = q.char_totals;
  const int c       = blockIdx.y;
  const int64_t k   = blockIdx.x;
  const uint32_t* a = agg + static_cast<int64_t>(c) * ngroups;
  uint32_t* bs      = q.base + static_cast<int64_t>(c) * ngroups;
  // this thread's groups first (their loads overlap the prefix pass below)
  const int64_t g0 = k * kGsChunk + static_cast<int64_t>(threadIdx.x) * kGsPer;
  uint32_t v[kGsPer];
#pragma unroll
  for (int j = 0; j < kGsPer; ++j) v[j] = (g0 + j < ngroups) ? a[g0 + j] : 0u;
  // chars of this column before the chunk (<= 3 chunks of 16 KB for a 2 GiB batch of wide rows)
  int64_t pre = 0;
  for (int64_t i = threadIdx.x; i < k * kGsChunk; i += kGsThreads) pre += a[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) pre += __shfl_down_sync(0xffffffffu, pre, o);
  if (lane_id() == 0) s_warp[warp_id()] = pre;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t t = 0;
    for (int i = 0; i < kGsThreads / 32; ++i) t += s_warp[i];
    s_pre = t;
  }
  __syncthreads();
  pre = s_pre;
  __syncthreads();
  int64_t tsum = 0;
#pragma unroll
  for (int j = 0; j < kGsPer; ++j) tsum += v[j];
  int64_t x = tsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane_id() >= o) x += y;
  }
  if (lane_id() == 31) s_warp[warp_id()] = x;
  __syncthreads();
  int64_t wpre = 0;
  for (int i = 0; i < warp_id(); ++i) wpre += s_warp[i];
  int64_t run = pre + wpre + x - tsum;
#pragma unroll
  for (int j = 0; j < kGsPer; ++j) {
    const int64_t g = g0 + j;
    if (g < ngroups) {
      bs[g] = static_cast<uint32_t>(run);  // exclusive: chars before group g
      run += v[j];
      if (g == ngroups - 1) {
        if (char_totals) char_totals[tab.scol[c]] = run;
        if (run > INT32_MAX) atomicOr(&q.sync_words[1], 2u);  // cudf strings offsets are int32
      }
    }
  }
  // ---- what phase 1 reports besides the offsets.  Every CTA of this grid takes a few columns: exact null counts (sum of
  // the per-CTA partials of from_rows_wide_kernel, one thread per partial) and zeros for the non-STRING entries of
  // char_totals; the last CTA to finish writes the status word.
  {
    const int ncta = gridDim.x * gridDim.y;
    const int me   = blockIdx.y * gridDim.x + blockIdx.x;
    for (int col = me; col < q.ncols; col += ncta) {
      if (q.null_counts) {
        int64_t nn = 0;
        for (int b = threadIdx.x; b < q.parts; b += kGsThreads) nn += q.null_part[static_cast<size_t>(b) * q.ncols + col];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) nn += __shfl_down_sync(0xffffffffu, nn, o);
        __syncthreads();
        if (lane_id() == 0) s_warp[warp_id()] = nn;
        __syncthreads();
        if (threadIdx.x == 0) {
          int64_t t = 0;
          for (int i = 0; i < kGsThreads / 32; ++i) t += s_warp[i];
          q.null_counts[col] = t;
        }
      }
      if (char_totals && threadIdx.x == 0 && !((q.str_bits[col >> 6] >> (col & 63)) & 1ull)) char_totals[col] = 0;
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_ticket = atomicAdd(&q.sync_words[0], 1u);
  __syncthreads();
  if (s_ticket != gridDim.x * gridDim.y - 1 || !char_totals) return;
  __threadfence();
  int bad = 0;
  for (int b = threadIdx.x; b < q.parts; b += kGsThreads) bad |= q.bad_part[b];
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) char_totals[q.ncols] = (*reinterpret_cast<volatile uint32_t*>(&q.sync_words[1])) | (bad ? 1u : 0u);
}

// ---- host side -----------------------------------------------------------------------------------------
// Plans the slabs of a schema.  Returns false (wide.enabled stays false) when the schema is not a wide
// variable-width table or the kernel's tables would not fit shared memory.
bool plan_wide(srj_plan* plan)
{
  WidePlan& wp = plan->wide;
  wp.enabled   = false;
  const int nc = plan->num_columns, nstr = plan->num_string_columns;
  const int spr      = plan->size_per_row;
  if (nstr < 8 || spr < 512 || nc > kWMaxCols) return false;
  const int slab_cap = 3200;
  int nslabs         = (spr + slab_cap - 1) / slab_cap;
  nslabs             = std::max(1, std::min(nslabs, 16));
  // first column of each slab: the first one starting at or after i * spr / nslabs
  std::vector<int> first(nslabs + 1, nc);
  first[0] = 0;
  for (int i = 1, c = 0; i < nslabs; ++i) {
    const int target = static_cast<int>(static_cast<int64_t>(i) * spr / nslabs);
    while (c < nc && plan->col_start[c] < target) ++c;
    first[i] = c;
  }
  std::vector<int> sidx_of(nc, -1);
  for (int s = 0; s < nstr; ++s) sidx_of[plan->string_columns[s]] = s;
  wp.entries.clear();
  wp.slabs.assign(nslabs, WideSlab{});
  int maxlen = 0;
  for (int i = 0; i < nslabs; ++i) {
    WideSlab& sl = wp.slabs[i];
    const int c0 = first[i], c1 = first[i + 1];
    int begin = c0 < nc ? plan->col_start[c0] : plan->validity_offset;
    int end   = begin;
    for (int c = c0; c < c1; ++c) end = std::max(end, plan->col_start[c] + plan->col_size[c]);
    // the pair before the slab's first STRING column must be staged too (canonical-layout check)
    for (int c = c0; c < c1; ++c)
      if (sidx_of[c] > 0) {
        begin = std::min(begin, plan->col_start[plan->string_columns[sidx_of[c] - 1]]);
        break;
      }
    if (i == nslabs - 1) end = spr;  // validity bytes
    const int nominal = c0 < nc ? plan->col_start[c0] : plan->validity_offset;
    if (nominal - begin > 128) return false;  // sparse strings: the whole-row kernel serves this schema
    sl.begin = begin & ~7;
    sl.end   = (end + 7) & ~7;
    maxlen   = std::max(maxlen, sl.end - sl.begin);
    // entries of the slab by width class 16, 8, 4, 2, 1, STRING
    for (int k = 0; k < 6; ++k) {
      sl.cb[k] = static_cast<int32_t>(wp.entries.size());
      for (int c = c0; c < c1; ++c) {
        const bool str = sidx_of[c] >= 0;
        const int want = k < 5 ? (16 >> k) : 0;
        if (str ? (k == 5) : (k < 5 && plan->col_size[c] == want))
          wp.entries.push_back(WideEntry{plan->col_start[c], c, sidx_of[c], i});
      }
    }
    sl.cb[6] = static_cast<int32_t>(wp.entries.size());
  }
  int pitch = (maxlen + 16 + 15) & ~15;
  if (((pitch >> 4) & 1) == 0) pitch += 16;  // odd multiple of 16 bytes: consecutive rows start 4 banks apart
  const size_t tables = wp.entries.size() * sizeof(WDesc) + kWMaxStages * sizeof(WHdr) + 2 * kWMaxStages * 8 +
                        static_cast<size_t>(nc) * 12 + nslabs * sizeof(WideSlab) + static_cast<size_t>(nstr) * 4 +
                        static_cast<size_t>(nslabs) * 6 * 16 * 2 + 256;
  const size_t budget = 232448;
  if (tables > 64 * 1024) return false;
  int NS = 3;  // two when three would leave tiles of fewer than 64 rows
  int R  = 0;
  for (;;) {
    const size_t avail = budget - tables;
    const size_t per   = static_cast<size_t>(pitch) + 4;  // payload + row position
    R                  = static_cast<int>((avail / NS - kWSlack) / per) / 32 * 32;
    if (R >= 64 || NS == 2) break;
    --NS;
  }
  R = std::min(R, 32 * kWMaxG);
  if (R < 32) return false;
  wp.R       = R;
  wp.G       = R / 32;
  wp.pitch   = pitch;
  wp.nstages = NS;
  wp.nslabs  = nslabs;
  wp.enabled = true;
  return true;
}

size_t wide_plan_blob_bytes(const srj_plan* plan)
{
  return plan->wide.enabled ? plan->wide.entries.size() * sizeof(WideEntry) + plan->wide.slabs.size() * sizeof(WideSlab) + 16 : 0;
}

// Workspace of a convert_from_rows call pair (srj_from_rows_workspace_bytes): group totals and group bases of the
// STRING columns (phase 2 reads the bases), per-CTA null counts and flags, two sync words.
static int64_t wide_groups_bytes(const srj_plan* plan, int64_t num_rows)
{
  return (static_cast<int64_t>(plan->num_string_columns) * ((num_rows + 31) / 32) * 4 + 15) & ~int64_t{15};
}
int64_t wide_workspace_bytes(const srj_plan* plan, int64_t num_rows)
{
  return 2 * wide_groups_bytes(plan, num_rows) + static_cast<int64_t>(kWMaxGrid) * (plan->num_columns + 1) * 4 + 16;
}
const uint32_t* wide_workspace_bases(const srj_plan* plan, int64_t num_rows, const void* workspace)
{
  return reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(workspace) + wide_groups_bytes(plan, num_rows));
}

static size_t wide_smem_bytes(const srj_plan* plan)
{
  const WidePlan& wp = plan->wide;
  size_t b           = static_cast<size_t>(wp.nstages) * (static_cast<size_t>(wp.R) * wp.pitch + kWSlack);
  b += wp.entries.size() * sizeof(WDesc) + static_cast<size_t>(wp.nstages) * sizeof(WHdr) + 2 * kWMaxStages * 8;
  b += static_cast<size_t>(plan->num_columns) * 8 + wp.slabs.size() * sizeof(WideSlab);
  b += static_cast<size_t>(wp.nstages) * wp.R * 4 + static_cast<size_t>(plan->num_columns) * 4;
  b += static_cast<size_t>(plan->num_string_columns) * 4;
  b += wp.slabs.size() * 6 * 16 * 2 + 16;  // first-unit table (<= 16 consumer warps)
  return (b + 127) & ~size_t{127};
}

template <int NCW>
static int launch_wide_variant(const WideParams& p, const WidePtrTab& tab, unsigned grid, size_t smem, cudaStream_t stream)
{
  auto go = [&](auto kern) -> int {
    SRJ_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    kern<<<grid, (NCW + kWProducers) * 32, smem, stream>>>(p, tab);
    return SRJ_OK;
  };
  switch (p.G) {
    case 1: return go(from_rows_wide_kernel<NCW, 1>);
    case 2: return go(from_rows_wide_kernel<NCW, 2>);
    case 3: return go(from_rows_wide_kernel<NCW, 3>);
    default: return go(from_rows_wide_kernel<NCW, 4>);
  }
}

// cols: the caller's output columns (host array).  d_scratch: the call pair's workspace (wide_workspace_bytes()).
int launch_from_rows_wide(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets, int64_t rows_bytes,
                          int64_t num_rows, const srj_column* cols, int64_t* d_null_counts, int64_t* d_char_totals,
                          void* d_scratch, cudaStream_t stream)
{
  if (num_rows == 0) return SRJ_OK;
  const WidePlan& wp = plan->wide;
  const int nc = plan->num_columns, nstr = plan->num_string_columns;
  int dev = 0, nsm = 0;
  SRJ_CUDA_TRY(cudaGetDevice(&dev));
  SRJ_CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  const int64_t ntiles = (num_rows + wp.R - 1) / wp.R;
  const unsigned grid  = static_cast<unsigned>(std::min<int64_t>(std::min(nsm, kWMaxGrid), ntiles));
  WidePtrTab tab;
  WideScanTab stab;
  for (int c = 0; c < nc; ++c) {
    tab.col[c]  = plan->type_ids[c] == SRJ_STRING ? static_cast<void*>(cols[c].offsets) : cols[c].data;
    tab.mask[c] = cols[c].null_mask;
  }
  for (int s = 0; s < nstr; ++s) {
    stab.offs[s] = cols[plan->string_columns[s]].offsets;
    stab.scol[s] = plan->string_columns[s];
  }
  WideParams p{};
  p.rows            = rows;
  p.row_offsets     = row_offsets;
  p.rows_bytes      = rows_bytes;
  p.num_rows        = num_rows;
  p.ngroups         = (num_rows + 31) / 32;
  p.ncols           = nc;
  p.nstr            = nstr;
  p.size_per_row    = plan->size_per_row;
  p.validity_offset = plan->validity_offset;
  p.R               = wp.R;
  p.G               = wp.G;
  p.pitch           = wp.pitch;
  p.nstages         = wp.nstages;
  p.nslabs          = wp.nslabs;
  p.nent            = static_cast<int32_t>(wp.entries.size());
  p.entries         = wp.d_entries;
  p.slabs           = wp.d_slabs;
  p.string_start    = plan->d_string_start;
  p.want_nulls      = d_null_counts != nullptr;
  uint8_t* sc       = static_cast<uint8_t*>(d_scratch);
  const int64_t agg_bytes = wide_groups_bytes(plan, num_rows);
  p.agg             = reinterpret_cast<uint32_t*>(sc);
  uint32_t* d_base  = reinterpret_cast<uint32_t*>(sc + agg_bytes);
  p.null_part       = reinterpret_cast<int32_t*>(sc + 2 * agg_bytes);
  p.bad_part        = p.null_part + static_cast<size_t>(kWMaxGrid) * nc;
  p.sync_words      = reinterpret_cast<uint32_t*>(p.bad_part + kWMaxGrid);
  const size_t smem = wide_smem_bytes(plan);
  const int rc = launch_wide_variant<12>(p, tab, grid, smem, stream);
  if (rc != SRJ_OK) return rc;
  WideScanParams q{};
  q.agg         = p.agg;
  q.base        = d_base;
  q.ngroups     = p.ngroups;
  q.num_rows    = num_rows;
  q.char_totals = d_char_totals;
  q.null_counts = d_null_counts;
  q.null_part   = p.null_part;
  q.bad_part    = p.bad_part;
  q.sync_words  = p.sync_words;
  q.parts       = static_cast<int32_t>(grid);
  q.ncols       = nc;
  q.nstr        = nstr;
  for (int s2 = 0; s2 < nstr; ++s2) q.str_bits[plan->string_columns[s2] >> 6] |= 1ull << (plan->string_columns[s2] & 63);
  const int64_t nchunks = (p.ngroups + kGsChunk - 1) / kGsChunk;
  wide_group_scan_kernel<<<dim3(static_cast<unsigned>(nchunks), nstr), kGsThreads, 0, stream>>>(q, stab);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj
