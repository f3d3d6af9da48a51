// zorder.cu -- ZOrder.interleaveBits and ZOrder.hilbertIndex on the device (reference zorder.cu, ZOrder.java):
// Delta Lake's InterleaveBits (OPTIMIZE ... ZORDER BY) and Skilling's Hilbert index for Hilbert clustering.
//
// Both produce, per row, the bit stream of N values of B bits each read MSB first and column-interleaved: stream
// position i holds bit B - 1 - i / N of value i % N.  interleaveBits writes that stream as the row's N * W bytes
// (B = 8W, byte 0 = positions 0..7); hilbertIndex reads its N * numBits <= 64 positions as an integer.
//
// interleave_word builds 32 positions of the stream at a time.  The positions of value c inside one word are u, u + N,
// u + 2N, ... (u < min(N, 32)), so each value contributes one run of at most ceil(32 / N) consecutive bits.  The run is
// cut out with one shift and spread to stride N by log2(ceil(32 / N)) shift / mask steps whose masks depend on N only
// (computed on the host): the GPU has no PDEP.  A row has ceil(N * W / 4) words of min(N, 32) steps each: O(N^2 * W / 4)
// steps for N <= 32 (one per value and word), one step per output bit beyond that.
//
// interleave_bits_kernel: lane = row, a warp owns 32 consecutive rows, i.e. one contiguous span of 32 * N * W output
// bytes.  Values are loaded with lane = row (coalesced), validity with one mask word per 32 rows and column.  When a row
// has at most kStageBytes bytes the warp builds its span in shared memory (big-endian words from PRMT) and writes it with
// 16-byte stores; wider rows go straight to global memory a word at a time.  The kernel also writes the offsets r * N * W.
// Tables wider than kZColsPerLaunch columns (rows of > 128 bytes, so never staged) take one launch per column chunk;
// the later launches OR their bits into the words the earlier ones wrote.
//
// hilbert_index_kernel: lane = row.  Skilling, "Programming the Hilbert curve" (AIP Conf. Proc. 707, 2004):
// AxesToTranspose (inverse undo, then Gray encode), then the transposed coordinates are read out through the same
// interleave_word with B = numBits.  The N <= 64 coordinates of N * numBits <= 64 bits live in two registers: X[0] and a
// 64-bit word holding X[1..N-1] at numBits-bit strides, indexed by shifts (no local memory).
#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"

namespace srj {
namespace {

constexpr int kZThreads       = 256;
constexpr int kZWarps         = kZThreads / 32;
constexpr int kStageBytes     = 128;   // rows up to this many bytes are staged per warp in shared memory (4 KB per warp)
constexpr int kZColsPerLaunch = 224;   // column descriptors per launch (kernel parameters stay under 4 KB)
constexpr int kHilbertMaxCols = 64;    // numBits >= 1 and N * numBits <= 64

// What interleave_word needs to know about N (host-computed, srj::zorder_spread)
struct ZSpread {
  int32_t n;          // values per row
  int32_t steps;      // dilation steps: ceil(log2(ceil(32 / N)))
  int32_t n32, j32;   // 32 % N and 32 / N: moving one word along the stream
  uint32_t mask[5];   // step s: x = (x | x << shift[s]) & mask[s], s from steps - 1 down to 0
  int32_t shift[5];
  uint8_t k[32];      // k[u] = ceil((32 - u) / N): stream positions of one value in a word whose first is at u
};

struct ZCol {
  const uint8_t* data;
  const uint32_t* mask;
};

struct InterleaveParams {
  ZCol cols[kZColsPerLaunch];   // columns [c_begin, c_end) of this launch
  ZSpread sp;
  int32_t c_begin, c_end;
  int32_t row_bytes;            // N * W
  int32_t first;                // 1: writes every byte; 0: ORs into the bytes of an earlier launch
  int64_t rows;
  int32_t* offsets;             // rows + 1 entries (first launch only, else NULL); may be unaligned
  uint8_t* out;
};

struct HilbertParams {
  ZCol cols[kHilbertMaxCols];
  ZSpread sp;
  int32_t bits;
  int32_t pad;
  int64_t rows;
  uint8_t* out;                 // int64 per row; may be unaligned
};

// Spread the low bits of x to stride N (bit i -> bit i * N), for x < 2^ceil(32 / N)
__device__ __forceinline__ uint32_t dilate(uint32_t x, const ZSpread& sp)
{
#pragma unroll
  for (int s = 4; s >= 0; --s)
    if (s < sp.steps) x = (x | (x << sp.shift[s])) & sp.mask[s];
  return x;
}

// Stream positions [32k, 32k + 32) of a row as a word whose bit 31 is position 32k.  c0 = 32k % N and j00 = 32k / N.
// get(c, lo, K) returns bits [lo, lo + K) of value c (LSB-indexed), K <= 32.  Positions past the last value bit are 0.
template <class Get>
__device__ __forceinline__ uint32_t interleave_word(const Get& get, const ZSpread& sp, int vbits, int c0, int j00)
{
  const int n   = sp.n;
  const int lim = n < 32 ? n : 32;
  uint32_t w    = 0;
  for (int u = 0; u < lim; ++u) {
    int c  = c0 + u;
    int j0 = j00;            // MSB-first index of the first bit of value c in this word
    if (c >= n) {
      c -= n;
      ++j0;
    }
    const int K = min(static_cast<int>(sp.k[u]), vbits - j0);
    if (K <= 0) continue;
    const uint32_t e = get(c, vbits - j0 - K, K);
    w |= dilate(e, sp) << (31 - u - (K - 1) * n);
  }
  return w;
}

__device__ __forceinline__ uint32_t low_bits(int K) { return K >= 32 ? ~0u : (1u << K) - 1u; }

template <int W>
struct ZValue;
template <> struct ZValue<1> { using T = uint32_t; __device__ static T load(const uint8_t* p, int64_t r) { return __ldg(p + r); } };
template <> struct ZValue<2> {
  using T = uint32_t;
  __device__ static T load(const uint8_t* p, int64_t r) { return __ldg(reinterpret_cast<const uint16_t*>(p) + r); }
};
template <> struct ZValue<4> {
  using T = uint32_t;
  __device__ static T load(const uint8_t* p, int64_t r) { return __ldg(reinterpret_cast<const uint32_t*>(p) + r); }
};
template <> struct ZValue<8> {
  using T = uint64_t;
  __device__ static T load(const uint8_t* p, int64_t r) { return __ldg(reinterpret_cast<const unsigned long long*>(p) + r); }
};
template <> struct ZValue<16> {   // two 8-byte loads: the column needs 8-byte alignment only
  using T = unsigned __int128;
  __device__ static T load(const uint8_t* p, int64_t r)
  {
    const auto* q = reinterpret_cast<const unsigned long long*>(p) + 2 * r;
    return (static_cast<T>(__ldg(q + 1)) << 64) | __ldg(q);
  }
};

__device__ __forceinline__ void store_i32(int32_t* p, int32_t v)
{
  if ((reinterpret_cast<uintptr_t>(p) & 3) == 0) {
    *p = v;
  } else {
    auto* b = reinterpret_cast<uint8_t*>(p);
#pragma unroll
    for (int i = 0; i < 4; ++i) b[i] = static_cast<uint8_t>(static_cast<uint32_t>(v) >> (8 * i));
  }
}

template <int W>
__global__ void __launch_bounds__(kZThreads) interleave_bits_kernel(const __grid_constant__ InterleaveParams p)
{
  __shared__ __align__(16) uint8_t stage[kZWarps][32 * kStageBytes + 16];
  using T            = typename ZValue<W>::T;
  const int lane     = threadIdx.x & 31;
  const int warp     = threadIdx.x >> 5;
  const int64_t r0   = (static_cast<int64_t>(blockIdx.x) * kZWarps + warp) * 32;
  if (r0 >= p.rows) return;                                    // the whole warp leaves together
  const int64_t r    = r0 + lane;
  const bool live    = r < p.rows;
  const int rb       = p.row_bytes;
  const bool staged  = rb <= kStageBytes;
  uint8_t* const g0  = p.out + r0 * rb;                        // the warp's span
  if (p.offsets && live) {
    store_i32(p.offsets + r, static_cast<int32_t>(r * rb));
    if (r == p.rows - 1) store_i32(p.offsets + r + 1, static_cast<int32_t>((r + 1) * rb));
  }
  // shared-memory byte of global address a: a - (g0 & ~15), so that 16-byte-aligned global words are aligned here too
  uint8_t* const st   = stage[warp];
  const int st_row    = static_cast<int>(reinterpret_cast<uintptr_t>(g0) & 15) + lane * rb;

  // bits [lo, lo + K) of the value of column c in this row; a null is 0 (one mask word per 32 rows and column)
  auto get = [&](int c, int lo, int K) -> uint32_t {
    if (c < p.c_begin || c >= p.c_end) return 0u;
    const ZCol& col = p.cols[c - p.c_begin];
    if (col.mask && !((__ldg(col.mask + (r0 >> 5)) >> lane) & 1u)) return 0u;
    const T v = ZValue<W>::load(col.data, r);
    return static_cast<uint32_t>(v >> lo) & low_bits(K);
  };

  const int nwords = (rb + 3) >> 2;
  int c0 = 0, j00 = 0;
  for (int k = 0; k < nwords; ++k) {
    if (live) {
      const uint32_t w = interleave_word(get, p.sp, 8 * W, c0, j00);
      const int nb     = min(4, rb - 4 * k);
      if (staged) {
        uint8_t* d = st + st_row + 4 * k;
        if (nb == 4 && (reinterpret_cast<uintptr_t>(d) & 3) == 0) {
          *reinterpret_cast<uint32_t*>(d) = __byte_perm(w, 0, 0x0123);   // big-endian
        } else {
          for (int i = 0; i < nb; ++i) d[i] = static_cast<uint8_t>(w >> (24 - 8 * i));
        }
      } else if (p.first || w) {
        uint8_t* d = g0 + static_cast<int64_t>(lane) * rb + 4 * k;
        if (nb == 4 && (reinterpret_cast<uintptr_t>(d) & 3) == 0) {
          auto* d4 = reinterpret_cast<uint32_t*>(d);
          *d4      = __byte_perm(w, 0, 0x0123) | (p.first ? 0u : *d4);
        } else {
          for (int i = 0; i < nb; ++i) d[i] = static_cast<uint8_t>(w >> (24 - 8 * i)) | (p.first ? 0 : d[i]);
        }
      }
    }
    c0 += p.sp.n32;
    j00 += p.sp.j32;
    if (c0 >= p.sp.n) {
      c0 -= p.sp.n;
      ++j00;
    }
  }
  if (!staged) return;
  __syncwarp();
  const int64_t span  = tmin<int64_t>(32, p.rows - r0) * rb;
  const uintptr_t gb  = reinterpret_cast<uintptr_t>(g0);
  const uintptr_t ge  = gb + static_cast<uintptr_t>(span);
  const uintptr_t sb  = gb & ~uintptr_t{15};
  const uintptr_t a0  = (gb + 15) & ~uintptr_t{15};
  const uintptr_t a1  = ge & ~uintptr_t{15};
  for (uintptr_t a = gb + lane; a < tmin(a0, ge); a += 32) *reinterpret_cast<uint8_t*>(a) = st[a - sb];
  for (uintptr_t a = a0 + 16 * lane; a < a1; a += 512)
    *reinterpret_cast<uint4*>(a) = *reinterpret_cast<const uint4*>(st + (a - sb));
  for (uintptr_t a = tmax(a0, a1) + lane; a < ge; a += 32) *reinterpret_cast<uint8_t*>(a) = st[a - sb];
}

__global__ void __launch_bounds__(kZThreads) hilbert_index_kernel(const __grid_constant__ HilbertParams p)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kZThreads + threadIdx.x;
  if (r >= p.rows) return;
  const int b          = p.bits;
  const int n          = p.sp.n;
  const uint32_t vmask = low_bits(b);
  // X[0] in x0; X[i] (i >= 1) in bits [(i - 1) * b, i * b) of xs
  uint32_t x0 = 0;
  uint64_t xs = 0;
  for (int c = 0; c < n; ++c) {
    const ZCol& col = p.cols[c];
    const bool ok   = !col.mask || ((__ldg(col.mask + (r >> 5)) >> (r & 31)) & 1u);
    const uint32_t v = ok ? __ldg(reinterpret_cast<const uint32_t*>(col.data) + r) & vmask : 0u;
    if (c == 0) x0 = v;
    else xs |= static_cast<uint64_t>(v) << ((c - 1) * b);
  }
  auto X = [&](int i) -> uint32_t { return i == 0 ? x0 : static_cast<uint32_t>(xs >> ((i - 1) * b)) & vmask; };

  // AxesToTranspose, inverse undo: for Q = 2^(b-1) .. 2, for each axis i: invert the low bits of X[0] when bit Q of
  // X[i] is set, else exchange the low bits of X[0] and X[i]
  for (int q = b - 1; q >= 1; --q) {
    const uint32_t Q = 1u << q, P = Q - 1u;
    if (x0 & Q) x0 ^= P;                                         // i = 0: the exchange with itself does nothing
    for (int i = 1; i < n; ++i) {
      const uint32_t xi = X(i);
      if (xi & Q) {
        x0 ^= P;
      } else {
        const uint32_t t = (x0 ^ xi) & P;
        x0 ^= t;
        xs ^= static_cast<uint64_t>(t) << ((i - 1) * b);
      }
    }
  }
  // Gray encode: X[i] ^= X[i - 1] in order, then every axis ^= t
  uint32_t prev = x0;
  for (int i = 1; i < n; ++i) {
    xs ^= static_cast<uint64_t>(prev) << ((i - 1) * b);
    prev = X(i);
  }
  uint32_t t = 0;
  for (int q = b - 1; q >= 1; --q)
    if (prev & (1u << q)) t ^= (1u << q) - 1u;
  x0 ^= t;
  for (int i = 1; i < n; ++i) xs ^= static_cast<uint64_t>(t) << ((i - 1) * b);

  auto get = [&](int c, int lo, int K) -> uint32_t { return (X(c) >> lo) & low_bits(K); };
  const int total  = n * b;
  const uint32_t h = interleave_word(get, p.sp, b, 0, 0);
  const uint32_t l = total > 32 ? interleave_word(get, p.sp, b, p.sp.n32, p.sp.j32) : 0u;
  const uint64_t v = ((static_cast<uint64_t>(h) << 32) | l) >> (64 - total);
  uint8_t* d       = p.out + 8 * r;
  if ((reinterpret_cast<uintptr_t>(d) & 7) == 0) {
    *reinterpret_cast<uint64_t*>(d) = v;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) d[i] = static_cast<uint8_t>(v >> (8 * i));
  }
}

ZSpread zorder_spread(int32_t n)
{
  ZSpread sp{};
  sp.n           = n;
  sp.n32         = 32 % n;
  sp.j32         = 32 / n;
  const int kmax = (32 + n - 1) / n;
  while ((1 << sp.steps) < kmax) ++sp.steps;
  for (int s = 0; s < sp.steps; ++s) {
    const int g = 1 << s;
    uint32_t m  = 0;
    for (int i = 0; i < kmax; ++i) m |= 1u << (i + (i & ~(g - 1)) * (n - 1));   // where bit i sits after step s
    sp.mask[s]  = m;
    sp.shift[s] = g * (n - 1);
  }
  for (int u = 0; u < 32 && u < n; ++u) sp.k[u] = static_cast<uint8_t>((31 - u) / n + 1);
  return sp;
}

}  // namespace

// out_offsets: rows + 1 int32 (r * ncols * elem_bytes); out: rows * ncols * elem_bytes bytes.  Either may be unaligned.
static int launch_interleave_bits(const srj_column* cols, int32_t ncols, int64_t rows, int32_t elem_bytes, int32_t* out_offsets, uint8_t* out,
                           cudaStream_t stream)
{
  if (rows == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(out_offsets, 0, 4, stream));
    return SRJ_OK;
  }
  InterleaveParams p{};
  p.sp        = zorder_spread(ncols);
  p.row_bytes = ncols * elem_bytes;
  p.rows      = rows;
  p.out       = out;
  const int64_t tiles = (rows + 31) / 32;
  const unsigned grid = static_cast<unsigned>((tiles + kZWarps - 1) / kZWarps);
  for (int32_t c0 = 0; c0 < ncols; c0 += kZColsPerLaunch) {
    p.c_begin = c0;
    p.c_end   = tmin(ncols, c0 + kZColsPerLaunch);
    p.first   = c0 == 0;
    p.offsets = c0 == 0 ? out_offsets : nullptr;
    for (int32_t c = p.c_begin; c < p.c_end; ++c)
      p.cols[c - c0] = ZCol{static_cast<const uint8_t*>(cols[c].data), cols[c].null_mask};
    switch (elem_bytes) {
      case 1: interleave_bits_kernel<1><<<grid, kZThreads, 0, stream>>>(p); break;
      case 2: interleave_bits_kernel<2><<<grid, kZThreads, 0, stream>>>(p); break;
      case 4: interleave_bits_kernel<4><<<grid, kZThreads, 0, stream>>>(p); break;
      case 8: interleave_bits_kernel<8><<<grid, kZThreads, 0, stream>>>(p); break;
      default: interleave_bits_kernel<16><<<grid, kZThreads, 0, stream>>>(p); break;
    }
    SRJ_CUDA_TRY(cudaGetLastError());
  }
  return SRJ_OK;
}

static int launch_hilbert_index(int32_t num_bits, const srj_column* cols, int32_t ncols, int64_t rows, int64_t* out, cudaStream_t stream)
{
  if (rows == 0) return SRJ_OK;
  HilbertParams p{};
  p.sp   = zorder_spread(ncols);
  p.bits = num_bits;
  p.rows = rows;
  p.out  = reinterpret_cast<uint8_t*>(out);
  for (int32_t c = 0; c < ncols; ++c) p.cols[c] = ZCol{static_cast<const uint8_t*>(cols[c].data), cols[c].null_mask};
  hilbert_index_kernel<<<static_cast<unsigned>((rows + kZThreads - 1) / kZThreads), kZThreads, 0, stream>>>(p);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

// zorder.cu:141-159: at least one column, fixed-width, one type id, the output within INT32_MAX bytes (a logic_error in
// the reference, so SRJ_EINVAL rather than SRJ_EOVERFLOW).  *elem_bytes = W.
static int interleave_check(const char* what, const srj_column* cols, int32_t n, int64_t rows, int32_t* elem_bytes)
{
  if (n <= 0 || !cols) { set_error("%s: The input table must have at least one column.", what); return SRJ_EINVAL; }
  if (rows < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  const int32_t w = type_width(cols[0].type_id);
  if (w == 0) { set_error("%s: Only fixed width columns can be used (type id %d)", what, cols[0].type_id); return SRJ_EUNSUPPORTED; }
  for (int32_t c = 0; c < n; ++c)
    if (cols[c].type_id != cols[0].type_id) { set_error("%s: All columns of the input table must be the same type.", what); return SRJ_EINVAL; }
  if (check_rows(what, cols, n, rows) != SRJ_OK) return SRJ_EINVAL;
  if (rows * static_cast<int64_t>(w) * n > INT32_MAX) { set_error("%s: Input is too large to process", what); return SRJ_EINVAL; }
  *elem_bytes = w;
  return SRJ_OK;
}

int srj_interleave_bits_sizes(const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t* total_bytes)
{
  SRJ_API_RANGE();
  if (!total_bytes) { set_error("interleave_bits_sizes: bad argument"); return SRJ_EINVAL; }
  int32_t w    = 0;
  const int rc = interleave_check("interleave_bits_sizes", cols, num_columns, num_rows, &w);
  if (rc != SRJ_OK) return rc;
  *total_bytes = num_rows * w * num_columns;
  return SRJ_OK;
}

int srj_interleave_bits(const srj_column* cols, int32_t num_columns, int64_t num_rows, int32_t* out_offsets, uint8_t* out_bytes, void* stream)
{
  SRJ_API_RANGE();
  int32_t w = 0;
  int rc    = interleave_check("interleave_bits", cols, num_columns, num_rows, &w);
  if (rc != SRJ_OK) return rc;
  for (int32_t c = 0; c < num_columns; ++c)
    if ((rc = check_data("interleave_bits", "column", cols[c], c)) != SRJ_OK) return rc;
  if ((rc = check_out("interleave_bits", "output offsets", out_offsets, 1)) != SRJ_OK) return rc;
  if ((rc = check_out("interleave_bits", "output bytes", out_bytes, 1, num_rows > 0)) != SRJ_OK) return rc;
  return launch_interleave_bits(cols, num_columns, num_rows, w, out_offsets, out_bytes, static_cast<cudaStream_t>(stream));
}

// zorder.cu:226-237
int srj_hilbert_index(int32_t num_bits, const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "hilbert_index";
  if (num_bits <= 0 || num_bits > 32) { set_error("%s: the number of bits must be >0 and <= 32.", what); return SRJ_EINVAL; }
  if (static_cast<int64_t>(num_bits) * num_columns > 64) { set_error("%s: we only support up to 64 bits of output right now.", what); return SRJ_EINVAL; }
  if (num_columns <= 0 || !cols) { set_error("%s: at least one column is required.", what); return SRJ_EINVAL; }
  if (num_rows < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  for (int32_t c = 0; c < num_columns; ++c) {
    if (cols[c].type_id != SRJ_INT32) { set_error("%s: All columns of the input table must be INT32.", what); return SRJ_EUNSUPPORTED; }
    if (cols[c].size != num_rows) { set_error("%s: column %d has %lld rows, expected %lld", what, c, static_cast<long long>(cols[c].size), static_cast<long long>(num_rows)); return SRJ_EINVAL; }
  }
  int rc = SRJ_OK;
  for (int32_t c = 0; c < num_columns; ++c)
    if ((rc = check_data(what, "column", cols[c], c)) != SRJ_OK) return rc;
  if ((rc = check_out(what, "output", out, 1, num_rows > 0)) != SRJ_OK) return rc;
  return launch_hilbert_index(num_bits, cols, num_columns, num_rows, out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
