// kudo.cu -- the reference's Kudo shuffle wire format for flat tables (SURVEY §8f rank 2): split a table at row indices
// into P self-describing partitions laid back to back in one buffer (shuffle_split, src/main/cpp/src/shuffle_split.hpp:60-136,
// shuffle_split.cu:640-690,940-1075) and assemble such partitions back into one table (shuffle_assemble,
// shuffle_split.hpp:174-189).  The bytes are the format of kudo/KudoSerializer.java:49-171:
//   partition = header | hasValidity bits | validity | offsets | data
//   header    = "KUD0", row offset, row count, validity length, offsets length, total length, column count: seven
//               BIG-ENDIAN 32-bit integers (kudo/KudoTableHeader.java:186-200); then (ncols + 7) / 8 bytes, bit c = column
//               c carries validity in this partition (it has a mask and the partition has rows)
//   validity  = per such column the mask bytes [row / 8, (row + n - 1) / 8] copied as they are (the reader skips row % 8
//               bits, kudo/SlicedValidityBufferInfo.java:63-77); the section is padded so that header + validity is a
//               multiple of 4 (KudoSerializer.java:497-499)
//   offsets   = per STRING column the n + 1 raw int32 offsets (not rebased), when n > 0; data = per column n * size bytes
//               or the chars; both sections padded to 4
// Flat tables only (fixed-width, decimals, STRING): the nested walk of the reference is not restated.
//
// Kernels: a thread per partition sizes it (and, for assemble, parses its header); one CTA per (column, partition)
// moves that column's three buffers with the widest accesses the two addresses allow; validity bits of assembled
// partitions reach the output words with atomicOr (a partition starts at an arbitrary row).
#include <algorithm>
#include <vector>

#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"

namespace srj {

constexpr int kKudoMaxCols   = 256;
constexpr uint32_t kKudoMagic = 0x4B554430u;

struct KCol {
  uint8_t* data;        // fixed-width values or chars
  uint8_t* mask;        // validity bytes (bit r%8 of byte r/8), or NULL
  int32_t* offsets;     // STRING
  int32_t size;         // element bytes, 0 for STRING
  int32_t sidx;         // index among the STRING columns, or -1
};

__host__ __device__ __forceinline__ int64_t pad4(int64_t x) { return (x + 3) & ~int64_t{3}; }
__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }
__host__ __device__ __forceinline__ int kudo_header_bytes(int ncols) { return 28 + (ncols + 7) / 8; }

// bytes of the three buffers of column c for rows [s, s + n)
__device__ __forceinline__ void kudo_col_sizes(const KCol& c, int32_t s, int32_t n, int64_t& v, int64_t& o, int64_t& d)
{
  v = (c.mask && n > 0) ? (s + n - 1) / 8 - s / 8 + 1 : 0;
  if (c.size == 0) {
    o = n > 0 ? 4 * (static_cast<int64_t>(n) + 1) : 0;
    d = c.offsets ? static_cast<int64_t>(c.offsets[s + n]) - c.offsets[s] : 0;
  } else {
    o = 0;
    d = static_cast<int64_t>(n) * c.size;
  }
}

// cooperative byte copy by the CTA.  The destination is written with aligned 16-byte stores; the source is read with
// aligned 16-byte loads when it is congruent to the destination mod 16, else as aligned 32-bit words funnel-shifted
// into place (the buffers of a Kudo partition have no alignment guarantees: KudoSerializer.java:157-159).
__device__ void cta_copy_bytes(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, int64_t n)
{
  const int tid = threadIdx.x, nt = blockDim.x;
  if (n <= 0) return;
  const uintptr_t da = reinterpret_cast<uintptr_t>(dst);
  const int64_t head = tmin<int64_t>(n, (16 - (da & 15)) & 15);
  for (int64_t i = tid; i < head; i += nt) dst[i] = src[i];
  const uintptr_t sa = reinterpret_cast<uintptr_t>(src + head);
  int64_t body       = (n - head) >> 4;
  uint4* d16         = reinterpret_cast<uint4*>(dst + head);
  if ((sa & 15) == 0) {
    const uint4* s16 = reinterpret_cast<const uint4*>(src + head);
    for (int64_t i = tid; i < body; i += nt) d16[i] = s16[i];
  } else {
    if (body > 0) --body;   // the last chunk's fifth word could lie past the source: it goes with the tail bytes
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(sa & ~uintptr_t{3});
    const uint32_t sh  = static_cast<uint32_t>(sa & 3) * 8u;
    for (int64_t i = tid; i < body; i += nt) {
      const uint32_t* w = sw + 4 * i;
      const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
      d16[i] = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
    }
  }
  for (int64_t i = head + body * 16 + tid; i < n; i += nt) dst[i] = src[i];
}

// ---- split ---------------------------------------------------------------------------------------------------------------
// *bad: bit 0 = a partition too large for the header, or splits not increasing; bit 1 = a split outside [0, num_rows]
__global__ void __launch_bounds__(256) kudo_split_sizes_kernel(const KCol* __restrict__ cols, int ncols, const int32_t* __restrict__ splits, int P,
                                                              int64_t num_rows, int64_t* __restrict__ part_sizes, int32_t* __restrict__ bad)
{
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= P) return;
  const int32_t s = splits[p], n = splits[p + 1] - s;
  // checked before any column is read: the STRING sizes read offsets[s] and offsets[s + n]
  if (s < 0 || splits[p + 1] > num_rows || n < 0) {
    part_sizes[p] = 0;
    atomicOr(bad, n < 0 ? 1 : 2);
    return;
  }
  int64_t V = 0, O = 0, D = 0;
  for (int c = 0; c < ncols; ++c) {
    int64_t v, o, d;
    kudo_col_sizes(cols[c], s, n, v, o, d);
    V += v;
    O += o;
    D += d;
  }
  const int hs  = kudo_header_bytes(ncols);
  part_sizes[p] = pad4(hs + V) + pad4(O) + pad4(D);
  // the header holds the section lengths as 32-bit integers (KudoTableHeaderCalc.java:70-77: toIntExact)
  if (pad4(hs + V) - hs + pad4(O) + pad4(D) > INT32_MAX) atomicOr(bad, 1);
}

// exclusive scan of P + 1 int64 in place by one CTA (P <= a few 10^4); element P receives the total
__global__ void __launch_bounds__(1024) i64_scan_small_kernel(int64_t* v, int n)
{
  __shared__ int64_t s_warp[32];
  __shared__ int64_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = lane_id(), w = warp_id();
  for (int b = 0; b < n + 1; b += 1024) {
    const int i     = b + threadIdx.x;
    const int64_t x = i < n ? v[i] : 0;
    int64_t inc     = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
      int64_t t = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += y;
      }
      s_warp[lane] = t;
    }
    __syncthreads();
    const int64_t base = s_carry + (w > 0 ? s_warp[w - 1] : 0);
    if (i <= n) v[i] = base + inc - x;
    __syncthreads();
    if (threadIdx.x == 0) s_carry += s_warp[31];
    __syncthreads();
  }
}

int launch_i64_scan_small(int64_t* v, int n, cudaStream_t stream)
{
  i64_scan_small_kernel<<<1, 1024, 0, stream>>>(v, n);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

__global__ void __launch_bounds__(256) kudo_split_kernel(const KCol* __restrict__ cols, int ncols, const int32_t* __restrict__ splits,
                                                        const int64_t* __restrict__ part_offsets, uint8_t* __restrict__ out)
{
  const int c = blockIdx.x, p = blockIdx.y;
  const int32_t s = splits[p], n = splits[p + 1] - s;
  const int hs   = kudo_header_bytes(ncols);
  uint8_t* part  = out + part_offsets[p];
  // where this column's buffers go: the sizes of the columns before it (and, for the section starts, of all columns)
  __shared__ int64_t s_pos[6];   // V, O, D before column c; V, O, D of the partition
  if (threadIdx.x == 0) {
    int64_t bv = 0, bo = 0, bd = 0, V = 0, O = 0, D = 0;
    for (int k = 0; k < ncols; ++k) {
      int64_t v, o, d;
      kudo_col_sizes(cols[k], s, n, v, o, d);
      if (k < c) { bv += v; bo += o; bd += d; }
      V += v; O += o; D += d;
    }
    s_pos[0] = bv; s_pos[1] = bo; s_pos[2] = bd; s_pos[3] = V; s_pos[4] = O; s_pos[5] = D;
  }
  __syncthreads();
  const int64_t V = s_pos[3], O = s_pos[4], D = s_pos[5];
  const int64_t vlen = pad4(hs + V) - hs, olen = pad4(O), dlen = pad4(D);
  uint8_t* v_at = part + hs;
  uint8_t* o_at = v_at + vlen;
  uint8_t* d_at = o_at + olen;
  if (c == 0) {
    // header (big endian), hasValidity bits, and the zero padding of the three sections
    if (threadIdx.x < 7) {
      const uint32_t f[7] = {kKudoMagic, static_cast<uint32_t>(s), static_cast<uint32_t>(n), static_cast<uint32_t>(vlen), static_cast<uint32_t>(olen),
                             static_cast<uint32_t>(vlen + olen + dlen), static_cast<uint32_t>(ncols)};
      reinterpret_cast<uint32_t*>(part)[threadIdx.x] = bswap32(f[threadIdx.x]);   // partitions start 4-byte aligned
    }
    for (int b = threadIdx.x; b < (ncols + 7) / 8; b += 256) {
      uint32_t bits = 0;
      for (int k = 8 * b; k < tmin(ncols, 8 * b + 8); ++k) bits |= (cols[k].mask && n > 0 ? 1u : 0u) << (k - 8 * b);
      part[28 + b] = static_cast<uint8_t>(bits);
    }
    if (threadIdx.x < 12) {
      const int sec     = threadIdx.x / 4, k = threadIdx.x % 4;
      uint8_t* end      = sec == 0 ? v_at + V : sec == 1 ? o_at + O : d_at + D;
      const int64_t pad = sec == 0 ? vlen - V : sec == 1 ? olen - O : dlen - D;
      if (k < pad) end[k] = 0;
    }
  }
  const KCol col = cols[c];
  int64_t v, o, d;
  kudo_col_sizes(col, s, n, v, o, d);
  if (v) cta_copy_bytes(v_at + s_pos[0], col.mask + s / 8, v);
  if (o) cta_copy_bytes(o_at + s_pos[1], reinterpret_cast<const uint8_t*>(col.offsets + s), o);
  if (d) cta_copy_bytes(d_at + s_pos[2], col.size ? col.data + static_cast<int64_t>(s) * col.size : col.data + col.offsets[s], d);
}

// ---- assemble ------------------------------------------------------------------------------------------------------------
struct KPartInfo {   // per partition, parsed from its header
  int32_t row_offset, rows, vlen, olen;
};

__device__ __forceinline__ uint32_t ld_be32(const uint8_t* p) { return (uint32_t{p[0]} << 24) | (uint32_t{p[1]} << 16) | (uint32_t{p[2]} << 8) | p[3]; }
__device__ __forceinline__ int32_t ld_le32(const uint8_t* p) { return static_cast<int32_t>(uint32_t{p[0]} | (uint32_t{p[1]} << 8) | (uint32_t{p[2]} << 16) | (uint32_t{p[3]} << 24)); }

// positions (from the start of the partition) of column c's buffers; *chars = bytes of its data buffer
__device__ void kudo_locate(const uint8_t* part, const KPartInfo& pi, const int32_t* sizes /* element size per column, 0 = STRING */, int ncols, int c,
                            bool* has_v, int64_t* v_at, int64_t* o_at, int64_t* d_at, int64_t* dbytes)
{
  const int hs = kudo_header_bytes(ncols);
  const int n = pi.rows, s = pi.row_offset;
  const int64_t vb = n > 0 ? (s + n - 1) / 8 - s / 8 + 1 : 0;
  int64_t v = hs, o = hs + pi.vlen, d = hs + static_cast<int64_t>(pi.vlen) + pi.olen;
  for (int k = 0; k <= c; ++k) {
    const bool hv = (part[28 + k / 8] >> (k % 8)) & 1;
    int64_t db;
    const int64_t ob = (sizes[k] == 0 && n > 0) ? 4 * (static_cast<int64_t>(n) + 1) : 0;
    if (sizes[k] == 0) db = ob ? static_cast<int64_t>(ld_le32(part + o + 4 * n)) - ld_le32(part + o) : 0;
    else db = static_cast<int64_t>(n) * sizes[k];
    if (k == c) {
      *has_v = hv;
      *v_at = v; *o_at = o; *d_at = d; *dbytes = db;
      return;
    }
    if (hv) v += vb;
    o += ob;
    d += db;
  }
}

// thread per partition: header -> KPartInfo, rows; *bad set on a malformed header
__global__ void __launch_bounds__(256) kudo_parse_kernel(const uint8_t* __restrict__ buf, const int64_t* __restrict__ part_offsets, int P, int ncols,
                                                        KPartInfo* __restrict__ info, int64_t* __restrict__ row_base /* [P + 1]: rows, scanned later */,
                                                        int32_t* __restrict__ bad)
{
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= P) return;
  const uint8_t* h = buf + part_offsets[p];
  KPartInfo pi{static_cast<int32_t>(ld_be32(h + 4)), static_cast<int32_t>(ld_be32(h + 8)), static_cast<int32_t>(ld_be32(h + 12)),
               static_cast<int32_t>(ld_be32(h + 16))};
  if (ld_be32(h) != kKudoMagic || static_cast<int>(ld_be32(h + 24)) != ncols || pi.rows < 0 || pi.row_offset < 0) {
    atomicExch(bad, 1);
    pi.rows = 0;
  }
  info[p]     = pi;
  row_base[p] = pi.rows;
}

// chars of every (STRING column, partition): thread per STRING column walks the partitions (exclusive prefix in place)
__global__ void __launch_bounds__(64) kudo_chars_kernel(const uint8_t* __restrict__ buf, const int64_t* __restrict__ part_offsets, int P, int ncols,
                                                       const int32_t* __restrict__ sizes, const int32_t* __restrict__ scols, int nstr,
                                                       const KPartInfo* __restrict__ info, int64_t* __restrict__ chars_base /* [nstr][P + 1] */)
{
  const int k = blockIdx.x * 64 + threadIdx.x;
  if (k >= nstr) return;
  int64_t run = 0;
  for (int p = 0; p < P; ++p) {
    bool hv;
    int64_t v, o, d, db;
    kudo_locate(buf + part_offsets[p], info[p], sizes, ncols, scols[k], &hv, &v, &o, &d, &db);
    chars_base[static_cast<int64_t>(k) * (P + 1) + p] = run;
    run += db;
  }
  chars_base[static_cast<int64_t>(k) * (P + 1) + P] = run;
}

__global__ void __launch_bounds__(256) kudo_assemble_kernel(const uint8_t* __restrict__ buf, const int64_t* __restrict__ part_offsets, int P, int ncols,
                                                           const int32_t* __restrict__ sizes, const KCol* __restrict__ out, const KPartInfo* __restrict__ info,
                                                           const int64_t* __restrict__ row_base, const int64_t* __restrict__ chars_base)
{
  const int c = blockIdx.x, p = blockIdx.y;
  const KPartInfo pi = info[p];
  const int n = pi.rows;
  if (n == 0) return;
  const uint8_t* part = buf + part_offsets[p];
  __shared__ int64_t s_at[4];
  __shared__ bool s_hv;
  if (threadIdx.x == 0) kudo_locate(part, pi, sizes, ncols, c, &s_hv, &s_at[0], &s_at[1], &s_at[2], &s_at[3]);
  __syncthreads();
  const KCol col   = out[c];
  const int64_t rb = row_base[p];
  // ---- validity: output bits [rb, rb + n) <- input bits [row_offset % 8, ... ) of the partition's bytes, or ones ----
  if (col.mask) {
    const uint8_t* vb   = part + s_at[0];
    const int shift     = pi.row_offset & 7;
    uint32_t* om        = reinterpret_cast<uint32_t*>(col.mask);
    const int64_t w0    = rb >> 5, w1 = (rb + n - 1) >> 5;
    for (int64_t w = w0 + threadIdx.x; w <= w1; w += 256) {
      const int64_t r_lo = tmax<int64_t>(rb, w << 5), r_hi = tmin<int64_t>(rb + n, (w + 1) << 5);   // rows of this word
      uint32_t bits = 0;
      if (s_hv) {
        const int64_t i0 = r_lo - rb + shift;   // first input bit
        uint64_t acc     = 0;
        const int64_t nbytes = ((i0 & 7) + (r_hi - r_lo) + 7) >> 3;   // <= 5
        for (int64_t b = 0; b < nbytes; ++b) acc |= static_cast<uint64_t>(vb[(i0 >> 3) + b]) << (8 * b);
        bits = static_cast<uint32_t>(acc >> (i0 & 7));
      } else {
        bits = 0xffffffffu;
      }
      const int cnt = static_cast<int>(r_hi - r_lo);
      if (cnt < 32) bits &= (1u << cnt) - 1u;
      bits <<= (r_lo & 31);
      if (bits) atomicOr(om + w, bits);
    }
  }
  // ---- offsets + chars, or fixed-width data ----
  if (sizes[c] == 0) {
    const uint8_t* ob = part + s_at[1];
    int sidx          = col.sidx;
    const int64_t cb  = chars_base[static_cast<int64_t>(sidx) * (P + 1) + p];
    const int32_t o0  = ld_le32(ob);
    for (int i = threadIdx.x; i <= n; i += 256) col.offsets[rb + i] = static_cast<int32_t>(cb + (ld_le32(ob + 4 * static_cast<int64_t>(i)) - o0));
    cta_copy_bytes(col.data + cb, part + s_at[2], s_at[3]);
  } else {
    cta_copy_bytes(col.data + rb * sizes[c], part + s_at[2], s_at[3]);
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------------
// workspace: [KCol x 256 | sizes int32 x 256 | scols int32 x 256 | bad flag (64 B) | KPartInfo x P | row_base int64 x (P + 1) | chars_base int64 x nstr x (P + 1)]
struct KudoWs {
  KCol* cols;
  int32_t* sizes;
  int32_t* scols;
  int32_t* bad;
  KPartInfo* info;
  int64_t* row_base;
  int64_t* chars_base;
};
static KudoWs kudo_ws(void* workspace, int P)
{
  uint8_t* w = static_cast<uint8_t*>(workspace);
  KudoWs k;
  k.cols  = reinterpret_cast<KCol*>(w);
  w += kKudoMaxCols * sizeof(KCol);
  k.sizes = reinterpret_cast<int32_t*>(w);
  w += kKudoMaxCols * 4;
  k.scols = reinterpret_cast<int32_t*>(w);
  w += kKudoMaxCols * 4;
  k.bad = reinterpret_cast<int32_t*>(w);
  w += 64;
  k.info = reinterpret_cast<KPartInfo*>(w);
  w += (static_cast<size_t>(P) * sizeof(KPartInfo) + 63) & ~size_t{63};
  k.row_base = reinterpret_cast<int64_t*>(w);
  w += ((static_cast<size_t>(P) + 1) * 8 + 63) & ~size_t{63};
  k.chars_base = reinterpret_cast<int64_t*>(w);
  return k;
}
static int64_t kudo_workspace_bytes(int32_t ncols, int32_t P)
{
  return static_cast<int64_t>(kKudoMaxCols) * (sizeof(KCol) + 8) + 64 + static_cast<int64_t>(P) * sizeof(KPartInfo) + 64 +
         (static_cast<int64_t>(P) + 1) * 8 + 64 + static_cast<int64_t>(std::max(ncols, 1)) * (static_cast<int64_t>(P) + 1) * 8 + 256;
}

static int kudo_upload(const srj_column* cols, int32_t ncols, const KudoWs& ws, int* nstr_out, cudaStream_t stream)
{
  if (ncols <= 0 || ncols > kKudoMaxCols) return SRJ_EUNSUPPORTED;
  KCol h[kKudoMaxCols];
  int32_t sizes[kKudoMaxCols], scols[kKudoMaxCols];
  int nstr = 0;
  for (int c = 0; c < ncols; ++c) {
    const int sz = type_width(cols[c].type_id);   // STRING: 0
    if (sz == 0 && cols[c].type_id != SRJ_STRING) return SRJ_EUNSUPPORTED;
    h[c].data    = static_cast<uint8_t*>(cols[c].data);
    h[c].mask    = reinterpret_cast<uint8_t*>(cols[c].null_mask);
    h[c].offsets = cols[c].offsets;
    h[c].size    = sz;
    h[c].sidx    = sz == 0 ? nstr : -1;
    sizes[c]     = sz;
    if (sz == 0) scols[nstr++] = c;
  }
  SRJ_CUDA_TRY(cudaMemcpyAsync(ws.cols, h, sizeof(KCol) * ncols, cudaMemcpyHostToDevice, stream));
  SRJ_CUDA_TRY(cudaMemcpyAsync(ws.sizes, sizes, 4 * ncols, cudaMemcpyHostToDevice, stream));
  if (nstr) SRJ_CUDA_TRY(cudaMemcpyAsync(ws.scols, scols, 4 * nstr, cudaMemcpyHostToDevice, stream));
  *nstr_out = nstr;
  return SRJ_OK;
}

static int launch_kudo_split_sizes(const srj_column* cols, int32_t ncols, int64_t num_rows, const int32_t* d_splits, int32_t P, int64_t* d_part_offsets,
                            int64_t* h_total, void* workspace, cudaStream_t stream)
{
  const KudoWs ws = kudo_ws(workspace, P);
  int nstr = 0;
  const int rc = kudo_upload(cols, ncols, ws, &nstr, stream);
  if (rc != SRJ_OK) return rc;
  SRJ_CUDA_TRY(cudaMemsetAsync(ws.bad, 0, 4, stream));
  kudo_split_sizes_kernel<<<(P + 255) / 256, 256, 0, stream>>>(ws.cols, ncols, d_splits, P, num_rows, d_part_offsets, ws.bad);
  i64_scan_small_kernel<<<1, 1024, 0, stream>>>(d_part_offsets, P);
  SRJ_CUDA_TRY(cudaGetLastError());
  int32_t bad = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(h_total, d_part_offsets + P, 8, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaMemcpyAsync(&bad, ws.bad, 4, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  return (bad & 2) ? SRJ_EINVAL : bad ? SRJ_EOVERFLOW : SRJ_OK;
}

static int launch_kudo_split(const srj_column* cols, int32_t ncols, const int32_t* d_splits, int32_t P, const int64_t* d_part_offsets, uint8_t* out,
                      void* workspace, cudaStream_t stream)
{
  const KudoWs ws = kudo_ws(workspace, P);
  int nstr = 0;
  const int rc = kudo_upload(cols, ncols, ws, &nstr, stream);
  if (rc != SRJ_OK) return rc;
  kudo_split_kernel<<<dim3(ncols, P), 256, 0, stream>>>(ws.cols, ncols, d_splits, d_part_offsets, out);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_kudo_assemble_sizes(const uint8_t* buf, const int64_t* d_part_offsets, int32_t P, const int32_t* type_ids, int32_t ncols, int64_t* h_rows,
                               int64_t* h_char_totals, void* workspace, cudaStream_t stream)
{
  const KudoWs ws = kudo_ws(workspace, P);
  if (ncols <= 0 || ncols > kKudoMaxCols) return SRJ_EUNSUPPORTED;
  int32_t sizes[kKudoMaxCols], scols[kKudoMaxCols];
  int nstr = 0;
  for (int c = 0; c < ncols; ++c) {
    sizes[c] = type_width(type_ids[c]);   // STRING: 0
    if (sizes[c] == 0 && type_ids[c] != SRJ_STRING) return SRJ_EUNSUPPORTED;
    if (sizes[c] == 0) scols[nstr++] = c;
    h_char_totals[c] = 0;
  }
  SRJ_CUDA_TRY(cudaMemcpyAsync(ws.sizes, sizes, 4 * ncols, cudaMemcpyHostToDevice, stream));
  if (nstr) SRJ_CUDA_TRY(cudaMemcpyAsync(ws.scols, scols, 4 * nstr, cudaMemcpyHostToDevice, stream));
  SRJ_CUDA_TRY(cudaMemsetAsync(ws.bad, 0, 4, stream));
  kudo_parse_kernel<<<(P + 255) / 256, 256, 0, stream>>>(buf, d_part_offsets, P, ncols, ws.info, ws.row_base, ws.bad);
  i64_scan_small_kernel<<<1, 1024, 0, stream>>>(ws.row_base, P);
  if (nstr) kudo_chars_kernel<<<(nstr + 63) / 64, 64, 0, stream>>>(buf, d_part_offsets, P, ncols, ws.sizes, ws.scols, nstr, ws.info, ws.chars_base);
  SRJ_CUDA_TRY(cudaGetLastError());
  int32_t bad = 0;
  std::vector<int64_t> totals(static_cast<size_t>(std::max(nstr, 1)));
  SRJ_CUDA_TRY(cudaMemcpyAsync(&bad, ws.bad, 4, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaMemcpyAsync(h_rows, ws.row_base + P, 8, cudaMemcpyDeviceToHost, stream));
  for (int k = 0; k < nstr; ++k)
    SRJ_CUDA_TRY(cudaMemcpyAsync(&totals[k], ws.chars_base + static_cast<int64_t>(k) * (P + 1) + P, 8, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  if (bad) return SRJ_EINVAL;
  for (int k = 0; k < nstr; ++k) h_char_totals[scols[k]] = totals[k];
  return SRJ_OK;
}

static int launch_kudo_assemble(const uint8_t* buf, const int64_t* d_part_offsets, int32_t P, const srj_column* out, int32_t ncols, int64_t total_rows,
                         void* workspace, cudaStream_t stream)
{
  const KudoWs ws = kudo_ws(workspace, P);
  int nstr = 0;
  const int rc = kudo_upload(out, ncols, ws, &nstr, stream);   // (sizes / scols are rewritten with the same values)
  if (rc != SRJ_OK) return rc;
  for (int c = 0; c < ncols; ++c) {
    if (out[c].null_mask && total_rows > 0) SRJ_CUDA_TRY(cudaMemsetAsync(out[c].null_mask, 0, static_cast<size_t>((total_rows + 31) / 32) * 4, stream));
    if (out[c].type_id == SRJ_STRING && total_rows == 0) SRJ_CUDA_TRY(cudaMemsetAsync(out[c].offsets, 0, 4, stream));
  }
  if (P > 0) kudo_assemble_kernel<<<dim3(ncols, P), 256, 0, stream>>>(buf, d_part_offsets, P, ncols, ws.sizes, ws.cols, ws.info, ws.row_base, ws.chars_base);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

int64_t srj_kudo_workspace_bytes(int32_t num_columns, int32_t num_partitions) { return kudo_workspace_bytes(std::max(num_columns, 0), std::max(num_partitions, 0)); }

static int kudo_check(const char* what, int32_t ncols, int32_t P, const void* a, const void* b, const void* ws)
{
  if (ncols <= 0 || P < 0 || !a || !b || !ws) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (ncols > 256 || P > 65535) { set_error("%s: at most 256 columns and 65535 partitions", what); return SRJ_EUNSUPPORTED; }
  return SRJ_OK;
}

int srj_kudo_split_sizes(const srj_column* cols, int32_t num_columns, int64_t num_rows, const int32_t* d_splits, int32_t num_partitions,
                         int64_t* d_partition_offsets, int64_t* total_bytes, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = kudo_check("kudo_split_sizes", num_columns, num_partitions, cols, d_partition_offsets, workspace);
  if (rc != SRJ_OK) return rc;
  if (!d_splits || !total_bytes || num_rows < 0 || num_rows > INT32_MAX) { set_error("kudo_split_sizes: bad argument"); return SRJ_EINVAL; }
  if ((rc = check_rows("kudo_split_sizes", cols, num_columns, num_rows)) != SRJ_OK) return rc;
  rc = launch_kudo_split_sizes(cols, num_columns, num_rows, d_splits, num_partitions, d_partition_offsets, total_bytes, workspace,
                               static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EUNSUPPORTED) set_error("kudo_split_sizes: only fixed-width, decimal and STRING columns");
  else if (rc == SRJ_EINVAL) set_error("kudo_split_sizes: the splits must lie in [0, %lld]", static_cast<long long>(num_rows));
  else if (rc == SRJ_EOVERFLOW) set_error("kudo_split_sizes: a partition exceeds the 32-bit section lengths of the Kudo header, or the splits are not increasing");
  return rc;
}

int srj_kudo_split(const srj_column* cols, int32_t num_columns, int64_t num_rows, const int32_t* d_splits, int32_t num_partitions,
                   const int64_t* d_partition_offsets, uint8_t* out, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = kudo_check("kudo_split", num_columns, num_partitions, cols, d_partition_offsets, workspace);
  if (rc != SRJ_OK) return rc;
  if (!d_splits) { set_error("kudo_split: bad argument"); return SRJ_EINVAL; }
  if ((rc = check_out("kudo_split", "output", out, 4, num_partitions > 0)) != SRJ_OK) return rc;
  if (num_partitions == 0) return SRJ_OK;
  (void)num_rows;
  rc = launch_kudo_split(cols, num_columns, d_splits, num_partitions, d_partition_offsets, out, workspace, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EUNSUPPORTED) set_error("kudo_split: only fixed-width, decimal and STRING columns");
  return rc;
}

int srj_kudo_assemble_sizes(const uint8_t* partitions, const int64_t* d_partition_offsets, int32_t num_partitions, const int32_t* type_ids,
                            int32_t num_columns, int64_t* total_rows, int64_t* char_totals, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = kudo_check("kudo_assemble_sizes", num_columns, num_partitions, type_ids, d_partition_offsets, workspace);
  if (rc != SRJ_OK) return rc;
  if ((num_partitions > 0 && !partitions) || !total_rows || !char_totals) { set_error("kudo_assemble_sizes: bad argument"); return SRJ_EINVAL; }
  rc = launch_kudo_assemble_sizes(partitions, d_partition_offsets, num_partitions, type_ids, num_columns, total_rows, char_totals, workspace,
                                  static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EINVAL) set_error("kudo_assemble_sizes: a partition does not start with a Kudo header of %d columns", num_columns);
  else if (rc == SRJ_EUNSUPPORTED) set_error("kudo_assemble_sizes: only fixed-width, decimal and STRING columns");
  else if (rc == SRJ_OK && *total_rows > INT32_MAX) { set_error("kudo_assemble_sizes: %lld rows exceed a column", static_cast<long long>(*total_rows)); return SRJ_EOVERFLOW; }
  return rc;
}

int srj_kudo_assemble(const uint8_t* partitions, const int64_t* d_partition_offsets, int32_t num_partitions, const srj_column* out,
                      int32_t num_columns, int64_t total_rows, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = kudo_check("kudo_assemble", num_columns, num_partitions, out, d_partition_offsets, workspace);
  if (rc != SRJ_OK) return rc;
  if ((rc = check_rows("kudo_assemble", out, num_columns, total_rows)) != SRJ_OK) return rc;
  rc = launch_kudo_assemble(partitions, d_partition_offsets, num_partitions, out, num_columns, total_rows, workspace, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EUNSUPPORTED) set_error("kudo_assemble: only fixed-width, decimal and STRING columns");
  return rc;
}

}  // extern "C"
