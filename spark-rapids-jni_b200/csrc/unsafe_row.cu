// unsafe_row.cu -- columns <-> Apache Spark UnsafeRow (SURVEY §8f rank 3: what BASELINE.json's metric literally
// names; the reference repo only speaks its own JCUDF row format, RowConversion.java:44-117, which the plugin adapts to
// Spark through CudfUnsafeRow).  The format is Apache Spark's, restated from its published sources
// (sql/catalyst/.../expressions/UnsafeRow.java and .../codegen/UnsafeRowWriter.java, branch-3.5):
//
//   row = [ null bitset : ceil(numFields / 64) 8-byte little-endian words, bit i SET = field i is NULL ]
//         [ one 8-byte slot per field                                                                    ]
//         [ variable-length region, every entry padded with zeros to a multiple of 8 bytes             ]
//   slot of a fixed-width field : the value in the low bytes, little endian, the rest of the slot zero (UnsafeRowWriter
//         zeroes the slot before a 1/2/4-byte write); decimals of precision <= 18 (DECIMAL32 / DECIMAL64) hold the
//         unscaled value as a 64-bit long; a NULL field's slot is 0 (setNullAt).
//   slot of a STRING            : (offset << 32) | length, offset from the start of the row; a NULL string has slot 0
//         and no bytes in the variable region.
//   slot of a DECIMAL128 (precision > 18): 16 bytes are ALWAYS reserved in the variable region (zeroed), holding the
//         unscaled value as BigInteger.toByteArray() -- big-endian two's complement, minimal length; the slot is
//         (offset << 32) | number of bytes, or (offset << 32) | 0 with the null bit set for a NULL.
//   Rows are a multiple of 8 bytes; variable-length entries follow in field order.  Floating-point payloads are copied
//   bit for bit (like the reference's row conversion, which moves bytes).
// No vector of this format exists in the reference repository: parity is pinned on hand-derived known answers of the rules
// above (the CPU restatement and its known-answer tests live with the test infrastructure) -- "parity unpinned".
//
// Kernels (lane = row: column accesses coalesced, row accesses strided but sector-local -- a thread walks its row):
//   ur_sizes_kernel      : bytes of every row (+ a grand total for the INT32_MAX check)
//   ur_to_rows_kernel    : bitset, slots, variable region
//   ur_from_rows_kernel  : slots -> fixed-width values / string lengths (scanned into offsets afterwards), null masks + counts
//   ur_chars_kernel      : chars of every STRING column (a warp per 32 rows, lane = byte)
#include <algorithm>

#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"

namespace srj {

constexpr int kUrStage   = 12 * 1024;  // shared-memory stage of a warp: its 32 rows when they are <= 384 bytes on average
constexpr int kUrBatch   = 16;         // fields whose column loads are in flight together (to_rows)
constexpr int kUrMaxCols = 256;  // fields of an UnsafeRow schema handled here (descriptor table in constant kernel parameters)

enum UrKind : int32_t { kUrFixed = 0, kUrString = 1, kUrDec128 = 2 };

struct UrCol {
  const uint8_t* data;      // to_rows: column data / chars; from_rows: output data (non-const use)
  const uint32_t* mask;     // NULL = all valid
  const int32_t* offsets;   // STRING
  int32_t kind;
  int32_t width;            // bytes of a fixed-width value in its column
  int32_t sext;             // 1: sign-extend to 64 bits (decimals <= 18 digits are longs in the row)
  int32_t pad;
};

struct UrTable {
  UrCol* cols;  // device [ncols]
  int32_t ncols, bitset_bytes, fixed_bytes, ndec;
};

__device__ __forceinline__ bool ur_valid(const uint32_t* mask, int64_t r) { return !mask || ((mask[r >> 5] >> (r & 31)) & 1u); }

__device__ __forceinline__ uint64_t ur_load_fixed(const UrCol& c, int64_t r)
{
  switch (c.width) {
    case 1: return c.data[r];
    case 2: return reinterpret_cast<const uint16_t*>(c.data)[r];
    case 4: {
      const uint32_t v = reinterpret_cast<const uint32_t*>(c.data)[r];
      return c.sext ? static_cast<uint64_t>(static_cast<int64_t>(static_cast<int32_t>(v))) : v;
    }
    default: return reinterpret_cast<const uint64_t*>(c.data)[r];
  }
}

// BigInteger.toByteArray() length of a 128-bit two's complement value: the fewest bytes that keep the sign bit
__device__ __forceinline__ int ur_dec_nbytes(uint64_t lo, uint64_t hi)
{
  const bool neg = static_cast<int64_t>(hi) < 0;
  const uint64_t h = neg ? ~hi : hi, l = neg ? ~lo : lo;   // leading bits equal to the sign become zeros
  const int lz = h ? __clzll(h) : 64 + (l ? __clzll(l) : 64);
  const int bits = 128 - lz + 1;                            // magnitude bits + one sign bit
  return (bits + 7) >> 3;                                   // 1 .. 16
}

// ---- sizes -------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ur_sizes_kernel(const UrTable t, int64_t n, int32_t* __restrict__ sizes, unsigned long long* __restrict__ total)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x;
  int64_t sz      = 0;
  if (r < n) {
    sz = t.fixed_bytes + 16 * t.ndec;
    for (int c = 0; c < t.ncols; ++c) {
      const UrCol col = t.cols[c];
      if (col.kind == kUrString && ur_valid(col.mask, r)) sz += (col.offsets[r + 1] - col.offsets[r] + 7) & ~7;
    }
    sizes[r] = static_cast<int32_t>(sz);
  }
  // grand total (warp reduce, one atomic per warp)
  unsigned long long s = static_cast<unsigned long long>(sz);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if (lane_id() == 0 && s) atomicAdd(total, s);
}

// ---- columns -> rows -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ur_to_rows_kernel(const UrTable t, int64_t n, const int32_t* __restrict__ row_offsets, int64_t row_stride,
                                                        uint8_t* __restrict__ rows, int stage)
{
  // The 32 rows of a warp are one contiguous byte range of the output: when it fits the warp's shared-memory stage the
  // rows are assembled there (a thread walking its row touches shared memory, not 32 scattered sectors per instruction)
  // and leave with coalesced 8-byte stores; larger ranges are written in place.
  extern __shared__ __align__(16) uint8_t s_stage[];
  UrCol* s_cols = reinterpret_cast<UrCol*>(s_stage + 8 * stage);       // the column descriptors, once per CTA
  for (int i = threadIdx.x; i < t.ncols; i += 256) s_cols[i] = t.cols[i];
  __syncthreads();
  const int lane = lane_id();
  for (int64_t blk = blockIdx.x; blk * 256 < n; blk += gridDim.x) {
  const int64_t r     = blk * 256 + threadIdx.x;
  const int64_t rw0   = r - lane;                                          // first row of the warp
  if (rw0 >= n) continue;
  __syncwarp();
  const int64_t rw1   = tmin<int64_t>(n, rw0 + 32);
  const int64_t b0    = row_offsets ? static_cast<int64_t>(row_offsets[rw0]) : rw0 * row_stride;
  const int64_t b1    = row_offsets ? static_cast<int64_t>(row_offsets[rw1]) : rw1 * row_stride;
  const bool staged   = b1 - b0 <= stage;
  uint8_t* wstage     = s_stage + static_cast<size_t>(warp_id()) * stage;
  if (r < n) {
  const int64_t myoff = row_offsets ? static_cast<int64_t>(row_offsets[r]) : r * row_stride;
  uint8_t* row        = staged ? wstage + (myoff - b0) : rows + myoff;
  uint64_t* slots     = reinterpret_cast<uint64_t*>(row + t.bitset_bytes);
  uint32_t cursor   = static_cast<uint32_t>(t.fixed_bytes);
  uint64_t nullbits = 0;
  // the column loads of kUrBatch fields are issued together (a thread walking its fields one dependent load at a time is
  // bound by DRAM latency): values are read whether or not the field is valid, the slot keeps 0 for a NULL
  for (int c0 = 0; c0 < t.ncols; c0 += kUrBatch) {
  uint64_t pv[kUrBatch];
  uint32_t pmask[kUrBatch];   // the mask WORDS: tested only after every load of the batch is in flight
#pragma unroll
  for (int j = 0; j < kUrBatch; ++j) {
    pv[j]    = 0;
    pmask[j] = 0xffffffffu;
    if (c0 + j < t.ncols) {
      const UrCol pc = s_cols[c0 + j];
      if (pc.mask) pmask[j] = __ldg(pc.mask + (r >> 5));
      if (pc.kind == kUrFixed) pv[j] = ur_load_fixed(pc, r);
    }
  }
#pragma unroll
  for (int j = 0; j < kUrBatch; ++j) {
    const int c = c0 + j;
    if (c >= t.ncols) break;
    const UrCol col  = s_cols[c];
    const bool valid = (pmask[j] >> (r & 31)) & 1u;
    uint64_t slot    = 0;
    if (col.kind == kUrFixed) {
      if (valid) slot = pv[j];
    } else if (col.kind == kUrString) {
      if (valid) {
        const int32_t o0 = col.offsets[r], len = col.offsets[r + 1] - o0;
        slot             = (static_cast<uint64_t>(cursor) << 32) | static_cast<uint32_t>(len);
        uint8_t* dst     = row + cursor;
        const int padded = (len + 7) & ~7;
        if (padded) *reinterpret_cast<uint64_t*>(dst + padded - 8) = 0;   // zero the last word: the padding bytes
        for (int i = 0; i < len; ++i) dst[i] = col.data[o0 + i];
        cursor += padded;
      }
    } else {  // DECIMAL128: 16 bytes always reserved (UnsafeRowWriter.write(ordinal, Decimal, precision, scale))
      uint64_t* dst = reinterpret_cast<uint64_t*>(row + cursor);
      dst[0] = dst[1] = 0;
      int nb = 0;
      if (valid) {
        const uint64_t lo = reinterpret_cast<const uint64_t*>(col.data)[2 * r], hi = reinterpret_cast<const uint64_t*>(col.data)[2 * r + 1];
        nb                = ur_dec_nbytes(lo, hi);
        uint8_t* b        = row + cursor;
        for (int i = 0; i < nb; ++i) {   // big endian: byte i is byte (nb - 1 - i) of the little-endian value
          const int k = nb - 1 - i;
          b[i]        = static_cast<uint8_t>((k < 8 ? lo >> (8 * k) : hi >> (8 * (k - 8))) & 0xff);
        }
      }
      slot = (static_cast<uint64_t>(cursor) << 32) | static_cast<uint32_t>(nb);
      cursor += 16;
    }
    if (!valid) nullbits |= 1ull << (c & 63);
    slots[c] = slot;
    if ((c & 63) == 63 || c == t.ncols - 1) {
      reinterpret_cast<uint64_t*>(row)[c >> 6] = nullbits;
      nullbits                                = 0;
    }
  }
  }
  }
  if (staged) {
    __syncwarp();
    uint64_t* g        = reinterpret_cast<uint64_t*>(rows + b0);
    const uint64_t* sm = reinterpret_cast<const uint64_t*>(wstage);
    for (int64_t i = lane; i < (b1 - b0) >> 3; i += 32) g[i] = sm[i];
  }
  }
}

// ---- rows -> columns (slots) ---------------------------------------------------------------------------------------------
struct UrOut {
  uint8_t* data;        // fixed / DECIMAL128 output
  uint32_t* mask;       // may be NULL
  int32_t* offsets;     // STRING: receives the lengths (element r), scanned afterwards
  int32_t kind, width, sext, pad;
};
struct UrOutTable {
  UrOut* cols;
  int32_t ncols, bitset_bytes, fixed_bytes, ndec;
};

__global__ void __launch_bounds__(256) ur_from_rows_kernel(const UrOutTable t, int64_t n, const uint8_t* __restrict__ rows,
                                                          const int32_t* __restrict__ row_offsets, int64_t row_stride,
                                                          unsigned long long* __restrict__ null_counts, int stage)
{
  extern __shared__ __align__(16) uint8_t s_stage[];
  // the column descriptors and the CTA's null counts live in shared memory behind the warps' stages
  UrOut* s_cols = reinterpret_cast<UrOut*>(s_stage + 8 * stage);
  int* s_nulls  = reinterpret_cast<int*>(s_cols + t.ncols);
  for (int i = threadIdx.x; i < t.ncols; i += 256) {
    s_cols[i]  = t.cols[i];
    s_nulls[i] = 0;
  }
  __syncthreads();
  const int lane = lane_id();
  for (int64_t blk = blockIdx.x; blk * 256 < n; blk += gridDim.x) {
  const int64_t r  = blk * 256 + threadIdx.x;
  const bool live  = r < n;
  const int64_t rw0 = r - lane;
  if (rw0 >= n) continue;   // whole warp past the end
  __syncwarp();             // the previous block's reads of this warp's stage are done
  const int64_t rw1 = tmin<int64_t>(n, rw0 + 32);
  const int64_t b0  = row_offsets ? static_cast<int64_t>(row_offsets[rw0]) : rw0 * row_stride;
  const int64_t b1  = row_offsets ? static_cast<int64_t>(row_offsets[rw1]) : rw1 * row_stride;
  const bool staged = b1 - b0 <= stage;
  uint8_t* wstage   = s_stage + static_cast<size_t>(warp_id()) * stage;
  if (staged) {   // the warp's 32 rows are one contiguous byte range: coalesced into shared memory, parsed from there
    const uint64_t* g = reinterpret_cast<const uint64_t*>(rows + b0);
    uint64_t* sm      = reinterpret_cast<uint64_t*>(wstage);
    for (int64_t i = lane; i < (b1 - b0) >> 3; i += 32) sm[i] = g[i];
    __syncwarp();
  }
  const int64_t myoff = live ? (row_offsets ? static_cast<int64_t>(row_offsets[r]) : r * row_stride) : b0;
  const uint8_t* row  = staged ? wstage + (myoff - b0) : rows + myoff;
  const uint64_t* slots = reinterpret_cast<const uint64_t*>(row + t.bitset_bytes);
  uint64_t nullbits = 0;
  for (int c = 0; c < t.ncols; ++c) {
    if ((c & 63) == 0) nullbits = live ? reinterpret_cast<const uint64_t*>(row)[c >> 6] : 0;
    const UrOut col   = s_cols[c];
    const bool valid  = live && !((nullbits >> (c & 63)) & 1ull);
    const uint64_t sl = live ? slots[c] : 0;
    if (live) {
      if (col.kind == kUrFixed) {
        switch (col.width) {
          case 1: col.data[r] = static_cast<uint8_t>(sl); break;
          case 2: reinterpret_cast<uint16_t*>(col.data)[r] = static_cast<uint16_t>(sl); break;
          case 4: reinterpret_cast<uint32_t*>(col.data)[r] = static_cast<uint32_t>(sl); break;
          default: reinterpret_cast<uint64_t*>(col.data)[r] = sl; break;
        }
      } else if (col.kind == kUrString) {
        col.offsets[r] = valid ? static_cast<int32_t>(sl & 0xffffffffu) : 0;
      } else {
        uint64_t lo = 0, hi = 0;
        if (valid) {
          const uint8_t* b = row + (sl >> 32);
          const int nb     = static_cast<int>(sl & 0xffffffffu);
          const bool neg   = nb > 0 && (b[0] & 0x80);
          lo = hi = neg ? ~0ull : 0ull;   // sign extension
          for (int i = 0; i < nb; ++i) {
            const int k      = nb - 1 - i;
            const uint64_t v = b[i];
            if (k < 8) lo = (lo & ~(0xffull << (8 * k))) | (v << (8 * k));
            else hi = (hi & ~(0xffull << (8 * (k - 8)))) | (v << (8 * (k - 8)));
          }
        }
        reinterpret_cast<uint64_t*>(col.data)[2 * r]     = lo;
        reinterpret_cast<uint64_t*>(col.data)[2 * r + 1] = hi;
      }
    }
    const unsigned word = __ballot_sync(0xffffffffu, valid);
    if (lane == 0 && r < n) {
      if (col.mask) col.mask[r >> 5] = word;
      const int rows_here = static_cast<int>(tmin<int64_t>(32, n - r));
      const int nulls     = rows_here - __popc(word);
      if (nulls) atomicAdd(&s_nulls[c], nulls);
    }
  }
  }
  __syncthreads();
  if (null_counts)
    for (int i = threadIdx.x; i < t.ncols; i += 256)
      if (s_nulls[i]) atomicAdd(null_counts + i, static_cast<unsigned long long>(s_nulls[i]));
}

// chars of one STRING column: a warp per 32 rows, lane = destination byte (the rows' strings are contiguous in the
// output), source row by a shuffle search over the 32 starts
__global__ void __launch_bounds__(256) ur_chars_kernel(const uint8_t* __restrict__ rows, const int32_t* __restrict__ row_offsets, int64_t row_stride,
                                                      int64_t n, int32_t slot_offset, int32_t null_word, int32_t null_bit,
                                                      const int32_t* __restrict__ out_off, uint8_t* __restrict__ out_chars)
{
  const int lane = lane_id();
  for (int64_t d0 = (static_cast<int64_t>(blockIdx.x) * 8 + warp_id()) * 32; d0 < n; d0 += static_cast<int64_t>(gridDim.x) * 256) {
    const int last    = static_cast<int>(tmin<int64_t>(32, n - d0)) - 1;
    const int64_t d   = tmin<int64_t>(d0 + lane, n - 1);
    const uint8_t* row = rows + (row_offsets ? static_cast<int64_t>(row_offsets[d]) : d * row_stride);
    const uint64_t sl = *reinterpret_cast<const uint64_t*>(row + slot_offset);
    const bool isnull = (reinterpret_cast<const uint64_t*>(row)[null_word] >> null_bit) & 1ull;
    const uint64_t src = reinterpret_cast<uint64_t>(row) + (isnull ? 0 : (sl >> 32));
    const int32_t ob  = out_off[d0];
    const int32_t pe  = out_off[d] - ob;
    const int32_t T   = out_off[d0 + last + 1] - ob;
    for (int32_t q = lane; q < ((T + 31) & ~31); q += 32) {
      int j = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const int cand  = j + step;
        const int32_t v = __shfl_sync(0xffffffffu, pe, cand & 31);
        if (cand <= last && v <= q) j = cand;
      }
      const int32_t pj  = __shfl_sync(0xffffffffu, pe, j);
      const uint64_t sj = __shfl_sync(0xffffffffu, src, j);
      if (q < T) out_chars[ob + q] = *reinterpret_cast<const uint8_t*>(sj + (q - pj));
    }
  }
}

// shared-memory stage of a warp: its 32 rows.  Fixed-size rows: exactly that (more CTAs stay resident); rows with
// strings: kUrStage (larger 32-row ranges are handled in place)
static int ur_stage(const int32_t* d_row_offsets, int fixed_row_bytes)
{
  if (d_row_offsets) return kUrStage;
  return std::min(kUrStage, (32 * fixed_row_bytes + 15) & ~15);
}

static unsigned ur_grid(int64_t n) { return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, int64_t{sm_count()} * 8))); }

// ---- host side -------------------------------------------------------------------------------------------------------------
static bool ur_classify(int32_t type_id, int32_t* kind, int32_t* width, int32_t* sext)
{
  *sext = 0;
  switch (type_id) {
    case SRJ_INT8: case SRJ_UINT8: case SRJ_BOOL8: *kind = kUrFixed; *width = 1; return true;
    case SRJ_INT16: case SRJ_UINT16: *kind = kUrFixed; *width = 2; return true;
    case SRJ_INT32: case SRJ_UINT32: case SRJ_FLOAT32: case SRJ_TIMESTAMP_DAYS: *kind = kUrFixed; *width = 4; return true;
    case SRJ_DECIMAL32: *kind = kUrFixed; *width = 4; *sext = 1; return true;
    case SRJ_INT64: case SRJ_UINT64: case SRJ_FLOAT64: case SRJ_TIMESTAMP_SECONDS: case SRJ_TIMESTAMP_MILLISECONDS:
    case SRJ_TIMESTAMP_MICROSECONDS: case SRJ_TIMESTAMP_NANOSECONDS: case SRJ_DECIMAL64: *kind = kUrFixed; *width = 8; return true;
    case SRJ_DECIMAL128: *kind = kUrDec128; *width = 16; return true;
    case SRJ_STRING: *kind = kUrString; *width = 0; return true;
    default: return false;
  }
}

static int unsafe_row_layout(const int32_t* type_ids, int32_t ncols, int32_t* bitset_bytes, int32_t* fixed_bytes, int32_t* ndec, int32_t* nstr)
{
  if (ncols <= 0 || ncols > kUrMaxCols) return SRJ_EUNSUPPORTED;
  *ndec = *nstr = 0;
  for (int c = 0; c < ncols; ++c) {
    int32_t k, w, s;
    if (!ur_classify(type_ids[c], &k, &w, &s)) return SRJ_EUNSUPPORTED;
    *ndec += k == kUrDec128;
    *nstr += k == kUrString;
  }
  *bitset_bytes = ((ncols + 63) / 64) * 8;   // UnsafeRow.calculateBitSetWidthInBytes
  *fixed_bytes  = *bitset_bytes + 8 * ncols;
  return SRJ_OK;
}

// workspace: [UrCol table | 8-byte total | scan partials]
static int64_t unsafe_row_workspace_bytes(int32_t ncols, int64_t n)
{
  return static_cast<int64_t>(kUrMaxCols) * sizeof(UrCol) + 64 + (i32_scan_nchunks(n + 1) + 64) * 4;
}

static int ur_upload(const srj_column* cols, int32_t ncols, void* workspace, UrTable* t, cudaStream_t stream)
{
  UrCol h[kUrMaxCols];
  int32_t types[kUrMaxCols];
  if (ncols <= 0 || ncols > kUrMaxCols) return SRJ_EUNSUPPORTED;   // before the type ids are copied into types[]
  for (int c = 0; c < ncols; ++c) types[c] = cols[c].type_id;
  int32_t nstr = 0;
  const int rc = unsafe_row_layout(types, ncols, &t->bitset_bytes, &t->fixed_bytes, &t->ndec, &nstr);
  if (rc != SRJ_OK) return rc;
  for (int c = 0; c < ncols; ++c) {
    ur_classify(cols[c].type_id, &h[c].kind, &h[c].width, &h[c].sext);
    h[c].data    = static_cast<const uint8_t*>(cols[c].data);
    h[c].mask    = cols[c].null_mask;
    h[c].offsets = cols[c].offsets;
    h[c].pad     = 0;
  }
  t->ncols = ncols;
  t->cols  = static_cast<UrCol*>(workspace);
  // pageable host -> device copy of a stack table: the runtime stages it before returning, the table may go out of scope
  SRJ_CUDA_TRY(cudaMemcpyAsync(workspace, h, sizeof(UrCol) * ncols, cudaMemcpyHostToDevice, stream));
  return SRJ_OK;
}

static int launch_unsafe_row_sizes(const srj_column* cols, int32_t ncols, int64_t n, int32_t* d_row_offsets, void* workspace, int64_t* h_total,
                            cudaStream_t stream)
{
  UrTable t{};
  int rc = ur_upload(cols, ncols, workspace, &t, stream);
  if (rc != SRJ_OK) return rc;
  auto* d_total = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(workspace) + kUrMaxCols * sizeof(UrCol));
  SRJ_CUDA_TRY(cudaMemsetAsync(d_total, 0, 8, stream));
  if (n > 0) {
    ur_sizes_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(t, n, d_row_offsets, d_total);
    SRJ_CUDA_TRY(cudaGetLastError());
  }
  unsigned long long total = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  *h_total = static_cast<int64_t>(total);
  if (total > static_cast<unsigned long long>(INT32_MAX)) return SRJ_EOVERFLOW;
  // sizes -> offsets (exclusive scan in place, grand total into element n)
  int32_t* sums = reinterpret_cast<int32_t*>(d_total + 8);
  if (n == 0) {
    SRJ_CUDA_TRY(cudaMemsetAsync(d_row_offsets, 0, 4, stream));
    return SRJ_OK;
  }
  return launch_i32_exclusive_scan(d_row_offsets, n, sums, d_row_offsets + n, stream);
}

static int launch_unsafe_to_rows(const srj_column* cols, int32_t ncols, int64_t n, const int32_t* d_row_offsets, uint8_t* rows, void* workspace,
                          cudaStream_t stream)
{
  UrTable t{};
  const int rc = ur_upload(cols, ncols, workspace, &t, stream);
  if (rc != SRJ_OK) return rc;
  if (n == 0) return SRJ_OK;
  const int stage   = ur_stage(d_row_offsets, t.fixed_bytes + 16 * t.ndec);
  const size_t smem = 8 * static_cast<size_t>(stage) + static_cast<size_t>(ncols) * (sizeof(UrCol) + 4) + 16;
  SRJ_CUDA_TRY(cudaFuncSetAttribute(ur_to_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * kUrStage + kUrMaxCols * (sizeof(UrCol) + 4) + 16));
  ur_to_rows_kernel<<<ur_grid(n), 256, smem, stream>>>(t, n, d_row_offsets, t.fixed_bytes + 16 * t.ndec, rows, stage);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_unsafe_from_rows(const srj_column* out, int32_t ncols, int64_t n, const uint8_t* rows, const int32_t* d_row_offsets,
                            int64_t* d_null_counts, void* workspace, cudaStream_t stream)
{
  UrTable t{};
  int rc = ur_upload(out, ncols, workspace, &t, stream);   // UrCol and UrOut share their layout
  if (rc != SRJ_OK) return rc;
  static_assert(sizeof(UrCol) == sizeof(UrOut), "descriptor layouts must match");
  if (d_null_counts) SRJ_CUDA_TRY(cudaMemsetAsync(d_null_counts, 0, sizeof(int64_t) * ncols, stream));
  int32_t* sums = reinterpret_cast<int32_t*>(static_cast<uint8_t*>(workspace) + kUrMaxCols * sizeof(UrCol) + 64);
  if (n > 0) {
    UrOutTable ot{reinterpret_cast<UrOut*>(t.cols), t.ncols, t.bitset_bytes, t.fixed_bytes, t.ndec};
    const int stage   = ur_stage(d_row_offsets, t.fixed_bytes + 16 * t.ndec);
    const size_t smem = 8 * static_cast<size_t>(stage) + static_cast<size_t>(ncols) * (sizeof(UrCol) + 4) + 16;
    SRJ_CUDA_TRY(cudaFuncSetAttribute(ur_from_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * kUrStage + kUrMaxCols * (sizeof(UrCol) + 4) + 16));
    ur_from_rows_kernel<<<ur_grid(n), 256, smem, stream>>>(ot, n, rows, d_row_offsets, t.fixed_bytes + 16 * t.ndec,
                                                                                   reinterpret_cast<unsigned long long*>(d_null_counts), stage);
    SRJ_CUDA_TRY(cudaGetLastError());
  }
  for (int c = 0; c < ncols; ++c) {
    if (out[c].type_id != SRJ_STRING) continue;
    if (n == 0) {
      SRJ_CUDA_TRY(cudaMemsetAsync(out[c].offsets, 0, 4, stream));
      continue;
    }
    rc = launch_i32_exclusive_scan(out[c].offsets, n, sums, out[c].offsets + n, stream);
    if (rc != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

static int launch_unsafe_from_rows_strings(const srj_column* out, int32_t ncols, int64_t n, const uint8_t* rows, const int32_t* d_row_offsets,
                                    cudaStream_t stream)
{
  int32_t types[kUrMaxCols];
  if (ncols > kUrMaxCols) return SRJ_EUNSUPPORTED;
  for (int c = 0; c < ncols; ++c) types[c] = out[c].type_id;
  int32_t bitset = 0, fixed = 0, ndec = 0, nstr = 0;
  const int rc = unsafe_row_layout(types, ncols, &bitset, &fixed, &ndec, &nstr);
  if (rc != SRJ_OK) return rc;
  if (n == 0) return SRJ_OK;
  const unsigned grid = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, int64_t{sm_count()} * 16)));
  for (int c = 0; c < ncols; ++c) {
    if (out[c].type_id != SRJ_STRING) continue;
    ur_chars_kernel<<<grid, 256, 0, stream>>>(rows, d_row_offsets, fixed + 16 * ndec, n, bitset + 8 * c, c >> 6, c & 63, out[c].offsets,
                                             static_cast<uint8_t*>(out[c].data));
  }
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

int srj_unsafe_row_layout(const int32_t* type_ids, int32_t num_columns, int32_t* bitset_bytes, int32_t* fixed_bytes)
{
  if (!type_ids || !bitset_bytes || !fixed_bytes) { set_error("unsafe_row_layout: bad argument"); return SRJ_EINVAL; }
  int32_t ndec = 0, nstr = 0, fb = 0;
  const int rc = unsafe_row_layout(type_ids, num_columns, bitset_bytes, &fb, &ndec, &nstr);
  if (rc != SRJ_OK) { set_error("unsafe_row_layout: 1..256 columns of fixed-width, decimal or STRING type"); return rc; }
  *fixed_bytes = fb + 16 * ndec;   // every DECIMAL128 field reserves 16 bytes of the variable region
  return SRJ_OK;
}

int64_t srj_unsafe_row_workspace_bytes(int32_t num_columns, int64_t num_rows) { return unsafe_row_workspace_bytes(num_columns, std::max<int64_t>(0, num_rows)); }

static int ur_check(const char* what, const srj_column* cols, int32_t ncols, int64_t n, const void* workspace)
{
  if (ncols <= 0 || n < 0 || !cols || !workspace) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (n > INT32_MAX) { set_error("%s: more than INT32_MAX rows", what); return SRJ_EOVERFLOW; }
  return check_rows(what, cols, ncols, n);
}

int srj_unsafe_row_sizes(const srj_column* cols, int32_t num_columns, int64_t num_rows, int32_t* d_row_offsets, int64_t* total_bytes,
                         void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = ur_check("unsafe_row_sizes", cols, num_columns, num_rows, workspace);
  if (rc != SRJ_OK) return rc;
  if (!d_row_offsets || !total_bytes) { set_error("unsafe_row_sizes: bad argument"); return SRJ_EINVAL; }
  rc = launch_unsafe_row_sizes(cols, num_columns, num_rows, d_row_offsets, workspace, total_bytes, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EOVERFLOW) set_error("unsafe_row_sizes: %lld bytes of rows exceed one LIST<INT8> column (INT32_MAX): convert fewer rows per call", static_cast<long long>(*total_bytes));
  else if (rc == SRJ_EUNSUPPORTED) set_error("unsafe_row_sizes: unsupported column type or more than 256 columns");
  return rc;
}

int srj_convert_to_unsafe_rows(const srj_column* cols, int32_t num_columns, int64_t num_rows, const int32_t* d_row_offsets, uint8_t* rows,
                               void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = ur_check("convert_to_unsafe_rows", cols, num_columns, num_rows, workspace);
  if (rc != SRJ_OK) return rc;
  if ((rc = check_out("convert_to_unsafe_rows", "rows buffer", rows, 8, num_rows > 0)) != SRJ_OK) return rc;
  if (!d_row_offsets)
    for (int32_t c = 0; c < num_columns; ++c)
      if (cols[c].type_id == SRJ_STRING) { set_error("convert_to_unsafe_rows: STRING columns need the row offsets of srj_unsafe_row_sizes"); return SRJ_EINVAL; }
  rc = launch_unsafe_to_rows(cols, num_columns, num_rows, d_row_offsets, rows, workspace, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EUNSUPPORTED) set_error("convert_to_unsafe_rows: unsupported column type or more than 256 columns");
  return rc;
}

int srj_convert_from_unsafe_rows(const uint8_t* rows, const int32_t* d_row_offsets, int64_t num_rows, const srj_column* out, int32_t num_columns,
                                 int64_t* d_null_counts, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = ur_check("convert_from_unsafe_rows", out, num_columns, num_rows, workspace);
  if (rc != SRJ_OK) return rc;
  if ((rc = check_out("convert_from_unsafe_rows", "rows buffer", rows, 8, num_rows > 0)) != SRJ_OK) return rc;
  if (!d_row_offsets)
    for (int32_t c = 0; c < num_columns; ++c)
      if (out[c].type_id == SRJ_STRING) { set_error("convert_from_unsafe_rows: variable-width rows need their offsets"); return SRJ_EINVAL; }
  rc = launch_unsafe_from_rows(out, num_columns, num_rows, rows, d_row_offsets, d_null_counts, workspace, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EUNSUPPORTED) set_error("convert_from_unsafe_rows: unsupported column type or more than 256 columns");
  return rc;
}

int srj_convert_from_unsafe_rows_strings(const uint8_t* rows, const int32_t* d_row_offsets, int64_t num_rows, const srj_column* out,
                                         int32_t num_columns, void* stream)
{
  SRJ_API_RANGE();
  if (num_columns <= 0 || num_rows < 0 || !out || (num_rows > 0 && (!rows || !d_row_offsets))) { set_error("convert_from_unsafe_rows_strings: bad argument"); return SRJ_EINVAL; }
  if (check_out("convert_from_unsafe_rows_strings", "rows buffer", rows, 8, false) != SRJ_OK) return SRJ_EINVAL;
  return launch_unsafe_from_rows_strings(out, num_columns, num_rows, rows, d_row_offsets, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
