/*
 * srj_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * A plain-C restatement of the reference's algorithms for the row<->columnar hot path
 * (JCUDF row format) and the Spark-compatible row hashes.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load this library; the product
 * (libsrj_b200.so) never links, loads or calls it.
 *
 * Parity pinning:
 *   - hashes: PINNED by the reference's Spark-derived golden vectors
 *       src/main/cpp/tests/hash.cpp:268-297,411-412,686-811,971-977 and
 *       src/test/java/com/nvidia/spark/rapids/jni/HashTest.java:54-180,273-405,576-700
 *     (tests/test_oracle_hash_golden.py).
 *   - row layout: pinned by src/main/cpp/tests/row_conversion.cpp:457-498 (PivotLikeLayout)
 *     and the Javadoc example RowConversion.java:77-105 (tests/test_oracle_rows.py).
 *   - DECIMAL128 / STRING row bytes: "PARITY UNPINNED" by any reference test (none exists,
 *     SURVEY.md 8c); the restatement follows the cited code paths and is checked by
 *     round-trip identity.
 *
 * Every function cites the reference file:line it follows.  Paths are relative to
 * the reference repository's root; RC = src/main/cpp/src/row_conversion.cu.
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* cudf type ids: thirdparty/cudf/cpp/include/cudf/types.hpp:191-224 */
enum {
  T_EMPTY = 0, T_INT8, T_INT16, T_INT32, T_INT64, T_UINT8, T_UINT16, T_UINT32, T_UINT64,
  T_FLOAT32, T_FLOAT64, T_BOOL8, T_TS_DAYS, T_TS_S, T_TS_MS, T_TS_US, T_TS_NS,
  T_DUR_DAYS, T_DUR_S, T_DUR_MS, T_DUR_US, T_DUR_NS, T_DICT32, T_STRING, T_LIST,
  T_DEC32, T_DEC64, T_DEC128, T_STRUCT
};

typedef struct {
  int32_t type_id;
  int32_t scale;
  int64_t size;         /* rows */
  void* data;           /* fixed-width values, or chars for STRING */
  uint32_t* null_mask;  /* bit i%32 of word i/32, 1 = valid; NULL = all valid (bit.hpp:48-106) */
  int32_t* offsets;     /* STRING only: size+1 offsets */
} orc_col;

#define ORC_OK 0
#define ORC_EINVAL (-1)
#define ORC_EUNSUPPORTED (-2)
#define ORC_EOVERFLOW (-3)

#define JCUDF_ROW_ALIGNMENT 8                 /* RC:63 */
#define MAX_BATCH_SIZE ((uint64_t)INT32_MAX)  /* RC:65 */

static int64_t round_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

/* size_of(): thirdparty/cudf/cpp/include/cudf/utilities/traits.hpp (fixed-width types) */
int32_t orc_size_of(int32_t t)
{
  switch (t) {
    case T_INT8: case T_UINT8: case T_BOOL8: return 1;
    case T_INT16: case T_UINT16: return 2;
    case T_INT32: case T_UINT32: case T_FLOAT32: case T_TS_DAYS: case T_DUR_DAYS: case T_DEC32:
      return 4;
    case T_INT64: case T_UINT64: case T_FLOAT64: case T_TS_S: case T_TS_MS: case T_TS_US:
    case T_TS_NS: case T_DUR_S: case T_DUR_MS: case T_DUR_US: case T_DUR_NS: case T_DEC64:
      return 8;
    case T_DEC128: return 16;
    default: return 0; /* not fixed width */
  }
}

static int is_valid(const uint32_t* m, int64_t i) { return !m || ((m[i >> 5] >> (i & 31)) & 1u); }

/*
 * compute_column_information  -- RC:1332-1371.
 * starts has ncols+1 entries (last = validity offset); returns size_per_row (unpadded) or <0.
 * STRING is "compound": 8 bytes (uint32 offset, uint32 length), aligned to 4 (RC:1346-1351).
 */
int32_t orc_compute_layout(const int32_t* types, int32_t ncols, int32_t* starts, int32_t* sizes)
{
  int64_t size_per_row = 0;
  for (int32_t i = 0; i < ncols; ++i) {
    int compound = (types[i] == T_STRING);
    int32_t sz = compound ? 8 : orc_size_of(types[i]);
    if (sz == 0) return ORC_EUNSUPPORTED; /* LIST/STRUCT/DICTIONARY: RowConversion.java:131 */
    int32_t al = compound ? 4 : sz;
    size_per_row = round_up(size_per_row, al);
    starts[i] = (int32_t)size_per_row;
    sizes[i] = sz;
    size_per_row += sz;
    if (size_per_row > INT32_MAX) return ORC_EOVERFLOW;
  }
  starts[ncols] = (int32_t)size_per_row;               /* validity offset, RC:1359-1361 */
  size_per_row += (ncols + 7) / 8;                     /* byte-aligned validity, RC:1363-1365 */
  return (int32_t)size_per_row;
}

/*
 * Per-row byte size of the JCUDF row -- RC:246-254 (strings) / RC:2026-2027 (fixed width):
 *   round_up(size_per_row + sum(strlen over string columns), 8)
 */
int orc_row_sizes(const orc_col* cols, int32_t ncols, int64_t nrows, int32_t size_per_row,
                  uint64_t* row_sizes)
{
  for (int64_t r = 0; r < nrows; ++r) {
    uint64_t s = 0;
    for (int32_t c = 0; c < ncols; ++c)
      if (cols[c].type_id == T_STRING) s += (uint64_t)(cols[c].offsets[r + 1] - cols[c].offsets[r]);
    row_sizes[r] = (uint64_t)round_up((int64_t)(size_per_row + s), JCUDF_ROW_ALIGNMENT);
  }
  return ORC_OK;
}

/*
 * build_batches -- RC:1466-1557.
 *   cumulative = inclusive_scan(row_sizes); per batch: lower_bound over
 *   (cumulative[i] - cumulative[last_row_end]) for MAX_BATCH_SIZE, then round the cut DOWN to a
 *   multiple of 32 rows unless it is the end of the table (RC:1500-1517).
 * boundaries gets num_batches+1 entries (first = 0); returns num_batches (0 for an empty table,
 * where the reference is UB: SURVEY App. C.4), or <0.
 * Divergence (documented): when the reference's cut would produce a batch > INT32_MAX bytes
 * (its off-by-one on the first row of the batch, e.g. 8-byte rows x 2^28) we step the cut back
 * by 32 rows instead of overflowing the int32 offsets.
 */
int32_t orc_build_batches(const uint64_t* row_sizes, int64_t nrows, int64_t* boundaries,
                          int32_t max_batches)
{
  if (nrows == 0) { boundaries[0] = 0; return 0; }
  uint64_t* cum = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)nrows);
  if (!cum) return ORC_EINVAL;
  uint64_t acc = 0;
  for (int64_t i = 0; i < nrows; ++i) { acc += row_sizes[i]; cum[i] = acc; }
  int32_t nb = 0;
  int64_t last = 0;
  boundaries[0] = 0;
  while (last < nrows) {
    /* lower_bound: first i in [last, nrows) with cum[i]-cum[last] >= MAX_BATCH_SIZE */
    int64_t lo = last, hi = nrows;
    while (lo < hi) {
      int64_t mid = lo + (hi - lo) / 2;
      if (cum[mid] - cum[last] < MAX_BATCH_SIZE) lo = mid + 1; else hi = mid;
    }
    int64_t batch_size = lo - last;
    int64_t row_end = (lo == nrows) ? last + batch_size : last + (batch_size / 32) * 32;
    /* overflow guard (divergence noted above) */
    for (;;) {
      uint64_t bytes = cum[row_end - 1] - (last ? cum[last - 1] : 0);
      if (bytes <= MAX_BATCH_SIZE) break;
      int64_t n = row_end - last;
      int64_t back = (n % 32) ? (n % 32) : 32;
      row_end -= back;
      if (row_end <= last) { free(cum); return ORC_EOVERFLOW; }
    }
    if (row_end <= last) { free(cum); return ORC_EOVERFLOW; } /* single row > 2 GiB */
    if (nb >= max_batches) { free(cum); return ORC_EINVAL; }
    boundaries[++nb] = row_end;
    last = row_end;
  }
  free(cum);
  return nb;
}

/*
 * convert_to_rows for ONE batch [row_start, row_start+row_count) -- RC:1762-1982.
 *   fixed-width fields   copy_to_rows          RC:574-688 (value bytes copied bit for bit)
 *   validity             copy_validity_to_rows RC:706-798 (bit c%8 of byte c/8, 1 = valid,
 *                                               unused high bits 0: RC:753-766)
 *   strings              copy_strings_to_rows  RC:816-861 ((uint32 offset, uint32 len) pair at the
 *                                               column's slot; chars appended in column order from
 *                                               byte size_per_row, no padding between them)
 *   row offsets          build_batches exclusive scan within the batch, RC:1526-1532
 * Padding bytes are undefined in the reference (SURVEY App. C.2); the oracle (and the product)
 * write zeros.  DECIMAL128: 16 bytes little-endian at its 16-aligned start (App. A.6; the
 * reference's general kernel mis-copies it, RC:660-665 -- "parity unpinned").
 * A null field's bytes are whatever the source column holds (copied blindly, App. A.6).
 */
int orc_convert_to_rows(const orc_col* cols, int32_t ncols, int64_t row_start, int64_t row_count,
                        int32_t* out_offsets /* row_count+1 */, uint8_t* out_data,
                        int64_t out_capacity)
{
  int32_t* types = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  int32_t* starts = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols + 1));
  int32_t* sizes = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  for (int32_t c = 0; c < ncols; ++c) types[c] = cols[c].type_id;
  int32_t spr = orc_compute_layout(types, ncols, starts, sizes);
  if (spr < 0) { free(types); free(starts); free(sizes); return spr; }
  int32_t voff = starts[ncols];
  uint64_t off = 0;
  int rc = ORC_OK;
  for (int64_t i = 0; i < row_count; ++i) {
    int64_t r = row_start + i;
    uint64_t var = 0;
    for (int32_t c = 0; c < ncols; ++c)
      if (types[c] == T_STRING) var += (uint64_t)(cols[c].offsets[r + 1] - cols[c].offsets[r]);
    uint64_t rsz = (uint64_t)round_up((int64_t)(spr + var), JCUDF_ROW_ALIGNMENT);
    if (off + rsz > (uint64_t)out_capacity || off + rsz > MAX_BATCH_SIZE) { rc = ORC_EOVERFLOW; break; }
    out_offsets[i] = (int32_t)off;
    uint8_t* row = out_data + off;
    memset(row, 0, rsz);
    uint32_t soff = (uint32_t)spr; /* RC:838: initial offset to variable-width data */
    for (int32_t c = 0; c < ncols; ++c) {
      if (types[c] == T_STRING) {
        int32_t s0 = cols[c].offsets[r];
        uint32_t len = (uint32_t)(cols[c].offsets[r + 1] - s0);
        memcpy(row + starts[c], &soff, 4);      /* RC:848 */
        memcpy(row + starts[c] + 4, &len, 4);   /* RC:849 */
        memcpy(row + soff, (const uint8_t*)cols[c].data + s0, len); /* RC:851-857 */
        soff += len;
      } else {
        memcpy(row + starts[c], (const uint8_t*)cols[c].data + (size_t)r * sizes[c], sizes[c]);
      }
      if (is_valid(cols[c].null_mask, r)) row[voff + c / 8] |= (uint8_t)(1u << (c % 8));
    }
    off += rsz;
  }
  if (rc == ORC_OK) out_offsets[row_count] = (int32_t)off;
  free(types); free(starts); free(sizes);
  return rc;
}

/*
 * convert_from_rows, phase 1 -- RC:2149-2372: fixed-width fields (copy_from_rows RC:879-969),
 * validity (copy_validity_from_rows RC:987-1094: tail bits of the last mask word are 0), and for
 * STRING columns the lengths (second uint32 of the pair) turned into offsets by an exclusive
 * scan (RC:2375-2388).  `row_offsets` NULL => fixed-width table, rows at stride
 * round_up(size_per_row, 8) (RC:279-289, 2317); else the LIST offsets are used (RC:2345).
 * cols[c].data must hold nrows*size bytes for fixed-width columns; cols[c].offsets nrows+1 ints
 * for STRING; cols[c].null_mask ceil(nrows/32) words (always written: RC:2220,2241).
 * char_totals[c] (if non-NULL) receives the chars size of STRING column c (RC:2390-2391).
 */
int orc_convert_from_rows_fixed(const uint8_t* rows, const int32_t* row_offsets, int64_t nrows,
                                orc_col* cols, int32_t ncols, int64_t* null_counts,
                                int64_t* char_totals)
{
  int32_t* types = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  int32_t* starts = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols + 1));
  int32_t* sizes = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  for (int32_t c = 0; c < ncols; ++c) types[c] = cols[c].type_id;
  int32_t spr = orc_compute_layout(types, ncols, starts, sizes);
  if (spr < 0) { free(types); free(starts); free(sizes); return spr; }
  int32_t voff = starts[ncols];
  int64_t stride = round_up(spr, JCUDF_ROW_ALIGNMENT);
  int64_t words = (nrows + 31) / 32;
  for (int32_t c = 0; c < ncols; ++c) {
    memset(cols[c].null_mask, 0, sizeof(uint32_t) * (size_t)words);
    if (null_counts) null_counts[c] = 0;
    if (types[c] == T_STRING) cols[c].offsets[0] = 0;
  }
  int rc = ORC_OK;
  for (int64_t r = 0; r < nrows && rc == ORC_OK; ++r) {
    const uint8_t* row = rows + (row_offsets ? (int64_t)row_offsets[r] : r * stride);
    for (int32_t c = 0; c < ncols; ++c) {
      if (types[c] == T_STRING) {
        uint32_t len;
        memcpy(&len, row + starts[c] + 4, 4);
        int64_t nxt = (int64_t)cols[c].offsets[r] + (int64_t)len;
        if (nxt > INT32_MAX) { rc = ORC_EOVERFLOW; break; }
        cols[c].offsets[r + 1] = (int32_t)nxt;
      } else {
        memcpy((uint8_t*)cols[c].data + (size_t)r * sizes[c], row + starts[c], sizes[c]);
      }
      if ((row[voff + c / 8] >> (c % 8)) & 1u) cols[c].null_mask[r >> 5] |= 1u << (r & 31);
      else if (null_counts) null_counts[c]++;
    }
  }
  if (char_totals)
    for (int32_t c = 0; c < ncols; ++c)
      char_totals[c] = (types[c] == T_STRING) ? cols[c].offsets[nrows] : 0;
  free(types); free(starts); free(sizes);
  return rc;
}

/*
 * convert_from_rows, phase 2 -- copy_strings_from_rows RC:1110-1150: chars of row r, column c are
 * copied from row + pair.offset (the FIRST uint32 of the pair, RC:1143) for pair.len bytes to
 * chars + offsets[r].
 */
int orc_convert_from_rows_strings(const uint8_t* rows, const int32_t* row_offsets, int64_t nrows,
                                  orc_col* cols, int32_t ncols)
{
  int32_t* types = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  int32_t* starts = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols + 1));
  int32_t* sizes = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  for (int32_t c = 0; c < ncols; ++c) types[c] = cols[c].type_id;
  int32_t spr = orc_compute_layout(types, ncols, starts, sizes);
  if (spr < 0) { free(types); free(starts); free(sizes); return spr; }
  int64_t stride = round_up(spr, JCUDF_ROW_ALIGNMENT);
  for (int64_t r = 0; r < nrows; ++r) {
    const uint8_t* row = rows + (row_offsets ? (int64_t)row_offsets[r] : r * stride);
    for (int32_t c = 0; c < ncols; ++c) {
      if (types[c] != T_STRING) continue;
      uint32_t so, len;
      memcpy(&so, row + starts[c], 4);
      memcpy(&len, row + starts[c] + 4, 4);
      memcpy((uint8_t*)cols[c].data + cols[c].offsets[r], row + so, len);
    }
  }
  free(types); free(starts); free(sizes);
  return ORC_OK;
}

/* ------------------------------------------------------------------------------------------
 * Hashes
 * ---------------------------------------------------------------------------------------- */

/* to_java_bigdecimal -- hash/hash.cuh:64-107: minimal big-endian two's complement bytes */
static int dec128_java_bytes(const uint8_t le[16], uint8_t out[16])
{
  int neg = (le[15] & 0x80) != 0;
  uint8_t zero = neg ? 0xff : 0x00;
  int length = 16;
  while (length > 0 && le[length - 1] == zero) --length; /* find_if_not from the top byte */
  if (length < 1) length = 1;                             /* hash.cuh:90-91 */
  if (length < 16 && (neg ^ ((le[length - 1] & 0x80) != 0))) ++length; /* hash.cuh:99-101 */
  for (int i = 0; i < length; ++i) out[i] = le[length - 1 - i];          /* reverse_copy :106 */
  return length;
}

/* normalize_nans / normalize_nans_and_zeros -- hash/hash.cuh:34-57 */
static uint32_t f32_norm(uint32_t bits, int zeros)
{
  float f; memcpy(&f, &bits, 4);
  if (zeros && f == 0.0f) return 0u;
  if (f != f) return 0x7fc00000u; /* numeric_limits<float>::quiet_NaN() */
  return bits;
}
static uint64_t f64_norm(uint64_t bits, int zeros)
{
  double d; memcpy(&d, &bits, 8);
  if (zeros && d == 0.0) return 0ull;
  if (d != d) return 0x7ff8000000000000ull;
  return bits;
}

/* ---- XXH64: hash/xxhash64.cu:73-199 ---- */
#define XP1 0x9E3779B185EBCA87ull
#define XP2 0xC2B2AE3D27D4EB4Full
#define XP3 0x165667B19E3779F9ull
#define XP4 0x85EBCA77C2B2AE63ull
#define XP5 0x27D4EB2F165667C5ull
static uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
static uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

uint64_t orc_xxh64_bytes(const uint8_t* data, int64_t n, uint64_t seed)
{
  int64_t off = 0;
  uint64_t h;
  if (n >= 32) { /* xxhash64.cu:127-172 */
    uint64_t v1 = seed + XP1 + XP2, v2 = seed + XP2, v3 = seed, v4 = seed - XP1;
    int64_t limit = n - 32;
    do {
      v1 = rotl64(v1 + rd64(data + off) * XP2, 31) * XP1; off += 8;
      v2 = rotl64(v2 + rd64(data + off) * XP2, 31) * XP1; off += 8;
      v3 = rotl64(v3 + rd64(data + off) * XP2, 31) * XP1; off += 8;
      v4 = rotl64(v4 + rd64(data + off) * XP2, 31) * XP1; off += 8;
    } while (off <= limit);
    h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = (h ^ (rotl64(v1 * XP2, 31) * XP1)) * XP1 + XP4;
    h = (h ^ (rotl64(v2 * XP2, 31) * XP1)) * XP1 + XP4;
    h = (h ^ (rotl64(v3 * XP2, 31) * XP1)) * XP1 + XP4;
    h = (h ^ (rotl64(v4 * XP2, 31) * XP1)) * XP1 + XP4;
  } else {
    h = seed + XP5; /* :174 */
  }
  h += (uint64_t)n;
  /* compute_remaining_bytes :85-117 */
  for (; off + 8 <= n; off += 8) {
    uint64_t k1 = rotl64(rd64(data + off) * XP2, 31) * XP1;
    h ^= k1;
    h = rotl64(h, 27) * XP1 + XP4;
  }
  if (off + 4 <= n) {
    h ^= (uint64_t)rd32(data + off) * XP1;
    h = rotl64(h, 23) * XP2 + XP3;
    off += 4;
  }
  for (; off < n; ++off) {
    h ^= (uint64_t)data[off] * XP5;
    h = rotl64(h, 11) * XP1;
  }
  /* finalize :181-189 */
  h ^= h >> 33; h *= XP2; h ^= h >> 29; h *= XP3; h ^= h >> 32;
  return h;
}

/* ---- Murmur3_x86_32 with Spark's tail: hash/murmur_hash.cuh:67-119 ---- */
static uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
uint32_t orc_murmur3_bytes(const uint8_t* data, int32_t len, uint32_t seed)
{
  const uint32_t c1 = 0xcc9e2d51u, c2 = 0x1b873593u, c3 = 0xe6546b64u;
  uint32_t h = seed;
  int32_t nblocks = len / 4;
  for (int32_t i = 0; i < nblocks; ++i) {
    uint32_t k1 = rd32(data + 4 * i);
    k1 *= c1; k1 = rotl32(k1, 15); k1 *= c2;
    h ^= k1; h = rotl32(h, 13); h = h * 5 + c3;
  }
  for (int32_t i = nblocks * 4; i < len; ++i) { /* Spark tail: each byte sign-extended, :72-93 */
    uint32_t k1 = (uint32_t)(int32_t)(int8_t)data[i];
    k1 *= c1; k1 = rotl32(k1, 15); k1 *= c2;
    h ^= k1; h = rotl32(h, 13); h = h * 5 + c3;
  }
  h ^= (uint32_t)len;
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16; /* fmix32 :42-50 */
  return h;
}

/*
 * Element -> bytes-to-hash for xxhash64 / murmur (they share the type rules):
 *   xxhash64.cu:201-273 and murmur_hash.cuh:130-205.  zeros=1 for xxhash64 (normalises -0.0,
 *   xxhash64.cu:231-241), zeros=0 for murmur (murmur_hash.cuh:163-173).
 * Returns the byte count, or <0 for unsupported types (nested / dictionary).
 */
static int elem_bytes(const orc_col* c, int64_t r, int zeros, uint8_t buf[16], const uint8_t** ext)
{
  *ext = NULL;
  const uint8_t* d = (const uint8_t*)c->data;
  switch (c->type_id) {
    case T_BOOL8: { uint32_t v = d[r] != 0; memcpy(buf, &v, 4); return 4; }
    case T_INT8: { uint32_t v = (uint32_t)(int32_t)((const int8_t*)d)[r]; memcpy(buf, &v, 4); return 4; }
    case T_UINT8: { uint32_t v = d[r]; memcpy(buf, &v, 4); return 4; }
    case T_INT16: { uint32_t v = (uint32_t)(int32_t)((const int16_t*)d)[r]; memcpy(buf, &v, 4); return 4; }
    case T_UINT16: { uint32_t v = ((const uint16_t*)d)[r]; memcpy(buf, &v, 4); return 4; }
    case T_FLOAT32: { uint32_t v = f32_norm(((const uint32_t*)d)[r], zeros); memcpy(buf, &v, 4); return 4; }
    case T_FLOAT64: { uint64_t v = f64_norm(((const uint64_t*)d)[r], zeros); memcpy(buf, &v, 8); return 8; }
    case T_DEC32: { uint64_t v = (uint64_t)(int64_t)((const int32_t*)d)[r]; memcpy(buf, &v, 8); return 8; }
    case T_DEC64: { memcpy(buf, d + 8 * r, 8); return 8; }
    case T_DEC128: return dec128_java_bytes(d + 16 * r, buf);
    case T_STRING: { *ext = d + c->offsets[r]; return c->offsets[r + 1] - c->offsets[r]; }
    default: {
      int32_t sz = orc_size_of(c->type_id);
      if (sz == 4 || sz == 8) { memcpy(buf, d + (size_t)sz * r, sz); return sz; } /* compute<T> :72-76 */
      return ORC_EUNSUPPORTED;
    }
  }
}

/* xxhash64 row hash -- hash/xxhash64.cu:310-323,352-353,550-579: h = seed; per column: null keeps h */
int orc_xxhash64(const orc_col* cols, int32_t ncols, int64_t nrows, int64_t seed, int64_t* out)
{
  int rc = ORC_OK;
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < nrows; ++r) {
    uint64_t h = (uint64_t)seed;
    for (int32_t c = 0; c < ncols; ++c) {
      if (!is_valid(cols[c].null_mask, r)) continue;
      uint8_t buf[16]; const uint8_t* ext;
      int n = elem_bytes(&cols[c], r, 1, buf, &ext);
      if (n < 0) { rc = n; continue; }
      h = orc_xxh64_bytes(ext ? ext : buf, n, h);
    }
    out[r] = (int64_t)h;
  }
  return rc;
}

/* murmur_hash3_32 row hash -- hash/murmur_hash.cu:76-86,111-117,191-221 */
int orc_murmur3_32(const orc_col* cols, int32_t ncols, int64_t nrows, uint32_t seed, int32_t* out)
{
  int rc = ORC_OK;
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < nrows; ++r) {
    uint32_t h = seed;
    for (int32_t c = 0; c < ncols; ++c) {
      if (!is_valid(cols[c].null_mask, r)) continue;
      uint8_t buf[16]; const uint8_t* ext;
      int n = elem_bytes(&cols[c], r, 0, buf, &ext);
      if (n < 0) { rc = n; continue; }
      h = orc_murmur3_bytes(ext ? ext : buf, n, h);
    }
    out[r] = (int32_t)h;
  }
  return rc;
}

/* hive hash -- hash/hive_hash.cu:42-152 (element), :179-191 (fold h = 31*h + x), :201-203 (null -> 0) */
static int hive_elem(const orc_col* c, int64_t r, int32_t* out)
{
  const uint8_t* d = (const uint8_t*)c->data;
  switch (c->type_id) {
    case T_BOOL8: *out = d[r] != 0; return 0;
    case T_INT8: *out = ((const int8_t*)d)[r]; return 0;
    case T_INT16: *out = ((const int16_t*)d)[r]; return 0;
    case T_INT32: case T_TS_DAYS: *out = ((const int32_t*)d)[r]; return 0;
    case T_INT64: { uint64_t k = ((const uint64_t*)d)[r]; *out = (int32_t)((k >> 32) ^ k); return 0; }
    case T_FLOAT32: *out = (int32_t)f32_norm(((const uint32_t*)d)[r], 0); return 0;
    case T_FLOAT64: { uint64_t k = f64_norm(((const uint64_t*)d)[r], 0); *out = (int32_t)((k >> 32) ^ k); return 0; }
    case T_TS_US: { /* :135-152, C++ truncating / and % */
      int64_t t = ((const int64_t*)d)[r];
      int64_t ts = t / 1000000, tns = (t % 1000000) * 1000;
      uint64_t res = ((uint64_t)ts << 30) | (uint64_t)tns;
      *out = (int32_t)((res >> 32) ^ res);
      return 0;
    }
    case T_STRING: { /* :49-56 */
      uint32_t h = 0;
      for (int32_t i = c->offsets[r]; i < c->offsets[r + 1]; ++i) h = h * 31u + (uint32_t)(int32_t)(int8_t)d[i];
      *out = (int32_t)h;
      return 0;
    }
    default: return ORC_EUNSUPPORTED; /* :63-66 CUDF_UNREACHABLE */
  }
}

int orc_hive_hash(const orc_col* cols, int32_t ncols, int64_t nrows, int32_t* out)
{
  int rc = ORC_OK;
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < nrows; ++r) {
    uint32_t h = 0;
    for (int32_t c = 0; c < ncols; ++c) {
      int32_t x = 0;
      if (is_valid(cols[c].null_mask, r)) { int e = hive_elem(&cols[c], r, &x); if (e < 0) rc = e; }
      h = 31u * h + (uint32_t)x;
    }
    out[r] = (int32_t)h;
  }
  return rc;
}

/* ---- single-element entry points for the nested-type restatement in oracle.py (LIST / STRUCT keys: the tree walk is
 * done in Python over small tables; xxhash64.cu:446-506, murmur_hash.cu:119-144, hive_hash.cu:363-433) ------------- */
uint64_t orc_xx_elem(const orc_col* c, int64_t r, uint64_t h)   /* a null element keeps the accumulator */
{
  if (!is_valid(c->null_mask, r)) return h;
  uint8_t buf[16]; const uint8_t* ext;
  int n = elem_bytes(c, r, 1, buf, &ext);
  return n < 0 ? h : orc_xxh64_bytes(ext ? ext : buf, n, h);
}
uint32_t orc_mm_elem(const orc_col* c, int64_t r, uint32_t h)
{
  if (!is_valid(c->null_mask, r)) return h;
  uint8_t buf[16]; const uint8_t* ext;
  int n = elem_bytes(c, r, 0, buf, &ext);
  return n < 0 ? h : orc_murmur3_bytes(ext ? ext : buf, n, h);
}
int32_t orc_hive_leaf(const orc_col* c, int64_t r)              /* a null element hashes to 0 */
{
  int32_t x = 0;
  if (is_valid(c->null_mask, r)) hive_elem(c, r, &x);
  return x;
}

/* ------------------------------------------------------------------------------------------
 * CPU baseline ("Spark InternalRow -> ColumnarBatch on host cores", BASELINE.md section 3):
 * the same per-row / per-field loops as above, one contiguous row range per thread.  Used only
 * by bench.py's cpu_baseline and --impl reference legs.
 * ---------------------------------------------------------------------------------------- */
int orc_num_threads(void)
{
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* fixed-width row->column, threaded over 32-row-aligned ranges (mask words never shared) */
int orc_from_rows_fixed_mt(const uint8_t* rows, int64_t nrows, orc_col* cols, int32_t ncols, int nthreads)
{
  int32_t* types = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  int32_t* starts = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols + 1));
  int32_t* sizes = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  for (int32_t c = 0; c < ncols; ++c) types[c] = cols[c].type_id;
  int32_t spr = orc_compute_layout(types, ncols, starts, sizes);
  if (spr < 0) { free(types); free(starts); free(sizes); return spr; }
  for (int32_t c = 0; c < ncols; ++c) if (types[c] == T_STRING) { free(types); free(starts); free(sizes); return ORC_EUNSUPPORTED; }
  int32_t voff = starts[ncols];
  int64_t stride = round_up(spr, JCUDF_ROW_ALIGNMENT);
  int64_t nblk = (nrows + 31) / 32;
  if (nthreads < 1) nthreads = 1;
#pragma omp parallel for schedule(static) num_threads(nthreads)
  for (int64_t b = 0; b < nblk; ++b) {
    int64_t r0 = b * 32, r1 = r0 + 32 > nrows ? nrows : r0 + 32;
    for (int32_t c = 0; c < ncols; ++c) cols[c].null_mask[b] = 0;
    for (int64_t r = r0; r < r1; ++r) {
      const uint8_t* row = rows + r * stride;
      for (int32_t c = 0; c < ncols; ++c) {
        /* per field: isNullAt -> putNull / typed put */
        if ((row[voff + c / 8] >> (c % 8)) & 1u) cols[c].null_mask[b] |= 1u << (r & 31);
        memcpy((uint8_t*)cols[c].data + (size_t)r * sizes[c], row + starts[c], sizes[c]);
      }
    }
  }
  free(types); free(starts); free(sizes);
  return ORC_OK;
}

/* general (strings allowed) row->column, threaded; string offsets need a serial scan, so the
 * threaded part is phase 1 lengths + fixed fields, then scan, then chars. */
int orc_from_rows_mt(const uint8_t* rows, const int32_t* row_offsets, int64_t nrows, orc_col* cols,
                     int32_t ncols, int nthreads)
{
  int32_t* types = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  int32_t* starts = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols + 1));
  int32_t* sizes = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  for (int32_t c = 0; c < ncols; ++c) types[c] = cols[c].type_id;
  int32_t spr = orc_compute_layout(types, ncols, starts, sizes);
  if (spr < 0) { free(types); free(starts); free(sizes); return spr; }
  int32_t voff = starts[ncols];
  int64_t stride = round_up(spr, JCUDF_ROW_ALIGNMENT);
  int64_t nblk = (nrows + 31) / 32;
  if (nthreads < 1) nthreads = 1;
#pragma omp parallel for schedule(static) num_threads(nthreads)
  for (int64_t b = 0; b < nblk; ++b) {
    int64_t r0 = b * 32, r1 = r0 + 32 > nrows ? nrows : r0 + 32;
    for (int32_t c = 0; c < ncols; ++c) cols[c].null_mask[b] = 0;
    for (int64_t r = r0; r < r1; ++r) {
      const uint8_t* row = rows + (row_offsets ? (int64_t)row_offsets[r] : r * stride);
      for (int32_t c = 0; c < ncols; ++c) {
        if ((row[voff + c / 8] >> (c % 8)) & 1u) cols[c].null_mask[b] |= 1u << (r & 31);
        if (types[c] == T_STRING) memcpy(&cols[c].offsets[r + 1], row + starts[c] + 4, 4);
        else memcpy((uint8_t*)cols[c].data + (size_t)r * sizes[c], row + starts[c], sizes[c]);
      }
    }
  }
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads)
  for (int32_t c = 0; c < ncols; ++c) {
    if (types[c] != T_STRING) continue;
    int32_t acc = 0;
    cols[c].offsets[0] = 0;
    for (int64_t r = 0; r < nrows; ++r) { acc += cols[c].offsets[r + 1]; cols[c].offsets[r + 1] = acc; }
  }
  if (cols && ncols) {
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (int64_t r = 0; r < nrows; ++r) {
      const uint8_t* row = rows + (row_offsets ? (int64_t)row_offsets[r] : r * stride);
      for (int32_t c = 0; c < ncols; ++c) {
        if (types[c] != T_STRING || !cols[c].data) continue;
        uint32_t so, len;
        memcpy(&so, row + starts[c], 4);
        memcpy(&len, row + starts[c] + 4, 4);
        memcpy((uint8_t*)cols[c].data + cols[c].offsets[r], row + so, len);
      }
    }
  }
  free(types); free(starts); free(sizes);
  return ORC_OK;
}

/* column->row for a batch whose offsets are already known, threaded over rows */
int orc_to_rows_mt(const orc_col* cols, int32_t ncols, int64_t row_start, int64_t row_count,
                   const int32_t* offsets, uint8_t* out_data, int nthreads)
{
  int32_t* types = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  int32_t* starts = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols + 1));
  int32_t* sizes = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ncols ? ncols : 1));
  for (int32_t c = 0; c < ncols; ++c) types[c] = cols[c].type_id;
  int32_t spr = orc_compute_layout(types, ncols, starts, sizes);
  if (spr < 0) { free(types); free(starts); free(sizes); return spr; }
  int32_t voff = starts[ncols];
  if (nthreads < 1) nthreads = 1;
#pragma omp parallel for schedule(static) num_threads(nthreads)
  for (int64_t i = 0; i < row_count; ++i) {
    int64_t r = row_start + i;
    uint8_t* row = out_data + offsets[i];
    memset(row, 0, (size_t)(offsets[i + 1] - offsets[i]));
    uint32_t soff = (uint32_t)spr;
    for (int32_t c = 0; c < ncols; ++c) {
      if (types[c] == T_STRING) {
        int32_t s0 = cols[c].offsets[r];
        uint32_t len = (uint32_t)(cols[c].offsets[r + 1] - s0);
        memcpy(row + starts[c], &soff, 4);
        memcpy(row + starts[c] + 4, &len, 4);
        memcpy(row + soff, (const uint8_t*)cols[c].data + s0, len);
        soff += len;
      } else {
        memcpy(row + starts[c], (const uint8_t*)cols[c].data + (size_t)r * sizes[c], sizes[c]);
      }
      if (is_valid(cols[c].null_mask, r)) row[voff + c / 8] |= (uint8_t)(1u << (c % 8));
    }
  }
  free(types); free(starts); free(sizes);
  return ORC_OK;
}
