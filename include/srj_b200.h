/*
 * srj_b200.h -- C ABI of libsrj_b200.so: the H100-native (sm_90a) replacement for the
 * row<->columnar + Spark row-hash hot path of NVIDIA/spark-rapids-jni.
 *
 * This is the drop-in boundary (SURVEY.md 8b).  Every entry point below is what the reference's
 * JNI layer for this path would bind; each cites the reference interface it replaces.  Paths are
 * relative to the reference tree; RC = src/main/cpp/src/row_conversion.cu.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only.  All data pointers are DEVICE pointers owned by the
 *     caller (the JNI shim allocates them with rmm exactly where the reference does); functions
 *     whose name ends in _host take HOST pointers and stage through the device themselves.
 *   - Every function returns SRJ_OK (0) or a negative srj_status; nothing throws across the
 *     boundary.  srj_last_error() returns a thread-local message for the last failure.
 *     The JNI shim maps codes to the reference's exception classes (INTEGRATION.md):
 *       SRJ_EINVAL/SRJ_EUNSUPPORTED -> ai.rapids.cudf.CudfException (cudf::logic_error, error.hpp:233-239)
 *       SRJ_EOVERFLOW -> CudfColumnSizeOverflowException, SRJ_ENOMEM -> OutOfMemoryError,
 *       SRJ_ECUDA -> CudaException / CudaFatalException.
 *   - Work is enqueued on the caller's `stream` (the reference uses the per-thread default
 *     stream, CMakeLists.txt:322-326); functions are re-entrant and keep no global mutable state.
 *     Functions documented "synchronizes" block until `stream` is idle because they return
 *     host-visible sizes (the reference synchronises at the same points: RC:1534-1544, 2389).
 *   - Bitmasks are cudf bitmasks: uint32 words, bit (i % 32) of word (i / 32), 1 = valid
 *     (thirdparty/cudf/cpp/include/cudf/utilities/bit.hpp:48-106).  NULL mask = all valid.
 *   - Row counts are int64 at this ABI; the JNI shim passes cudf::size_type (int32) values.
 */
#ifndef SRJ_B200_H
#define SRJ_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SRJ_API __attribute__((visibility("default")))
#else
#define SRJ_API
#endif

/* ---- status codes --------------------------------------------------------------------------- */
typedef enum srj_status {
  SRJ_OK           = 0,
  SRJ_EINVAL       = -1, /* bad argument / layout precondition (CUDF_EXPECTS -> cudf::logic_error)  */
  SRJ_EUNSUPPORTED = -2, /* type not supported on this path (RowConversion.java:131, hive_hash.cu:63) */
  SRJ_EOVERFLOW    = -3, /* a column would exceed the int32 size_type limit (std::overflow_error)    */
  SRJ_ECUDA        = -4, /* CUDA runtime error (cudf::cuda_error)                                    */
  SRJ_ENOMEM       = -5  /* device allocation failed (rmm::out_of_memory)                            */
} srj_status;

/* ---- cudf type ids: thirdparty/cudf/cpp/include/cudf/types.hpp:191-224 ----------------------- */
typedef enum srj_type_id {
  SRJ_EMPTY = 0, SRJ_INT8, SRJ_INT16, SRJ_INT32, SRJ_INT64, SRJ_UINT8, SRJ_UINT16, SRJ_UINT32, SRJ_UINT64,
  SRJ_FLOAT32, SRJ_FLOAT64, SRJ_BOOL8, SRJ_TIMESTAMP_DAYS, SRJ_TIMESTAMP_SECONDS,
  SRJ_TIMESTAMP_MILLISECONDS, SRJ_TIMESTAMP_MICROSECONDS, SRJ_TIMESTAMP_NANOSECONDS,
  SRJ_DURATION_DAYS, SRJ_DURATION_SECONDS, SRJ_DURATION_MILLISECONDS, SRJ_DURATION_MICROSECONDS,
  SRJ_DURATION_NANOSECONDS, SRJ_DICTIONARY32, SRJ_STRING, SRJ_LIST, SRJ_DECIMAL32, SRJ_DECIMAL64,
  SRJ_DECIMAL128, SRJ_STRUCT, SRJ_NUM_TYPE_IDS
} srj_type_id;

/*
 * srj_column: the cudf::column_view fields this path reads/writes
 * (thirdparty/cudf/cpp/include/cudf/column/column_view.hpp:237-244).  One struct serves inputs and
 * outputs; for outputs the caller allocates every buffer and the library fills it.
 *   fixed-width column : data = size * size_of(type) bytes
 *   STRING column      : data = chars, offsets = int32[size + 1]   (RC:1919-1923, 2421-2428)
 *   LIST column        : offsets = int32[size + 1], children[0] = the element column     (hash entry points only)
 *   STRUCT column      : children[0 .. num_children) = the fields, each `size` rows        (hash entry points only)
 * Sliced views (offset != 0) are not supported, as in the reference (RC:1809-1811).
 */
typedef struct srj_column {
  int32_t type_id;     /* srj_type_id                                        */
  int32_t scale;       /* decimals only; carried, never interpreted           */
  int64_t size;        /* rows                                                */
  void* data;          /* device                                              */
  uint32_t* null_mask; /* device, ceil(size/32) words, or NULL (= all valid)  */
  int32_t* offsets;    /* device, STRING / LIST                               */
  const struct srj_column* children; /* HOST array of child descriptors (LIST / STRUCT), else NULL */
  int32_t num_children;
  int32_t reserved;
} srj_column;

/* One output batch of convert_to_rows = one LIST<INT8> column of <= INT32_MAX bytes (RC:174-190). */
typedef struct srj_row_batch {
  int64_t row_start; /* first table row in this batch                     */
  int64_t row_count; /* rows in this batch (multiple of 32 except the last, RC:1515-1517) */
  int64_t num_bytes; /* size of the INT8 child                            */
} srj_row_batch;

/* ---- library --------------------------------------------------------------------------------- */
SRJ_API const char* srj_version(void);
SRJ_API const char* srj_last_error(void);
SRJ_API const char* srj_status_string(int status);

/* ---- layout: compute_column_information, RC:1332-1371 ---------------------------------------- */
typedef struct srj_layout {
  int32_t num_columns;
  int32_t num_string_columns;
  int32_t validity_offset;    /* byte offset of the validity bytes in a row                 */
  int32_t size_per_row;       /* validity_offset + ceil(ncols/8): UNPADDED fixed+validity   */
  int32_t fixed_row_size;     /* round_up(size_per_row, 8): the row stride of a fixed-width-only table */
  int32_t reserved;
} srj_layout;

/* col_starts/col_sizes (each num_columns entries) may be NULL. */
SRJ_API int srj_compute_layout(const int32_t* type_ids, int32_t num_columns, srj_layout* out,
                               int32_t* col_starts, int32_t* col_sizes);

/*
 * A plan caches the per-schema device metadata (column starts/sizes, width-class schedule) so the
 * hot calls do no host->device metadata traffic.  Create once per schema per device (the JNI shim
 * keeps a small schema-keyed cache); destroy when done.  Plans are immutable => thread-safe.
 */
typedef struct srj_plan srj_plan;
SRJ_API int srj_plan_create(const int32_t* type_ids, const int32_t* scales /* may be NULL */,
                            int32_t num_columns, srj_plan** out);
SRJ_API void srj_plan_destroy(srj_plan* plan);
SRJ_API int srj_plan_layout(const srj_plan* plan, srj_layout* out);

/* ---- convert_to_rows: RowConversion.convertToRows / RC:1994-2055 ------------------------------ */
/*
 * Step 1 (synchronizes when the table has STRING columns): per-row sizes (RC:201-257) and the
 * <= 2 GiB / 32-row batch cut (build_batches, RC:1466-1557).  `workspace` must hold
 * srj_to_rows_workspace_bytes(plan, num_rows) bytes (0 for fixed-width-only tables) and must be
 * passed unchanged to step 2.  Writes up to max_batches entries; *num_batches gets the count
 * (0 for an empty table: the caller then returns one empty LIST column, SURVEY App. C.4).
 */
SRJ_API int64_t srj_to_rows_workspace_bytes(const srj_plan* plan, int64_t num_rows);
SRJ_API int srj_to_rows_plan_batches(const srj_plan* plan, const srj_column* cols, int64_t num_rows,
                                     void* workspace, srj_row_batch* batches, int32_t max_batches,
                                     int32_t* num_batches, void* stream);
/*
 * Step 2 (async): fill each batch's LIST offsets child (int32[row_count + 1]) and INT8 data child
 * (num_bytes).  Fuses copy_to_rows + copy_validity_to_rows + copy_strings_to_rows
 * (RC:574-688, 706-798, 816-861).  Padding bytes are written as zeros (undefined in the reference).
 * `workspace` is the buffer step 1 filled: its cumulative row sizes are only read, the scratch
 * words behind them (scan partials, dead after step 1) carry a 4-byte device flag of the fast
 * variable-width kernel -- so two step-2 calls must not share one workspace concurrently.
 */
SRJ_API int srj_convert_to_rows(const srj_plan* plan, const srj_column* cols, int64_t num_rows,
                                const void* workspace, const srj_row_batch* batches,
                                int32_t num_batches, int32_t* const* batch_offsets,
                                uint8_t* const* batch_data, void* stream);

/* ---- convert_from_rows: RowConversion.convertFromRows / RC:2149-2441 -------------------------- */
/*
 * Phase 1 (async): fixed-width columns, every column's validity mask, exact null counts
 * (replaces fixup_null_counts, RC:2130-2136) and, for STRING columns, the offsets child
 * (lengths + exclusive scan, RC:2375-2388).  Fuses copy_from_rows + copy_validity_from_rows
 * (RC:879-969, 987-1094).
 *   rows        : the LIST's INT8 child
 *   row_offsets : the LIST's offsets child (int32[num_rows + 1]) or NULL for a fixed-width-only
 *                 schema, where rows are read at stride fixed_row_size exactly as the reference
 *                 does (RC:2317; it ignores the offsets there too, SURVEY App. C.5)
 *   rows_bytes  : size of `rows`; checked against size_per_row * num_rows (RC:2197)
 *   cols        : num_columns outputs; data (fixed-width), null_mask and (STRING) offsets must be
 *                 allocated; STRING data (chars) may be NULL in this phase
 *   d_null_counts : device int64[num_columns] or NULL
 *   d_char_totals : device int64[num_columns + 1] or NULL.  Entries [0, num_columns) receive the chars size
 *                 of each STRING column (0 for the others); the caller reads them back (that read is the
 *                 one sync the reference also has, RC:2389) to size the chars.  Entry [num_columns] is a
 *                 status word for phase 2: bit 0 set = some row does not use the canonical string layout
 *                 (pair.offset != size_per_row + lengths of the preceding STRING columns); phase 2 then
 *                 follows the stored pair offsets exactly like copy_strings_from_rows (RC:1143) instead of
 *                 its fast path.  Bit 1 set = a STRING column's chars exceed INT32_MAX (the caller maps it to
 *                 SRJ_EOVERFLOW / CudfColumnSizeOverflowException; the totals themselves are exact int64).
 *                 The STRING offsets children are complete only after phase 2.
 * If hash_kind != SRJ_HASH_NONE the row hash of the listed key columns is computed in the same call, from
 * the key columns just written, and written to hash_out (int64 for xxhash64, int32 otherwise): the fused
 * from_rows + partition-hash of BASELINE config 4.  Keys must be fixed-width columns.
 */
/*
 * Workspace of one phase-1 / phase-2 call pair: srj_from_rows_workspace_bytes(plan, num_rows) bytes of device memory
 * (0 for schemas that need none; then NULL may be passed).  Phase 1 leaves there what phase 2 needs besides the
 * offsets children (for wide tables: the chars of every STRING column before each 32-row group -- the offsets
 * children themselves hold group-local sums between the two calls and are finished by phase 2), so the same
 * buffer must be passed to both calls and must not be shared by two conversions in flight.
 */
SRJ_API int64_t srj_from_rows_workspace_bytes(const srj_plan* plan, int64_t num_rows);

typedef enum srj_hash_kind { SRJ_HASH_NONE = 0, SRJ_HASH_XXHASH64 = 1, SRJ_HASH_MURMUR3_32 = 2, SRJ_HASH_HIVE = 3 } srj_hash_kind;

typedef struct srj_fused_hash {
  int32_t kind;            /* srj_hash_kind */
  int32_t num_keys;        /* <= 16 */
  int32_t key_columns[16]; /* indices into the schema, hashed in this order */
  int64_t seed;            /* xxhash64: int64 seed; murmur: low 32 bits; hive: ignored */
  void* out;               /* device, num_rows elements */
} srj_fused_hash;

SRJ_API int srj_convert_from_rows_fixed(const srj_plan* plan, const uint8_t* rows,
                                        const int32_t* row_offsets, int64_t rows_bytes,
                                        int64_t num_rows, const srj_column* cols,
                                        int64_t* d_null_counts, int64_t* d_char_totals,
                                        const srj_fused_hash* hash /* may be NULL */, void* workspace,
                                        void* stream);
/* Phase 2 (async): gather the chars of every STRING column (copy_strings_from_rows, RC:1110-1150).
 * d_char_totals is the buffer phase 1 filled (its status word selects the fast path); NULL = always
 * follow the stored pair offsets. */
SRJ_API int srj_convert_from_rows_strings(const srj_plan* plan, const uint8_t* rows,
                                          const int32_t* row_offsets, int64_t rows_bytes, int64_t num_rows,
                                          const srj_column* cols, const int64_t* d_char_totals,
                                          const void* workspace, void* stream);

/* ---- row hashes: Hash.xxhash64 / murmurHash32 / hiveHash, hash/hash.hpp:40-74 ------------------ */
#define SRJ_DEFAULT_XXHASH64_SEED 42 /* hash/hash.hpp:27 */
#define SRJ_MAX_STACK_DEPTH 8        /* hash/hash.hpp:28: nesting limit of LIST / STRUCT keys */
SRJ_API int srj_get_max_stack_depth(void); /* Hash.getMaxStackDepth, HashJni.cpp:26-30 */
/* out has no null mask (xxhash64.cu:556-562).  num_columns == 0 or num_rows == 0 is a no-op.
 * LIST / STRUCT keys are hashed like the reference (xxhash64.cu:446-506, murmur_hash.cu:119-144,
 * hive_hash.cu:363-433): xxhash64 / murmur chain the leaf values depth first (nulls keep the accumulator; murmur
 * rejects LIST<STRUCT>, murmur_hash.cu:167-187), hive folds 31 * h + x over the fields of a struct and over the
 * elements of a list.  Nesting beyond SRJ_MAX_STACK_DEPTH returns SRJ_EINVAL (CudfException). */
SRJ_API int srj_xxhash64(const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t seed,
                         int64_t* out, void* stream);
SRJ_API int srj_murmur_hash3_32(const srj_column* cols, int32_t num_columns, int64_t num_rows,
                                uint32_t seed, int32_t* out, void* stream);
SRJ_API int srj_hive_hash(const srj_column* cols, int32_t num_columns, int64_t num_rows, int32_t* out,
                          void* stream);

/* ---- SHA-2 of a STRING column, nulls preserved: Hash.sha{224,256,384,512}NullsPreserved, hash/sha.cpp:31-49 ----------
 * FIPS 180-4 SHA-224 / SHA-256 / SHA-384 / SHA-512 of each row's bytes as lowercase hex: 56 / 64 / 96 / 128 chars per
 * valid row (the empty string hashes normally).  A null row gives a null output row of zero length; the output mask equals
 * the input's.  Two steps, like the other STRING outputs:
 *   srj_sha2_workspace_bytes : bytes of the sizes call's workspace (needed only when the input has a null mask).
 *   srj_sha2_sizes           : d_out_offsets[rows + 1] of the output and *total_chars (host).  Without an input mask the
 *                              offsets are width x row and the call does not synchronise; with one it scans the mask
 *                              and reads the valid count back (one stream synchronisation).  SRJ_EOVERFLOW when the chars
 *                              would exceed INT32_MAX (nothing is written then).
 *   srj_sha2_hash            : (async) writes the chars into out->data (16-byte aligned; may be NULL only when
 *                              *total_chars was 0) at out->offsets (the sizes call's output), and copies the input mask to
 *                              out->null_mask when out has one (all valid when the input has none).  An input with a
 *                              mask needs an output mask.
 * digest_bits is 224, 256, 384 or 512 (else SRJ_EINVAL); the input must be one STRING column (else SRJ_EUNSUPPORTED),
 * <= INT32_MAX rows.  The output null count equals the input's.
 */
SRJ_API int64_t srj_sha2_workspace_bytes(int64_t num_rows);
SRJ_API int srj_sha2_sizes(int32_t digest_bits, const srj_column* input, int32_t* d_out_offsets, int64_t* total_chars, void* workspace,
                           void* stream);
SRJ_API int srj_sha2_hash(int32_t digest_bits, const srj_column* input, const srj_column* out, void* stream);

/* ---- Hash.hostCrc32, hash/HashJni.cpp:143-157: zlib crc32 on the HOST ------------------------------------------------
 * *out = crc32(crc, buf[0 .. len)), equal to zlib's crc32 and java.util.zip.CRC32, chaining from a previous value.
 * buf may be NULL only when len == 0; len < 0 or a NULL buffer with len > 0 is SRJ_EINVAL.  Touches no device.
 */
SRJ_API int srj_host_crc32(uint32_t crc, const void* buf, int64_t len, uint32_t* out);

/* ---- Spark BloomFilter: BloomFilter.create / put / merge / probe, bloom_filter.hpp:32-162, bloom_filter.cu:288-497 ------
 * The serialized filter of Spark's BloomFilterImpl.writeTo, big-endian throughout:
 *   V1: int32 {1, num_hashes, num_longs} (12 bytes), then num_longs longs
 *   V2: int32 {2, num_hashes, seed, num_longs} (16 bytes), then num_longs longs
 * Bit p lives in bit p % 64 of long p / 64; every position is taken modulo num_longs * 64.  A key x sets / tests the k
 * positions of Spark's double hashing over h1 = Murmur3 hashLong(x, seed) and h2 = hashLong(x, h1) (seed 0 for V1): V1
 * with 32-bit combined hashes, V2 with 64-bit ones (bloom_filter.cu:70-152).
 *   srj_bloom_filter_sizes : (host only, no device) num_longs = ceil(bits / 64) and the serialized size.  SRJ_EINVAL for a
 *                            version other than 1 / 2, num_hashes <= 0, bits <= 0, bits > INT32_MAX * 64 (the JNI shim
 *                            throws IllegalArgumentException for these) or a size over INT32_MAX bytes.
 *   srj_bloom_filter_init  : writes the header and zeroes the bit array of `filter` (the sizes call's total_bytes).
 *   srj_bloom_filter_put   : sets the bits of every valid row of `input`; null rows are skipped.
 *   srj_bloom_filter_probe : out[r] (BOOL8) = 1 when all the bits of row r are set.  The input mask is copied to out_mask
 *                            when out_mask is not NULL (all valid when the input has none); an input with a mask needs
 *                            out_mask.  Values under null rows are unspecified.  The output null count is the input's.
 *   srj_bloom_filter_merge : `filters` holds num_filters serialized filters back to back (the child of a LIST<UINT8>
 *                            column); `out` (filters_bytes / num_filters bytes) receives the first one's header and the
 *                            word-wise OR of all bit arrays.  SRJ_EINVAL when the first header does not parse, when
 *                            filters_bytes != num_filters x its size, or when any header differs from the first (version,
 *                            num_hashes, seed or size).  The workspace holds srj_bloom_filter_merge_workspace_bytes() bytes.
 * put / probe / merge read the filter's 16 header bytes back to the host once and synchronise the stream for it (the
 * reference does the same in every call, bloom_filter.cu:201-203); merge reads its header-check flag back with that same
 * synchronisation.  Errors of put / probe: a truncated filter, an unknown version, a bit array that is empty or whose size
 * disagrees with filter_bytes, and (V1) num_longs * 64 > INT32_MAX are SRJ_EINVAL; an input that is not one INT64 column is
 * SRJ_EUNSUPPORTED.  Filter and output buffers must be 4-byte aligned.
 */
#define SRJ_BLOOM_FILTER_VERSION_1 1
#define SRJ_BLOOM_FILTER_VERSION_2 2
SRJ_API int srj_bloom_filter_sizes(int32_t version, int32_t num_hashes, int64_t bits, int32_t* num_longs, int64_t* total_bytes);
SRJ_API int srj_bloom_filter_init(int32_t version, int32_t num_hashes, int32_t num_longs, int32_t seed, uint8_t* filter, void* stream);
SRJ_API int srj_bloom_filter_put(uint8_t* filter, int64_t filter_bytes, const srj_column* input, void* stream);
SRJ_API int srj_bloom_filter_probe(const uint8_t* filter, int64_t filter_bytes, const srj_column* input, uint8_t* out,
                                   uint32_t* out_mask, void* stream);
SRJ_API int64_t srj_bloom_filter_merge_workspace_bytes(void);
SRJ_API int srj_bloom_filter_merge(const uint8_t* filters, int64_t filters_bytes, int32_t num_filters, uint8_t* out, void* workspace,
                                   void* stream);

/* ---- ZOrder.interleaveBits / hilbertIndex, ZOrder.java:29-87, zorder.cu:137-267 --------------------------------------
 * Both read a row's N values MSB first, column-interleaved: stream position i holds bit B - 1 - i / N of column i % N,
 * where a value is its little-endian bytes as an unsigned B-bit integer (two's complement, raw IEEE bits) and a null row
 * counts as 0.
 *   srj_interleave_bits_sizes : (host only, no device) *total_bytes = num_rows * N * W.  Checks every argument of
 *                               srj_interleave_bits: N >= 1 columns of num_rows rows each, one fixed-width type id for all
 *                               of them (DECIMAL scales are not compared); W is its size.  SRJ_EUNSUPPORTED for a type that
 *                               is not fixed-width, SRJ_EINVAL for the rest, including num_rows * N * W > INT32_MAX.
 *   srj_interleave_bits       : (async) Delta Lake's InterleaveBits, B = 8W: row r is the N * W bytes
 *                               out_bytes[r * N * W ..) holding the stream (byte 0 = positions 0..7, MSB first), and
 *                               out_offsets[0 .. num_rows] = r * N * W: the offsets and chars of a LIST<UINT8> column
 *                               with no null mask.
 *   srj_hilbert_index         : (async) out[r] = the Hilbert index of the point (X[0] .. X[N-1]) of row r, B = num_bits,
 *                               X[c] = the INT32 value's low num_bits bits: Skilling's AxesToTranspose with Gray encoding
 *                               (AIP Conf. Proc. 707, 2004), then the stream of the transposed coordinates read as an
 *                               N * num_bits-bit integer.  SRJ_EINVAL for num_bits outside [1, 32], num_bits * N > 64,
 *                               N < 1 or a row count that differs; SRJ_EUNSUPPORTED for a column that is not INT32.
 * Inputs need element alignment (8 bytes for DECIMAL128); the outputs may be unaligned.  No synchronisation.
 */
SRJ_API int srj_interleave_bits_sizes(const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t* total_bytes);
SRJ_API int srj_interleave_bits(const srj_column* cols, int32_t num_columns, int64_t num_rows, int32_t* out_offsets, uint8_t* out_bytes,
                                void* stream);
SRJ_API int srj_hilbert_index(int32_t num_bits, const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t* out,
                              void* stream);

/* ---- Iceberg partition transforms: IcebergBucket / IcebergTruncate / IcebergDateTimeUtil ------------------------------
 * Reference iceberg/iceberg_bucket.cu:388-457, iceberg_truncate.cu:141-238, iceberg_datetime_util.cu:137-248.  Every
 * result has the input's rows; out_mask (ceil(rows / 32) words) receives a copy of the input's null mask (all ones when
 * the input has none) and may be NULL only when the input has no mask.  The null count is the input's.
 *   srj_iceberg_bucket       : (async) out[r] = (murmur3_x86_32(bytes, 0) & INT32_MAX) % num_buckets, 0 for a null row.
 *                              Bytes: INT32 / TIMESTAMP_DAYS widened to int64, INT64 / TIMESTAMP_MICROSECONDS: 8 bytes
 *                              little-endian; DECIMAL32/64/128: BigInteger.toByteArray() of the unscaled value; STRING:
 *                              the chars; LIST<UINT8>: the child bytes.  SRJ_EINVAL for num_buckets <= 0,
 *                              SRJ_EUNSUPPORTED for another type or a LIST whose child is not UINT8.
 *   srj_iceberg_truncate_workspace_bytes : bytes of srj_iceberg_truncate_sizes' workspace.
 *   srj_iceberg_truncate_sizes : STRING / LIST<UINT8> only: d_out_offsets[0 .. rows] of the output and *total_bytes (host;
 *                              synchronises the stream once).  A null row has zero length.  STRING keeps the bytes before
 *                              the (width+1)-th byte that is not a UTF-8 continuation byte (all of them when there is
 *                              none); LIST<UINT8> keeps min(len, width) bytes.
 *   srj_iceberg_truncate     : (async) INT32, INT64, DECIMAL32/64/128: out->data[r] = v - (((v % W) + W) % W) in the
 *                              storage type (W = width sign-extended, % truncated, + and - wrapping), 0 for a null row.
 *                              STRING: out->offsets (from the sizes call) and the chars in out->data; LIST<UINT8>:
 *                              out->offsets and the bytes in out->children[0].data.  SRJ_EINVAL for width == 0
 *                              (integral) or width <= 0 (STRING / LIST) and for a LIST child with a null mask;
 *                              SRJ_EUNSUPPORTED for another type.
 *   srj_iceberg_datetime     : (async) transform SRJ_ICEBERG_YEARS / MONTHS / DAYS / HOURS of a TIMESTAMP_DAYS (not
 *                              HOURS) or TIMESTAMP_MICROSECONDS column: years and months since 1970-01 (proleptic
 *                              Gregorian), days since 1970-01-01, hours since the epoch (wrapping to int32), from the
 *                              floored day / hour.  out is int32 per row (TIMESTAMP_DAYS for DAYS).  Rows under nulls are
 *                              computed from their bits.  SRJ_EINVAL for an unknown transform, SRJ_EUNSUPPORTED for
 *                              another type.
 * Fixed-width inputs and outputs need element alignment (8 bytes for DECIMAL128); offsets need 4 bytes.
 */
#define SRJ_ICEBERG_YEARS 0
#define SRJ_ICEBERG_MONTHS 1
#define SRJ_ICEBERG_DAYS 2
#define SRJ_ICEBERG_HOURS 3
SRJ_API int srj_iceberg_bucket(const srj_column* input, int32_t num_buckets, int32_t* out, uint32_t* out_mask, void* stream);
SRJ_API int64_t srj_iceberg_truncate_workspace_bytes(int64_t num_rows);
SRJ_API int srj_iceberg_truncate_sizes(const srj_column* input, int32_t width, int32_t* d_out_offsets, int64_t* total_bytes,
                                       void* workspace, void* stream);
SRJ_API int srj_iceberg_truncate(const srj_column* input, int32_t width, const srj_column* out, void* stream);
SRJ_API int srj_iceberg_datetime(int32_t transform, const srj_column* input, int32_t* out, uint32_t* out_mask, void* stream);

/* ---- DecimalUtils: DECIMAL128 multiply, divide, integral divide, remainder, add and subtract -------------------------
 * Reference decimal_utils.cu:529-1167 (multiply_decimal128 .. sub_decimal128).  a and b are DECIMAL128 columns with the
 * same row count; a value is v * 10^scale (cudf scale).  Every row, null or not, is computed from the bits under it in
 * 256-bit two's complement, as the reference does:
 *   SRJ_DECIMAL_MULTIPLY       : a * b rounded HALF_UP to out_scale; with interim_cast, first rounded to 38 digits when
 *                                it has more (Spark's SPARK-40129 behaviour).  A row whose scale-up would pass 38 digits
 *                                overflows with value 0.
 *   SRJ_DECIMAL_DIVIDE         : a / b rounded HALF_UP to out_scale.
 *   SRJ_DECIMAL_INTEGER_DIVIDE : a / b truncated at out_scale (0 for Spark's div); out is int64 per row, the low 64 bits
 *                                of the quotient, whose overflow flag is judged on the whole quotient.
 *   SRJ_DECIMAL_REMAINDER      : a - (a div b) * b at out_scale, with the sign of a (Java's BigDecimal.remainder).
 *   SRJ_DECIMAL_ADD / SUBTRACT : a + b or a - b at min(a.scale, b.scale), then rounded HALF_UP to out_scale.
 * overflow[r] (BOOL8) is 1 when |result| >= 10^38 or b is 0 (divide family; value 0).  out holds 16 bytes per row (8 for
 * INTEGER_DIVIDE): the low bits of the result.  When a or b has a null mask, out_mask (ceil(rows / 32) words) receives the
 * AND of the masks and *null_count its null count, read back with one stream synchronisation; otherwise *null_count (if
 * given) is 0, out_mask is not written and the call is asynchronous.  Both output columns take that mask.
 * SRJ_EUNSUPPORTED when a or b is not DECIMAL128; SRJ_EINVAL for an unknown op, differing row counts, a missing buffer,
 * and for the scale combinations whose rows would need a power of ten the reference cannot represent (multiply:
 * out_scale - (a.scale + b.scale) > 38; divide: out_scale - (a.scale - b.scale) outside [-114, 38]; remainder: a divisor
 * or dividend shift above 38 or below -76; add / subtract: |a.scale - b.scale| > 76, or out_scale more than 38 above or
 * 76 below min(a.scale, b.scale)).  Inputs need 8-byte alignment, out 8 bytes, out_mask 4; overflow may be unaligned.
 */
#define SRJ_DECIMAL_MULTIPLY 0
#define SRJ_DECIMAL_DIVIDE 1
#define SRJ_DECIMAL_INTEGER_DIVIDE 2
#define SRJ_DECIMAL_REMAINDER 3
#define SRJ_DECIMAL_ADD 4
#define SRJ_DECIMAL_SUBTRACT 5
SRJ_API int srj_decimal128_binary(int32_t op, const srj_column* a, const srj_column* b, int32_t out_scale, int32_t interim_cast,
                                  uint8_t* overflow, void* out, uint32_t* out_mask, int64_t* null_count, void* stream);

/* ---- DateTimeUtils: Julian / Gregorian rebase and date / timestamp truncation ------------------------------------------
 * Reference datetime_rebase.cu:342-372, datetime_truncate.cu:327-376.  Inputs are TIMESTAMP_DAYS (int32 days since
 * 1970-01-01) or TIMESTAMP_MICROSECONDS (int64 microseconds since the epoch, UTC); out has the input's type.  Dates go
 * through y/m/d with the year reduced to int16, as the reference's cuda::std::chrono::year does (DESIGN 3.6j).
 *   srj_datetime_rebase   : (async) SRJ_DATETIME_GREGORIAN_TO_JULIAN: a day's proleptic Gregorian y/m/d read as a Julian
 *                           date (1582-10-05 .. 14 -> 1582-10-15; from 1582-10-15 on unchanged); JULIAN_TO_GREGORIAN: the
 *                           reverse (unchanged from day -141427 on).  Micros: unchanged from 1582-10-15T00:00Z on, else the
 *                           floored day is rebased and the time of day reattached, wrapping in int64.  Rows under nulls
 *                           are computed from their bits.  out_mask (ceil(rows / 32) words) receives a copy of the input's
 *                           mask (all ones when it has none) and may be NULL only when the input has no mask; the null
 *                           count is the input's.
 *   srj_datetime_truncate : exactly one of format_col (a STRING column) and format (format_len bytes) is given.  Formats
 *                           are ASCII case-insensitive: YEAR / YYYY / YY, QUARTER, MONTH / MM / MON, WEEK (the Monday on
 *                           or before), and for TIMESTAMP_MICROSECONDS only DAY / DD, HOUR, MINUTE, SECOND, MILLISECOND,
 *                           MICROSECOND (the time of day floored).  A row whose format is anything else is null.  Null
 *                           rows hold 0.
 *                           format: (async) rows = datetime rows.  A format that fits the type: out_mask receives a copy of
 *                           the input's mask (may be NULL when it has none) and *null_count = -1, meaning the input's null
 *                           count, which the caller holds.  Otherwise the result is all null: out and out_mask are zeroed
 *                           (out_mask is needed) and *null_count = rows.
 *                           format_col: rows = format rows; the datetime has one row, applied to every row, or as many as
 *                           the format.  A row is null when its datetime, its format or the format's parse is.  out_mask is
 *                           needed; *null_count is read back (one stream synchronisation).
 *                           SRJ_EUNSUPPORTED for a datetime that is not a timestamp of days or microseconds or a format
 *                           column that is not STRING; SRJ_EINVAL for other row counts or a missing null_count.
 * Both: zero rows touch nothing.  SRJ_EINVAL for a missing or misaligned buffer (data and out at their element, offsets
 * and out_mask at 4 bytes).
 */
#define SRJ_DATETIME_GREGORIAN_TO_JULIAN 0
#define SRJ_DATETIME_JULIAN_TO_GREGORIAN 1
SRJ_API int srj_datetime_rebase(int32_t direction, const srj_column* input, void* out, uint32_t* out_mask, void* stream);
SRJ_API int srj_datetime_truncate(const srj_column* datetime, const srj_column* format_col, const char* format, int32_t format_len,
                                  void* out, uint32_t* out_mask, int64_t* null_count, void* stream);

/* ---- GpuTimeZoneDB: timestamps to and from a time zone, one zone per row, and ORC's writer -> reader zones -------------
 * Reference timezones.cu, datetime_utils.cuh:278-588.  A time zone table is the two columns GpuTimeZoneDB.loadData builds,
 * one row per zone:
 *   fixed_transitions : LIST<STRUCT<utcInstant INT64, localInstant INT64, offset INT32>> (offsets, children[0] the STRUCT
 *                       with its three fields as children), seconds: entry 0 is (INT64_MIN, INT64_MIN, the first offset),
 *                       then one entry per transition, ascending; localInstant is utc + offsetAfter for a gap and utc +
 *                       offsetBefore for an overlap, offset is offsetAfter.
 *   dst_rules         : LIST<INT32> (offsets, children[0] the INT32 column) of the same row count: 0 ints, or two rules of
 *                       (month, dayOfMonthIndicator, dayOfWeek 0 = Monday .. 6 or -1, secondsFromMidnight, offsetBefore,
 *                       offsetAfter).
 * A value's seconds s are truncated toward zero.  When the zone has rules and s is above its last instant (localInstant
 * converting to UTC, utcInstant from UTC), the rules of year(floor(s / 86400)) give the offset; otherwise the last entry
 * whose instant is <= s.  The result is value -/+ offset in the value's unit, wrapping in int64.
 *   srj_timezone_convert       : SRJ_TIMEZONE_TO_UTC / FROM_UTC of a TIMESTAMP_SECONDS / MILLISECONDS / MICROSECONDS /
 *                                NANOSECONDS column in zone tz_index; out has its type and out_mask (ceil(rows / 32) words,
 *                                may be NULL only when the input has no mask) a copy of its mask (all ones without one).
 *                                Reads the zone's bounds back (one stream synchronisation), then runs asynchronously.
 *                                SRJ_EINVAL for a tz_index outside the table, or a zone without entries or with a rule list
 *                                of other than 0 or 12 ints.
 *   srj_timezone_convert_multi : one zone per row, for string-to-timestamp casts: seconds (INT64), micros (INT32), invalid
 *                                (BOOL8 / UINT8), tz_type (UINT8), tz_offset (INT32) and tz_indices (INT32), all of one row
 *                                count; input masks are not read.  A row is null when invalid; tz_type 1 (a fixed offset)
 *                                gives seconds - tz_offset, any other the zone tz_indices[row] converted to UTC (null when the
 *                                index is outside the table or the zone malformed).  Then micros are added with the
 *                                reference's overflow check; an overflow is null.  out (TIMESTAMP_MICROSECONDS) holds 0 under
 *                                nulls; out_mask is needed; *null_count is read back (one stream synchronisation).
 *   srj_orc_convert_timezones  : (async) ORC's SerializationUtils.convertBetweenTimezones of a TIMESTAMP_MICROSECONDS column.
 *                                Each zone is (transitions INT64 ms, offsets INT32 ms, raw offset ms); NULL transitions and
 *                                offsets mean a fixed offset.  The offset at a millisecond is an exact match's, else the
 *                                previous transition's, the raw offset before the first and from the last on.
 *                                result = us + (w - r') * 1000 with ms = us / 1000 truncated, w the writer's offset at ms, r
 *                                the reader's, r' the reader's at ms + w - r.  out_mask as srj_timezone_convert.
 * All: zero rows touch nothing after the host-side checks.  SRJ_EUNSUPPORTED for an input of another type; SRJ_EINVAL for a
 * table of another layout, mismatched row counts, or a missing or misaligned buffer (data and out at their element,
 * offsets and masks at 4 bytes).
 */
#define SRJ_TIMEZONE_TO_UTC 0
#define SRJ_TIMEZONE_FROM_UTC 1
SRJ_API int srj_timezone_convert(int32_t direction, const srj_column* input, const srj_column* fixed_transitions, const srj_column* dst_rules,
                                 int32_t tz_index, void* out, uint32_t* out_mask, void* stream);
SRJ_API int srj_timezone_convert_multi(const srj_column* seconds, const srj_column* micros, const srj_column* invalid, const srj_column* tz_type,
                                       const srj_column* tz_offset, const srj_column* fixed_transitions, const srj_column* dst_rules,
                                       const srj_column* tz_indices, int64_t* out, uint32_t* out_mask, int64_t* null_count, void* stream);
SRJ_API int srj_orc_convert_timezones(const srj_column* input, const srj_column* writer_transitions, const srj_column* writer_offsets,
                                      int32_t writer_raw_offset, const srj_column* reader_transitions, const srj_column* reader_offsets,
                                      int32_t reader_raw_offset, void* out, uint32_t* out_mask, void* stream);

/* ---- CastStrings: string to timestamp (first phase) and string to date -------------------------------------------------
 * Reference cast_string_to_datetime.cu (Spark 3.5's SparkDateTimeUtils).  Both trim bytes <= 32 and 127 from each end.
 *   srj_cast_parse_timestamps : (async) parses [+-]yyyy[y][y][-m[m][-d[d][( |T)[h]h:[m]m:[s]s[.fraction][zone]]]], or a
 *                               time alone ("T..." or "h:m..."), into the six columns of CastStrings'
 *                               parseTimestampStringsToIntermediate, one row per input row:
 *                               result UINT8 (0 ok, 1 invalid), seconds INT64 (the local date-time as seconds from the
 *                               epoch), micros INT32 (the first 6 fraction digits), tz_type UINT8 (0 none, 1 fixed, 2 other,
 *                               3 invalid), tz_offset INT32 (seconds, fixed zones), tz_index INT32 (-1 when none).
 *                               Zones: Z; [+-]h[h], [+-]hh[mm[ss]], [+-]h[h]:m[m], [+-]h[h]:mm:ss up to 18:00:00; UT, UTC,
 *                               GMT, GMT0 and those prefixes followed by an offset; any other name is looked up in
 *                               tz_name_map, a STRUCT<name STRING, index INT32> sorted by name bytes (further fields are
 *                               ignored), and a name it lacks makes the row invalid.  A row without a zone takes type 2 and
 *                               default_tz_index.  A time alone takes its date from default_epoch_day without a zone, from
 *                               now_seconds + offset with a fixed zone, and from now_seconds converted into a named zone with
 *                               the time zone table (fixed_transitions / dst_rules, the layout of srj_timezone_convert).
 *                               The version (spark_platform 0 = vanilla Spark, 1 = Databricks) selects Spark 3.2.0's
 *                               offsets (a one-digit minute is rejected, "+hh:mm" right after the time is read with a sign
 *                               of 1 for '+' and 0 for '-') and, from Spark 4.0 / Databricks 14.3, rejects spaces before
 *                               "Thh:mm:ss".  Years outside [-300000, 300000] and invalid dates or times are invalid.
 *                               A null row is invalid (0, 0, 0 and -1 elsewhere) whatever bytes its offsets span.
 *                               Defined where the reference's is not: a default_tz_index outside the table is SRJ_EINVAL;
 *                               a time alone whose named zone maps outside the table, or to a malformed zone, is invalid;
 *                               a tenth segment of a Spark 3.2.0 string is dropped.
 *   srj_cast_parse_dates      : [+-]yyyy[y][y][y][-[m]m[-[d]d[( |T)anything]]] into TIMESTAMP_DAYS.  A row is null when the
 *                               input row is, when it does not parse, or when its year is outside [-10^7, 10^7] or its day
 *                               count outside int32.  out holds 0 under nulls; out_mask is needed; *null_count is read back
 *                               (one stream synchronisation).
 * Both: zero rows touch nothing after the host-side checks.  A STRING column (the input, the map's names) may have NULL
 * chars only when its offsets span no byte; such a column with rows is checked by reading its first and last offsets back
 * (one stream synchronisation, on that path alone).  SRJ_EINVAL for an input that is not STRING, a name map that is
 * not STRUCT<STRING, INT32>, STRING offsets that span bytes with NULL chars, a time zone table of another layout, or a missing or misaligned buffer (outputs at their
 * element, masks and offsets at 4 bytes).
 */
#define SRJ_SPARK_VANILLA 0
#define SRJ_SPARK_DATABRICKS 1
SRJ_API int srj_cast_parse_timestamps(const srj_column* input, const srj_column* tz_name_map, const srj_column* fixed_transitions,
                                      const srj_column* dst_rules, int32_t default_tz_index, int64_t default_epoch_day, int64_t now_seconds,
                                      int32_t spark_platform, int32_t spark_major, int32_t spark_minor, int32_t spark_patch,
                                      uint8_t* out_result, int64_t* out_seconds, int32_t* out_micros, uint8_t* out_tz_type,
                                      int32_t* out_tz_offset, int32_t* out_tz_index, void* stream);
SRJ_API int srj_cast_parse_dates(const srj_column* input, int32_t* out, uint32_t* out_mask, int64_t* null_count, void* stream);

/* ---- JoinPrimitives: hash inner join and the outer / semi / anti gather-map builders --------------------------------
 * Reference join_primitives.cu:203-227 (hash_inner_join over cudf::hash_join) and 358-576 (the helpers).  Gather maps are
 * int32 device arrays; INT32_MIN marks the missing side of an outer row.
 *   srj_hash_join_workspace_bytes : bytes of the join's workspace (build table, per-row counts, tile offsets).
 *   srj_hash_inner_join_size      : builds a hash table on the right keys, counts every left row's matches and returns the
 *                                   pair count in *num_pairs (one stream synchronisation).  Keys are equal when every
 *                                   column is: integers, timestamps, durations and decimals by value, BOOL8 as bool,
 *                                   FLOAT32 / FLOAT64 with every NaN equal and -0.0 == 0.0, STRING by length and bytes.
 *                                   With nulls_equal a null equals a null of the same column; without it a row with a null
 *                                   key matches nothing.  Either side with zero rows: *num_pairs = 0 before any other check.
 *   srj_hash_inner_join           : (async) with the same arguments and the workspace the size call filled, writes
 *                                   left_map / right_map (num_pairs each): every pair of rows with equal keys once, the left
 *                                   map non-decreasing (the order of the right rows of one left row is unspecified).
 *   SRJ_EINVAL for zero key columns on a side, differing column counts, types or decimal scales, more than INT32_MAX rows,
 *   columns of one side with differing row counts, a missing or misaligned buffer (data at its element, at most 8 bytes;
 *   offsets and masks at 4); SRJ_EUNSUPPORTED for LIST / STRUCT (or other non-flat) keys and more than SRJ_MAX_JOIN_KEYS
 *   key columns.
 *
 *   srj_join_mask_workspace_bytes : bytes of one match mask over table_rows rows (a counter, the bitmask, compaction scratch).
 *   srj_join_mark                 : (async) clears the mask, then sets the bit of every row 0 <= map[i] < table_rows names
 *                                   and counts the distinct rows set.
 *   srj_join_matched_counts       : matched[i] = the count of workspaces[i] (one stream synchronisation for all of them).
 *   srj_join_compact              : (async) out = the ascending rows whose bit is set (matched != 0) or clear (matched == 0).
 *   srj_join_make_outer           : (async) out_left / out_right = the inner pairs, then every unmatched left row with
 *                                   INT32_MIN on the right, then (right_ws != NULL: full outer) every unmatched right row with
 *                                   INT32_MIN on the left.  The workspaces are marked with the maps; left_unmatched /
 *                                   right_unmatched are the table rows minus their matched counts.
 *   srj_join_matched_rows         : (async) out[r] (BOOL8, table_rows bytes) = 1 when an in-range map entry names r, else 0.
 * Maps must be 4-byte aligned; a map may be NULL only when its length is 0.  SRJ_EINVAL for a negative length or table
 * size, a table size above INT32_MAX, or a missing buffer.  Zero rows touch nothing.
 */
#define SRJ_MAX_JOIN_KEYS 32
SRJ_API int64_t srj_hash_join_workspace_bytes(int64_t left_rows, int64_t right_rows);
SRJ_API int srj_hash_inner_join_size(const srj_column* left_keys, int32_t num_left_keys, const srj_column* right_keys, int32_t num_right_keys,
                                     int32_t nulls_equal, int64_t* num_pairs, void* workspace, void* stream);
SRJ_API int srj_hash_inner_join(const srj_column* left_keys, int32_t num_left_keys, const srj_column* right_keys, int32_t num_right_keys,
                                int32_t nulls_equal, int32_t* left_map, int32_t* right_map, void* workspace, void* stream);
SRJ_API int64_t srj_join_mask_workspace_bytes(int64_t table_rows);
SRJ_API int srj_join_mark(const int32_t* map, int64_t map_len, int64_t table_rows, void* workspace, void* stream);
SRJ_API int srj_join_matched_counts(const void* const* workspaces, int32_t count, int64_t* matched, void* stream);
SRJ_API int srj_join_compact(const void* workspace, int64_t table_rows, int32_t matched, int32_t* out, void* stream);
SRJ_API int srj_join_make_outer(const int32_t* left_map, const int32_t* right_map, int64_t map_len, int64_t left_rows, int64_t right_rows,
                                const void* left_ws, int64_t left_unmatched, const void* right_ws, int64_t right_unmatched,
                                int32_t* out_left, int32_t* out_right, void* stream);
SRJ_API int srj_join_matched_rows(const int32_t* map, int64_t map_len, int64_t table_rows, uint8_t* out, void* stream);

/* ---- Histogram: percentile and median from value-frequency histograms, and createHistogramIfValid ------------------
 * Reference histogram.cu (Spark's Percentile).  A null_mask counts as nulls here: pass NULL for a column without nulls.
 *   srj_percentile_workspace_bytes     : bytes of the workspace of the two percentile calls.
 *   srj_percentile_from_histogram_size : input is LIST<STRUCT<value T, count INT64>> (children[0] the STRUCT, its
 *                                        children the values and the counts; offsets[0] may be > 0).  T is INT8..INT64,
 *                                        UINT8..UINT64, FLOAT32, FLOAT64 or BOOL8.  Sorts the rows by length into the
 *                                        workspace, returns in *valid_rows the rows holding a non-null value (0 when
 *                                        num_percentages is 0) and in *num_values the doubles of the output (see below);
 *                                        one stream synchronisation.  The list's own mask is not read: a null list is an
 *                                        empty one.
 *   srj_percentile_from_histogram      : with the same arguments and the workspace the size call filled, writes per
 *                                        valid row and percentage p (in order): the non-null values ordered ascending
 *                                        (NaN after +inf, every NaN equal, -0.0 before 0.0, BOOL8 nonzero = true), acc
 *                                        the running sum of their counts, position = (acc.last - 1) * p, lower / higher
 *                                        = floor / ceil(position); the elements at ranks lower + 1 and higher + 1 are
 *                                        the first whose acc reaches the rank (the last element when none does); the
 *                                        result is the lower element when lower == higher or both are equal in T, else
 *                                        (higher - position) * lo + (position - lower) * hi, each product rounded.
 *                                        Flat output (output_as_lists 0): out = rows * P doubles, row-major, 0.0 under
 *                                        null rows; rows doubles, all null, when P is 0 or the rows reference no element
 *                                        (the reference's early return).  out_mask has one bit per double, each null
 *                                        where its row is (ceil(num_values / 32) words).  List output: out = valid_rows
 *                                        * P doubles, out_offsets = rows + 1 (a null row is an empty list), out_mask one
 *                                        bit per row (ceil(rows / 32) words).  One stream synchronisation (it reads back
 *                                        the tiers and the list of rows longer than SRJ_HISTOGRAM_CTA_ELEMENTS, at most
 *                                        16 bytes per SRJ_HISTOGRAM_CTA_ELEMENTS + 1 elements); each such row takes a
 *                                        radix select with one launch sequence of its own.
 *   Both: SRJ_EINVAL for an input that is not LIST ("The input column must be of type LIST."), a STRUCT child with
 *   nulls, not a STRUCT or not of two children, counts with nulls or not INT64 (the reference's messages, in its order);
 *   SRJ_EOVERFLOW when rows * num_percentages > INT32_MAX; SRJ_EUNSUPPORTED for another T; SRJ_EINVAL for a missing
 *   or misaligned buffer.  Zero rows touch nothing.  Negative counts give unspecified values.
 *
 *   srj_histogram_workspace_bytes      : bytes of the workspace of the two create calls.
 *   srj_histogram_create_size          : checks the frequencies (INT64, no nulls, the values' size; the reference's
 *                                        messages) and the values (any fixed-width type, else SRJ_EUNSUPPORTED), then
 *                                        flags negative and zero frequencies on the device (one stream synchronisation).
 *                                        A negative one is SRJ_EINVAL ("The input frequencies must not contain negative
 *                                        values.") and nothing is written.  *out_rows = the output's element rows (the
 *                                        rows, or for lists the rows with frequency > 0); *value_nulls = the null
 *                                        values among them.
 *   srj_histogram_create               : (async) with the same values, frequencies and output_as_lists, and the workspace
 *                                        the size call filled (its zero flag and keep flags are read on the device).
 *                                        out_values (*out_rows elements of the values' type) and out_frequencies
 *                                        (*out_rows INT64) must hold *out_rows elements; when *out_rows > 0 they must be
 *                                        present, which this call cannot check: the count is on the device.
 *                                        output_as_lists 0: STRUCT<values, frequencies> of every row; a value is null where
 *                                        it was or where its frequency is 0, and when some frequency is 0 every null
 *                                        value's frequency becomes 1; out_values_mask (ceil(rows / 32) words) is needed.
 *                                        output_as_lists 1: one single-element list per row with frequency > 0, an empty
 *                                        list for the others (out_offsets rows + 1); the child keeps the values' nulls and
 *                                        the frequencies; out_values_mask (ceil(*out_rows / 32) words, only those are
 *                                        written) is needed when the values have a mask.  Zero rows touch nothing.
 */
#define SRJ_HISTOGRAM_CTA_ELEMENTS 8192
SRJ_API int64_t srj_percentile_workspace_bytes(int64_t num_rows, int64_t num_elements, int32_t num_percentages);
SRJ_API int srj_percentile_from_histogram_size(const srj_column* input, int32_t num_percentages, int32_t output_as_lists, int64_t* valid_rows,
                                               int64_t* num_values, void* workspace, void* stream);
SRJ_API int srj_percentile_from_histogram(const srj_column* input, const double* percentages, int32_t num_percentages,
                                          int32_t output_as_lists, double* out, uint32_t* out_mask, int32_t* out_offsets, void* workspace,
                                          void* stream);
SRJ_API int64_t srj_histogram_workspace_bytes(int64_t num_rows);
SRJ_API int srj_histogram_create_size(const srj_column* values, const srj_column* frequencies, int32_t output_as_lists, int64_t* out_rows,
                                      int64_t* value_nulls, void* workspace, void* stream);
SRJ_API int srj_histogram_create(const srj_column* values, const srj_column* frequencies, int32_t output_as_lists, void* out_values,
                                 uint32_t* out_values_mask, int64_t* out_frequencies, int32_t* out_offsets, void* workspace, void* stream);

/* ---- Arithmetic: Spark's multiply with ANSI / try overflow handling, and round / bround ----------------------------
 * Reference multiply.cu, round_float.cu and cudf's round/round.cu.  A null_mask counts as nulls here: pass NULL for a
 * column without nulls.  Both calls set *error_row to -1 first.
 *   srj_multiply : left * right, each a column or a scalar.  An operand with a scalar validity (a device byte, non-zero =
 *                  valid, as cudf::scalar::validity_data() holds it) is a scalar: its data is its one device value and its
 *                  size and mask are not read.  Rows = the column operand's size.  Types INT8, INT16, INT32, INT64, FLOAT32,
 *                  FLOAT64, the same on both sides.  An integer row overflows when its exact product is outside the type:
 *                  by default it wraps; with is_try_mode it is null; with is_ansi_mode *error_row is the smallest
 *                  overflowing row with both operands valid (-1 when none) and the output is not a result.  Floats are IEEE
 *                  products in every mode.  A row is null when an operand is (a null scalar: every row); a null row holds
 *                  0.  out: rows elements of the type, aligned to the element.  out_mask: ceil(rows / 32) words, 4-byte
 *                  aligned, needed when the result can hold nulls (an operand has a mask or is a scalar, or try mode on an
 *                  integer type), else it may be NULL (when given, it is written).  *null_count: the output's nulls when
 *                  the result can hold nulls, else 0.  The null count and the error row are read back together (one
 *                  stream synchronisation) when either is needed; otherwise the call is asynchronous.  Errors, in this
 *                  order: SRJ_EINVAL for two scalars or differing types, SRJ_EUNSUPPORTED for another type, SRJ_EINVAL for
 *                  differing row counts (column * column), for is_ansi_mode with is_try_mode, and for a missing or
 *                  misaligned buffer.
 *   srj_round    : (async, unless ANSI on an integer type with decimal_places < 0: one stream synchronisation for
 *                  *error_row) rounds to decimal_places with method SRJ_ROUND_HALF_UP or SRJ_ROUND_HALF_EVEN.  Zero rows
 *                  return SRJ_OK before any check.  FLOAT32 / FLOAT64: n = T(pow(10, |dp|)); dp == 0: round / rint;
 *                  dp > 0: modf, then int_part + round(frac * n) / n; dp < 0: round(e / n) * n; each operation rounded
 *                  to nearest in T.  INT8..INT64: dp >= 0 copies; dp < 0 rounds to a multiple of 10^-dp (HALF_UP away
 *                  from zero, HALF_EVEN to the even multiple), the exact result wrapped to the type; with is_ansi_mode
 *                  *error_row is the smallest valid row whose exact result is outside the type.  DECIMAL32 / 64 / 128
 *                  (ANSI ignored): the output's scale is -dp; the same scale copies; a larger input scale multiplies by
 *                  10^k, wrapping; a scale movement k above 9 / 18 / 38 digits gives zeros; else the storage integer is
 *                  rounded and divided by 10^k exactly.  out: rows elements of the input's type, aligned to the element
 *                  (8 bytes at most).  out_mask (ceil(rows / 32) words, 4-byte aligned) receives a copy of the input's
 *                  mask, all ones when it has none, and may be NULL only when the input has no mask.  SRJ_EUNSUPPORTED
 *                  for another type, then SRJ_EINVAL for another method and for a missing or misaligned buffer.
 */
#define SRJ_ROUND_HALF_UP 0
#define SRJ_ROUND_HALF_EVEN 1
SRJ_API int srj_multiply(const srj_column* left, const uint8_t* left_scalar_valid, const srj_column* right, const uint8_t* right_scalar_valid,
                         int32_t is_ansi_mode, int32_t is_try_mode, void* out, uint32_t* out_mask, int64_t* null_count, int64_t* error_row,
                         void* stream);
SRJ_API int srj_round(const srj_column* input, int32_t decimal_places, int32_t method, int32_t is_ansi_mode, void* out, uint32_t* out_mask,
                      int64_t* error_row, void* stream);

/* ---- DecimalUtils.floatingPointToDecimal: Spark's CAST(float / double AS DECIMAL) ----------------------------------
 * Reference decimal_utils.cu:1174-1417 over cudf's fixed_point/detail/floating_conversion.hpp, bit for bit inside the
 * domain below, the reference's integer wraps included.  input: FLOAT32 or FLOAT64 (a null_mask counts as nulls);
 * out_type_id: SRJ_DECIMAL32 / 64 / 128 with `precision` digits at cudf `scale` (the value is out * 10^scale).  A null,
 * NaN or infinite row is null and holds 0; any other value is scaled and rounded as Spark does (a double rounds half up
 * after half a unit in the last place is added, a float at the edge of its precision), and a result not strictly inside
 * (-10^precision, 10^precision) is null, holds 0 and fails.  out: rows elements of the output type, aligned to the
 * element (8 bytes at most); out_mask: ceil(rows / 32) words, 4-byte aligned, always written; *null_count its nulls.
 * One stream synchronisation reads back *null_count and *failure_row.
 * Defined here where the reference is not:
 *   - *failure_row is the smallest failing row, or -1 (the reference stores some failing row, racing between threads);
 *   - the domain: precision 1..9 (DECIMAL32), 1..18 (DECIMAL64), 1..38 (DECIMAL128), and scale in [-precision, 38]
 *     (Spark scale -38 .. precision, the legacy negative scales included), where every power of ten the reference forms
 *     for the bound and the scale factor fits the type; outside it SRJ_EINVAL before any launch;
 *   - the reference divides DECIMAL64 rows whose last-digit exponent is 63 by 10^64 mod 2^64 = 0; the quotient is all
 *     ones here, so those rows (|x| near 2^210 * 10^-scale) fail.
 * Errors, in this order: SRJ_EINVAL for a NULL input, null_count or failure_row; SRJ_EUNSUPPORTED for an input that is
 * not FLOAT32 / FLOAT64 or an output type that is not DECIMAL32 / 64 / 128; SRJ_EINVAL for a precision or scale outside
 * the domain and a negative row count; zero rows return SRJ_OK here, touching nothing; then SRJ_EINVAL for missing or
 * misaligned input data, output or output mask.
 */
SRJ_API int srj_float_to_fixed_point(const srj_column* input, int32_t out_type_id, int32_t precision, int32_t scale, void* out,
                                     uint32_t* out_mask, int64_t* null_count, int64_t* failure_row, void* stream);

/* ---- NumberConverter and CastStrings' radix casts: Spark's conv(), bin() and hex() ---------------------------------
 * Reference number_converter.cu (Spark 3.5's NumberConverter), cast_long_to_binary_string.cu, hex.cu and
 * CastStringJni.cpp's fromIntegersWithBase (cudf's from_integers / integers_to_hex, then the extract ^0?([0-9a-fA-F]+)$).
 * Every output is a STRING column: d_out_offsets int32[rows + 1] and its chars.  Each op except bytesToHex is a sizes call
 * (lengths, exclusive scan, one stream synchronisation to read back *total_chars) and a write call (async) taking the
 * same arguments, the offsets and the workspace the sizes call filled.  A result of more than INT32_MAX chars returns
 * SRJ_EOVERFLOW from the sizes call (its offsets are then not a column).
 *
 *   srj_conv_*         : NumberConverter.convert / isConvertOverflow.  input is a STRING column, or NULL with a scalar
 *                        string of scalar_len bytes at the device pointer `scalar` (scalar_len < 0: a null scalar,
 *                        SRJ_EINVAL).  from_base / to_base are INT32 columns, or NULL with the int from / to.  A scalar
 *                        input needs at least one base column; the output has the column arguments' rows, and base
 *                        columns of other row counts are SRJ_EINVAL.  A row is null when its input or a base is null,
 *                        when from is outside [2, 36] or |to| outside [2, 36] (every row when both are scalars), or when
 *                        the string is empty after trimming ' ' from both ends.  Otherwise an optional '-' and the
 *                        digits below `from` (0-9, A-Z, a-z) that follow it accumulate in 64 bits; the first other byte
 *                        ends the number.  On overflow (past 2^64 - 1) the value is all ones.  A negative input with
 *                        to > 0 is negated (all ones stays); with to < 0 a value with its top bit set is negated and the
 *                        result gets a '-', as does a negative input.  Digits are upper case, "0" for zero.
 *                        srj_conv_sizes writes the offsets, out_mask (ceil(rows / 32) words, always) and *null_count;
 *                        srj_conv writes the chars.  srj_conv_overflow sets *overflow to 1 when a non-null row with valid
 *                        bases overflows (Spark's ANSI error), else 0; it synchronizes.
 *   srj_long_to_binary_* : CastStrings.fromLongToBinary.  INT64 only: the 64-bit two's complement in binary without
 *                        leading zeros, "0" for zero.
 *   srj_integers_to_string_* : CastStrings.fromIntegersWithBase.  INT8..INT64, UINT8..UINT64.  base 10: decimal with '-'
 *                        for negative values; base 16: upper-case hex of the value's own width without leading zeros ("0"
 *                        for zero, INT8 -1 -> "FF").  Another base is SRJ_EINVAL ("Bases supported 10, 16; Actual: N",
 *                        checked before the type; the JNI shim throws the reference's CastException on row 0).
 *   srj_bytes_to_hex_* : CastStrings.bytesToHex.  STRING, or LIST<UINT8> read as its child's bytes: each byte becomes two
 *                        upper-case hex digits.  The offsets are twice the input's, rebased to 0, so a null row keeps its
 *                        span; its chars hold the hex of its bytes.  No workspace.
 * For bin, fromIntegersWithBase and bytesToHex the output mask is a copy of the input's: out->null_mask is needed when
 * the input has a mask and is not written when it has none.  Null rows of bin and fromIntegersWithBase have length 0.
 * Workspaces: srj_conv_workspace_bytes(rows) (it keeps each row's parsed value), srj_long_to_binary_workspace_bytes and
 * srj_integers_to_string_workspace_bytes (the scan's), 8-byte aligned.
 * Defined here where the reference is not: the base-column row check, the chars under null bytesToHex rows, and
 * SRJ_EOVERFLOW past INT32_MAX chars.  Errors: SRJ_EUNSUPPORTED for another input or base type; SRJ_EINVAL for a NULL or
 * misaligned buffer, a bad row count or base, and the scalar cases above.
 */
SRJ_API int64_t srj_conv_workspace_bytes(int64_t num_rows);
SRJ_API int srj_conv_sizes(const srj_column* input, const uint8_t* scalar, int32_t scalar_len, const srj_column* from_base, int32_t from,
                           const srj_column* to_base, int32_t to, int32_t* d_out_offsets, uint32_t* out_mask, int64_t* null_count,
                           int64_t* total_chars, void* workspace, void* stream);
SRJ_API int srj_conv(const srj_column* input, const uint8_t* scalar, int32_t scalar_len, const srj_column* from_base, int32_t from,
                     const srj_column* to_base, int32_t to, const int32_t* d_out_offsets, uint8_t* out_chars, const void* workspace,
                     void* stream);
SRJ_API int srj_conv_overflow(const srj_column* input, const uint8_t* scalar, int32_t scalar_len, const srj_column* from_base, int32_t from,
                              const srj_column* to_base, int32_t to, int32_t* overflow, void* stream);
SRJ_API int64_t srj_long_to_binary_workspace_bytes(int64_t num_rows);
SRJ_API int srj_long_to_binary_sizes(const srj_column* input, int32_t* d_out_offsets, int64_t* total_chars, void* workspace, void* stream);
SRJ_API int srj_long_to_binary(const srj_column* input, const srj_column* out, void* stream);
SRJ_API int64_t srj_integers_to_string_workspace_bytes(int64_t num_rows);
SRJ_API int srj_integers_to_string_sizes(const srj_column* input, int32_t base, int32_t* d_out_offsets, int64_t* total_chars, void* workspace,
                                         void* stream);
SRJ_API int srj_integers_to_string(const srj_column* input, int32_t base, const srj_column* out, void* stream);
SRJ_API int srj_bytes_to_hex_sizes(const srj_column* input, int32_t* d_out_offsets, int64_t* total_chars, void* stream);
SRJ_API int srj_bytes_to_hex(const srj_column* input, const srj_column* out, void* stream);

/* ---- multi-GPU configuration (SURVEY 8e: row-range shards + one all-gather of per-column chunks) ---------------- */
/* ---- Spark HashPartitioning on the device (SURVEY 8f rank 1) ---------------------------------------------------
 * The consumer of Hash.murmurHash32: GpuHashPartitioning computes pmod(murmur3_32(42, keys), P) per row and then
 * partitions the batch (cudf Table.partition) into the P slices shuffle_split takes
 * (src/main/cpp/src/shuffle_split.hpp:60-189: a table plus exactly these split offsets).
 *
 *   srj_partition_workspace_bytes : bytes of the caller-provided workspace of the calls below.
 *   srj_hash_partition            : d_partition_ids[r] = pmod(murmur3_32(seed, keys of row r), P) (null keys keep the
 *                                   accumulator, hash/murmur_hash.cu:111-117); then srj_partition_plan.
 *   srj_partition_plan            : ids -> d_partition_offsets[P + 1] (row index where each partition starts; [P] = rows)
 *                                   and the STABLE partition maps: d_scatter_map[src] = dest, d_gather_map[dest] = src
 *                                   (rows of one partition keep their input order).  Ids outside [0, P) are reduced
 *                                   with Spark's pmod in place.  <= INT32_MAX rows, <= 16384 partitions.  The workspace
 *                                   keeps the plan's tile order: pass it, unmodified, to srj_partition_columns.
 *   srj_partition_columns         : (same num_partitions, maps and workspace as the plan) moves fixed-width data and
 *                                   null masks into `out`; for STRING columns writes the
 *                                   output offsets (out.offsets[rows] = the chars the column needs: read it, allocate
 *                                   out.data, then call srj_partition_strings).  d_null_counts (device int64[ncols],
 *                                   may be NULL) receives the null count of every column that has a mask.
 *   srj_partition_strings         : the chars of every STRING column.
 * All pointers device pointers owned by the caller; asynchronous on `stream`.
 */
SRJ_API int64_t srj_partition_workspace_bytes(int64_t num_rows, int32_t num_partitions);
SRJ_API int srj_hash_partition(const srj_column* keys, int32_t num_keys, int64_t num_rows, uint32_t seed, int32_t num_partitions,
                               int32_t* d_partition_ids, int32_t* d_partition_offsets, int32_t* d_scatter_map,
                               int32_t* d_gather_map, void* workspace, void* stream);
SRJ_API int srj_partition_plan(int32_t* d_partition_ids, int64_t num_rows, int32_t num_partitions, int32_t* d_partition_offsets,
                               int32_t* d_scatter_map, int32_t* d_gather_map, void* workspace, void* stream);
SRJ_API int srj_partition_columns(const srj_column* in, const srj_column* out, int32_t num_columns, int64_t num_rows,
                                  int32_t num_partitions, const int32_t* d_scatter_map, const int32_t* d_gather_map,
                                  int64_t* d_null_counts, void* workspace, void* stream);
SRJ_API int srj_partition_strings(const srj_column* in, const srj_column* out, int32_t num_columns, int64_t num_rows,
                                  const int32_t* d_gather_map, void* stream);

/* ---- Kudo shuffle wire format: split / assemble (SURVEY 8f rank 2) -------------------------------------------------
 * shuffle_split / shuffle_assemble of the reference (src/main/cpp/src/shuffle_split.hpp:60-189) for FLAT tables
 * (fixed-width, decimal, STRING columns): a table is cut at `splits` (P + 1 row indices, e.g. the partition offsets
 * of srj_hash_partition) into P partitions written back to back, each in the Kudo format of
 * kudo/KudoSerializer.java:49-171 (header "KUD0" + 6 big-endian ints + hasValidity bits | validity | offsets | data);
 * assemble concatenates partitions (of one or several splits) back into one table.
 *   srj_kudo_split_sizes    : d_partition_offsets[P + 1] (byte offset of every partition) and *total_bytes (host; one
 *                             stream synchronisation).  SRJ_EINVAL when a split lies outside [0, num_rows],
 *                             SRJ_EOVERFLOW when the splits decrease or a partition overflows the header's lengths.
 *   srj_kudo_split          : writes the partitions into `out` (total_bytes, 4-byte aligned).
 *   srj_kudo_assemble_sizes : parses the headers; *total_rows and, per STRING column, char_totals[c] (host arrays);
 *                             SRJ_EINVAL on a malformed header.  The workspace keeps what srj_kudo_assemble needs.
 *   srj_kudo_assemble       : fills `out` (total_rows rows per column; null masks, where given, are produced for every
 *                             column -- partitions without validity contribute valid rows).
 * <= 256 columns, <= 65535 partitions.  LIST / STRUCT columns are not supported (SRJ_EUNSUPPORTED).
 */
SRJ_API int64_t srj_kudo_workspace_bytes(int32_t num_columns, int32_t num_partitions);
SRJ_API int srj_kudo_split_sizes(const srj_column* cols, int32_t num_columns, int64_t num_rows, const int32_t* d_splits,
                                 int32_t num_partitions, int64_t* d_partition_offsets, int64_t* total_bytes, void* workspace,
                                 void* stream);
SRJ_API int srj_kudo_split(const srj_column* cols, int32_t num_columns, int64_t num_rows, const int32_t* d_splits,
                           int32_t num_partitions, const int64_t* d_partition_offsets, uint8_t* out, void* workspace, void* stream);
SRJ_API int srj_kudo_assemble_sizes(const uint8_t* partitions, const int64_t* d_partition_offsets, int32_t num_partitions,
                                    const int32_t* type_ids, int32_t num_columns, int64_t* total_rows, int64_t* char_totals,
                                    void* workspace, void* stream);
SRJ_API int srj_kudo_assemble(const uint8_t* partitions, const int64_t* d_partition_offsets, int32_t num_partitions,
                              const srj_column* out, int32_t num_columns, int64_t total_rows, void* workspace, void* stream);

/* ---- Apache Spark UnsafeRow codec (SURVEY 8f rank 3) -----------------------------------------------------------
 * The row format Spark's own operators consume (org.apache.spark.sql.catalyst.expressions.UnsafeRow /
 * codegen.UnsafeRowWriter); the reference speaks only JCUDF (RowConversion.java:44-117) and leaves the adaptation to
 * the plugin's CudfUnsafeRow.  Row = null bitset (ceil(n/64) 8-byte words, bit SET = NULL) | one 8-byte slot per
 * field | variable region (strings: (offset << 32) | length, padded to 8; DECIMAL128: 16 bytes always reserved,
 * BigInteger.toByteArray() big-endian minimal bytes, slot (offset << 32) | byte count).  DECIMAL32/64 are longs.
 * Supported: the fixed-width types of the row path, STRING, DECIMAL32/64/128; <= 256 columns; rows 8-byte aligned.
 *
 *   srj_unsafe_row_layout   : bitset bytes and the size of a row without its strings.
 *   srj_unsafe_row_sizes    : d_row_offsets[rows + 1] (byte offset of every row) and *total_bytes (host; the call
 *                             synchronises the stream once); SRJ_EOVERFLOW beyond INT32_MAX bytes.
 *   srj_convert_to_unsafe_rows   : columns -> rows (d_row_offsets may be NULL for tables without STRING columns:
 *                                  rows are then fixed_bytes apart).
 *   srj_convert_from_unsafe_rows : rows -> fixed-width / decimal values, null masks (+ counts), and for STRING
 *                                  columns the output offsets (out.offsets[rows] = chars needed: read it, allocate
 *                                  out.data, then call srj_convert_from_unsafe_rows_strings).
 */
SRJ_API int srj_unsafe_row_layout(const int32_t* type_ids, int32_t num_columns, int32_t* bitset_bytes, int32_t* fixed_bytes);
SRJ_API int64_t srj_unsafe_row_workspace_bytes(int32_t num_columns, int64_t num_rows);
SRJ_API int srj_unsafe_row_sizes(const srj_column* cols, int32_t num_columns, int64_t num_rows, int32_t* d_row_offsets,
                                 int64_t* total_bytes, void* workspace, void* stream);
SRJ_API int srj_convert_to_unsafe_rows(const srj_column* cols, int32_t num_columns, int64_t num_rows, const int32_t* d_row_offsets,
                                       uint8_t* rows, void* workspace, void* stream);
SRJ_API int srj_convert_from_unsafe_rows(const uint8_t* rows, const int32_t* d_row_offsets, int64_t num_rows, const srj_column* out,
                                         int32_t num_columns, int64_t* d_null_counts, void* workspace, void* stream);
SRJ_API int srj_convert_from_unsafe_rows_strings(const uint8_t* rows, const int32_t* d_row_offsets, int64_t num_rows,
                                                 const srj_column* out, int32_t num_columns, void* stream);

/*
 * After the NCCL all-gather of every rank's packed column slab, add to the STRING offsets of rank r's rows the chars
 * the ranks before r hold for that column, so that the gathered chunks form one column.  No reference counterpart
 * (the reference has no collective); the plugin-side caller owns the NCCL communicator.
 *   gathered     : [world][slab_bytes] device buffer (the all-gather's output)
 *   d_offs_at    : device int64[num_string_columns]: byte offset of each STRING column's int32 offsets[rows + 1] in a slab
 *   d_scol       : device int32[num_string_columns]: schema column of each STRING column
 *   d_totals     : device int64[world][num_columns + 1]: every rank's d_char_totals, all-gathered
 */
SRJ_API int srj_shard_rebase_offsets(void* gathered, int64_t slab_bytes, const int64_t* d_offs_at, const int32_t* d_scol,
                                     const int64_t* d_totals, int64_t rows_per_shard, int32_t num_columns,
                                     int32_t num_string_columns, int32_t world, void* stream);

/* ---- host-buffer entry points (end-to-end path: H2D + convert + D2H inside the call) ---------------------- */
/*
 * What a caller holding HOST buffers uses (the plugin's row<->columnar transitions hand over host memory: the
 * reference's consumers copy to the device, call convertFromRows / convertToRows, copy back).  Device staging
 * buffers and streams live in a small per-plan pool and are reused by later calls (no cudaMalloc per call); calls are
 * re-entrant (concurrent calls take different pool entries) and synchronize before returning.  Pinned host buffers
 * give full PCIe speed.  Two calls in flight on two threads overlap one's H2D with the other's D2H (full duplex).
 *
 * srj_host_alloc_fn: the library calls it when an output buffer's size is known only during the call; it returns HOST
 * memory of `bytes` bytes (JNI shim: HostMemoryBuffer.allocate) or NULL on failure (-> SRJ_ENOMEM).
 *   from_rows: index = schema column of a STRING column -> its chars buffer
 *   to_rows  : index = 2 * batch -> int32 offsets[row_count + 1] of the batch, 2 * batch + 1 -> its row bytes
 */
typedef void* (*srj_host_alloc_fn)(void* ctx, int32_t index, int64_t bytes);

/*
 * Rows -> columns.  h_rows / h_row_offsets are the LIST's children in host memory (h_row_offsets may be NULL for a
 * fixed-width-only schema: rows at stride fixed_row_size); rows_bytes = size of h_rows.  h_cols[i].data / null_mask /
 * offsets are HOST buffers to fill (null_mask may be NULL to skip it); a STRING column's data pointer is an OUTPUT:
 * obtained from `alloc` and stored into h_cols[i].data.  Fixed-width-only schemas are streamed through the device in
 * chunks of `chunk_rows` rows (0 = library default) so that H2D, kernel and D2H of consecutive chunks overlap.
 */
SRJ_API int srj_convert_from_rows_host(const srj_plan* plan, const uint8_t* h_rows, const int32_t* h_row_offsets,
                                       int64_t rows_bytes, int64_t num_rows, srj_column* h_cols, int64_t* h_null_counts,
                                       int64_t chunk_rows, srj_host_alloc_fn alloc, void* alloc_ctx);
/*
 * Columns -> rows.  h_cols are HOST columns; batches[] receives the <= 2 GiB batch cut (build_batches, RC:1466-1557),
 * h_batch_offsets[b] / h_batch_data[b] the host buffers obtained from `alloc` for each batch.
 */
SRJ_API int srj_convert_to_rows_host(const srj_plan* plan, const srj_column* h_cols, int64_t num_rows,
                                     srj_row_batch* batches, int32_t max_batches, int32_t* num_batches,
                                     int32_t** h_batch_offsets, uint8_t** h_batch_data, srj_host_alloc_fn alloc,
                                     void* alloc_ctx);

#ifdef __cplusplus
}
#endif
#endif /* SRJ_B200_H */
