// kernels.hpp -- host-side launchers implemented in the .cu files.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/srj_b200.h"
#include "plan.hpp"

namespace srj {

// from_rows.cu
int launch_from_rows(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets, int64_t rows_bytes,
                     int64_t num_rows, void* const* d_ent_dst, uint32_t* const* d_masks, int64_t* d_null_counts,
                     int64_t* d_status, cudaStream_t stream);

size_t from_rows_smem_bytes(const Tiling& tl, int nentries, int ncols, int nstr);  // dynamic shared memory of from_rows_kernel

// from_rows_wide.cu: wide variable-width tables (per-row TMA slabs; offsets leave as group-local inclusive sums +
// absolute group bases, finished by phase 2)
bool plan_wide(srj_plan* plan);
int64_t wide_workspace_bytes(const srj_plan* plan, int64_t num_rows);
const uint32_t* wide_workspace_bases(const srj_plan* plan, int64_t num_rows, const void* workspace);  // [nstr][ngroups]
int launch_from_rows_wide(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets, int64_t rows_bytes,
                          int64_t num_rows, const srj_column* cols /* host array of the output columns */,
                          int64_t* d_null_counts, int64_t* d_char_totals, void* d_scratch /* wide_workspace_bytes() */,
                          cudaStream_t stream);

// strings.cu
// In-place inclusive scan of the int32 lengths stored at offsets[c][1..n] for every STRING column
// (offsets[c][0] = 0), per-column totals to d_char_totals[schema col] (int64), a total beyond INT32_MAX sets bit 1 of *d_status.
int launch_string_offsets_scan(int32_t* const* d_offsets /* device array [nstr] */, const int32_t* d_string_cols,
                               int nstr, int64_t num_rows, int64_t* d_char_totals, int64_t* d_status,
                               void* d_partials /* int64 [nstr * nchunks] */, cudaStream_t stream);
int64_t string_scan_partials_bytes(int nstr, int64_t num_rows);
// copy_strings_from_rows replacement.  cols = the caller's columns (host array); d_tab = device table
// [offsets nstr][chars nstr], needed (and uploaded by the caller) only when !strings_fast_path().
int launch_strings_from_rows(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets,
                             int64_t rows_bytes, int64_t num_rows, const srj_column* cols, void* const* d_tab,
                             const int64_t* d_status,
                             const uint32_t* d_bases /* non-NULL: offsets hold group-local inclusive sums, the chars before
                                                        each 32-row group are d_bases[nstr][ngroups] (wide tables) */,
                             cudaStream_t stream);
bool strings_wide_eligible(const srj_plan* plan);
bool strings_fast_path(const srj_plan* plan, const int64_t* d_status);

// to_rows.cu
int launch_row_sizes(const srj_plan* plan, const int32_t* const* d_str_offsets, int64_t num_rows,
                     uint64_t* d_cum_sizes, cudaStream_t stream);
// batch cut on the device: d_out = int64[1 + 3 * max_batches]
int launch_batch_cut(const uint64_t* d_cum, int64_t num_rows, int32_t max_batches, int64_t* d_out, cudaStream_t stream);
int launch_to_rows(const srj_plan* plan, const void* const* d_col_data, const uint32_t* const* d_masks,
                   const int32_t* const* d_str_offsets, const uint8_t* const* d_str_chars, int64_t row_start,
                   int64_t row_count, const uint64_t* d_cum_sizes /* NULL for fixed */, int32_t* out_offsets,
                   uint8_t* out_data, int64_t out_bytes, cudaStream_t stream,
                   const void* const* h_col_data /* host copy of the column pointers (alignment checks) */,
                   int32_t* d_fail_flag /* 4 bytes of device scratch (variable-width tables), may be NULL */);
// to_rows_var.cu: wide rows with STRING columns.  *launched = 0: table not eligible, nothing was launched.
int launch_to_rows_var(const srj_plan* plan, const void* const* d_col_data, const uint32_t* const* d_masks,
                       const int32_t* const* d_str_offsets, const uint8_t* const* d_str_chars, int64_t row_start,
                       int64_t row_count, const int32_t* out_offsets, uint8_t* out_data, int64_t out_bytes,
                       int32_t* d_fail_flag, cudaStream_t stream, const void* const* h_col_data, int* launched);

// hash_nested.cu: tables with LIST / STRUCT key columns
bool hash_has_nested(const srj_column* cols, int32_t num_columns);
int launch_hash_nested(int kind, const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t seed, void* out,
                       void* d_scratch, void* h_pinned, size_t scratch_bytes, cudaStream_t stream);

// hash.cu
int launch_hash(int kind, const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t seed, void* out,
                cudaStream_t stream);

// ---- partition.cu: Spark HashPartitioning (ids, stable partition maps, moving the columns) ----
int64_t partition_workspace_bytes(int64_t num_rows, int32_t num_partitions);
int launch_partition_plan(int32_t* d_ids, int64_t num_rows, int32_t num_partitions, int32_t* d_part_offsets, int32_t* d_scatter_map,
                          int32_t* d_gather_map, void* workspace, cudaStream_t stream);
int launch_partition_scatter_fixed(const void* in, void* out, int elem_size, const int32_t* d_scatter_map, int64_t n, cudaStream_t stream);
int launch_partition_gather_mask(const uint32_t* in, uint32_t* out, const int32_t* d_gather_map, int64_t n, unsigned long long* d_null_count,
                                 cudaStream_t stream);
int launch_partition_move_tiles(const srj_column* in, const srj_column* out, const int* elem_size, int32_t ncols, int64_t n, int32_t P,
                                const int32_t* d_scatter_map, const void* workspace, unsigned long long* d_null_counts, cudaStream_t stream);
int launch_partition_string_offsets(const int32_t* in_off, int32_t* out_off, const int32_t* d_gather_map, int64_t n, void* scan_ws,
                                    cudaStream_t stream);
int launch_partition_gather_chars(const uint8_t* in_chars, const int32_t* in_off, uint8_t* out_chars, const int32_t* out_off,
                                  const int32_t* d_gather_map, int64_t n, cudaStream_t stream);

// exclusive scan of int32 in place (partition.cu); `sums` = i32_scan_nchunks(n) ints of scratch; *tail (may be NULL) <- grand total
int64_t i32_scan_nchunks(int64_t n);
int launch_i32_exclusive_scan(int32_t* v, int64_t n, int32_t* sums, int32_t* tail, cudaStream_t stream);

// ---- unsafe_row.cu: columns <-> Apache Spark UnsafeRow ----
int unsafe_row_layout(const int32_t* type_ids, int32_t ncols, int32_t* bitset_bytes, int32_t* fixed_bytes, int32_t* ndec, int32_t* nstr);
int64_t unsafe_row_workspace_bytes(int32_t ncols, int64_t n);
int launch_unsafe_row_sizes(const srj_column* cols, int32_t ncols, int64_t n, int32_t* d_row_offsets, void* workspace, int64_t* h_total,
                            cudaStream_t stream);
int launch_unsafe_to_rows(const srj_column* cols, int32_t ncols, int64_t n, const int32_t* d_row_offsets, uint8_t* rows, void* workspace,
                          cudaStream_t stream);
int launch_unsafe_from_rows(const srj_column* out, int32_t ncols, int64_t n, const uint8_t* rows, const int32_t* d_row_offsets,
                            int64_t* d_null_counts, void* workspace, cudaStream_t stream);
int launch_unsafe_from_rows_strings(const srj_column* out, int32_t ncols, int64_t n, const uint8_t* rows, const int32_t* d_row_offsets,
                                    cudaStream_t stream);

// ---- sha2.cu: SHA-224/256/384/512 of a STRING column as lowercase hex, nulls preserved ----
int32_t sha2_hex_width(int32_t digest_bits);    // hex chars per valid row, 0 for an unknown digest
int64_t sha2_workspace_bytes(int64_t n);
// output offsets (width x valid rows before each row) and, on the host, the chars total; SRJ_EOVERFLOW beyond INT32_MAX
int launch_sha2_sizes(int32_t digest_bits, const srj_column& in, int32_t* d_offsets, int64_t* h_total, void* workspace, cudaStream_t stream);
int launch_sha2(int32_t digest_bits, const srj_column& in, const srj_column& out, cudaStream_t stream);

// ---- bloom_filter.cu: Spark's serialized V1 / V2 bloom filter (init, put, probe, merge) ----
struct BloomHeader {
  int32_t version, num_hashes, seed, num_longs;   // seed is 0 for V1
};
// m with x % bits == x - mulhi(x, m) * bits, minus bits once more when that is >= bits (32-bit x for V1, 64-bit for V2)
uint64_t bloom_reciprocal(int32_t version, uint64_t bits);
int launch_bloom_init(const BloomHeader& h, uint8_t* buf, cudaStream_t stream);
int launch_bloom_put(const BloomHeader& h, uint8_t* buf, const srj_column& in, cudaStream_t stream);
int launch_bloom_probe(const BloomHeader& h, const uint8_t* buf, const srj_column& in, uint8_t* out, uint32_t* out_mask, cudaStream_t stream);
// header copy, header check (*d_flag <- 1 on a mismatch) and the word-wise OR of `nfilters` filters `stride` bytes apart
int launch_bloom_merge(const uint8_t* child, int64_t stride, int32_t nfilters, int hdr_bytes, uint8_t* out, int32_t* d_flag, cudaStream_t stream);

// ---- zorder.cu: ZOrder.interleaveBits / hilbertIndex (the caller has checked every argument) ----
// out_offsets: rows + 1 int32 (r * ncols * elem_bytes); out: rows * ncols * elem_bytes bytes.  Either may be unaligned.
int launch_interleave_bits(const srj_column* cols, int32_t ncols, int64_t rows, int32_t elem_bytes, int32_t* out_offsets, uint8_t* out,
                           cudaStream_t stream);
int launch_hilbert_index(int32_t num_bits, const srj_column* cols, int32_t ncols, int64_t rows, int64_t* out, cudaStream_t stream);

// ---- iceberg.cu: Iceberg's bucket / truncate / date-time transforms (the caller has checked every argument) ----
// out_mask (NULL: none) gets a copy of the input's mask, all ones when the input has none.
int launch_iceberg_bucket(const srj_column& in, int32_t num_buckets, int32_t* out, uint32_t* out_mask, cudaStream_t stream);
int launch_iceberg_truncate_fixed(const srj_column& in, int32_t width, void* out, uint32_t* out_mask, cudaStream_t stream);
int64_t iceberg_truncate_workspace_bytes(int64_t n);
// STRING / LIST<UINT8>: d_offsets[0 .. n] and *h_total (reads the total back: one stream synchronisation)
int launch_iceberg_truncate_sizes(const srj_column& in, int32_t width, int32_t* d_offsets, int64_t* h_total, void* workspace,
                                  cudaStream_t stream);
int launch_iceberg_truncate_bytes(const srj_column& in, const int32_t* out_offsets, uint8_t* out_bytes, uint32_t* out_mask, cudaStream_t stream);
int launch_iceberg_datetime(int32_t transform, const srj_column& in, int32_t* out, uint32_t* out_mask, cudaStream_t stream);

// ---- decimal.cu: DecimalUtils' DECIMAL128 arithmetic (the caller has checked every argument and scale) ----
// Writes out_mask (the AND of the input masks) and *null_count when an input has a mask, reading the count back (one
// stream synchronisation); otherwise *null_count = 0 and out_mask is untouched.
int launch_decimal128_binary(int32_t op, const srj_column& a, const srj_column& b, int32_t out_scale, bool interim_cast, uint8_t* ovf,
                             void* out, uint32_t* out_mask, int64_t* null_count, cudaStream_t stream);
// A device counter of the calling host thread on the current device, allocated once; a call that uses it reads it back
// before it returns.
int null_counter(unsigned long long** out);

// ---- datetime.cu: DateTimeUtils' rebase and truncation (the caller has checked every argument) ----
// Truncation formats, in the reference's order of families; TIMESTAMP_DAYS accepts kDtYear .. kDtWeek.
enum DtFormat : int32_t {
  kDtYear, kDtQuarter, kDtMonth, kDtWeek, kDtDay, kDtHour, kDtMinute, kDtSecond, kDtMillisecond, kDtMicrosecond, kDtInvalid
};
// the format named by len bytes at s (ASCII case-insensitive), kDtInvalid when none
int32_t datetime_parse_format(const char* s, int32_t len);
bool datetime_format_fits(int32_t fmt, bool micros);
// out_mask (NULL: none) gets a copy of the input's mask, all ones when the input has none
int launch_datetime_rebase(int32_t direction, const srj_column& in, void* out, uint32_t* out_mask, cudaStream_t stream);
// a format that does not fit the type zeroes out and out_mask (which must then be given); otherwise as the rebase
int launch_datetime_truncate_scalar(int32_t fmt, const srj_column& in, void* out, uint32_t* out_mask, cudaStream_t stream);
// fmt.size rows; dt has one row (broadcast) or fmt.size.  Writes out, out_mask and *null_count (one read-back).
int launch_datetime_truncate_column(const srj_column& dt, const srj_column& fmt, void* out, uint32_t* out_mask, int64_t* null_count,
                                    cudaStream_t stream);

// ---- timezone.cu: GpuTimeZoneDB's conversions (the caller has checked every argument and the table's layout) ----
// reads the zone's bounds back (one synchronisation), checks it has an entry and 0 or 12 rule integers, then launches
int launch_timezone_convert(bool to_utc, const srj_column& in, const srj_column& fixed, const srj_column& dst, int32_t tz_index, void* out,
                            uint32_t* out_mask, cudaStream_t stream);
// in[0..5]: seconds, micros, invalid, tz type, tz offset, tz indices.  Writes out, out_mask and *null_count (one read-back).
int launch_timezone_convert_multi(const srj_column* in, const srj_column& fixed, const srj_column& dst, int64_t* out, uint32_t* out_mask,
                                  int64_t* null_count, cudaStream_t stream);
// a table of 0 transitions is a fixed offset (its pointers may be NULL)
int launch_orc_convert_timezones(const srj_column& in, const int64_t* wt, const int32_t* wo, int32_t wn, int32_t wraw, const int64_t* rt,
                                 const int32_t* ro, int32_t rn, int32_t rraw, void* out, uint32_t* out_mask, cudaStream_t stream);

// ---- cast_datetime.cu: CastStrings' string-to-timestamp and string-to-date parses (the caller has checked every argument) ----
// name_map: STRUCT<STRING, INT32>; fixed / dst: the time zone table; default_tz inside the table.  Asynchronous.
int launch_cast_parse_timestamps(const srj_column& in, const srj_column& name_map, const srj_column& fixed, const srj_column& dst,
                                 int32_t default_tz, int64_t default_epoch_day, int64_t now, bool is_320, bool is_400, uint8_t* result,
                                 int64_t* seconds, int32_t* micros, uint8_t* tz_type, int32_t* tz_offset, int32_t* tz_index,
                                 cudaStream_t stream);
// writes out, out_mask and *null_count (one read-back)
int launch_cast_parse_dates(const srj_column& in, int32_t* out, uint32_t* out_mask, int64_t* null_count, cudaStream_t stream);

// ---- join.cu: JoinPrimitives' hash inner join and gather-map helpers (the caller has checked every argument) ----
constexpr int32_t kMaxJoinKeys = SRJ_MAX_JOIN_KEYS;
int32_t join_key_width(int32_t type_id);      // bytes of a fixed-width key type, 0 for any other
int64_t hash_join_workspace_bytes(int64_t left_rows, int64_t right_rows);
// builds the table on the right keys, counts each left row's matches and reads the pair count back (one synchronisation)
int launch_hash_join_size(const srj_column* left, const srj_column* right, int32_t ncols, int64_t left_rows, int64_t right_rows, bool nulls_equal,
                          int64_t* num_pairs, void* workspace, cudaStream_t stream);
// writes the pairs from the table and counts launch_hash_join_size left in the workspace
int launch_hash_join(const srj_column* left, const srj_column* right, int32_t ncols, int64_t left_rows, int64_t right_rows, int32_t* left_map,
                     int32_t* right_map, void* workspace, cudaStream_t stream);
int64_t join_mask_workspace_bytes(int64_t rows);
int launch_join_mark(const int32_t* map, int64_t n, int64_t rows, void* workspace, cudaStream_t stream);
int read_join_matched(const void* const* workspaces, int32_t count, int64_t* matched, cudaStream_t stream);
int launch_join_compact(const void* workspace, int64_t rows, bool set, int32_t* out, cudaStream_t stream);
int launch_join_fill(int32_t* out, int64_t n, int32_t value, cudaStream_t stream);
int launch_join_matched_rows(const int32_t* map, int64_t n, int64_t rows, uint8_t* out, cudaStream_t stream);

// ---- kudo.cu: the Kudo shuffle wire format for flat tables (split / assemble) ----
// exclusive scan of v[0 .. n] in place by one CTA (n up to a few 10^5); v[n] receives the total
int launch_i64_scan_small(int64_t* v, int n, cudaStream_t stream);
int64_t kudo_workspace_bytes(int32_t ncols, int32_t P);
int launch_kudo_split_sizes(const srj_column* cols, int32_t ncols, int64_t num_rows, const int32_t* d_splits, int32_t P, int64_t* d_part_offsets,
                            int64_t* h_total, void* workspace, cudaStream_t stream);
int launch_kudo_split(const srj_column* cols, int32_t ncols, const int32_t* d_splits, int32_t P, const int64_t* d_part_offsets, uint8_t* out,
                      void* workspace, cudaStream_t stream);
int launch_kudo_assemble_sizes(const uint8_t* buf, const int64_t* d_part_offsets, int32_t P, const int32_t* type_ids, int32_t ncols, int64_t* h_rows,
                               int64_t* h_char_totals, void* workspace, cudaStream_t stream);
int launch_kudo_assemble(const uint8_t* buf, const int64_t* d_part_offsets, int32_t P, const srj_column* out, int32_t ncols, int64_t total_rows,
                         void* workspace, cudaStream_t stream);

}  // namespace srj
