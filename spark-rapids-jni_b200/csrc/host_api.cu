// host_api.cu -- the host-buffer entry points of include/srj_b200.h (srj_convert_from_rows_host,
// srj_convert_to_rows_host): H2D, the device conversion through the same C ABI the device callers use, D2H.
// Device staging (buffers + streams) comes from a small per-plan pool and is reused: no cudaMalloc / cudaFree /
// stream creation on the steady-state path.  No kernels here.
#include <algorithm>
#include <cstring>
#include <vector>

#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"
#include "plan.hpp"

namespace srj {

namespace {

// RAII lease of one arena of the plan's pool: the first free one, else wait for arena 0.
struct ArenaLease {
  HostArena* a = nullptr;
  explicit ArenaLease(const srj_plan* plan)
  {
    for (auto& x : plan->host_pool.a)
      if (x.busy.try_lock()) { a = &x; return; }
    plan->host_pool.a[0].busy.lock();
    a = &plan->host_pool.a[0];
  }
  ~ArenaLease() { a->busy.unlock(); }
  int streams()
  {
    for (auto& s : a->st)
      if (!s) SRJ_CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return SRJ_OK;
  }
  int reserve(int which, size_t bytes)
  {
    if (a->d_cap[which] >= bytes) return SRJ_OK;
    if (a->d_buf[which]) { for (auto& s : a->st) if (s) cudaStreamSynchronize(s); cudaFree(a->d_buf[which]); }
    a->d_buf[which] = nullptr;
    a->d_cap[which] = 0;
    const size_t cap = (bytes + bytes / 8 + (size_t{1} << 20)) & ~size_t{255};   // grow-only, with slack
    SRJ_CUDA_TRY(cudaMalloc(&a->d_buf[which], cap));
    a->d_cap[which] = cap;
    return SRJ_OK;
  }
  int reserve_pinned(size_t bytes)
  {
    if (a->h_cap >= bytes) return SRJ_OK;
    if (a->h_pin) cudaFreeHost(a->h_pin);
    a->h_pin = nullptr;
    a->h_cap = 0;
    SRJ_CUDA_TRY(cudaMallocHost(&a->h_pin, bytes + 4096));
    a->h_cap = bytes + 4096;
    return SRJ_OK;
  }
  uint8_t* buf(int which) const { return static_cast<uint8_t*>(a->d_buf[which]); }
};

size_t align256(size_t v) { return (v + 255) & ~size_t{255}; }

// ---- fixed-width schemas: chunks pipelined over three streams (H2D | kernel | D2H of consecutive chunks overlap) -----
int from_rows_host_fixed(const srj_plan* plan, ArenaLease& L, const uint8_t* h_rows, int64_t num_rows, srj_column* h_cols,
                         int64_t* h_null_counts, int64_t chunk_rows)
{
  const int nc    = plan->num_columns;
  const int64_t S = plan->fixed_row_size;
  if (chunk_rows <= 0) {
    // ~1/12 of the input per chunk, between 32 MB and 1 GB of rows (larger chunks are faster): per chunk the copies
    // have a fixed cost and the first H2D / last D2H are not overlapped
    const int64_t cbytes = std::min<int64_t>(1ll << 30, std::max<int64_t>(32ll << 20, num_rows * S / 12));
    chunk_rows = std::max<int64_t>(32 * 1024, cbytes / S);
  }
  const int64_t T = plan->tiling.tile_rows >= 32 ? plan->tiling.tile_rows : 32;
  chunk_rows      = (chunk_rows + T - 1) / T * T;
  chunk_rows      = std::min<int64_t>(chunk_rows, (num_rows + T - 1) / T * T);
  constexpr int kSlots = 3;
  const int nslots     = static_cast<int>(std::min<int64_t>(kSlots, (num_rows + chunk_rows - 1) / chunk_rows));
  // per slot: row chunk | every column chunk + mask chunk (256-byte aligned pieces) | the pointer table
  std::vector<size_t> off_data(nc), off_mask(nc);
  size_t col_bytes = 0;
  for (int c = 0; c < nc; ++c) {
    off_data[c] = col_bytes;
    col_bytes += align256(static_cast<size_t>(chunk_rows) * plan->col_size[c]);
    off_mask[c] = col_bytes;
    col_bytes += align256(static_cast<size_t>(chunk_rows) / 8 + 4);
  }
  const size_t nent     = plan->fr_entries.size();
  const size_t tab_slot = align256(sizeof(void*) * (nent + nc));
  const size_t row_slot = align256(static_cast<size_t>(chunk_rows) * S);
  int rc;
  if ((rc = L.streams()) != SRJ_OK) return rc;
  if ((rc = L.reserve(0, row_slot * nslots)) != SRJ_OK) return rc;
  if ((rc = L.reserve(1, col_bytes * nslots)) != SRJ_OK) return rc;
  if ((rc = L.reserve(2, tab_slot * nslots + align256(sizeof(int64_t) * nc))) != SRJ_OK) return rc;
  if ((rc = L.reserve_pinned(tab_slot * nslots)) != SRJ_OK) return rc;
  int64_t* d_nulls = reinterpret_cast<int64_t*>(L.buf(2) + tab_slot * nslots);
  cudaStream_t s0  = L.a->st[0];
  SRJ_CUDA_TRY(cudaMemsetAsync(d_nulls, 0, sizeof(int64_t) * nc, s0));
  for (int s = 0; s < nslots; ++s) {
    void** tab = reinterpret_cast<void**>(static_cast<uint8_t*>(L.a->h_pin) + tab_slot * s);
    for (size_t e = 0; e < nent; ++e) tab[e] = L.buf(1) + col_bytes * s + off_data[plan->fr_entries[e].column];
    for (int c = 0; c < nc; ++c) tab[nent + c] = L.buf(1) + col_bytes * s + off_mask[c];
  }
  SRJ_CUDA_TRY(cudaMemcpyAsync(L.buf(2), L.a->h_pin, tab_slot * nslots, cudaMemcpyHostToDevice, s0));
  SRJ_CUDA_TRY(cudaStreamSynchronize(s0));   // tables + zeroed counters are in place before the chunk streams start
  int64_t k = 0;
  for (int64_t r0 = 0; r0 < num_rows; r0 += chunk_rows, ++k) {
    const int s       = static_cast<int>(k % nslots);
    cudaStream_t st   = L.a->st[s];
    const int64_t n   = std::min(chunk_rows, num_rows - r0);
    uint8_t* d_rows   = L.buf(0) + row_slot * s;
    void** d_tab      = reinterpret_cast<void**>(L.buf(2) + tab_slot * s);
    uint8_t* d_cols   = L.buf(1) + col_bytes * s;
    SRJ_CUDA_TRY(cudaMemcpyAsync(d_rows, h_rows + r0 * S, static_cast<size_t>(n) * S, cudaMemcpyHostToDevice, st));
    // the kernel sees a chunk-local table whose last mask word is zero-tailed; chunk starts are multiples of 32
    rc = launch_from_rows(plan, d_rows, nullptr, n * S, n, d_tab, reinterpret_cast<uint32_t* const*>(d_tab + nent), d_nulls, nullptr, st);
    if (rc != SRJ_OK) return rc;
    for (int c = 0; c < nc; ++c) {
      SRJ_CUDA_TRY(cudaMemcpyAsync(static_cast<uint8_t*>(h_cols[c].data) + r0 * plan->col_size[c], d_cols + off_data[c],
                                   static_cast<size_t>(n) * plan->col_size[c], cudaMemcpyDeviceToHost, st));
      if (h_cols[c].null_mask)
        SRJ_CUDA_TRY(cudaMemcpyAsync(h_cols[c].null_mask + r0 / 32, d_cols + off_mask[c], static_cast<size_t>((n + 31) / 32) * 4,
                                     cudaMemcpyDeviceToHost, st));
    }
  }
  for (int s = 0; s < nslots; ++s) SRJ_CUDA_TRY(cudaStreamSynchronize(L.a->st[s]));
  if (h_null_counts) SRJ_CUDA_TRY(cudaMemcpy(h_null_counts, d_nulls, sizeof(int64_t) * nc, cudaMemcpyDeviceToHost));
  return SRJ_OK;
}

// ---- schemas with STRING columns: one batch resident on the device (H2D -> phase 1 -> sizes -> phase 2 -> D2H) --------
int from_rows_host_var(const srj_plan* plan, ArenaLease& L, const uint8_t* h_rows, const int32_t* h_offs, int64_t rows_bytes,
                       int64_t num_rows, srj_column* h_cols, int64_t* h_null_counts, srj_host_alloc_fn alloc, void* ctx)
{
  const int nc = plan->num_columns;
  const int64_t n = num_rows;
  if (!h_offs) { set_error("convert_from_rows_host: a schema with STRING columns needs the LIST offsets"); return SRJ_EINVAL; }
  if (!alloc) { set_error("convert_from_rows_host: a schema with STRING columns needs the chars allocator"); return SRJ_EINVAL; }
  const size_t words = static_cast<size_t>((n + 31) / 32);
  // outputs: per column data (fixed) or offsets (STRING), then masks
  std::vector<size_t> at_data(nc), at_mask(nc);
  size_t out_bytes = 0;
  for (int c = 0; c < nc; ++c) {
    at_data[c] = out_bytes;
    out_bytes += align256(plan->type_ids[c] == SRJ_STRING ? static_cast<size_t>(n + 1) * 4 : static_cast<size_t>(n) * plan->col_size[c]);
  }
  for (int c = 0; c < nc; ++c) { at_mask[c] = out_bytes; out_bytes += align256(words * 4); }
  const size_t ws_bytes  = static_cast<size_t>(srj_from_rows_workspace_bytes(plan, n));
  const size_t at_offs   = 0;
  const size_t at_ws     = align256(static_cast<size_t>(n + 1) * 4);
  const size_t at_cnt    = at_ws + align256(ws_bytes);
  const size_t misc      = at_cnt + align256(static_cast<size_t>(2 * nc + 1) * 8);
  int rc;
  if ((rc = L.streams()) != SRJ_OK) return rc;
  if ((rc = L.reserve(0, static_cast<size_t>(rows_bytes) + 64)) != SRJ_OK) return rc;
  if ((rc = L.reserve(1, out_bytes)) != SRJ_OK) return rc;
  if ((rc = L.reserve(2, misc)) != SRJ_OK) return rc;
  if ((rc = L.reserve_pinned(static_cast<size_t>(2 * nc + 1) * 8)) != SRJ_OK) return rc;
  cudaStream_t st  = L.a->st[0];
  uint8_t* d_rows  = L.buf(0);
  int32_t* d_offs  = reinterpret_cast<int32_t*>(L.buf(2) + at_offs);
  void* d_ws       = L.buf(2) + at_ws;
  int64_t* d_nulls = reinterpret_cast<int64_t*>(L.buf(2) + at_cnt);
  int64_t* d_tot   = d_nulls + nc;
  SRJ_CUDA_TRY(cudaMemcpyAsync(d_offs, h_offs, static_cast<size_t>(n + 1) * 4, cudaMemcpyHostToDevice, st));
  SRJ_CUDA_TRY(cudaMemcpyAsync(d_rows, h_rows, static_cast<size_t>(rows_bytes), cudaMemcpyHostToDevice, st));
  std::vector<srj_column> dc(nc);
  for (int c = 0; c < nc; ++c) {
    dc[c]           = srj_column{plan->type_ids[c], plan->scales[c], n, nullptr, reinterpret_cast<uint32_t*>(L.buf(1) + at_mask[c]), nullptr};
    if (plan->type_ids[c] == SRJ_STRING) dc[c].offsets = reinterpret_cast<int32_t*>(L.buf(1) + at_data[c]);
    else dc[c].data = L.buf(1) + at_data[c];
  }
  rc = srj_convert_from_rows_fixed(plan, d_rows, d_offs, rows_bytes, n, dc.data(), d_nulls, d_tot, nullptr, d_ws, st);
  if (rc != SRJ_OK) return rc;
  int64_t* h_cnt = static_cast<int64_t*>(L.a->h_pin);
  SRJ_CUDA_TRY(cudaMemcpyAsync(h_cnt, d_nulls, static_cast<size_t>(2 * nc + 1) * 8, cudaMemcpyDeviceToHost, st));
  // the fixed-width columns and every mask can leave while the sizes are read and the chars are gathered
  cudaStream_t st2 = L.a->st[1];
  cudaEvent_t ev;
  SRJ_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  cudaEventRecord(ev, st);
  cudaStreamWaitEvent(st2, ev, 0);
  for (int c = 0; c < nc; ++c) {
    if (plan->type_ids[c] != SRJ_STRING && h_cols[c].data)
      cudaMemcpyAsync(h_cols[c].data, L.buf(1) + at_data[c], static_cast<size_t>(n) * plan->col_size[c], cudaMemcpyDeviceToHost, st2);
    if (h_cols[c].null_mask) cudaMemcpyAsync(h_cols[c].null_mask, L.buf(1) + at_mask[c], words * 4, cudaMemcpyDeviceToHost, st2);
  }
  SRJ_CUDA_TRY(cudaStreamSynchronize(st));   // the read of RC:2389
  cudaEventDestroy(ev);
  if (h_cnt[2 * nc] & 2) { cudaStreamSynchronize(st2); set_error("convert_from_rows_host: a STRING column exceeds the int32 chars limit"); return SRJ_EOVERFLOW; }
  std::vector<size_t> at_chars(nc, 0);
  size_t chars_bytes = 0;
  for (int c = 0; c < nc; ++c)
    if (plan->type_ids[c] == SRJ_STRING) {
      at_chars[c] = chars_bytes;
      chars_bytes += align256(static_cast<size_t>(h_cnt[nc + c]));
    }
  if ((rc = L.reserve(3, chars_bytes + 256)) != SRJ_OK) { cudaStreamSynchronize(st2); return rc; }
  for (int c = 0; c < nc; ++c)
    if (plan->type_ids[c] == SRJ_STRING) {
      dc[c].data     = L.buf(3) + at_chars[c];
      h_cols[c].data = h_cnt[nc + c] > 0 ? alloc(ctx, c, h_cnt[nc + c]) : nullptr;
      if (h_cnt[nc + c] > 0 && !h_cols[c].data) { cudaStreamSynchronize(st2); set_error("convert_from_rows_host: the chars allocator failed for column %d", c); return SRJ_ENOMEM; }
    }
  rc = srj_convert_from_rows_strings(plan, d_rows, d_offs, rows_bytes, n, dc.data(), d_tot, d_ws, st);
  if (rc != SRJ_OK) { cudaStreamSynchronize(st2); return rc; }
  for (int c = 0; c < nc; ++c)
    if (plan->type_ids[c] == SRJ_STRING) {
      if (h_cols[c].offsets) SRJ_CUDA_TRY(cudaMemcpyAsync(h_cols[c].offsets, dc[c].offsets, static_cast<size_t>(n + 1) * 4, cudaMemcpyDeviceToHost, st));
      if (h_cnt[nc + c] > 0)
        SRJ_CUDA_TRY(cudaMemcpyAsync(h_cols[c].data, dc[c].data, static_cast<size_t>(h_cnt[nc + c]), cudaMemcpyDeviceToHost, st));
    }
  SRJ_CUDA_TRY(cudaStreamSynchronize(st));
  SRJ_CUDA_TRY(cudaStreamSynchronize(st2));
  if (h_null_counts) std::memcpy(h_null_counts, h_cnt, sizeof(int64_t) * nc);
  return SRJ_OK;
}

}  // namespace
}  // namespace srj

using namespace srj;

extern "C" {

int srj_convert_from_rows_host(const srj_plan* plan, const uint8_t* h_rows, const int32_t* h_row_offsets, int64_t rows_bytes,
                               int64_t num_rows, srj_column* h_cols, int64_t* h_null_counts, int64_t chunk_rows,
                               srj_host_alloc_fn alloc, void* alloc_ctx)
{
  SRJ_API_RANGE();
  int rc = check_cols(plan, h_cols, num_rows, "convert_from_rows_host");
  if (rc != SRJ_OK) return rc;
  const int nc = plan->num_columns;
  if (h_null_counts) std::fill(h_null_counts, h_null_counts + nc, 0);
  if (num_rows == 0) return SRJ_OK;
  if (!h_rows) { set_error("convert_from_rows_host: rows is null"); return SRJ_EINVAL; }
  if (static_cast<int64_t>(plan->fixed_row_size) * num_rows > rows_bytes) { set_error("convert_from_rows_host: The layout of the data appears to be off"); return SRJ_EINVAL; }
  for (int c = 0; c < nc; ++c) {
    const bool str = plan->type_ids[c] == SRJ_STRING;
    if (!str && !h_cols[c].data) { set_error("convert_from_rows_host: column %d has no data buffer", c); return SRJ_EINVAL; }
    if (str && !h_cols[c].offsets) { set_error("convert_from_rows_host: STRING column %d has no offsets buffer", c); return SRJ_EINVAL; }
  }
  ArenaLease L(plan);
  if (plan->num_string_columns == 0) return from_rows_host_fixed(plan, L, h_rows, num_rows, h_cols, h_null_counts, chunk_rows);
  return from_rows_host_var(plan, L, h_rows, h_row_offsets, rows_bytes, num_rows, h_cols, h_null_counts, alloc, alloc_ctx);
}

int srj_convert_to_rows_host(const srj_plan* plan, const srj_column* h_cols, int64_t num_rows, srj_row_batch* batches,
                             int32_t max_batches, int32_t* num_batches, int32_t** h_batch_offsets, uint8_t** h_batch_data,
                             srj_host_alloc_fn alloc, void* alloc_ctx)
{
  SRJ_API_RANGE();
  int rc = check_cols(plan, h_cols, num_rows, "convert_to_rows_host");
  if (rc != SRJ_OK) return rc;
  if (!batches || !num_batches || max_batches < 1 || !h_batch_offsets || !h_batch_data || !alloc) { set_error("convert_to_rows_host: bad argument"); return SRJ_EINVAL; }
  *num_batches = 0;
  if (num_rows == 0) return SRJ_OK;
  const int nc       = plan->num_columns;
  const int64_t n    = num_rows;
  const size_t words = static_cast<size_t>((n + 31) / 32);
  ArenaLease L(plan);
  if ((rc = L.streams()) != SRJ_OK) return rc;
  cudaStream_t st = L.a->st[0];
  // inputs on the device: data / offsets / masks / chars
  std::vector<size_t> at_data(nc), at_mask(nc), at_offs(nc), bytes_data(nc);
  size_t in_bytes = 0;
  for (int c = 0; c < nc; ++c) {
    const bool str = plan->type_ids[c] == SRJ_STRING;
    if (str && !h_cols[c].offsets) { set_error("convert_to_rows_host: STRING column %d has no offsets", c); return SRJ_EINVAL; }
    bytes_data[c] = str ? static_cast<size_t>(h_cols[c].offsets[n]) : static_cast<size_t>(n) * plan->col_size[c];
    if (bytes_data[c] && !h_cols[c].data) { set_error("convert_to_rows_host: column %d has no data", c); return SRJ_EINVAL; }
    at_data[c] = in_bytes; in_bytes += align256(bytes_data[c] + 16);
    at_mask[c] = in_bytes; in_bytes += h_cols[c].null_mask ? align256(words * 4) : 0;
    at_offs[c] = in_bytes; in_bytes += str ? align256(static_cast<size_t>(n + 1) * 4) : 0;
  }
  const size_t ws_bytes = static_cast<size_t>(srj_to_rows_workspace_bytes(plan, n));
  if ((rc = L.reserve(1, in_bytes)) != SRJ_OK) return rc;
  if ((rc = L.reserve(2, align256(ws_bytes) + 256)) != SRJ_OK) return rc;
  std::vector<srj_column> dc(nc);
  for (int c = 0; c < nc; ++c) {
    const bool str = plan->type_ids[c] == SRJ_STRING;
    dc[c] = srj_column{plan->type_ids[c], plan->scales[c], n, L.buf(1) + at_data[c], nullptr, nullptr};
    if (bytes_data[c]) SRJ_CUDA_TRY(cudaMemcpyAsync(dc[c].data, h_cols[c].data, bytes_data[c], cudaMemcpyHostToDevice, st));
    if (h_cols[c].null_mask) {
      dc[c].null_mask = reinterpret_cast<uint32_t*>(L.buf(1) + at_mask[c]);
      SRJ_CUDA_TRY(cudaMemcpyAsync(dc[c].null_mask, h_cols[c].null_mask, words * 4, cudaMemcpyHostToDevice, st));
    }
    if (str) {
      dc[c].offsets = reinterpret_cast<int32_t*>(L.buf(1) + at_offs[c]);
      SRJ_CUDA_TRY(cudaMemcpyAsync(dc[c].offsets, h_cols[c].offsets, static_cast<size_t>(n + 1) * 4, cudaMemcpyHostToDevice, st));
    }
  }
  void* d_ws = L.buf(2);
  rc = srj_to_rows_plan_batches(plan, dc.data(), n, d_ws, batches, max_batches, num_batches, st);   // synchronizes for STRING schemas
  if (rc != SRJ_OK) return rc;
  const int nb = *num_batches;
  size_t out_bytes = 0;
  std::vector<size_t> at_bo(nb), at_bd(nb);
  for (int b = 0; b < nb; ++b) {
    at_bo[b] = out_bytes; out_bytes += align256(static_cast<size_t>(batches[b].row_count + 1) * 4);
    at_bd[b] = out_bytes; out_bytes += align256(static_cast<size_t>(batches[b].num_bytes) + 16);
  }
  if ((rc = L.reserve(0, out_bytes)) != SRJ_OK) return rc;
  std::vector<int32_t*> d_bo(nb);
  std::vector<uint8_t*> d_bd(nb);
  for (int b = 0; b < nb; ++b) {
    d_bo[b]            = reinterpret_cast<int32_t*>(L.buf(0) + at_bo[b]);
    d_bd[b]            = L.buf(0) + at_bd[b];
    h_batch_offsets[b] = static_cast<int32_t*>(alloc(alloc_ctx, 2 * b, static_cast<int64_t>(batches[b].row_count + 1) * 4));
    h_batch_data[b]    = static_cast<uint8_t*>(alloc(alloc_ctx, 2 * b + 1, std::max<int64_t>(batches[b].num_bytes, 1)));
    if (!h_batch_offsets[b] || !h_batch_data[b]) { set_error("convert_to_rows_host: the batch allocator failed"); return SRJ_ENOMEM; }
  }
  rc = srj_convert_to_rows(plan, dc.data(), n, d_ws, batches, nb, d_bo.data(), d_bd.data(), st);
  if (rc != SRJ_OK) return rc;
  for (int b = 0; b < nb; ++b) {
    SRJ_CUDA_TRY(cudaMemcpyAsync(h_batch_offsets[b], d_bo[b], static_cast<size_t>(batches[b].row_count + 1) * 4, cudaMemcpyDeviceToHost, st));
    if (batches[b].num_bytes)
      SRJ_CUDA_TRY(cudaMemcpyAsync(h_batch_data[b], d_bd[b], static_cast<size_t>(batches[b].num_bytes), cudaMemcpyDeviceToHost, st));
  }
  SRJ_CUDA_TRY(cudaStreamSynchronize(st));
  return SRJ_OK;
}

}  // extern "C"
