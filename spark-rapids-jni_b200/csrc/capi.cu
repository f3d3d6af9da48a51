// capi.cu -- the extern "C" boundary declared in include/srj_b200.h: argument checking, plans,
// per-call pointer tables, launch sequencing.  No kernels here.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "common.cuh"
#include "hash_device.cuh"
#include "kernels.hpp"
#include "plan.hpp"

namespace srj {

static thread_local char g_err[512] = "";

// NVTX range of one C-ABI call (the reference wraps its entry points the same way: nvtx_ranges.hpp:24-46,
// SRJ_FUNC_RANGE); header-only NVTX v3, a no-op unless a profiler is attached.
struct ApiRange {
  explicit ApiRange(const char* name) { nvtxRangePushA(name); }
  ~ApiRange() { nvtxRangePop(); }
};
#define SRJ_API_RANGE() ::srj::ApiRange _srj_range(__func__)

void set_error(const char* fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what)
{
  set_error("CUDA error %d (%s) at %s", static_cast<int>(e), cudaGetErrorString(e), what);
  return e == cudaErrorMemoryAllocation ? SRJ_ENOMEM : SRJ_ECUDA;
}

int sm_count()
{
  int dev = 0, nsm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 132;  // H100 SXM; a failing device surfaces at the launch that follows
  return nsm;
}

static int size_of_type(int32_t t)
{
  switch (t) {
    case SRJ_INT8: case SRJ_UINT8: case SRJ_BOOL8: return 1;
    case SRJ_INT16: case SRJ_UINT16: return 2;
    case SRJ_INT32: case SRJ_UINT32: case SRJ_FLOAT32: case SRJ_TIMESTAMP_DAYS: case SRJ_DURATION_DAYS:
    case SRJ_DECIMAL32: return 4;
    case SRJ_INT64: case SRJ_UINT64: case SRJ_FLOAT64: case SRJ_TIMESTAMP_SECONDS: case SRJ_TIMESTAMP_MILLISECONDS:
    case SRJ_TIMESTAMP_MICROSECONDS: case SRJ_TIMESTAMP_NANOSECONDS: case SRJ_DURATION_SECONDS:
    case SRJ_DURATION_MILLISECONDS: case SRJ_DURATION_MICROSECONDS: case SRJ_DURATION_NANOSECONDS:
    case SRJ_DECIMAL64: return 8;
    case SRJ_DECIMAL128: return 16;
    default: return 0;
  }
}

// compute_column_information, RC:1332-1371
static int compute_layout(const int32_t* types, int32_t n, srj_layout* out, std::vector<int32_t>* starts,
                          std::vector<int32_t>* sizes)
{
  if (n < 0 || (n > 0 && !types)) { set_error("layout: bad schema"); return SRJ_EINVAL; }
  int64_t off = 0;
  int nstr    = 0;
  if (starts) starts->clear();
  if (sizes) sizes->clear();
  for (int32_t i = 0; i < n; ++i) {
    const bool compound = types[i] == SRJ_STRING;
    const int sz        = compound ? 8 : size_of_type(types[i]);
    if (sz == 0) {
      set_error("column %d: type id %d is not supported by the row format (only fixed-width and STRING, RowConversion.java:131)", i, types[i]);
      return SRJ_EUNSUPPORTED;
    }
    const int al = compound ? 4 : sz;
    off          = (off + al - 1) / al * al;
    if (starts) starts->push_back(static_cast<int32_t>(off));
    if (sizes) sizes->push_back(sz);
    off += sz;
    nstr += compound;
    if (off > INT32_MAX - 8) { set_error("layout: row too large"); return SRJ_EOVERFLOW; }
  }
  out->num_columns        = n;
  out->num_string_columns = nstr;
  out->validity_offset    = static_cast<int32_t>(off);
  off += (n + 7) / 8;
  out->size_per_row   = static_cast<int32_t>(off);
  out->fixed_row_size = static_cast<int32_t>((off + 7) / 8 * 8);
  out->reserved       = 0;
  return SRJ_OK;
}

// RAII lease of one TableRing slot (see plan.hpp).  upload() copies `host_bytes` of pointer tables to the
// device buffer; the device buffer may be larger (`total_bytes`) to carry device-only scratch behind them.
struct TableLease {
  const srj_plan* plan;
  cudaStream_t stream;
  TableSlot* slot = nullptr;
  TableLease(const srj_plan* p, cudaStream_t s) : plan(p), stream(s) {}
  int acquire(size_t total_bytes)
  {
    TableRing& r = plan->ring;
    {
      std::lock_guard<std::mutex> lk(r.mu);
      slot = &r.slots[r.next++ % TableRing::kSlots];
    }
    slot->busy.lock();  // > kSlots concurrent callers: the 9th waits for the 1st call to return
    if (slot->used) SRJ_CUDA_TRY(cudaEventSynchronize(slot->ev));  // previous user of this slot has drained
    if (!slot->ev) SRJ_CUDA_TRY(cudaEventCreateWithFlags(&slot->ev, cudaEventDisableTiming));
    if (slot->cap < total_bytes) {
      const size_t cap = std::max<size_t>(total_bytes * 2, 16384);
      if (slot->d_buf) cudaFree(slot->d_buf);
      if (slot->h_pinned) cudaFreeHost(slot->h_pinned);
      slot->d_buf = slot->h_pinned = nullptr;
      slot->cap = 0;
      SRJ_CUDA_TRY(cudaMalloc(&slot->d_buf, cap));
      SRJ_CUDA_TRY(cudaMallocHost(&slot->h_pinned, cap));
      slot->cap = cap;
    }
    return SRJ_OK;
  }
  void* host() const { return slot->h_pinned; }
  void* dev() const { return slot->d_buf; }
  int upload(size_t host_bytes)
  {
    SRJ_CUDA_TRY(cudaMemcpyAsync(slot->d_buf, slot->h_pinned, host_bytes, cudaMemcpyHostToDevice, stream));
    return SRJ_OK;
  }
  ~TableLease()
  {
    if (!slot) return;
    if (slot->ev) {
      cudaEventRecord(slot->ev, stream);
      slot->used = true;
    }
    slot->busy.unlock();
  }
};

// Phase 1 of a wide variable-width table runs from_rows_wide_kernel.
static bool use_wide_from_rows(const srj_plan* plan, const int32_t* row_offsets)
{
  return plan->wide.enabled && row_offsets != nullptr;
}

static int check_cols(const srj_plan* plan, const srj_column* cols, int64_t num_rows, const char* who)
{
  if (!plan || (plan->num_columns > 0 && !cols)) { set_error("%s: null argument", who); return SRJ_EINVAL; }
  if (num_rows < 0) { set_error("%s: negative row count", who); return SRJ_EINVAL; }
  for (int c = 0; c < plan->num_columns; ++c) {
    if (cols[c].type_id != plan->type_ids[c]) { set_error("%s: column %d type %d does not match the plan (%d)", who, c, cols[c].type_id, plan->type_ids[c]); return SRJ_EINVAL; }
    if (cols[c].size != num_rows) { set_error("%s: column %d has %lld rows, expected %lld", who, c, (long long)cols[c].size, (long long)num_rows); return SRJ_EINVAL; }
  }
  return SRJ_OK;
}

}  // namespace srj

using namespace srj;

extern "C" {

const char* srj_version(void) { return "srj_b200 0.1.0 (sm_90a)"; }
const char* srj_last_error(void) { return g_err; }
const char* srj_status_string(int s)
{
  switch (s) {
    case SRJ_OK: return "SRJ_OK";
    case SRJ_EINVAL: return "SRJ_EINVAL";
    case SRJ_EUNSUPPORTED: return "SRJ_EUNSUPPORTED";
    case SRJ_EOVERFLOW: return "SRJ_EOVERFLOW";
    case SRJ_ECUDA: return "SRJ_ECUDA";
    case SRJ_ENOMEM: return "SRJ_ENOMEM";
    default: return "SRJ_E?";
  }
}

int srj_compute_layout(const int32_t* type_ids, int32_t num_columns, srj_layout* out, int32_t* col_starts,
                       int32_t* col_sizes)
{
  if (!out) { set_error("layout: out is null"); return SRJ_EINVAL; }
  std::vector<int32_t> st, sz;
  const int rc = compute_layout(type_ids, num_columns, out, &st, &sz);
  if (rc != SRJ_OK) return rc;
  if (col_starts) std::copy(st.begin(), st.end(), col_starts);
  if (col_sizes) std::copy(sz.begin(), sz.end(), col_sizes);
  return SRJ_OK;
}

int srj_plan_create(const int32_t* type_ids, const int32_t* scales, int32_t num_columns, srj_plan** out)
{
  SRJ_API_RANGE();
  if (!out) { set_error("plan_create: out is null"); return SRJ_EINVAL; }
  *out = nullptr;
  srj_layout lay{};
  std::vector<int32_t> st, sz;
  int rc = compute_layout(type_ids, num_columns, &lay, &st, &sz);
  if (rc != SRJ_OK) return rc;
  auto* p               = new srj_plan();
  p->num_columns        = num_columns;
  p->num_string_columns = lay.num_string_columns;
  p->validity_offset    = lay.validity_offset;
  p->size_per_row       = lay.size_per_row;
  p->fixed_row_size     = lay.fixed_row_size;
  p->type_ids.assign(type_ids, type_ids + num_columns);
  p->scales.assign(num_columns, 0);
  if (scales) p->scales.assign(scales, scales + num_columns);
  p->col_start = st;
  p->col_size  = sz;
  std::vector<int32_t> string_start;
  for (int c = 0; c < num_columns; ++c)
    if (type_ids[c] == SRJ_STRING) {
      p->string_columns.push_back(c);
      string_start.push_back(st[c]);
    }
  // schedules: entries grouped by width class
  for (int k = 0; k < kNumClasses; ++k) {
    p->fr_class_begin[k] = static_cast<int32_t>(p->fr_entries.size());
    p->tr_class_begin[k] = static_cast<int32_t>(p->tr_entries.size());
    for (int c = 0; c < num_columns; ++c) {
      if (type_ids[c] == SRJ_STRING) {
        if (k == 2) p->fr_entries.push_back(Entry{st[c] + 4, c});  // the length word, RC:2163-2172
      } else if (class_of_size(sz[c]) == k) {
        p->fr_entries.push_back(Entry{st[c], c});
        p->tr_entries.push_back(Entry{st[c], c});
      }
    }
  }
  p->fr_class_begin[kNumClasses] = static_cast<int32_t>(p->fr_entries.size());
  p->tr_class_begin[kNumClasses] = static_cast<int32_t>(p->tr_entries.size());

  // from_rows tiling (shared memory budget 227 KB/CTA on sm_90)
  Tiling& tl = p->tiling;
  const int S = p->fixed_row_size;
  // Narrow rows (512 rows fit 64 KB): three 64 KB stages.  Wider rows: two 100 KB stages -- taller tiles mean longer
  // contiguous pieces per column and per CTA, which is what the DRAM likes once the part is warm.
  if (S <= 128) { tl.num_stages = 3; tl.stage_bytes = 64 * 1024; }
  else          { tl.num_stages = 2; tl.stage_bytes = 100 * 1024; }
  int fitrows = tl.stage_bytes / S;
  int R       = fitrows / 32 * 32;
  if (R > 512) R = 512;
  if (R >= 128) R = R / 128 * 128;  // 4 row groups per unit => predicate-free fast path
  if (R < 32) R = fitrows >= 16 ? 16 : 8;
  tl.tile_rows     = R;
  tl.rows_per_item = R >= 32 ? 32 : R;
  // The per-schema shared-memory tables (entry starts, column and mask pointers, null counters) come on top of the
  // stages: for very wide schemas shrink the stages until the kernel's request fits the 227 KB limit.
  {
    const int nent_fr = static_cast<int>(p->fr_entries.size());
    while (from_rows_smem_bytes(tl, nent_fr, num_columns, lay.num_string_columns) > 232448 && tl.stage_bytes > 8 * 1024) {
      tl.stage_bytes   = (tl.stage_bytes * 3 / 4) & ~127;
      int fit          = tl.stage_bytes / S;
      int r2           = fit / 32 * 32;
      if (r2 > 512) r2 = 512;
      if (r2 >= 128) r2 = r2 / 128 * 128;
      if (r2 < 32) r2 = fit >= 16 ? 16 : 8;
      tl.tile_rows     = r2;
      tl.rows_per_item = r2 >= 32 ? 32 : r2;
    }
    if (from_rows_smem_bytes(tl, nent_fr, num_columns, lay.num_string_columns) > 232448) {
      delete p;
      set_error("plan_create: schema too wide for the kernels' shared-memory tables (%d columns)", num_columns);
      return SRJ_EUNSUPPORTED;
    }
  }

  plan_wide(p);  // slabs of a wide variable-width table (from_rows_wide.cu); p->wide.enabled says whether it applies

  // device mirror
  {
    const cudaError_t e0 = cudaGetDevice(&p->device);
    if (e0 != cudaSuccess) { delete p; return cuda_fail(e0, "cudaGetDevice"); }
  }
  const size_t b_fr = p->fr_entries.size() * sizeof(Entry);
  const size_t b_tr = p->tr_entries.size() * sizeof(Entry);
  const size_t b_cs = static_cast<size_t>(num_columns) * 4;
  const size_t b_sc = p->string_columns.size() * 4;
  std::vector<int32_t> tr_chunk(p->tr_entries.size());
  {
    // staging layout of to_rows2: widest class first so that every piece stays 16-byte aligned
    int32_t acc = 0;
    for (int k = kNumClasses - 1; k >= 0; --k)
      for (int e = p->tr_class_begin[k]; e < p->tr_class_begin[k + 1]; ++e) { tr_chunk[e] = acc; acc += 1 << k; }
  }
  const size_t b_tc = tr_chunk.size() * 4;
  const size_t b_we = p->wide.enabled ? p->wide.entries.size() * sizeof(WideEntry) : 0;
  const size_t b_ws = p->wide.enabled ? p->wide.slabs.size() * sizeof(WideSlab) : 0;
  const size_t tot  = b_fr + b_tr + b_cs + 2 * b_sc + b_tc + b_we + b_ws + 96;
  std::vector<uint8_t> blob(tot, 0);
  size_t o = 0;
  auto put = [&](const void* src, size_t n) { size_t at = o; if (n) memcpy(blob.data() + o, src, n); o += (n + 7) & ~size_t{7}; return at; };
  const size_t o_fr = put(p->fr_entries.data(), b_fr);
  const size_t o_tr = put(p->tr_entries.data(), b_tr);
  const size_t o_cs = put(st.data(), b_cs);
  const size_t o_sc = put(p->string_columns.data(), b_sc);
  const size_t o_ss = put(string_start.data(), b_sc);
  const size_t o_tc = put(tr_chunk.data(), b_tc);
  const size_t o_we = put(p->wide.entries.data(), b_we);
  const size_t o_ws = put(p->wide.slabs.data(), b_ws);
  cudaError_t e = cudaMalloc(&p->d_blob, tot);
  if (e != cudaSuccess) { delete p; return cuda_fail(e, "cudaMalloc(plan)"); }
  e = cudaMemcpy(p->d_blob, blob.data(), tot, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { cudaFree(p->d_blob); delete p; return cuda_fail(e, "cudaMemcpy(plan)"); }
  auto* base        = static_cast<uint8_t*>(p->d_blob);
  p->d_fr_entries   = reinterpret_cast<const Entry*>(base + o_fr);
  p->d_tr_entries   = reinterpret_cast<const Entry*>(base + o_tr);
  p->d_col_start    = reinterpret_cast<const int32_t*>(base + o_cs);
  p->d_string_cols  = reinterpret_cast<const int32_t*>(base + o_sc);
  p->d_string_start = reinterpret_cast<const int32_t*>(base + o_ss);
  p->d_tr_chunk_off = reinterpret_cast<const int32_t*>(base + o_tc);
  p->wide.d_entries = reinterpret_cast<const WideEntry*>(base + o_we);
  p->wide.d_slabs   = reinterpret_cast<const WideSlab*>(base + o_ws);
  *out              = p;
  return SRJ_OK;
}

void srj_plan_destroy(srj_plan* plan)
{
  if (!plan) return;
  if (plan->d_blob) cudaFree(plan->d_blob);
  for (auto& ar : plan->host_pool.a) {
    for (auto& s : ar.st) if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    for (auto& d : ar.d_buf) if (d) cudaFree(d);
    if (ar.h_pin) cudaFreeHost(ar.h_pin);
  }
  for (auto& sl : plan->ring.slots) {
    if (sl.used && sl.ev) cudaEventSynchronize(sl.ev);
    if (sl.d_buf) cudaFree(sl.d_buf);
    if (sl.h_pinned) cudaFreeHost(sl.h_pinned);
    if (sl.ev) cudaEventDestroy(sl.ev);
  }
  delete plan;
}

int srj_plan_layout(const srj_plan* plan, srj_layout* out)
{
  if (!plan || !out) { set_error("plan_layout: null argument"); return SRJ_EINVAL; }
  out->num_columns        = plan->num_columns;
  out->num_string_columns = plan->num_string_columns;
  out->validity_offset    = plan->validity_offset;
  out->size_per_row       = plan->size_per_row;
  out->fixed_row_size     = plan->fixed_row_size;
  out->reserved           = 0;
  return SRJ_OK;
}

// ---------------------------------------------------------------------------------------------------
// convert_to_rows
// ---------------------------------------------------------------------------------------------------
static const int kRsChunkHost = 4096;  // must match kRsChunk in to_rows.cu

int64_t srj_to_rows_workspace_bytes(const srj_plan* plan, int64_t num_rows)
{
  if (!plan || plan->num_string_columns == 0 || num_rows <= 0) return 0;
  const int64_t nchunks = (num_rows + kRsChunkHost - 1) / kRsChunkHost;
  return (num_rows + nchunks) * 8;
}

int srj_to_rows_plan_batches(const srj_plan* plan, const srj_column* cols, int64_t num_rows, void* workspace,
                             srj_row_batch* batches, int32_t max_batches, int32_t* num_batches, void* stream_)
{
  SRJ_API_RANGE();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc              = check_cols(plan, cols, num_rows, "to_rows_plan_batches");
  if (rc != SRJ_OK) return rc;
  if (!batches || !num_batches || max_batches < 1) { set_error("to_rows_plan_batches: bad batch array"); return SRJ_EINVAL; }
  *num_batches = 0;
  if (num_rows == 0) return SRJ_OK;
  const uint64_t MAXB = INT32_MAX;  // MAX_BATCH_SIZE, RC:65
  if (plan->num_string_columns == 0) {
    // constant row size: build_batches (RC:1466-1557) in closed form.
    const uint64_t S = plan->fixed_row_size;
    int64_t last     = 0;
    while (last < num_rows) {
      // lower_bound over (i - last) * S >= MAXB  (cum[i] - cum[last] with cum inclusive)
      const int64_t k      = static_cast<int64_t>((MAXB + S - 1) / S);  // first i - last reaching MAXB
      const bool to_end    = last + k >= num_rows;
      int64_t rows         = to_end ? num_rows - last : k / 32 * 32;
      while (static_cast<uint64_t>(rows) * S > MAXB) rows -= (rows % 32) ? (rows % 32) : 32;  // overflow guard
      if (rows <= 0) { set_error("to_rows: a single row exceeds 2 GiB"); return SRJ_EOVERFLOW; }
      if (*num_batches >= max_batches) { set_error("to_rows: more than %d batches", max_batches); return SRJ_EINVAL; }
      batches[*num_batches] = srj_row_batch{last, rows, static_cast<int64_t>(static_cast<uint64_t>(rows) * S)};
      ++*num_batches;
      last += rows;
    }
    return SRJ_OK;
  }
  if (!workspace) { set_error("to_rows_plan_batches: workspace is null"); return SRJ_EINVAL; }
  // device: per-row sizes + inclusive scan
  const int nstr = plan->num_string_columns;
  std::vector<const int32_t*> h_off(nstr);
  for (int s = 0; s < nstr; ++s) {
    h_off[s] = cols[plan->string_columns[s]].offsets;
    if (!h_off[s]) { set_error("to_rows: STRING column %d has no offsets", plan->string_columns[s]); return SRJ_EINVAL; }
  }
  // pointer table of the STRING offsets + room for the batch list the device computes
  const int cap          = std::min<int>(max_batches, 4096);
  const size_t tab_bytes = (sizeof(void*) * nstr + 15) & ~size_t{15};
  const size_t out_bytes = sizeof(int64_t) * (1 + 3 * static_cast<size_t>(cap));
  TableLease sc(plan, stream);
  rc = sc.acquire(tab_bytes + out_bytes);
  if (rc != SRJ_OK) return rc;
  memcpy(sc.host(), h_off.data(), sizeof(void*) * nstr);
  rc = sc.upload(sizeof(void*) * nstr);
  if (rc != SRJ_OK) return rc;
  uint64_t* cum = static_cast<uint64_t*>(workspace);
  rc            = launch_row_sizes(plan, static_cast<const int32_t* const*>(sc.dev()), num_rows, cum, stream);
  if (rc != SRJ_OK) return rc;
  // build_batches on the device, one read-back (the sync of RC:1534-1544, once instead of once per batch)
  int64_t* d_out = reinterpret_cast<int64_t*>(static_cast<uint8_t*>(sc.dev()) + tab_bytes);
  int64_t* h_out = reinterpret_cast<int64_t*>(static_cast<uint8_t*>(sc.host()) + tab_bytes);
  rc             = launch_batch_cut(cum, num_rows, cap, d_out, stream);
  if (rc != SRJ_OK) return rc;
  const size_t first = sizeof(int64_t) * (1 + 3 * static_cast<size_t>(std::min(cap, 8)));   // nearly always one batch
  SRJ_CUDA_TRY(cudaMemcpyAsync(h_out, d_out, first, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  if (h_out[0] > 8) {
    SRJ_CUDA_TRY(cudaMemcpyAsync(h_out, d_out, sizeof(int64_t) * (1 + 3 * static_cast<size_t>(h_out[0])), cudaMemcpyDeviceToHost, stream));
    SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  if (h_out[0] == -1) { set_error("to_rows: a single row exceeds 2 GiB"); return SRJ_EOVERFLOW; }
  if (h_out[0] < 0) { set_error("to_rows: more than %d batches", cap); return SRJ_EINVAL; }
  *num_batches = static_cast<int32_t>(h_out[0]);
  for (int b = 0; b < *num_batches; ++b) batches[b] = srj_row_batch{h_out[1 + 3 * b], h_out[2 + 3 * b], h_out[3 + 3 * b]};
  return SRJ_OK;
}

int srj_convert_to_rows(const srj_plan* plan, const srj_column* cols, int64_t num_rows, const void* workspace,
                        const srj_row_batch* batches, int32_t num_batches, int32_t* const* batch_offsets,
                        uint8_t* const* batch_data, void* stream_)
{
  SRJ_API_RANGE();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc              = check_cols(plan, cols, num_rows, "convert_to_rows");
  if (rc != SRJ_OK) return rc;
  if (num_batches == 0 || num_rows == 0) return SRJ_OK;
  if (!batches || !batch_offsets || !batch_data) { set_error("convert_to_rows: null batch arrays"); return SRJ_EINVAL; }
  const int nc = plan->num_columns, nstr = plan->num_string_columns;
  if (nstr > 0 && !workspace) { set_error("convert_to_rows: workspace is null"); return SRJ_EINVAL; }
  // pointer tables: [col_data nc][masks nc][str_offsets nstr][str_chars nstr]
  std::vector<const void*> tab(2 * static_cast<size_t>(nc) + 2 * static_cast<size_t>(nstr));
  for (int c = 0; c < nc; ++c) {
    if (plan->type_ids[c] != SRJ_STRING && !cols[c].data) { set_error("convert_to_rows: column %d has no data", c); return SRJ_EINVAL; }
    tab[c]      = cols[c].data;
    tab[nc + c] = cols[c].null_mask;
  }
  for (int s = 0; s < nstr; ++s) {
    const srj_column& c = cols[plan->string_columns[s]];
    if (!c.offsets) { set_error("convert_to_rows: STRING column %d has no offsets", plan->string_columns[s]); return SRJ_EINVAL; }
    tab[2 * nc + s]        = c.offsets;
    tab[2 * nc + nstr + s] = c.data;
  }
  TableLease sc(plan, stream);
  rc = sc.acquire(tab.size() * sizeof(void*));
  if (rc != SRJ_OK) return rc;
  memcpy(sc.host(), tab.data(), tab.size() * sizeof(void*));
  rc = sc.upload(tab.size() * sizeof(void*));
  if (rc != SRJ_OK) return rc;
  auto** d = static_cast<const void**>(sc.dev());
  for (int b = 0; b < num_batches; ++b) {
    if (!batch_offsets[b] || (!batch_data[b] && batches[b].num_bytes > 0)) { set_error("convert_to_rows: batch %d buffers are null", b); return SRJ_EINVAL; }
    rc = launch_to_rows(plan, d, reinterpret_cast<const uint32_t* const*>(d + nc),
                        reinterpret_cast<const int32_t* const*>(d + 2 * nc),
                        reinterpret_cast<const uint8_t* const*>(d + 2 * nc + nstr), batches[b].row_start,
                        batches[b].row_count, nstr ? static_cast<const uint64_t*>(workspace) : nullptr,
                        batch_offsets[b], batch_data[b], batches[b].num_bytes, stream, tab.data(),
                        // the scan partials behind the cumulative sizes are dead after plan_batches: 4 bytes of
                        // them carry the "fast kernel gave up" flag
                        nstr ? reinterpret_cast<int32_t*>(const_cast<uint64_t*>(static_cast<const uint64_t*>(workspace)) + num_rows) : nullptr);
    if (rc != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

// ---------------------------------------------------------------------------------------------------
// convert_from_rows
// ---------------------------------------------------------------------------------------------------
int64_t srj_from_rows_workspace_bytes(const srj_plan* plan, int64_t num_rows)
{
  if (!plan || num_rows <= 0 || !plan->wide.enabled) return 0;
  return wide_workspace_bytes(plan, num_rows);
}

int srj_convert_from_rows_fixed(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets,
                                int64_t rows_bytes, int64_t num_rows, const srj_column* cols, int64_t* d_null_counts,
                                int64_t* d_char_totals, const srj_fused_hash* hash, void* workspace, void* stream_)
{
  SRJ_API_RANGE();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc              = check_cols(plan, cols, num_rows, "convert_from_rows");
  if (rc != SRJ_OK) return rc;
  const int nc = plan->num_columns, nstr = plan->num_string_columns;
  if (nstr > 0 && !row_offsets && num_rows > 0) { set_error("convert_from_rows: a schema with STRING columns needs the LIST offsets"); return SRJ_EINVAL; }
  if (nstr == 0) row_offsets = nullptr;  // fixed-width schemas ignore the offsets like the reference (RC:2317)
  // RC:2197: size_per_row * num_rows <= child.size()
  if (static_cast<int64_t>(plan->fixed_row_size) * num_rows > rows_bytes) {
    set_error("convert_from_rows: The layout of the data appears to be off (%lld rows x %d bytes > %lld)", (long long)num_rows, plan->fixed_row_size, (long long)rows_bytes);
    return SRJ_EINVAL;
  }
  if (num_rows > 0 && !rows) { set_error("convert_from_rows: rows is null"); return SRJ_EINVAL; }
  if (hash && hash->kind != SRJ_HASH_NONE) {
    if (hash->num_keys < 0 || hash->num_keys > 16 || !hash->out) { set_error("fused hash: bad key list / output"); return SRJ_EINVAL; }
    for (int k = 0; k < hash->num_keys; ++k) {
      const int c = hash->key_columns[k];
      if (c < 0 || c >= nc) { set_error("fused hash: key column %d out of range", c); return SRJ_EINVAL; }
      if (plan->type_ids[c] == SRJ_STRING) { set_error("fused hash: STRING keys are not supported in the fused path"); return SRJ_EUNSUPPORTED; }
      if (hash->kind == SRJ_HASH_HIVE && !hash::hive_supported(plan->type_ids[c])) { set_error("fused hive hash: unsupported key type %d", plan->type_ids[c]); return SRJ_EUNSUPPORTED; }
    }
  }
  for (int c = 0; c < nc; ++c) {
    if (plan->type_ids[c] == SRJ_STRING) {
      if (!cols[c].offsets) { set_error("convert_from_rows: STRING column %d has no offsets buffer", c); return SRJ_EINVAL; }
    } else if (!cols[c].data && num_rows > 0) {
      set_error("convert_from_rows: column %d has no data buffer", c); return SRJ_EINVAL;
    }
    if (!cols[c].null_mask && num_rows > 0) { set_error("convert_from_rows: column %d has no null mask buffer (always allocated, RC:2220)", c); return SRJ_EINVAL; }
  }
  // The hash of a "fused" call is the streaming hash kernel over the key columns just written (12 more bytes per row
  // for two integer keys, but the conversion kernel keeps its issue slots for the transpose and the hash its own
  // kernel shape), so wide variable-width tables keep their fast path too.
  auto hash_after = [&]() -> int {
    if (!hash || hash->kind == SRJ_HASH_NONE || num_rows == 0) return SRJ_OK;
    srj_column keys[16];
    for (int k = 0; k < hash->num_keys; ++k) keys[k] = cols[hash->key_columns[k]];
    return launch_hash(hash->kind, keys, hash->num_keys, num_rows, hash->seed, hash->out, stream);
  };
  if (use_wide_from_rows(plan, row_offsets)) {
    // wide variable-width table: per-row slabs; the pointer tables travel as kernel parameters and the kernels publish
    // null counts / totals / status themselves: no memset, no staging copy, no hidden allocation
    if (num_rows > 0 && !workspace) { set_error("convert_from_rows: this schema needs a workspace (srj_from_rows_workspace_bytes)"); return SRJ_EINVAL; }
    rc = launch_from_rows_wide(plan, rows, row_offsets, rows_bytes, num_rows, cols, d_null_counts, d_char_totals, workspace, stream);
    return rc != SRJ_OK ? rc : hash_after();
  }
  if (d_null_counts) SRJ_CUDA_TRY(cudaMemsetAsync(d_null_counts, 0, sizeof(int64_t) * nc, stream));
  if (d_char_totals) SRJ_CUDA_TRY(cudaMemsetAsync(d_char_totals, 0, sizeof(int64_t) * (nc + 1), stream));
  const size_t nent = plan->fr_entries.size();
  // pointer tables: [ent_dst nent][masks nc][str_offsets nstr] + scan partials
  std::vector<void*> tab(nent + nc + nstr);
  for (size_t e = 0; e < nent; ++e) {
    const int c = plan->fr_entries[e].column;
    tab[e]      = plan->type_ids[c] == SRJ_STRING ? static_cast<void*>(reinterpret_cast<uint8_t*>(cols[c].offsets) + 4)  // lengths land at offsets[1..n]
                                                  : cols[c].data;
  }
  for (int c = 0; c < nc; ++c) tab[nent + c] = cols[c].null_mask;
  for (int s = 0; s < nstr; ++s) tab[nent + nc + s] = cols[plan->string_columns[s]].offsets;
  const size_t tab_bytes  = (tab.size() * sizeof(void*) + 15) & ~size_t{15};
  const size_t part_bytes = static_cast<size_t>(string_scan_partials_bytes(nstr, num_rows));
  TableLease sc(plan, stream);
  rc = sc.acquire(tab_bytes + part_bytes + 16);
  if (rc != SRJ_OK) return rc;
  memcpy(sc.host(), tab.data(), tab.size() * sizeof(void*));
  rc = sc.upload(tab.size() * sizeof(void*));
  if (rc != SRJ_OK) return rc;
  auto** d = static_cast<void**>(sc.dev());
  rc = launch_from_rows(plan, rows, row_offsets, rows_bytes, num_rows, d, reinterpret_cast<uint32_t* const*>(d + nent),
                        d_null_counts, d_char_totals ? d_char_totals + nc : nullptr, stream);
  if (rc != SRJ_OK) return rc;
  if (nstr > 0) {
    uint8_t* tail = static_cast<uint8_t*>(sc.dev()) + tab_bytes;
    rc = launch_string_offsets_scan(reinterpret_cast<int32_t* const*>(d + nent + nc), plan->d_string_cols, nstr, num_rows,
                                    d_char_totals, d_char_totals ? d_char_totals + nc : nullptr, tail, stream);
    if (rc != SRJ_OK) return rc;
  }
  return hash_after();
}

int srj_convert_from_rows_strings(const srj_plan* plan, const uint8_t* rows, const int32_t* row_offsets,
                                  int64_t rows_bytes, int64_t num_rows, const srj_column* cols,
                                  const int64_t* d_char_totals, const void* workspace, void* stream_)
{
  SRJ_API_RANGE();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc              = check_cols(plan, cols, num_rows, "convert_from_rows_strings");
  if (rc != SRJ_OK) return rc;
  const int nstr = plan->num_string_columns;
  if (nstr == 0 || num_rows == 0) return SRJ_OK;
  if (!rows || !row_offsets) { set_error("convert_from_rows_strings: rows / offsets are null"); return SRJ_EINVAL; }
  for (int s = 0; s < nstr; ++s)
    if (!cols[plan->string_columns[s]].offsets) { set_error("convert_from_rows_strings: STRING column %d has no offsets", plan->string_columns[s]); return SRJ_EINVAL; }
  const int64_t* d_status = d_char_totals ? d_char_totals + plan->num_columns : nullptr;
  // wide tables: phase 1 (from_rows_wide.cu) left group-local offsets + the group bases in the workspace
  const uint32_t* d_bases = nullptr;
  if (plan->wide.enabled) {
    if (!workspace) { set_error("convert_from_rows_strings: this schema needs the workspace phase 1 filled"); return SRJ_EINVAL; }
    d_bases = wide_workspace_bases(plan, num_rows, workspace);
  }
  if (strings_fast_path(plan, d_status))   // pointer tables travel as kernel parameters
    return launch_strings_from_rows(plan, rows, row_offsets, rows_bytes, num_rows, cols, nullptr, d_status, d_bases, stream);
  std::vector<void*> tab(2 * static_cast<size_t>(nstr));
  for (int s = 0; s < nstr; ++s) {
    const srj_column& c = cols[plan->string_columns[s]];
    tab[s]        = c.offsets;
    tab[nstr + s] = c.data;  // may be NULL only when the column has no chars at all
  }
  TableLease sc(plan, stream);
  rc = sc.acquire(tab.size() * sizeof(void*));
  if (rc != SRJ_OK) return rc;
  memcpy(sc.host(), tab.data(), tab.size() * sizeof(void*));
  rc = sc.upload(tab.size() * sizeof(void*));
  if (rc != SRJ_OK) return rc;
  return launch_strings_from_rows(plan, rows, row_offsets, rows_bytes, num_rows, cols, static_cast<void* const*>(sc.dev()),
                                  d_status, d_bases, stream);
}

// ---------------------------------------------------------------------------------------------------
// hashes
// ---------------------------------------------------------------------------------------------------
int srj_get_max_stack_depth(void) { return SRJ_MAX_STACK_DEPTH; }

// Tables with LIST / STRUCT keys: the column trees are uploaded through a process-wide staging ring (there is no plan
// on the hash entry points) and hashed by hash_nested.cu.
static int hash_any(int kind, const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t seed, void* out, cudaStream_t stream)
{
  if (!hash_has_nested(cols, num_columns)) return launch_hash(kind, cols, num_columns, num_rows, seed, out, stream);
  if (num_columns == 0 || num_rows == 0) return SRJ_OK;
  static srj_plan staging{};              // only its pointer-table ring is used
  constexpr size_t kBytes = 256 * 1024;   // ~5000 tree nodes
  TableLease sc(&staging, stream);
  int rc = sc.acquire(kBytes);
  if (rc != SRJ_OK) return rc;
  return launch_hash_nested(kind, cols, num_columns, num_rows, seed, out, sc.dev(), sc.host(), kBytes, stream);
}

int srj_xxhash64(const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t seed, int64_t* out, void* stream)
{
  SRJ_API_RANGE();
  if (num_columns < 0 || num_rows < 0 || (num_columns > 0 && !cols) || (num_rows > 0 && !out)) { set_error("xxhash64: bad argument"); return SRJ_EINVAL; }
  return hash_any(SRJ_HASH_XXHASH64, cols, num_columns, num_rows, seed, out, static_cast<cudaStream_t>(stream));
}

int srj_murmur_hash3_32(const srj_column* cols, int32_t num_columns, int64_t num_rows, uint32_t seed, int32_t* out,
                        void* stream)
{
  SRJ_API_RANGE();
  if (num_columns < 0 || num_rows < 0 || (num_columns > 0 && !cols) || (num_rows > 0 && !out)) { set_error("murmur_hash3_32: bad argument"); return SRJ_EINVAL; }
  return hash_any(SRJ_HASH_MURMUR3_32, cols, num_columns, num_rows, seed, out, static_cast<cudaStream_t>(stream));
}

int srj_hive_hash(const srj_column* cols, int32_t num_columns, int64_t num_rows, int32_t* out, void* stream)
{
  SRJ_API_RANGE();
  if (num_columns < 0 || num_rows < 0 || (num_columns > 0 && !cols) || (num_rows > 0 && !out)) { set_error("hive_hash: bad argument"); return SRJ_EINVAL; }
  return hash_any(SRJ_HASH_HIVE, cols, num_columns, num_rows, 0, out, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// SHA-2 with nulls preserved (sha2.cu) and the host CRC32
// ---------------------------------------------------------------------------------------------------
int64_t srj_sha2_workspace_bytes(int64_t num_rows) { return sha2_workspace_bytes(std::max<int64_t>(0, num_rows)); }

static int sha2_check(const char* what, int32_t digest_bits, const srj_column* in)
{
  if (sha2_hex_width(digest_bits) == 0) { set_error("%s: digest_bits %d is not one of 224, 256, 384, 512", what, digest_bits); return SRJ_EINVAL; }
  if (!in) { set_error("%s: input is null", what); return SRJ_EINVAL; }
  if (in->type_id != SRJ_STRING) { set_error("%s: SHA-2 hashing requires a string column (type id %d)", what, in->type_id); return SRJ_EUNSUPPORTED; }
  if (in->size < 0 || in->size > INT32_MAX) { set_error("%s: %lld rows", what, static_cast<long long>(in->size)); return SRJ_EINVAL; }
  if (in->size > 0 && !in->offsets) { set_error("%s: the STRING column has no offsets", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

int srj_sha2_sizes(int32_t digest_bits, const srj_column* input, int32_t* d_out_offsets, int64_t* total_chars, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = sha2_check("sha2_sizes", digest_bits, input);
  if (rc != SRJ_OK) return rc;
  if (!d_out_offsets || !total_chars) { set_error("sha2_sizes: bad argument"); return SRJ_EINVAL; }
  if (input->null_mask && input->size > 0 && !workspace) { set_error("sha2_sizes: an input with a null mask needs the workspace (srj_sha2_workspace_bytes)"); return SRJ_EINVAL; }
  rc = launch_sha2_sizes(digest_bits, *input, d_out_offsets, total_chars, workspace, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EOVERFLOW)
    set_error("sha2_sizes: %lld chars of SHA-%d hex exceed one STRING column (INT32_MAX): hash fewer rows per call", static_cast<long long>(*total_chars), digest_bits);
  return rc;
}

int srj_sha2_hash(int32_t digest_bits, const srj_column* input, const srj_column* out, void* stream)
{
  SRJ_API_RANGE();
  int rc = sha2_check("sha2_hash", digest_bits, input);
  if (rc != SRJ_OK) return rc;
  if (!out || out->size != input->size || (input->size > 0 && !out->offsets)) { set_error("sha2_hash: the output needs the offsets of srj_sha2_sizes and the input's row count"); return SRJ_EINVAL; }
  if (input->null_mask && !out->null_mask && input->size > 0) { set_error("sha2_hash: the input has a null mask but the output has none"); return SRJ_EINVAL; }
  if (!input->null_mask && input->size > 0 && !out->data) { set_error("sha2_hash: the output has no chars buffer"); return SRJ_EINVAL; }
  if (reinterpret_cast<uintptr_t>(out->data) & 15) { set_error("sha2_hash: the output chars must be 16-byte aligned"); return SRJ_EINVAL; }
  return launch_sha2(digest_bits, *input, *out, static_cast<cudaStream_t>(stream));
}

// zlib's crc32 (reflected polynomial 0xEDB88320), slicing by 8: eight 256-entry tables, eight input bytes per step.
namespace {
struct Crc32Tables {
  uint32_t t[8][256];
  Crc32Tables()
  {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
      t[0][i] = c;
    }
    for (int s = 1; s < 8; ++s)
      for (int i = 0; i < 256; ++i) t[s][i] = (t[s - 1][i] >> 8) ^ t[0][t[s - 1][i] & 0xff];
  }
};
}  // namespace

int srj_host_crc32(uint32_t crc, const void* buf, int64_t len, uint32_t* out)
{
  SRJ_API_RANGE();
  if (!out || len < 0 || (!buf && len > 0)) { set_error("host_crc32: len must be >= 0, and the buffer may be NULL only when len is 0"); return SRJ_EINVAL; }
  static const Crc32Tables T;   // built once, thread-safe (function-local static)
  const auto* p = static_cast<const uint8_t*>(buf);
  uint32_t c    = ~crc;
  for (; len >= 8; len -= 8, p += 8) {   // little-endian host: the low word holds the first four bytes
    uint32_t lo, hi;
    memcpy(&lo, p, 4);
    memcpy(&hi, p + 4, 4);
    lo ^= c;
    c = T.t[7][lo & 0xff] ^ T.t[6][(lo >> 8) & 0xff] ^ T.t[5][(lo >> 16) & 0xff] ^ T.t[4][lo >> 24] ^ T.t[3][hi & 0xff] ^
        T.t[2][(hi >> 8) & 0xff] ^ T.t[1][(hi >> 16) & 0xff] ^ T.t[0][hi >> 24];
  }
  for (; len > 0; --len, ++p) c = T.t[0][(c ^ *p) & 0xff] ^ (c >> 8);
  *out = ~c;
  return SRJ_OK;
}

// ---------------------------------------------------------------------------------------------------
// Spark BloomFilter (bloom_filter.cu)
// ---------------------------------------------------------------------------------------------------
static int bloom_hdr_bytes(int32_t version) { return version == 2 ? 16 : 12; }   // bloom_filter.hpp:59-63

static int bloom_check_params(const char* what, int32_t version, int32_t num_hashes, int64_t num_longs)
{
  if (version != 1 && version != 2) { set_error("%s: Bloom filter version must be 1 or 2 (got %d)", what, version); return SRJ_EINVAL; }
  if (num_hashes <= 0) { set_error("%s: Bloom filters must have a positive hash count", what); return SRJ_EINVAL; }
  if (num_longs <= 0) { set_error("%s: Bloom filters must have a positive number of bits", what); return SRJ_EINVAL; }
  if (bloom_hdr_bytes(version) + 8 * num_longs > INT32_MAX) { set_error("%s: Bloom filter buffer size exceeds int32 range", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

// bloom_filter.cu:189-236 + the size checks of put / probe (bloom_filter.cu:340, 459): parse the serialized header of a
// filter of `bytes` bytes at device address `buf` (one read-back, one stream synchronisation)
static int bloom_read_header(const char* what, const uint8_t* buf, int64_t bytes, BloomHeader* h, cudaStream_t stream)
{
  if (bytes < 12 || !buf) { set_error("%s: Encountered truncated bloom filter", what); return SRJ_EINVAL; }
  if (reinterpret_cast<uintptr_t>(buf) & 3) { set_error("%s: the filter buffer must be 4-byte aligned", what); return SRJ_EINVAL; }
  uint32_t raw[4] = {0, 0, 0, 0};
  SRJ_CUDA_TRY(cudaMemcpyAsync(raw, buf, static_cast<size_t>(std::min<int64_t>(bytes, 16)), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  const auto be = [](uint32_t v) { return static_cast<int32_t>(__builtin_bswap32(v)); };
  h->version    = be(raw[0]);
  if (h->version != 1 && h->version != 2) { set_error("%s: Unexpected bloom filter version %d", what, h->version); return SRJ_EINVAL; }
  const int hdr = bloom_hdr_bytes(h->version);
  if (bytes < hdr) { set_error("%s: Encountered truncated bloom filter header", what); return SRJ_EINVAL; }
  h->num_hashes = be(raw[1]);
  h->seed       = h->version == 2 ? be(raw[2]) : 0;
  h->num_longs  = h->version == 2 ? be(raw[3]) : be(raw[2]);
  if (h->num_longs <= 0) { set_error("%s: Invalid empty bloom filter size", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

static int bloom_check_input(const char* what, const srj_column* in)
{
  if (!in) { set_error("%s: input is null", what); return SRJ_EINVAL; }
  if (in->type_id != SRJ_INT64) { set_error("%s: bloom filters take one INT64 column (type id %d)", what, in->type_id); return SRJ_EUNSUPPORTED; }
  if (in->size < 0 || (in->size > 0 && !in->data)) { set_error("%s: bad input column", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

// put / probe: the buffer must be exactly one filter, and V1 indexes with 31-bit positions (bloom_filter.cu:340-359, 459-471)
static int bloom_check_filter(const char* what, const BloomHeader& h, int64_t bytes)
{
  if (bytes != bloom_hdr_bytes(h.version) + 8 * static_cast<int64_t>(h.num_longs)) {
    set_error("%s: Encountered invalid/mismatched bloom filter buffer data", what);
    return SRJ_EINVAL;
  }
  if (h.version == 1 && 64 * static_cast<int64_t>(h.num_longs) > INT32_MAX) { set_error("%s: V1 bloom filter bit count exceeds int32 range", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

int srj_bloom_filter_sizes(int32_t version, int32_t num_hashes, int64_t bits, int32_t* num_longs, int64_t* total_bytes)
{
  SRJ_API_RANGE();
  if (!num_longs || !total_bytes) { set_error("bloom_filter_sizes: bad argument"); return SRJ_EINVAL; }
  // BloomFilterJni.cpp:40-47: Spark's BitArray holds at most INT32_MAX longs
  if (bits > static_cast<int64_t>(INT32_MAX) * 64) {
    set_error("bloom_filter_sizes: bloom filter bit count must be positive and less than or equal to the maximum supported size");
    return SRJ_EINVAL;
  }
  const int64_t longs = bits > 0 ? (bits + 63) / 64 : 0;
  const int rc        = bloom_check_params("bloom_filter_sizes", version, num_hashes, longs);
  if (rc != SRJ_OK) return rc;
  *num_longs   = static_cast<int32_t>(longs);
  *total_bytes = bloom_hdr_bytes(version) + 8 * longs;
  return SRJ_OK;
}

int srj_bloom_filter_init(int32_t version, int32_t num_hashes, int32_t num_longs, int32_t seed, uint8_t* filter, void* stream)
{
  SRJ_API_RANGE();
  const int rc = bloom_check_params("bloom_filter_init", version, num_hashes, num_longs);
  if (rc != SRJ_OK) return rc;
  if (!filter || (reinterpret_cast<uintptr_t>(filter) & 3)) { set_error("bloom_filter_init: the filter buffer must be a 4-byte aligned device pointer"); return SRJ_EINVAL; }
  return launch_bloom_init(BloomHeader{version, num_hashes, version == 2 ? seed : 0, num_longs}, filter, static_cast<cudaStream_t>(stream));
}

int srj_bloom_filter_put(uint8_t* filter, int64_t filter_bytes, const srj_column* input, void* stream)
{
  SRJ_API_RANGE();
  int rc = bloom_check_input("bloom_filter_put", input);
  if (rc != SRJ_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BloomHeader h{};
  if ((rc = bloom_read_header("bloom_filter_put", filter, filter_bytes, &h, st)) != SRJ_OK) return rc;
  if ((rc = bloom_check_filter("bloom_filter_put", h, filter_bytes)) != SRJ_OK) return rc;
  return launch_bloom_put(h, filter, *input, st);
}

int srj_bloom_filter_probe(const uint8_t* filter, int64_t filter_bytes, const srj_column* input, uint8_t* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  int rc = bloom_check_input("bloom_filter_probe", input);
  if (rc != SRJ_OK) return rc;
  if (input->size > 0 && !out) { set_error("bloom_filter_probe: the output is null"); return SRJ_EINVAL; }
  if (input->size > 0 && input->null_mask && !out_mask) { set_error("bloom_filter_probe: the input has a null mask but the output has none"); return SRJ_EINVAL; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BloomHeader h{};
  if ((rc = bloom_read_header("bloom_filter_probe", filter, filter_bytes, &h, st)) != SRJ_OK) return rc;
  if ((rc = bloom_check_filter("bloom_filter_probe", h, filter_bytes)) != SRJ_OK) return rc;
  return launch_bloom_probe(h, filter, *input, out, out_mask, st);
}

int64_t srj_bloom_filter_merge_workspace_bytes(void) { return 16; }

// bloom_filter.cu:374-449.  The stride of the filters is known from the sizes alone (filters_bytes / num_filters), and the
// header size follows from it (12 + 8 * num_longs is 4 mod 8, 16 + 8 * num_longs is 0 mod 8), so the header check and
// the OR are enqueued before the first header is read back; header and flag then come back with one synchronisation and
// the checks run in the reference's order.  On an error `out` holds garbage.
int srj_bloom_filter_merge(const uint8_t* filters, int64_t filters_bytes, int32_t num_filters, uint8_t* out, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "bloom_filter_merge";
  if (num_filters <= 0 || filters_bytes < 0 || (filters_bytes > 0 && !filters)) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (filters_bytes < 12) { set_error("%s: Encountered truncated bloom filter", what); return SRJ_EINVAL; }
  if (!workspace || !out) { set_error("%s: the output and the workspace are needed", what); return SRJ_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(filters) | reinterpret_cast<uintptr_t>(out)) & 3) { set_error("%s: the buffers must be 4-byte aligned", what); return SRJ_EINVAL; }
  cudaStream_t st       = static_cast<cudaStream_t>(stream);
  const int64_t stride  = filters_bytes / num_filters;
  const bool launched   = stride * num_filters == filters_bytes && stride >= 16 && stride % 4 == 0 && stride <= INT32_MAX;
  auto* d_flag          = static_cast<int32_t*>(workspace);
  if (launched) {
    const int rc = launch_bloom_merge(filters, stride, num_filters, stride % 8 == 4 ? 12 : 16, out, d_flag, st);
    if (rc != SRJ_OK) return rc;
  }
  int32_t flag    = 0;
  uint32_t raw[4] = {0, 0, 0, 0};
  SRJ_CUDA_TRY(cudaMemcpyAsync(raw, filters, static_cast<size_t>(std::min<int64_t>(filters_bytes, 16)), cudaMemcpyDeviceToHost, st));
  if (launched) SRJ_CUDA_TRY(cudaMemcpyAsync(&flag, d_flag, 4, cudaMemcpyDeviceToHost, st));
  SRJ_CUDA_TRY(cudaStreamSynchronize(st));
  const auto be = [](uint32_t v) { return static_cast<int32_t>(__builtin_bswap32(v)); };
  const int32_t version = be(raw[0]);
  if (version != 1 && version != 2) { set_error("%s: Unexpected bloom filter version %d", what, version); return SRJ_EINVAL; }
  const int hdr = bloom_hdr_bytes(version);
  if (filters_bytes < hdr) { set_error("%s: Encountered truncated bloom filter header", what); return SRJ_EINVAL; }
  const int64_t num_longs = version == 2 ? be(raw[3]) : be(raw[2]);
  if (num_longs <= 0) { set_error("%s: Invalid empty bloom filter size", what); return SRJ_EINVAL; }
  if (filters_bytes != (hdr + 8 * num_longs) * num_filters) { set_error("%s: Encountered invalid/mismatched bloom filter buffer data", what); return SRJ_EINVAL; }
  if (hdr + 8 * num_longs > INT32_MAX) { set_error("%s: Bloom filter buffer size exceeds int32 range", what); return SRJ_EINVAL; }
  if (!launched || flag) { set_error("%s: Mismatch of bloom filter parameters", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

// ---------------------------------------------------------------------------------------------------
// ZOrder: interleaveBits and hilbertIndex (zorder.cu)
// ---------------------------------------------------------------------------------------------------
// zorder.cu:141-159: at least one column, fixed-width, one type id, the output within INT32_MAX bytes (a logic_error in
// the reference, so SRJ_EINVAL rather than SRJ_EOVERFLOW).  *elem_bytes = W.
static int interleave_check(const char* what, const srj_column* cols, int32_t n, int64_t rows, int32_t* elem_bytes)
{
  if (n <= 0 || !cols) { set_error("%s: The input table must have at least one column.", what); return SRJ_EINVAL; }
  if (rows < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  const int32_t w = size_of_type(cols[0].type_id);
  if (w == 0) { set_error("%s: Only fixed width columns can be used (type id %d)", what, cols[0].type_id); return SRJ_EUNSUPPORTED; }
  for (int32_t c = 0; c < n; ++c) {
    if (cols[c].type_id != cols[0].type_id) { set_error("%s: All columns of the input table must be the same type.", what); return SRJ_EINVAL; }
    if (cols[c].size != rows) { set_error("%s: column %d has %lld rows, expected %lld", what, c, static_cast<long long>(cols[c].size), static_cast<long long>(rows)); return SRJ_EINVAL; }
  }
  if (rows * static_cast<int64_t>(w) * n > INT32_MAX) { set_error("%s: Input is too large to process", what); return SRJ_EINVAL; }
  *elem_bytes = w;
  return SRJ_OK;
}

// the data of every column present and aligned to its element (8 bytes for DECIMAL128: it is loaded as two longs)
static int zorder_check_data(const char* what, const srj_column* cols, int32_t n, int64_t rows, int32_t w)
{
  if (rows == 0) return SRJ_OK;
  const uintptr_t align = static_cast<uintptr_t>(w < 8 ? w : 8);
  for (int32_t c = 0; c < n; ++c)
    if (!cols[c].data || (reinterpret_cast<uintptr_t>(cols[c].data) & (align - 1))) {
      set_error("%s: column %d has no data or data not aligned to %d bytes", what, c, static_cast<int>(align));
      return SRJ_EINVAL;
    }
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
  if ((rc = zorder_check_data("interleave_bits", cols, num_columns, num_rows, w)) != SRJ_OK) return rc;
  if (!out_offsets || (num_rows > 0 && !out_bytes)) { set_error("interleave_bits: the output offsets and bytes are needed"); return SRJ_EINVAL; }
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
  const int rc = zorder_check_data(what, cols, num_columns, num_rows, 4);
  if (rc != SRJ_OK) return rc;
  if (num_rows > 0 && !out) { set_error("%s: the output is null", what); return SRJ_EINVAL; }
  return launch_hilbert_index(num_bits, cols, num_columns, num_rows, out, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// Iceberg partition transforms: bucket, truncate, year / month / day / hour (iceberg.cu)
// ---------------------------------------------------------------------------------------------------
static bool is_binary(const srj_column* c)
{
  return c->type_id == SRJ_LIST && c->num_children >= 1 && c->children && c->children[0].type_id == SRJ_UINT8;
}

static bool aligned_to(const void* p, int a) { return (reinterpret_cast<uintptr_t>(p) & static_cast<uintptr_t>(a - 1)) == 0; }

// the input's buffers for rows > 0: fixed-width data at its element alignment (8 bytes for DECIMAL128), STRING / LIST
// offsets at 4 bytes; with check_mask, an input with a mask needs an output mask
static int ice_check_buffers(const char* what, const srj_column* in, const uint32_t* out_mask, bool check_mask = true)
{
  if (in->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (in->size == 0) return SRJ_OK;
  if (in->type_id == SRJ_STRING || in->type_id == SRJ_LIST) {
    if (!in->offsets || !aligned_to(in->offsets, 4)) { set_error("%s: the input offsets are missing or not 4-byte aligned", what); return SRJ_EINVAL; }
  } else {
    const int a = std::min(size_of_type(in->type_id), 8);
    if (!in->data || !aligned_to(in->data, a)) { set_error("%s: the input data is missing or not aligned to %d bytes", what, a); return SRJ_EINVAL; }
  }
  if (check_mask && in->null_mask && !out_mask) { set_error("%s: the input has a null mask but no output mask was given", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

// iceberg_bucket.cu:393, 411-454
int srj_iceberg_bucket(const srj_column* input, int32_t num_buckets, int32_t* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_bucket";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (num_buckets <= 0) { set_error("%s: num_buckets must be positive", what); return SRJ_EINVAL; }
  switch (input->type_id) {
    case SRJ_INT32: case SRJ_INT64: case SRJ_DECIMAL32: case SRJ_DECIMAL64: case SRJ_DECIMAL128:
    case SRJ_TIMESTAMP_DAYS: case SRJ_TIMESTAMP_MICROSECONDS: case SRJ_STRING: break;
    case SRJ_LIST:
      if (is_binary(input)) break;
      set_error("%s: Binary type must be LIST of UINT8", what);
      return SRJ_EUNSUPPORTED;
    default: set_error("%s: Unsupported type for bucket transform: %d", what, input->type_id); return SRJ_EUNSUPPORTED;
  }
  const int rc = ice_check_buffers(what, input, out_mask);
  if (rc != SRJ_OK) return rc;
  if (input->size > 0 && (!out || !aligned_to(out, 4))) { set_error("%s: the output is missing or not 4-byte aligned", what); return SRJ_EINVAL; }
  return launch_iceberg_bucket(*input, num_buckets, out, out_mask, static_cast<cudaStream_t>(stream));
}

static bool truncate_integral(int32_t t)
{
  return t == SRJ_INT32 || t == SRJ_INT64 || t == SRJ_DECIMAL32 || t == SRJ_DECIMAL64 || t == SRJ_DECIMAL128;
}

// iceberg_truncate.cu:174-175, 202-213: STRING or LIST<UINT8> with a non-nullable child, width > 0
static int truncate_bytes_check(const char* what, const srj_column* in, int32_t width)
{
  if (in->type_id != SRJ_STRING && in->type_id != SRJ_LIST) { set_error("%s: Unsupported type for truncation", what); return SRJ_EUNSUPPORTED; }
  if (width <= 0) { set_error("%s: Length must be positive", what); return SRJ_EINVAL; }
  if (in->type_id == SRJ_LIST) {
    if (!is_binary(in)) { set_error("%s: Input must be LIST(UINT8)", what); return SRJ_EUNSUPPORTED; }
    if (in->children[0].null_mask) { set_error("%s: Child column of binary column must be non-nullable", what); return SRJ_EINVAL; }
  }
  return SRJ_OK;
}

int64_t srj_iceberg_truncate_workspace_bytes(int64_t num_rows) { return iceberg_truncate_workspace_bytes(std::max<int64_t>(0, num_rows)); }

int srj_iceberg_truncate_sizes(const srj_column* input, int32_t width, int32_t* d_out_offsets, int64_t* total_bytes, void* workspace,
                               void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_truncate_sizes";
  if (!input || !d_out_offsets || !total_bytes) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  int rc = truncate_bytes_check(what, input, width);
  if (rc != SRJ_OK) return rc;
  if ((rc = ice_check_buffers(what, input, nullptr, false)) != SRJ_OK) return rc;
  if (!aligned_to(d_out_offsets, 4)) { set_error("%s: the output offsets must be 4-byte aligned", what); return SRJ_EINVAL; }
  if (input->size > 0 && !workspace) { set_error("%s: the workspace is needed (srj_iceberg_truncate_workspace_bytes)", what); return SRJ_EINVAL; }
  return launch_iceberg_truncate_sizes(*input, width, d_out_offsets, total_bytes, workspace, static_cast<cudaStream_t>(stream));
}

// iceberg_truncate.cu:146-166 (integral), IcebergTruncateJni.cpp (the type switch)
int srj_iceberg_truncate(const srj_column* input, int32_t width, const srj_column* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_truncate";
  if (!input || !out) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (truncate_integral(input->type_id)) {
    if (width == 0) { set_error("%s: Width must not be zero", what); return SRJ_EINVAL; }
    const int rc = ice_check_buffers(what, input, out->null_mask);
    if (rc != SRJ_OK) return rc;
    if (input->size > 0 && (!out->data || !aligned_to(out->data, std::min(size_of_type(input->type_id), 8)))) {
      set_error("%s: the output data is missing or not aligned to its element", what);
      return SRJ_EINVAL;
    }
    return launch_iceberg_truncate_fixed(*input, width, out->data, out->null_mask, s);
  }
  int rc = truncate_bytes_check(what, input, width);
  if (rc != SRJ_OK) return rc;
  if ((rc = ice_check_buffers(what, input, out->null_mask)) != SRJ_OK) return rc;
  if (input->size == 0) return SRJ_OK;
  if (!out->offsets) { set_error("%s: the output needs the offsets of srj_iceberg_truncate_sizes", what); return SRJ_EINVAL; }
  if (input->type_id == SRJ_LIST && (out->num_children < 1 || !out->children)) { set_error("%s: the LIST output needs its UINT8 child", what); return SRJ_EINVAL; }
  uint8_t* bytes = static_cast<uint8_t*>(input->type_id == SRJ_LIST ? out->children[0].data : out->data);
  return launch_iceberg_truncate_bytes(*input, out->offsets, bytes, out->null_mask, s);
}

// iceberg_datetime_util.cu:137-248 and IcebergDateTimeUtil.java's type checks
int srj_iceberg_datetime(int32_t transform, const srj_column* input, int32_t* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "iceberg_datetime";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (transform < SRJ_ICEBERG_YEARS || transform > SRJ_ICEBERG_HOURS) { set_error("%s: unknown transform %d", what, transform); return SRJ_EINVAL; }
  const bool days = input->type_id == SRJ_TIMESTAMP_DAYS, micros = input->type_id == SRJ_TIMESTAMP_MICROSECONDS;
  if (!micros && !(days && transform != SRJ_ICEBERG_HOURS)) {
    set_error("%s: Input column must be of type TIMESTAMP_MICROSECONDS%s (type id %d)", what, transform == SRJ_ICEBERG_HOURS ? "" : " or TIMESTAMP_DAYS",
              input->type_id);
    return SRJ_EUNSUPPORTED;
  }
  const int rc = ice_check_buffers(what, input, out_mask);
  if (rc != SRJ_OK) return rc;
  if (input->size > 0 && (!out || !aligned_to(out, 4))) { set_error("%s: the output is missing or not 4-byte aligned", what); return SRJ_EINVAL; }
  return launch_iceberg_datetime(transform, *input, out, out_mask, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// DecimalUtils: DECIMAL128 multiply / divide / integral divide / remainder / add / subtract (decimal.cu)
// ---------------------------------------------------------------------------------------------------
// The scale combinations whose rows would reach pow_ten's CUDF_UNREACHABLE (k > 76) or divide by a truncated
// pow_ten(k).as_128_bits() (k > 38) in the reference, path by path; multiply keeps the reference's own
// check_scale_divisor (decimal_utils.cu:505-510).  Spark's type rules never produce them.
static const char* decimal_scale_error(int32_t op, int64_t sa, int64_t sb, int64_t so)
{
  switch (op) {
    case SRJ_DECIMAL_MULTIPLY: return so - (sa + sb) > 38 ? "divisor too big" : nullptr;
    case SRJ_DECIMAL_DIVIDE:
    case SRJ_DECIMAL_INTEGER_DIVIDE: {
      const int64_t x = so - (sa - sb);                 // > 0: round by 10^x; < -38: 10^38, then 10^(-x - 38)
      return x > 38 || x < -38 - 76 ? "the quotient scale needs a power of ten beyond 10^38 (divisor) or 10^76 (multiplier)" : nullptr;
    }
    case SRJ_DECIMAL_REMAINDER: {
      const int64_t ds = so - sb, ns = ds > 0 ? so - sa : sb - sa;
      return ds > 38 || ds < -76 || ns > 38 || ns < -76 ? "the remainder scale needs a power of ten beyond 10^38 (divisor) or 10^76 (multiplier)"
                                                        : nullptr;
    }
    default: {
      const int64_t inter = std::min(sa, sb), d = sa - sb;
      return d > 76 || d < -76 || inter - so > 76 || so - inter > 38 ? "the intermediate scale needs a power of ten beyond 10^38 (divisor) or 10^76 (multiplier)"
                                                                     : nullptr;
    }
  }
}

// decimal_utils.cu:967-1167 (multiply_decimal128 .. sub_decimal128)
int srj_decimal128_binary(int32_t op, const srj_column* a, const srj_column* b, int32_t out_scale, int32_t interim_cast, uint8_t* overflow,
                          void* out, uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "decimal128_binary";
  if (!a || !b) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (op < SRJ_DECIMAL_MULTIPLY || op > SRJ_DECIMAL_SUBTRACT) { set_error("%s: unknown op %d", what, op); return SRJ_EINVAL; }
  if (a->type_id != SRJ_DECIMAL128 || b->type_id != SRJ_DECIMAL128) { set_error("%s: not a DECIMAL128 column", what); return SRJ_EUNSUPPORTED; }
  if (a->size < 0 || a->size != b->size) { set_error("%s: inputs have mismatched row counts", what); return SRJ_EINVAL; }
  if (const char* e = decimal_scale_error(op, a->scale, b->scale, out_scale)) {
    set_error("%s: scales (%d, %d) -> %d: %s", what, a->scale, b->scale, out_scale, e);
    return SRJ_EINVAL;
  }
  if (a->size == 0) {
    if (null_count) *null_count = 0;
    return SRJ_OK;
  }
  if (!a->data || !b->data || !aligned_to(a->data, 8) || !aligned_to(b->data, 8)) { set_error("%s: the input data is missing or not 8-byte aligned", what); return SRJ_EINVAL; }
  if (!overflow) { set_error("%s: the overflow output is null", what); return SRJ_EINVAL; }
  if (!out || !aligned_to(out, 8)) { set_error("%s: the result output is missing or not 8-byte aligned", what); return SRJ_EINVAL; }
  if ((a->null_mask || b->null_mask) && (!out_mask || !aligned_to(out_mask, 4) || !null_count)) {
    set_error("%s: an input has a null mask but no output mask or null count was given", what);
    return SRJ_EINVAL;
  }
  return launch_decimal128_binary(op, *a, *b, out_scale, interim_cast != 0, overflow, out, out_mask, null_count, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// DateTimeUtils: calendar rebase and date / timestamp truncation (datetime.cu)
// ---------------------------------------------------------------------------------------------------
static bool is_datetime(int32_t t) { return t == SRJ_TIMESTAMP_DAYS || t == SRJ_TIMESTAMP_MICROSECONDS; }

// rows > 0: the datetime data and out at the element's alignment
static int datetime_check_data(const char* what, const srj_column* dt, const void* out)
{
  const int a = dt->type_id == SRJ_TIMESTAMP_DAYS ? 4 : 8;
  if (!dt->data || !aligned_to(dt->data, a)) { set_error("%s: the datetime data is missing or not aligned to %d bytes", what, a); return SRJ_EINVAL; }
  if (!out || !aligned_to(out, a)) { set_error("%s: the output is missing or not aligned to %d bytes", what, a); return SRJ_EINVAL; }
  return SRJ_OK;
}

// datetime_rebase.cu:342-372
int srj_datetime_rebase(int32_t direction, const srj_column* input, void* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "datetime_rebase";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (direction != SRJ_DATETIME_GREGORIAN_TO_JULIAN && direction != SRJ_DATETIME_JULIAN_TO_GREGORIAN) {
    set_error("%s: unknown direction %d", what, direction);
    return SRJ_EINVAL;
  }
  if (!is_datetime(input->type_id)) { set_error("%s: The input must be either day or microsecond timestamps to rebase.", what); return SRJ_EUNSUPPORTED; }
  if (input->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (input->size == 0) return SRJ_OK;
  const int rc = datetime_check_data(what, input, out);
  if (rc != SRJ_OK) return rc;
  if (input->null_mask && (!out_mask || !aligned_to(out_mask, 4))) { set_error("%s: the input has a null mask but no output mask was given", what); return SRJ_EINVAL; }
  return launch_datetime_rebase(direction, *input, out, out_mask, static_cast<cudaStream_t>(stream));
}

// datetime_truncate.cu:327-376
int srj_datetime_truncate(const srj_column* datetime, const srj_column* format_col, const char* format, int32_t format_len, void* out,
                          uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "datetime_truncate";
  if (!datetime || !null_count || (format_col == nullptr) == (format == nullptr) || (format && format_len < 0)) {
    set_error("%s: bad argument (give exactly one of a format column and a format string, and a null count)", what);
    return SRJ_EINVAL;
  }
  if (!is_datetime(datetime->type_id)) { set_error("%s: The date/time input must be either day or microsecond timestamps.", what); return SRJ_EUNSUPPORTED; }
  if (format_col && format_col->type_id != SRJ_STRING) { set_error("%s: The format input must be of string type.", what); return SRJ_EUNSUPPORTED; }
  if (datetime->size < 0 || (format_col && format_col->size < 0)) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (format_col && datetime->size != 1 && datetime->size != format_col->size) {
    set_error("%s: The input date/time column must have exactly one row or the same number of rows as the format column.", what);
    return SRJ_EINVAL;
  }
  const int64_t rows = format_col ? format_col->size : datetime->size;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows == 0) {
    *null_count = 0;
    return SRJ_OK;
  }
  const int rc = datetime_check_data(what, datetime, out);
  if (rc != SRJ_OK) return rc;
  if (format_col) {
    if (!format_col->offsets || !aligned_to(format_col->offsets, 4)) { set_error("%s: the format offsets are missing or not 4-byte aligned", what); return SRJ_EINVAL; }
    if (!out_mask || !aligned_to(out_mask, 4)) { set_error("%s: a format column needs an output mask", what); return SRJ_EINVAL; }
    return launch_datetime_truncate_column(*datetime, *format_col, out, out_mask, null_count, s);
  }
  const int32_t fmt = datetime_parse_format(format, format_len);
  const bool fits   = datetime_format_fits(fmt, datetime->type_id == SRJ_TIMESTAMP_MICROSECONDS);
  if ((!fits || datetime->null_mask) && (!out_mask || !aligned_to(out_mask, 4))) {
    set_error("%s: the result has nulls but no output mask was given", what);
    return SRJ_EINVAL;
  }
  *null_count = fits ? -1 : rows;
  return launch_datetime_truncate_scalar(fmt, *datetime, out, out_mask, s);
}

// ---------------------------------------------------------------------------------------------------
// GpuTimeZoneDB: time zone conversions (timezone.cu)
// ---------------------------------------------------------------------------------------------------
static bool is_timestamp_64(int32_t t) { return t >= SRJ_TIMESTAMP_SECONDS && t <= SRJ_TIMESTAMP_NANOSECONDS; }

// a flat column of type t (or of either type when t2 >= 0) with rows rows, its data aligned to its element when rows > 0
static int tz_check_flat(const char* what, const char* name, const srj_column* c, int32_t t, int32_t t2, int64_t rows)
{
  if (!c) { set_error("%s: the %s column is null", what, name); return SRJ_EINVAL; }
  if (c->type_id != t && c->type_id != t2) { set_error("%s: the %s column has type id %d", what, name, c->type_id); return SRJ_EINVAL; }
  if (c->size != rows) { set_error("%s: the %s column has %lld rows, not %lld", what, name, static_cast<long long>(c->size), static_cast<long long>(rows)); return SRJ_EINVAL; }
  const int a = size_of_type(c->type_id);
  if (rows > 0 && (!c->data || !aligned_to(c->data, a))) { set_error("%s: the %s data is missing or not aligned to %d bytes", what, name, a); return SRJ_EINVAL; }
  return SRJ_OK;
}

// the two columns of a time zone table (GpuTimeZoneDB.loadData's layout)
static int tz_check_table(const char* what, const srj_column* fixed, const srj_column* dst)
{
  if (!fixed || !dst) { set_error("%s: the time zone table is null", what); return SRJ_EINVAL; }
  if (fixed->type_id != SRJ_LIST || dst->type_id != SRJ_LIST || fixed->num_children < 1 || !fixed->children || dst->num_children < 1 || !dst->children) {
    set_error("%s: the time zone table must be LIST<STRUCT<INT64, INT64, INT32>> and LIST<INT32>", what);
    return SRJ_EINVAL;
  }
  if (fixed->size < 0 || fixed->size > INT32_MAX || dst->size != fixed->size) { set_error("%s: the time zone table's columns have mismatched row counts", what); return SRJ_EINVAL; }
  if (!fixed->offsets || !aligned_to(fixed->offsets, 4) || !dst->offsets || !aligned_to(dst->offsets, 4)) {
    set_error("%s: the time zone table's list offsets are missing or not 4-byte aligned", what);
    return SRJ_EINVAL;
  }
  const srj_column* s = &fixed->children[0];
  if (s->type_id != SRJ_STRUCT || s->num_children != 3 || !s->children) { set_error("%s: the transitions must be STRUCT<INT64, INT64, INT32>", what); return SRJ_EINVAL; }
  static const char* const names[3] = {"utcInstant", "localInstant", "offset"};
  for (int i = 0; i < 3; ++i) {
    const int rc = tz_check_flat(what, names[i], &s->children[i], i < 2 ? SRJ_INT64 : SRJ_INT32, -1, s->size);
    if (rc != SRJ_OK) return rc;
  }
  return tz_check_flat(what, "DST rules", &dst->children[0], SRJ_INT32, -1, dst->children[0].size);
}

// an input of type t with rows > 0 needs its data and out at 8 bytes, and out_mask when it has a mask
static int tz_check_io(const char* what, const srj_column* in, const void* out, const uint32_t* out_mask)
{
  if (in->size < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  if (in->size == 0) return SRJ_OK;
  if (!in->data || !aligned_to(in->data, 8)) { set_error("%s: the input data is missing or not 8-byte aligned", what); return SRJ_EINVAL; }
  if (!out || !aligned_to(out, 8)) { set_error("%s: the output is missing or not 8-byte aligned", what); return SRJ_EINVAL; }
  if ((in->null_mask && !out_mask) || (out_mask && !aligned_to(out_mask, 4))) { set_error("%s: the input has a null mask but no 4-byte aligned output mask was given", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

// timezones.cu:80-111, 494-539
int srj_timezone_convert(int32_t direction, const srj_column* input, const srj_column* fixed_transitions, const srj_column* dst_rules,
                         int32_t tz_index, void* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "timezone_convert";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (direction != SRJ_TIMEZONE_TO_UTC && direction != SRJ_TIMEZONE_FROM_UTC) { set_error("%s: unknown direction %d", what, direction); return SRJ_EINVAL; }
  if (!is_timestamp_64(input->type_id)) { set_error("%s: Unsupported timestamp unit for timezone conversion (type id %d)", what, input->type_id); return SRJ_EUNSUPPORTED; }
  int rc = tz_check_table(what, fixed_transitions, dst_rules);
  if (rc != SRJ_OK) return rc;
  if (tz_index < 0 || tz_index >= fixed_transitions->size) {
    set_error("%s: time zone index %d is outside the table of %lld zones", what, tz_index, static_cast<long long>(fixed_transitions->size));
    return SRJ_EINVAL;
  }
  if ((rc = tz_check_io(what, input, out, out_mask)) != SRJ_OK) return rc;
  return launch_timezone_convert(direction == SRJ_TIMEZONE_TO_UTC, *input, *fixed_transitions, *dst_rules, tz_index, out, out_mask,
                                 static_cast<cudaStream_t>(stream));
}

// timezones.cu:186-240
int srj_timezone_convert_multi(const srj_column* seconds, const srj_column* micros, const srj_column* invalid, const srj_column* tz_type,
                               const srj_column* tz_offset, const srj_column* fixed_transitions, const srj_column* dst_rules,
                               const srj_column* tz_indices, int64_t* out, uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "timezone_convert_multi";
  if (!seconds || !null_count) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (seconds->type_id != SRJ_INT64) { set_error("%s: seconds column must be of type INT64", what); return SRJ_EUNSUPPORTED; }
  if (micros && micros->type_id != SRJ_INT32) { set_error("%s: microseconds column must be of type INT32", what); return SRJ_EUNSUPPORTED; }
  const int64_t n = seconds->size;
  if (n < 0) { set_error("%s: bad row count", what); return SRJ_EINVAL; }
  int rc = tz_check_table(what, fixed_transitions, dst_rules);
  if (rc != SRJ_OK) return rc;
  const srj_column* cols[6] = {seconds, micros, invalid, tz_type, tz_offset, tz_indices};
  static const char* const names[6] = {"seconds", "microseconds", "invalid", "tz type", "tz offset", "tz indices"};
  static const int32_t types[6][2] = {{SRJ_INT64, -1}, {SRJ_INT32, -1}, {SRJ_BOOL8, SRJ_UINT8}, {SRJ_UINT8, -1}, {SRJ_INT32, -1}, {SRJ_INT32, -1}};
  for (int i = 0; i < 6; ++i)
    if ((rc = tz_check_flat(what, names[i], cols[i], types[i][0], types[i][1], n)) != SRJ_OK) return rc;
  if (n == 0) {
    *null_count = 0;
    return SRJ_OK;
  }
  if (!out || !aligned_to(out, 8)) { set_error("%s: the output is missing or not 8-byte aligned", what); return SRJ_EINVAL; }
  if (!out_mask || !aligned_to(out_mask, 4)) { set_error("%s: the output mask is missing or not 4-byte aligned", what); return SRJ_EINVAL; }
  const srj_column in[6] = {*seconds, *micros, *invalid, *tz_type, *tz_offset, *tz_indices};
  return launch_timezone_convert_multi(in, *fixed_transitions, *dst_rules, out, out_mask, null_count, static_cast<cudaStream_t>(stream));
}

// timezones.cu:380-486; a NULL table is a fixed offset
int srj_orc_convert_timezones(const srj_column* input, const srj_column* writer_transitions, const srj_column* writer_offsets,
                              int32_t writer_raw_offset, const srj_column* reader_transitions, const srj_column* reader_offsets,
                              int32_t reader_raw_offset, void* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "orc_convert_timezones";
  if (!input) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (input->type_id != SRJ_TIMESTAMP_MICROSECONDS) { set_error("%s: Input column must be of type TIMESTAMP_MICROSECONDS", what); return SRJ_EUNSUPPORTED; }
  const srj_column* tr[2] = {writer_transitions, reader_transitions};
  const srj_column* of[2] = {writer_offsets, reader_offsets};
  int32_t rows[2]         = {0, 0};
  for (int i = 0; i < 2; ++i) {
    const char* side = i ? "reader" : "writer";
    if (!tr[i] && !of[i]) continue;
    if (!tr[i] || !of[i]) { set_error("%s: the %s table needs both its transitions and its offsets", what, side); return SRJ_EINVAL; }
    if (tr[i]->size < 0 || tr[i]->size > INT32_MAX) { set_error("%s: bad %s table size", what, side); return SRJ_EINVAL; }
    int rc = tz_check_flat(what, i ? "reader transitions" : "writer transitions", tr[i], SRJ_INT64, -1, tr[i]->size);
    if (rc == SRJ_OK) rc = tz_check_flat(what, i ? "reader offsets" : "writer offsets", of[i], SRJ_INT32, -1, tr[i]->size);
    if (rc != SRJ_OK) return rc;
    rows[i] = static_cast<int32_t>(tr[i]->size);
  }
  const int rc = tz_check_io(what, input, out, out_mask);
  if (rc != SRJ_OK) return rc;
  auto ptr64 = [&](int i) { return rows[i] ? static_cast<const int64_t*>(tr[i]->data) : nullptr; };
  auto ptr32 = [&](int i) { return rows[i] ? static_cast<const int32_t*>(of[i]->data) : nullptr; };
  return launch_orc_convert_timezones(*input, ptr64(0), ptr32(0), rows[0], writer_raw_offset, ptr64(1), ptr32(1), rows[1], reader_raw_offset, out,
                                      out_mask, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// CastStrings: string to timestamp and string to date (cast_datetime.cu)
// ---------------------------------------------------------------------------------------------------
// a STRING column: int32 offsets[rows + 1] at 4 bytes.  Its chars may be NULL only when it holds none: a column with rows
// and NULL chars has its first and last offsets read back (one stream synchronisation, on that path alone) and is
// SRJ_EINVAL when they span any byte.
static int cast_check_strings(const char* what, const char* name, const srj_column* c, cudaStream_t stream)
{
  if (!c) { set_error("%s: the %s column is null", what, name); return SRJ_EINVAL; }
  if (c->type_id != SRJ_STRING) { set_error("%s: the %s column must be STRING (type id %d)", what, name, c->type_id); return SRJ_EINVAL; }
  if (c->size < 0 || c->size > INT32_MAX) { set_error("%s: bad %s row count", what, name); return SRJ_EINVAL; }
  if (c->size > 0 && (!c->offsets || !aligned_to(c->offsets, 4))) { set_error("%s: the %s offsets are missing or not 4-byte aligned", what, name); return SRJ_EINVAL; }
  if (c->null_mask && !aligned_to(c->null_mask, 4)) { set_error("%s: the %s null mask is not 4-byte aligned", what, name); return SRJ_EINVAL; }
  if (c->size > 0 && !c->data) {
    int32_t ends[2] = {0, 0};
    SRJ_CUDA_TRY(cudaMemcpyAsync(&ends[0], c->offsets, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    SRJ_CUDA_TRY(cudaMemcpyAsync(&ends[1], c->offsets + c->size, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
    if (ends[0] != ends[1]) { set_error("%s: the %s column has no chars but its offsets span %d bytes", what, name, ends[1] - ends[0]); return SRJ_EINVAL; }
  }
  return SRJ_OK;
}

static bool out_ok(const void* p, int a) { return p && aligned_to(p, a); }

// cast_string_to_datetime.cu:870-948, 1110-1133; version.hpp:64-68
int srj_cast_parse_timestamps(const srj_column* input, const srj_column* tz_name_map, const srj_column* fixed_transitions, const srj_column* dst_rules,
                              int32_t default_tz_index, int64_t default_epoch_day, int64_t now_seconds, int32_t spark_platform, int32_t spark_major,
                              int32_t spark_minor, int32_t spark_patch, uint8_t* out_result, int64_t* out_seconds, int32_t* out_micros,
                              uint8_t* out_tz_type, int32_t* out_tz_offset, int32_t* out_tz_index, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "cast_parse_timestamps";
  int rc           = cast_check_strings(what, "input", input, static_cast<cudaStream_t>(stream));
  if (rc != SRJ_OK) return rc;
  if (!tz_name_map || tz_name_map->type_id != SRJ_STRUCT || tz_name_map->num_children < 2 || !tz_name_map->children || tz_name_map->size < 0) {
    set_error("%s: the time zone name map must be STRUCT<STRING, INT32>", what);
    return SRJ_EINVAL;
  }
  const srj_column* names = &tz_name_map->children[0];
  if ((rc = cast_check_strings(what, "time zone name", names, static_cast<cudaStream_t>(stream))) != SRJ_OK) return rc;
  if (names->size != tz_name_map->size) { set_error("%s: the time zone name map's fields have mismatched row counts", what); return SRJ_EINVAL; }
  if ((rc = tz_check_flat(what, "time zone index", &tz_name_map->children[1], SRJ_INT32, -1, tz_name_map->size)) != SRJ_OK) return rc;
  if ((rc = tz_check_table(what, fixed_transitions, dst_rules)) != SRJ_OK) return rc;
  if (default_tz_index < 0 || default_tz_index >= fixed_transitions->size) {
    set_error("%s: default time zone index %d is outside the table of %lld zones", what, default_tz_index,
              static_cast<long long>(fixed_transitions->size));
    return SRJ_EINVAL;
  }
  const int64_t n = input->size;
  if (n == 0) return SRJ_OK;
  if (!out_ok(out_result, 1) || !out_ok(out_seconds, 8) || !out_ok(out_micros, 4) || !out_ok(out_tz_type, 1) || !out_ok(out_tz_offset, 4) ||
      !out_ok(out_tz_index, 4)) {
    set_error("%s: an output is missing or not aligned to its element", what);
    return SRJ_EINVAL;
  }
  // is_vanilla_320 and is_vanilla_400_or_later || is_databricks_14_3_or_later
  const auto ge = [&](int32_t a, int32_t b, int32_t c) {
    return spark_major > a || (spark_major == a && (spark_minor > b || (spark_minor == b && spark_patch >= c)));
  };
  const bool is_320 = spark_platform == SRJ_SPARK_VANILLA && spark_major == 3 && spark_minor == 2 && spark_patch == 0;
  const bool is_400 = (spark_platform == SRJ_SPARK_VANILLA && ge(4, 0, 0)) || (spark_platform == SRJ_SPARK_DATABRICKS && ge(14, 3, 0));
  return launch_cast_parse_timestamps(*input, *tz_name_map, *fixed_transitions, *dst_rules, default_tz_index, default_epoch_day, now_seconds, is_320,
                                      is_400, out_result, out_seconds, out_micros, out_tz_type, out_tz_offset, out_tz_index,
                                      static_cast<cudaStream_t>(stream));
}

// cast_string_to_datetime.cu:1034-1106, 1135-1140
int srj_cast_parse_dates(const srj_column* input, int32_t* out, uint32_t* out_mask, int64_t* null_count, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "cast_parse_dates";
  if (!null_count) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  const int rc = cast_check_strings(what, "input", input, static_cast<cudaStream_t>(stream));
  if (rc != SRJ_OK) return rc;
  if (input->size == 0) {
    *null_count = 0;
    return SRJ_OK;
  }
  if (!out_ok(out, 4) || !out_ok(out_mask, 4)) { set_error("%s: the output or its mask is missing or not 4-byte aligned", what); return SRJ_EINVAL; }
  return launch_cast_parse_dates(*input, out, out_mask, null_count, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// JoinPrimitives: hash inner join and the gather-map helpers (join.cu)
// ---------------------------------------------------------------------------------------------------
// join_primitives.cu:212-220 and cudf's validate_hash_join_probe: key counts first, an empty side returns empty, then the
// schema.  *rows[2] receive the row counts; *empty is set when either is 0 (nothing else was checked then).
static int join_check(const char* what, const srj_column* l, int32_t nl, const srj_column* r, int32_t nr, int64_t rows[2], bool* empty)
{
  if (!l || !r || nl < 0 || nr < 0) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (nl == 0) { set_error("%s: Left keys table must have at least one column", what); return SRJ_EINVAL; }
  if (nr == 0) { set_error("%s: Right keys table must have at least one column", what); return SRJ_EINVAL; }
  for (int side = 0; side < 2; ++side) {
    const srj_column* t = side ? r : l;
    const int32_t n     = side ? nr : nl;
    rows[side]          = t[0].size;
    for (int32_t c = 0; c < n; ++c)
      if (t[c].size < 0 || t[c].size != rows[side]) { set_error("%s: the %s key columns have differing or negative row counts", what, side ? "right" : "left"); return SRJ_EINVAL; }
  }
  *empty = rows[0] == 0 || rows[1] == 0;
  if (*empty) return SRJ_OK;
  for (int side = 0; side < 2; ++side) {
    const srj_column* t = side ? r : l;
    for (int32_t c = 0; c < (side ? nr : nl); ++c)
      if (t[c].type_id != SRJ_STRING && join_key_width(t[c].type_id) == 0) { set_error("%s: key type %d is not supported", what, t[c].type_id); return SRJ_EUNSUPPORTED; }
  }
  if (nl != nr) { set_error("%s: Mismatch in number of columns to be joined on", what); return SRJ_EINVAL; }
  if (nl > SRJ_MAX_JOIN_KEYS) { set_error("%s: more than %d key columns", what, SRJ_MAX_JOIN_KEYS); return SRJ_EUNSUPPORTED; }
  for (int32_t c = 0; c < nl; ++c)
    if (l[c].type_id != r[c].type_id || l[c].scale != r[c].scale) { set_error("%s: Mismatch in joining column data types", what); return SRJ_EINVAL; }
  if (rows[0] > INT32_MAX || rows[1] > INT32_MAX) { set_error("%s: more than INT32_MAX rows", what); return SRJ_EINVAL; }
  for (int side = 0; side < 2; ++side) {
    const srj_column* t = side ? r : l;
    for (int32_t c = 0; c < nl; ++c) {
      const bool str = t[c].type_id == SRJ_STRING;
      const int a    = str ? 1 : std::min(join_key_width(t[c].type_id), 8);
      if ((!t[c].data && !str) || !aligned_to(t[c].data, a) || (str && (!t[c].offsets || !aligned_to(t[c].offsets, 4))) ||
          !aligned_to(t[c].null_mask, 4)) {
        set_error("%s: key column %d of the %s table has a missing or misaligned buffer", what, c, side ? "right" : "left");
        return SRJ_EINVAL;
      }
    }
  }
  return SRJ_OK;
}

int64_t srj_hash_join_workspace_bytes(int64_t left_rows, int64_t right_rows)
{
  return hash_join_workspace_bytes(std::max<int64_t>(0, left_rows), std::max<int64_t>(0, right_rows));
}

int srj_hash_inner_join_size(const srj_column* left_keys, int32_t num_left_keys, const srj_column* right_keys, int32_t num_right_keys,
                             int32_t nulls_equal, int64_t* num_pairs, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "hash_inner_join_size";
  if (!num_pairs) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  int64_t rows[2];
  bool empty  = false;
  const int rc = join_check(what, left_keys, num_left_keys, right_keys, num_right_keys, rows, &empty);
  if (rc != SRJ_OK) return rc;
  *num_pairs = 0;
  if (empty) return SRJ_OK;
  if (!workspace) { set_error("%s: the workspace is needed (srj_hash_join_workspace_bytes)", what); return SRJ_EINVAL; }
  return launch_hash_join_size(left_keys, right_keys, num_left_keys, rows[0], rows[1], nulls_equal != 0, num_pairs, workspace,
                               static_cast<cudaStream_t>(stream));
}

int srj_hash_inner_join(const srj_column* left_keys, int32_t num_left_keys, const srj_column* right_keys, int32_t num_right_keys,
                        int32_t nulls_equal, int32_t* left_map, int32_t* right_map, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "hash_inner_join";
  int64_t rows[2];
  bool empty  = false;
  const int rc = join_check(what, left_keys, num_left_keys, right_keys, num_right_keys, rows, &empty);
  if (rc != SRJ_OK || empty) return rc;
  (void)nulls_equal;   // the size call's counts already hold it
  if (!workspace || !left_map || !right_map || !aligned_to(left_map, 4) || !aligned_to(right_map, 4)) {
    set_error("%s: a missing or misaligned map or workspace", what);
    return SRJ_EINVAL;
  }
  return launch_hash_join(left_keys, right_keys, num_left_keys, rows[0], rows[1], left_map, right_map, workspace, static_cast<cudaStream_t>(stream));
}

// a gather map of map_len entries (4-byte aligned; NULL only when empty) over a table of table_rows rows
static int join_check_map(const char* what, const int32_t* map, int64_t map_len, int64_t table_rows)
{
  if (map_len < 0 || table_rows < 0) { set_error("%s: Table sizes must be non-negative", what); return SRJ_EINVAL; }
  if (table_rows > INT32_MAX) { set_error("%s: more than INT32_MAX table rows", what); return SRJ_EINVAL; }
  if ((map_len > 0 && !map) || !aligned_to(map, 4)) { set_error("%s: the gather map is missing or not 4-byte aligned", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

int64_t srj_join_mask_workspace_bytes(int64_t table_rows) { return join_mask_workspace_bytes(std::max<int64_t>(0, table_rows)); }

int srj_join_mark(const int32_t* map, int64_t map_len, int64_t table_rows, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_mark";
  const int rc     = join_check_map(what, map, map_len, table_rows);
  if (rc != SRJ_OK) return rc;
  if (!workspace || !aligned_to(workspace, 8)) { set_error("%s: the workspace is missing or not 8-byte aligned", what); return SRJ_EINVAL; }
  return launch_join_mark(map, map_len, table_rows, workspace, static_cast<cudaStream_t>(stream));
}

int srj_join_matched_counts(const void* const* workspaces, int32_t count, int64_t* matched, void* stream)
{
  SRJ_API_RANGE();
  if (count < 0 || (count > 0 && (!workspaces || !matched))) { set_error("join_matched_counts: bad argument"); return SRJ_EINVAL; }
  for (int32_t i = 0; i < count; ++i)
    if (!workspaces[i]) { set_error("join_matched_counts: workspace %d is null", i); return SRJ_EINVAL; }
  if (count == 0) return SRJ_OK;
  return read_join_matched(workspaces, count, matched, static_cast<cudaStream_t>(stream));
}

int srj_join_compact(const void* workspace, int64_t table_rows, int32_t matched, int32_t* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_compact";
  const int rc     = join_check_map(what, nullptr, 0, table_rows);
  if (rc != SRJ_OK) return rc;
  if (table_rows == 0) return SRJ_OK;
  if (!workspace || !out || !aligned_to(out, 4)) { set_error("%s: a missing workspace or a missing or misaligned output", what); return SRJ_EINVAL; }
  return launch_join_compact(workspace, table_rows, matched != 0, out, static_cast<cudaStream_t>(stream));
}

// join_primitives.cu:358-461
int srj_join_make_outer(const int32_t* left_map, const int32_t* right_map, int64_t map_len, int64_t left_rows, int64_t right_rows,
                        const void* left_ws, int64_t left_unmatched, const void* right_ws, int64_t right_unmatched, int32_t* out_left,
                        int32_t* out_right, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_make_outer";
  int rc           = join_check_map(what, left_map, map_len, left_rows);
  if (rc != SRJ_OK || (rc = join_check_map(what, right_map, map_len, right_rows)) != SRJ_OK) return rc;
  const bool full = right_ws != nullptr;
  if (left_unmatched < 0 || left_unmatched > left_rows || (full && (right_unmatched < 0 || right_unmatched > right_rows))) {
    set_error("%s: unmatched counts outside the table sizes", what);
    return SRJ_EINVAL;
  }
  const int64_t total = map_len + left_unmatched + (full ? right_unmatched : 0);
  if (total == 0) return SRJ_OK;
  if (!left_ws || !out_left || !out_right || !aligned_to(out_left, 4) || !aligned_to(out_right, 4)) {
    set_error("%s: a missing workspace or a missing or misaligned output", what);
    return SRJ_EINVAL;
  }
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (map_len > 0) {
    SRJ_CUDA_TRY(cudaMemcpyAsync(out_left, left_map, static_cast<size_t>(map_len) * 4, cudaMemcpyDeviceToDevice, s));
    SRJ_CUDA_TRY(cudaMemcpyAsync(out_right, right_map, static_cast<size_t>(map_len) * 4, cudaMemcpyDeviceToDevice, s));
  }
  if (left_unmatched > 0) {
    if ((rc = launch_join_compact(left_ws, left_rows, false, out_left + map_len, s)) != SRJ_OK) return rc;
    if ((rc = launch_join_fill(out_right + map_len, left_unmatched, INT32_MIN, s)) != SRJ_OK) return rc;
  }
  if (full && right_unmatched > 0) {
    const int64_t at = map_len + left_unmatched;
    if ((rc = launch_join_compact(right_ws, right_rows, false, out_right + at, s)) != SRJ_OK) return rc;
    if ((rc = launch_join_fill(out_left + at, right_unmatched, INT32_MIN, s)) != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

// join_primitives.cu:549-576
int srj_join_matched_rows(const int32_t* map, int64_t map_len, int64_t table_rows, uint8_t* out, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "join_matched_rows";
  const int rc     = join_check_map(what, map, map_len, table_rows);
  if (rc != SRJ_OK) return rc;
  if (table_rows == 0) return SRJ_OK;
  if (!out) { set_error("%s: the output is null", what); return SRJ_EINVAL; }
  return launch_join_matched_rows(map, map_len, table_rows, out, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// Spark HashPartitioning: pmod(murmur3_32(seed, keys), P) + stable partition (partition.cu)
// ---------------------------------------------------------------------------------------------------
int64_t srj_partition_workspace_bytes(int64_t num_rows, int32_t num_partitions)
{
  return partition_workspace_bytes(num_rows, num_partitions);
}

int srj_partition_plan(int32_t* d_partition_ids, int64_t num_rows, int32_t num_partitions, int32_t* d_partition_offsets,
                       int32_t* d_scatter_map, int32_t* d_gather_map, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  if (num_rows < 0 || num_partitions <= 0 || !d_partition_offsets || (num_rows > 0 && (!d_partition_ids || !workspace))) {
    set_error("partition_plan: bad argument");
    return SRJ_EINVAL;
  }
  if (num_rows > INT32_MAX || num_partitions > (1 << 14)) {
    set_error("partition_plan: %lld rows / %d partitions exceed the int32 row index / 16384 partitions", static_cast<long long>(num_rows), num_partitions);
    return SRJ_EUNSUPPORTED;
  }
  return launch_partition_plan(d_partition_ids, num_rows, num_partitions, d_partition_offsets, d_scatter_map, d_gather_map, workspace,
                               static_cast<cudaStream_t>(stream));
}

int srj_hash_partition(const srj_column* keys, int32_t num_keys, int64_t num_rows, uint32_t seed, int32_t num_partitions,
                       int32_t* d_partition_ids, int32_t* d_partition_offsets, int32_t* d_scatter_map, int32_t* d_gather_map,
                       void* workspace, void* stream)
{
  SRJ_API_RANGE();
  if (num_keys <= 0 || !keys) { set_error("hash_partition: no key columns"); return SRJ_EINVAL; }
  if (num_rows > 0 && !d_partition_ids) { set_error("hash_partition: bad argument"); return SRJ_EINVAL; }
  // the partition count is checked before the keys are hashed: a refused call launches nothing
  if (num_partitions <= 0) { set_error("hash_partition: %d partitions", num_partitions); return SRJ_EINVAL; }
  if (num_partitions > (1 << 14)) { set_error("hash_partition: %d partitions exceed 16384 partitions", num_partitions); return SRJ_EUNSUPPORTED; }
  // the hashes go where the ids will be: part_ids_kernel turns them into ids in place
  int rc = hash_any(SRJ_HASH_MURMUR3_32, keys, num_keys, num_rows, seed, d_partition_ids, static_cast<cudaStream_t>(stream));
  if (rc != SRJ_OK) return rc;
  return srj_partition_plan(d_partition_ids, num_rows, num_partitions, d_partition_offsets, d_scatter_map, d_gather_map, workspace, stream);
}

int srj_partition_columns(const srj_column* in, const srj_column* out, int32_t num_columns, int64_t num_rows, int32_t num_partitions,
                          const int32_t* d_scatter_map, const int32_t* d_gather_map, int64_t* d_null_counts, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (num_columns < 0 || num_rows < 0 || num_partitions <= 0 || (num_columns > 0 && (!in || !out))) { set_error("partition_columns: bad argument"); return SRJ_EINVAL; }
  if (num_rows > 0 && (!d_scatter_map || !d_gather_map || !workspace)) { set_error("partition_columns: the maps and the plan's workspace are needed"); return SRJ_EINVAL; }
  if (d_null_counts && num_columns > 0) SRJ_CUDA_TRY(cudaMemsetAsync(d_null_counts, 0, sizeof(int64_t) * num_columns, st));
  std::vector<int> esz(static_cast<size_t>(num_columns), 0);
  for (int32_t c = 0; c < num_columns; ++c) {
    const srj_column& a = in[c];
    const srj_column& b = out[c];
    if (a.type_id != b.type_id || a.size != num_rows || b.size != num_rows) { set_error("partition_columns: column %d: type / size mismatch", c); return SRJ_EINVAL; }
    if (a.type_id == SRJ_STRING) {
      if (!a.offsets || !b.offsets) { set_error("partition_columns: STRING column %d needs offsets", c); return SRJ_EINVAL; }
    } else {
      esz[c] = size_of_type(a.type_id);
      if (esz[c] <= 0) { set_error("partition_columns: column %d: unsupported type %d", c, a.type_id); return SRJ_EUNSUPPORTED; }
      if (num_rows > 0 && (!a.data || !b.data)) { set_error("partition_columns: column %d: NULL data", c); return SRJ_EINVAL; }
    }
    if (a.null_mask && !b.null_mask) { set_error("partition_columns: column %d has a null mask but its output has none", c); return SRJ_EINVAL; }
    if (!a.null_mask && b.null_mask && num_rows > 0) SRJ_CUDA_TRY(cudaMemsetAsync(b.null_mask, 0xff, static_cast<size_t>((num_rows + 31) / 32) * 4, st));
  }
  // fixed-width data and every null mask: tile by tile, staged in destination order (plans of <= 1024 partitions) ...
  int rc = launch_partition_move_tiles(in, out, esz.data(), num_columns, num_rows, num_partitions, d_scatter_map, workspace,
                                       reinterpret_cast<unsigned long long*>(d_null_counts), st);
  if (rc == SRJ_EUNSUPPORTED) {
    // ... or row by row
    rc = SRJ_OK;
    for (int32_t c = 0; c < num_columns && rc == SRJ_OK && num_rows > 0; ++c) {
      if (esz[c] > 0) rc = launch_partition_scatter_fixed(in[c].data, out[c].data, esz[c], d_scatter_map, num_rows, st);
      if (rc == SRJ_OK && in[c].null_mask)
        rc = launch_partition_gather_mask(in[c].null_mask, out[c].null_mask, d_gather_map, num_rows,
                                          d_null_counts ? reinterpret_cast<unsigned long long*>(d_null_counts + c) : nullptr, st);
    }
  }
  if (rc != SRJ_OK) return rc;
  // STRING columns: the output offsets (lengths through the gather map, then a scan; partials behind the plan's tile order)
  for (int32_t c = 0; c < num_columns; ++c) {
    if (in[c].type_id != SRJ_STRING) continue;
    if (num_rows == 0) {
      SRJ_CUDA_TRY(cudaMemsetAsync(out[c].offsets, 0, 4, st));   // an empty STRING column still has its offsets[0] = 0
      continue;
    }
    rc = launch_partition_string_offsets(in[c].offsets, out[c].offsets, d_gather_map, num_rows, static_cast<int32_t*>(workspace) + num_rows, st);
    if (rc != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

int srj_partition_strings(const srj_column* in, const srj_column* out, int32_t num_columns, int64_t num_rows, const int32_t* d_gather_map,
                          void* stream)
{
  SRJ_API_RANGE();
  if (num_columns < 0 || num_rows < 0 || (num_columns > 0 && (!in || !out))) { set_error("partition_strings: bad argument"); return SRJ_EINVAL; }
  for (int32_t c = 0; c < num_columns; ++c) {
    if (in[c].type_id != SRJ_STRING || num_rows == 0) continue;
    if (!out[c].offsets || !in[c].offsets) { set_error("partition_strings: column %d: NULL offsets", c); return SRJ_EINVAL; }
    const int rc = launch_partition_gather_chars(static_cast<const uint8_t*>(in[c].data), in[c].offsets, static_cast<uint8_t*>(out[c].data),
                                                 out[c].offsets, d_gather_map, num_rows, static_cast<cudaStream_t>(stream));
    if (rc != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

// ---------------------------------------------------------------------------------------------------
// Apache Spark UnsafeRow codec (unsafe_row.cu)
// ---------------------------------------------------------------------------------------------------
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
  for (int32_t c = 0; c < ncols; ++c)
    if (cols[c].size != n) { set_error("%s: column %d has %lld rows, expected %lld", what, c, static_cast<long long>(cols[c].size), static_cast<long long>(n)); return SRJ_EINVAL; }
  return SRJ_OK;
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
  if ((num_rows > 0 && !rows) || (reinterpret_cast<uintptr_t>(rows) & 7)) { set_error("convert_to_unsafe_rows: rows must be 8-byte aligned"); return SRJ_EINVAL; }
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
  if ((num_rows > 0 && !rows) || (reinterpret_cast<uintptr_t>(rows) & 7)) { set_error("convert_from_unsafe_rows: rows must be 8-byte aligned"); return SRJ_EINVAL; }
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
  if (reinterpret_cast<uintptr_t>(rows) & 7) { set_error("convert_from_unsafe_rows_strings: rows must be 8-byte aligned"); return SRJ_EINVAL; }
  return launch_unsafe_from_rows_strings(out, num_columns, num_rows, rows, d_row_offsets, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// Kudo shuffle wire format: split / assemble (kudo.cu)
// ---------------------------------------------------------------------------------------------------
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
  for (int32_t c = 0; c < num_columns; ++c)
    if (cols[c].size != num_rows) { set_error("kudo_split_sizes: column %d: row count mismatch", c); return SRJ_EINVAL; }
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
  if (!d_splits || (num_partitions > 0 && !out) || (reinterpret_cast<uintptr_t>(out) & 3)) { set_error("kudo_split: out must be a 4-byte aligned device buffer"); return SRJ_EINVAL; }
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
  for (int32_t c = 0; c < num_columns; ++c)
    if (out[c].size != total_rows) { set_error("kudo_assemble: column %d: expected %lld rows", c, static_cast<long long>(total_rows)); return SRJ_EINVAL; }
  rc = launch_kudo_assemble(partitions, d_partition_offsets, num_partitions, out, num_columns, total_rows, workspace, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EUNSUPPORTED) set_error("kudo_assemble: only fixed-width, decimal and STRING columns");
  return rc;
}

}  // extern "C"
