// srj_jni_common.hpp -- what the two JNI translation units share: status -> Java exception mapping (the classes
// the reference throws, src/main/cpp/src/error.hpp:181-239), a per-schema plan cache, column_view -> srj_column.
#pragma once
#ifdef SRJ_JNI_STUBS
#include "jni_stub.h"
#include "cudf_abi_stub.hpp"
#else
#include <jni.h>
#include <cudf/column/column.hpp>
#include <cudf/column/column_factories.hpp>
#include <cudf/column/column_view.hpp>
#include <cudf/lists/lists_column_view.hpp>
#include <cudf/table/table_view.hpp>
#include <cudf/utilities/default_stream.hpp>
#include <rmm/device_buffer.hpp>
#include "cudf_jni_apis.hpp"
#endif

#include <exception>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/srj_b200.h"

namespace srjshim {

// SRJ_EINVAL / SRJ_EUNSUPPORTED -> CudfException (cudf::logic_error), SRJ_EOVERFLOW -> CudfColumnSizeOverflowException,
// SRJ_ENOMEM -> OutOfMemoryError, SRJ_ECUDA -> CudaException (error.hpp:181-239).  Returns true when it threw.
inline bool throw_if_error(JNIEnv* env, int status)
{
  if (status == SRJ_OK) return false;
  const char* cls = "ai/rapids/cudf/CudfException";
  if (status == SRJ_EOVERFLOW) cls = "ai/rapids/cudf/CudfColumnSizeOverflowException";
  else if (status == SRJ_ENOMEM) cls = "java/lang/OutOfMemoryError";
  else if (status == SRJ_ECUDA) cls = "ai/rapids/cudf/CudaException";
  if (!env->ExceptionCheck()) env->ThrowNew(env->FindClass(cls), srj_last_error());
  return true;
}

inline void throw_java(JNIEnv* env, const char* cls, const char* msg)
{
  if (!env->ExceptionCheck()) env->ThrowNew(env->FindClass(cls), msg);
}

// Throws com.nvidia.spark.rapids.jni.ExceptionWithRowIndex(row) through its (I)V constructor, as the reference's
// CATCH_EXCEPTION_WITH_ROW_INDEX does, after freeing the call's output buffers: an ANSI row error returns no column.
inline void throw_row_index(JNIEnv* env, int64_t row, std::vector<rmm::device_buffer*> outputs)
{
  for (rmm::device_buffer* b : outputs) *b = rmm::device_buffer{};
  if (env->ExceptionCheck()) return;
  jclass cls = env->FindClass("com/nvidia/spark/rapids/jni/ExceptionWithRowIndex");
  if (!cls) return;
  jmethodID ctor = env->GetMethodID(cls, "<init>", "(I)V");
  if (!ctor) return;
  jobject ex = env->NewObject(cls, ctor, static_cast<jint>(row));
  if (ex) env->Throw(static_cast<jthrowable>(ex));
}

// No C++ exception (rmm::out_of_memory, std::bad_alloc, ...) may leave a JNI function: map them to the Java classes.
// Call from a catch (...) block.
inline void throw_from_exception(JNIEnv* env)
{
  try {
    throw;
  } catch (const std::bad_alloc& e) {
    throw_java(env, "java/lang/OutOfMemoryError", e.what());
  } catch (const std::exception& e) {
    throw_java(env, "ai/rapids/cudf/CudfException", e.what());
  } catch (...) {
    throw_java(env, "ai/rapids/cudf/CudfException", "unknown C++ exception");
  }
}

// One srj_plan per (device, schema): plans are immutable and thread-safe, so concurrent Spark tasks share them.
inline const srj_plan* plan_for(const std::vector<int32_t>& types, const std::vector<int32_t>& scales, int* status)
{
  static std::mutex mu;
  static std::map<std::pair<std::vector<int32_t>, std::vector<int32_t>>, srj_plan*> cache;
  std::lock_guard<std::mutex> lk(mu);
  auto key = std::make_pair(types, scales);
  auto it  = cache.find(key);
  if (it != cache.end()) { *status = SRJ_OK; return it->second; }
  srj_plan* p = nullptr;
  *status     = srj_plan_create(types.data(), scales.data(), static_cast<int32_t>(types.size()), &p);
  if (*status == SRJ_OK) cache.emplace(std::move(key), p);
  return p;
}

// The cudf::column_view fields the C ABI reads (include/srj_b200.h: srj_column).  Sliced views are not supported,
// as in the reference (RC:1809-1811 passes raw null_mask()).
inline srj_column to_srj(const cudf::column_view& c)
{
  srj_column s{};
  s.type_id   = static_cast<int32_t>(c.type().id());
  s.scale     = c.type().scale();
  s.size      = c.size();
  s.null_mask = const_cast<uint32_t*>(c.null_mask());
  if (c.type().id() == cudf::type_id::STRING) {
    s.data    = const_cast<char*>(c.head<char>());                       // chars live in the parent's data (RC:1919-1923)
    s.offsets = c.num_children() > 0 ? const_cast<int32_t*>(c.child(0).head<int32_t>()) : nullptr;
  } else {
    s.data = const_cast<uint8_t*>(c.head<uint8_t>());
  }
  return s;
}

// to_srj for any input of the Iceberg transforms: a LIST<UINT8> (binary) column also gets its offsets and its element
// column, described in *child (which must outlive the returned descriptor's use)
inline srj_column to_srj_any(const cudf::column_view& c, srj_column* child)
{
  if (c.type().id() != cudf::type_id::LIST) return to_srj(c);
  srj_column s{};
  s.type_id   = SRJ_LIST;
  s.size      = c.size();
  s.null_mask = const_cast<uint32_t*>(c.null_mask());
  cudf::lists_column_view const lists(c);
  s.offsets          = const_cast<int32_t*>(lists.offsets().head<int32_t>());
  *child             = to_srj(lists.child());
  s.children         = child;
  s.num_children     = 1;
  return s;
}

// the two LIST columns of a time zone table as srj_timezone_convert takes them; the descriptors point into the struct itself
struct TzTable {
  srj_column fixed{}, dst{}, entries{}, fields[3]{}, rules{};
};

inline void to_srj_table(const cudf::table_view& t, TzTable* out)
{
  const cudf::column_view trans = t.column(0), dst = t.column(1);
  out->fixed.type_id = SRJ_LIST;
  out->fixed.size    = trans.size();
  const cudf::lists_column_view tl(trans);
  out->fixed.offsets = const_cast<int32_t*>(tl.offsets().head<int32_t>());
  const cudf::column_view st = tl.child();
  out->entries.type_id       = static_cast<int32_t>(st.type().id());
  out->entries.size          = st.size();
  for (int i = 0; i < 3 && i < st.num_children(); ++i) out->fields[i] = to_srj(st.child(i));
  out->entries.children      = out->fields;
  out->entries.num_children  = st.num_children() < 3 ? st.num_children() : 3;
  out->fixed.children        = &out->entries;
  out->fixed.num_children    = 1;
  out->dst.type_id           = SRJ_LIST;
  out->dst.size              = dst.size();
  const cudf::lists_column_view dl(dst);
  out->dst.offsets      = const_cast<int32_t*>(dl.offsets().head<int32_t>());
  out->rules            = to_srj(dl.child());
  out->dst.children     = &out->rules;
  out->dst.num_children = 1;
}

// a device buffer for a copy of the input's null mask (empty when the input has none)
inline rmm::device_buffer mask_like(const srj_column& in, rmm::cuda_stream_view stream)
{
  return rmm::device_buffer(in.null_mask ? static_cast<size_t>((in.size + 31) / 32) * 4 : 0, stream);
}

inline int32_t size_of_type(int32_t t)
{
  srj_layout l{};
  int32_t st = 0, sz = 0;
  return srj_compute_layout(&t, 1, &l, &st, &sz) == SRJ_OK ? sz : 0;
}

// blocking device -> host copy on `stream` (cudaMemcpyAsync + synchronize in the real build)
bool copy_to_host(void* dst, const void* src, size_t bytes, rmm::cuda_stream_view stream);
bool copy_from_host(void* dst, const void* src, size_t bytes, rmm::cuda_stream_view stream);

template <typename T>
jlong release_as_jlong(std::unique_ptr<T>&& p) { return reinterpret_cast<jlong>(p.release()); }   // jni_utils.hpp:34-46

}  // namespace srjshim
