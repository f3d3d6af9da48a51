// ZOrderJni.cpp -- com.nvidia.spark.rapids.jni.ZOrder over libsrj_b200.so: the two natives of ZOrder.java:85-87
// (reference ZOrderJni.cpp).  Inputs: a jlongArray of cudf::column_view*.  Outputs:
//   interleaveBits -> a heap cudf::column* LIST<UINT8> (INT32 offsets child, UINT8 child, no null mask)
//   hilbertIndex   -> a heap cudf::column* INT64 (no null mask)
// ZOrder.java handles zero columns itself; here they reach the C ABI, which rejects them (CudfException).  A null handle
// throws NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

// the views behind the handles; false when it threw
bool views_of(JNIEnv* env, jlongArray handles, std::vector<srj_column>* cols, int64_t* rows)
{
  if (!handles) { throw_java(env, "java/lang/NullPointerException", "array of column handles is null"); return false; }
  const int nc = env->GetArrayLength(handles);
  cols->resize(nc);
  *rows    = 0;
  jlong* h = env->GetLongArrayElements(handles, nullptr);
  for (int c = 0; c < nc; ++c) {
    auto const* v = reinterpret_cast<cudf::column_view const*>(h[c]);
    if (!v) {
      env->ReleaseLongArrayElements(handles, h, JNI_ABORT);
      throw_java(env, "java/lang/NullPointerException", "column handle is null");
      return false;
    }
    (*cols)[c] = to_srj(*v);
    if (c == 0) *rows = v->size();
  }
  env->ReleaseLongArrayElements(handles, h, JNI_ABORT);
  return true;
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_ZOrder_interleaveBits(JNIEnv* env, jclass, jlongArray handles)
{
  try {
    cudf::jni::auto_set_device(env);
    std::vector<srj_column> cols;
    int64_t n = 0;
    if (!views_of(env, handles, &cols, &n)) return 0;
    const int32_t nc = static_cast<int32_t>(cols.size());
    int64_t total    = 0;
    int st           = srj_interleave_bits_sizes(cols.data(), nc, n, &total);
    if (throw_if_error(env, st)) return 0;
    auto stream = cudf::get_default_stream();
    rmm::device_buffer offsets(static_cast<size_t>(n + 1) * 4, stream);
    rmm::device_buffer bytes(static_cast<size_t>(total), stream);
    st = srj_interleave_bits(cols.data(), nc, n, static_cast<int32_t*>(offsets.data()), static_cast<uint8_t*>(bytes.data()), stream.value());
    if (throw_if_error(env, st)) return 0;
    auto offsets_col = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::INT32}, static_cast<cudf::size_type>(n + 1),
                                                      std::move(offsets), rmm::device_buffer{}, 0);
    auto bytes_col   = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::UINT8}, static_cast<cudf::size_type>(total),
                                                      std::move(bytes), rmm::device_buffer{}, 0);
    return release_as_jlong(cudf::make_lists_column(static_cast<cudf::size_type>(n), std::move(offsets_col), std::move(bytes_col), 0,
                                                    rmm::device_buffer{}));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_ZOrder_hilbertIndex(JNIEnv* env, jclass, jint numBits, jlongArray handles)
{
  try {
    cudf::jni::auto_set_device(env);
    std::vector<srj_column> cols;
    int64_t n = 0;
    if (!views_of(env, handles, &cols, &n)) return 0;
    auto stream = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * 8, stream);
    const int st = srj_hilbert_index(numBits, cols.data(), static_cast<int32_t>(cols.size()), n, static_cast<int64_t*>(out.data()),
                                     stream.value());
    if (throw_if_error(env, st)) return 0;
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::INT64}, static_cast<cudf::size_type>(n),
                                                           std::move(out), rmm::device_buffer{}, 0));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
