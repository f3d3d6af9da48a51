// IcebergBucketJni.cpp -- com.nvidia.spark.rapids.jni.iceberg.IcebergBucket over libsrj_b200.so: the native of
// IcebergBucket.java (reference iceberg/IcebergBucketJni.cpp).  Input: one cudf::column_view* (INT32, INT64, DECIMAL32/64/128,
// TIMESTAMP_DAYS, TIMESTAMP_MICROSECONDS, STRING or LIST<UINT8>); output: a heap cudf::column* INT32 with the input's null
// mask and null count.  IcebergBucket.java rejects numBuckets <= 0 before the call; a null handle throws
// NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

using namespace srjshim;

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_iceberg_IcebergBucket_computeBucket(JNIEnv* env, jclass, jlong input_column,
                                                                                            jint num_buckets)
{
  if (!input_column) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& view = *reinterpret_cast<cudf::column_view const*>(input_column);
    srj_column child{};
    const srj_column in = to_srj_any(view, &child);
    const int64_t n     = view.size();
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * 4, stream);
    rmm::device_buffer mask = mask_like(in, stream);
    const int st = srj_iceberg_bucket(&in, num_buckets, static_cast<int32_t*>(out.data()), static_cast<uint32_t*>(mask.data()), stream.value());
    if (throw_if_error(env, st)) return 0;
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::INT32}, static_cast<cudf::size_type>(n),
                                                           std::move(out), std::move(mask), view.null_count()));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
