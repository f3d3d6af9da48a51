// IcebergDateTimeUtilJni.cpp -- com.nvidia.spark.rapids.jni.iceberg.IcebergDateTimeUtil over libsrj_b200.so: the four
// natives of IcebergDateTimeUtil.java (reference iceberg/IcebergDateTimeUtilJni.cpp).  Input: one cudf::column_view* of
// type TIMESTAMP_DAYS (not for hours) or TIMESTAMP_MICROSECONDS, which IcebergDateTimeUtil.java checks before the call;
// output: a heap cudf::column* INT32 (TIMESTAMP_DAYS for daysFromEpoch) with the input's null mask and null count.  A null
// handle throws NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

jlong datetime(JNIEnv* env, int32_t transform, jlong input)
{
  if (!input) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& view    = *reinterpret_cast<cudf::column_view const*>(input);
    const srj_column in = to_srj(view);
    const int64_t n     = view.size();
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * 4, stream);
    rmm::device_buffer mask = mask_like(in, stream);
    const int st = srj_iceberg_datetime(transform, &in, static_cast<int32_t*>(out.data()), static_cast<uint32_t*>(mask.data()), stream.value());
    if (throw_if_error(env, st)) return 0;
    const auto out_type = transform == SRJ_ICEBERG_DAYS ? cudf::type_id::TIMESTAMP_DAYS : cudf::type_id::INT32;
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{out_type}, static_cast<cudf::size_type>(n), std::move(out),
                                                           std::move(mask), view.null_count()));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_iceberg_IcebergDateTimeUtil_yearsFromEpoch(JNIEnv* env, jclass, jlong input)
{
  return datetime(env, SRJ_ICEBERG_YEARS, input);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_iceberg_IcebergDateTimeUtil_monthsFromEpoch(JNIEnv* env, jclass, jlong input)
{
  return datetime(env, SRJ_ICEBERG_MONTHS, input);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_iceberg_IcebergDateTimeUtil_daysFromEpoch(JNIEnv* env, jclass, jlong input)
{
  return datetime(env, SRJ_ICEBERG_DAYS, input);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_iceberg_IcebergDateTimeUtil_hoursFromEpoch(JNIEnv* env, jclass, jlong input)
{
  return datetime(env, SRJ_ICEBERG_HOURS, input);
}

}  // extern "C"
