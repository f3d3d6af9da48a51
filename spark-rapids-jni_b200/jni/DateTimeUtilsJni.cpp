// DateTimeUtilsJni.cpp -- com.nvidia.spark.rapids.jni.DateTimeUtils over libsrj_b200.so: the four natives of
// DateTimeUtils.java (reference DateTimeUtilsJni.cpp).  Inputs: cudf::column_view* handles of TIMESTAMP_DAYS or
// TIMESTAMP_MICROSECONDS (and a STRING format column, or a format jstring); output: a heap cudf::column* of the datetime's
// type.  The rebase keeps the input's null mask and null count; a truncation's result carries a mask only when it has
// nulls, as the reference's does.  A null handle throws NullPointerException; a null jstring is an empty format (all
// null); C-ABI errors map to the classes of srj_jni_common.hpp.
#include <cstring>

#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

jlong rebase(JNIEnv* env, int32_t direction, jlong input)
{
  if (!input) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& view    = *reinterpret_cast<cudf::column_view const*>(input);
    const srj_column in = to_srj(view);
    const int64_t n     = view.size();
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * (in.type_id == SRJ_TIMESTAMP_DAYS ? 4 : 8), stream);
    rmm::device_buffer mask = mask_like(in, stream);
    const int st = srj_datetime_rebase(direction, &in, out.data(), static_cast<uint32_t*>(mask.data()), stream.value());
    if (throw_if_error(env, st)) return 0;
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{view.type().id()}, static_cast<cudf::size_type>(n), std::move(out),
                                                           std::move(mask), view.null_count()));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

// format_col or format (format_len bytes) as srj_datetime_truncate takes them
jlong truncate(JNIEnv* env, jlong datetime, const srj_column* format_col, const char* format, int32_t format_len)
{
  auto const& view    = *reinterpret_cast<cudf::column_view const*>(datetime);
  const srj_column dt = to_srj(view);
  const int64_t n     = format_col ? format_col->size : view.size();
  auto stream         = cudf::get_default_stream();
  rmm::device_buffer out(static_cast<size_t>(n) * (dt.type_id == SRJ_TIMESTAMP_DAYS ? 4 : 8), stream);
  rmm::device_buffer mask(static_cast<size_t>((n + 31) / 32) * 4, stream);
  int64_t nulls = 0;
  const int st  = srj_datetime_truncate(&dt, format_col, format, format_len, out.data(), static_cast<uint32_t*>(mask.data()), &nulls,
                                        stream.value());
  if (throw_if_error(env, st)) return 0;
  if (nulls < 0) nulls = view.null_count();                   // the scalar format kept the input's mask
  if (nulls == 0) mask = rmm::device_buffer(0, stream);
  return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{view.type().id()}, static_cast<cudf::size_type>(n), std::move(out),
                                                         std::move(mask), static_cast<cudf::size_type>(nulls)));
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_DateTimeUtils_rebaseGregorianToJulian(JNIEnv* env, jclass, jlong input)
{
  return rebase(env, SRJ_DATETIME_GREGORIAN_TO_JULIAN, input);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_DateTimeUtils_rebaseJulianToGregorian(JNIEnv* env, jclass, jlong input)
{
  return rebase(env, SRJ_DATETIME_JULIAN_TO_GREGORIAN, input);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_DateTimeUtils_truncateWithColumnFormat(JNIEnv* env, jclass, jlong datetime,
                                                                                                jlong format)
{
  if (!datetime) { throw_java(env, "java/lang/NullPointerException", "input datetime is null"); return 0; }
  if (!format) { throw_java(env, "java/lang/NullPointerException", "input format is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    const srj_column fmt = to_srj(*reinterpret_cast<cudf::column_view const*>(format));
    return truncate(env, datetime, &fmt, nullptr, 0);
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_DateTimeUtils_truncateWithScalarFormat(JNIEnv* env, jclass, jlong datetime,
                                                                                                jstring format)
{
  if (!datetime) { throw_java(env, "java/lang/NullPointerException", "input datetime is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    const char* chars = format ? env->GetStringUTFChars(format, nullptr) : nullptr;   // as native_jstring reads it
    if (format && !chars) return 0;                                                    // OutOfMemoryError is pending
    std::string fmt = chars ? std::string(chars, std::strlen(chars)) : std::string();
    if (chars) env->ReleaseStringUTFChars(format, chars);
    return truncate(env, datetime, nullptr, fmt.c_str(), static_cast<int32_t>(fmt.size()));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
