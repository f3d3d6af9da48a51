// GpuTimeZoneDBJni.cpp -- com.nvidia.spark.rapids.jni.GpuTimeZoneDB over libsrj_b200.so: the four natives of
// GpuTimeZoneDB.java (reference GpuTimeZoneDBJni.cpp).  Inputs: cudf::column_view* and cudf::table_view* handles (the
// time zone table of GpuTimeZoneDB.getTimezoneInfo, or an ORC zone's (transitions, offsets) table); output: a heap
// cudf::column*.  The single-zone and ORC conversions keep the input's type, mask and null count; the per-row-zone cast
// returns TIMESTAMP_MICROSECONDS with a mask only when a row is null.  A null handle throws NullPointerException, except
// ORC's two tables (a null one is a fixed offset); C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

jlong convert(JNIEnv* env, int32_t direction, jlong input, jlong tz_info, jint tz_index)
{
  if (!input || !tz_info) { throw_java(env, "java/lang/NullPointerException", "column is null"); return 0; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& view = *reinterpret_cast<cudf::column_view const*>(input);
    auto const& info = *reinterpret_cast<cudf::table_view const*>(tz_info);
    if (info.num_columns() < 2) { throw_java(env, "ai/rapids/cudf/CudfException", "the timezone info table needs two columns"); return 0; }
    const srj_column in = to_srj(view);
    TzTable t;
    to_srj_table(info, &t);
    const int64_t n = view.size();
    auto stream     = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * 8, stream);
    rmm::device_buffer mask = mask_like(in, stream);
    const int st = srj_timezone_convert(direction, &in, &t.fixed, &t.dst, tz_index, out.data(), static_cast<uint32_t*>(mask.data()),
                                        stream.value());
    if (throw_if_error(env, st)) return 0;
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{view.type().id()}, static_cast<cudf::size_type>(n), std::move(out),
                                                           std::move(mask), view.null_count()));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_GpuTimeZoneDB_convertTimestampColumnToUTC(JNIEnv* env, jclass, jlong input,
                                                                                                   jlong tz_info, jint tz_index)
{
  return convert(env, SRJ_TIMEZONE_TO_UTC, input, tz_info, tz_index);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_GpuTimeZoneDB_convertUTCTimestampColumnToTimeZone(JNIEnv* env, jclass, jlong input,
                                                                                                           jlong tz_info, jint tz_index)
{
  return convert(env, SRJ_TIMEZONE_FROM_UTC, input, tz_info, tz_index);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_GpuTimeZoneDB_convertTimestampColumnToUTCWithTzCv(
  JNIEnv* env, jclass, jlong seconds, jlong micros, jlong invalid, jlong tz_type, jlong tz_offset, jlong tz_info, jlong tz_indices)
{
  const jlong handles[7]     = {seconds, micros, invalid, tz_type, tz_offset, tz_info, tz_indices};
  const char* const names[7] = {"seconds column is null", "microseconds column is null", "invalid column is null", "tz type column is null",
                                "tz offset column is null", "timezone info table is null", "tz indices column is null"};
  for (int i = 0; i < 7; ++i)
    if (!handles[i]) { throw_java(env, "java/lang/NullPointerException", names[i]); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    srj_column cols[6];
    const jlong col_handles[6] = {seconds, micros, invalid, tz_type, tz_offset, tz_indices};
    for (int i = 0; i < 6; ++i) cols[i] = to_srj(*reinterpret_cast<cudf::column_view const*>(col_handles[i]));
    auto const& info = *reinterpret_cast<cudf::table_view const*>(tz_info);
    if (info.num_columns() < 2) { throw_java(env, "ai/rapids/cudf/CudfException", "the timezone info table needs two columns"); return 0; }
    TzTable t;
    to_srj_table(info, &t);
    const int64_t n = cols[0].size;
    auto stream     = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * 8, stream);
    rmm::device_buffer mask(static_cast<size_t>((n + 31) / 32) * 4, stream);
    int64_t nulls = 0;
    const int st  = srj_timezone_convert_multi(&cols[0], &cols[1], &cols[2], &cols[3], &cols[4], &t.fixed, &t.dst, &cols[5],
                                               static_cast<int64_t*>(out.data()), static_cast<uint32_t*>(mask.data()), &nulls, stream.value());
    if (throw_if_error(env, st)) return 0;
    if (nulls == 0) mask = rmm::device_buffer(0, stream);                          // a mask only when some row is null
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::TIMESTAMP_MICROSECONDS}, static_cast<cudf::size_type>(n),
                                                           std::move(out), std::move(mask), static_cast<cudf::size_type>(nulls)));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_GpuTimeZoneDB_convertOrcTimezones(JNIEnv* env, jclass, jlong input, jlong writer_table,
                                                                                           jint writer_raw_offset, jlong reader_table,
                                                                                           jint reader_raw_offset)
{
  if (!input) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& view   = *reinterpret_cast<cudf::column_view const*>(input);
    const srj_column in = to_srj(view);
    srj_column tables[2][2]{};
    const jlong handles[2] = {writer_table, reader_table};
    for (int i = 0; i < 2; ++i) {
      if (!handles[i]) continue;
      auto const& t = *reinterpret_cast<cudf::table_view const*>(handles[i]);
      if (t.num_columns() < 2) { throw_java(env, "ai/rapids/cudf/CudfException", "an ORC time zone table needs two columns"); return 0; }
      tables[i][0] = to_srj(t.column(0));
      tables[i][1] = to_srj(t.column(1));
    }
    const int64_t n = view.size();
    auto stream     = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * 8, stream);
    rmm::device_buffer mask = mask_like(in, stream);
    const int st = srj_orc_convert_timezones(&in, writer_table ? &tables[0][0] : nullptr, writer_table ? &tables[0][1] : nullptr, writer_raw_offset,
                                             reader_table ? &tables[1][0] : nullptr, reader_table ? &tables[1][1] : nullptr, reader_raw_offset,
                                             out.data(), static_cast<uint32_t*>(mask.data()), stream.value());
    if (throw_if_error(env, st)) return 0;
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{view.type().id()}, static_cast<cudf::size_type>(n), std::move(out),
                                                           std::move(mask), view.null_count()));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
