// CastStringsJni.cpp -- com.nvidia.spark.rapids.jni.CastStrings' string-to-timestamp and string-to-date natives over
// libsrj_b200.so (reference CastStringJni.cpp:323-376).  Inputs: cudf::column_view* (the strings, the STRUCT<STRING, INT32>
// zone name map) and a cudf::table_view* (GpuTimeZoneDB.getTimezoneInfo's table); output: a heap cudf::column*, the
// six-field STRUCT of the first phase or a TIMESTAMP_DAYS column with a mask only when a row is null.  The current time
// that dates a string holding a time alone is read here, as the reference reads it.  A null handle throws
// NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

#include <chrono>

using namespace srjshim;

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_CastStrings_parseTimestampStringsToIntermediate(
  JNIEnv* env, jclass, jlong input_column, jint default_timezone_index, jlong default_epoch_day, jlong tz_name_to_index_map,
  jlong timezone_info_table, jint platform, jint major, jint minor, jint patch)
{
  if (!input_column) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }   // JNI_NULL_CHECK
  if (!tz_name_to_index_map) { throw_java(env, "java/lang/NullPointerException", "timezone name to index column is null"); return 0; }
  if (!timezone_info_table) { throw_java(env, "java/lang/NullPointerException", "timezone info table is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& view = *reinterpret_cast<cudf::column_view const*>(input_column);
    auto const& map  = *reinterpret_cast<cudf::column_view const*>(tz_name_to_index_map);
    auto const& info = *reinterpret_cast<cudf::table_view const*>(timezone_info_table);
    if (info.num_columns() < 2) { throw_java(env, "ai/rapids/cudf/CudfException", "the timezone info table needs two columns"); return 0; }
    const srj_column in = to_srj(view);
    srj_column fields[2]{};
    srj_column names{};
    names.type_id = static_cast<int32_t>(map.type().id());
    for (int i = 0; i < 2 && i < map.num_children(); ++i) fields[i] = to_srj(map.child(i));
    names.size         = map.size();
    names.children     = fields;
    names.num_children = map.num_children() < 2 ? map.num_children() : 2;
    TzTable t;
    to_srj_table(info, &t);
    const int64_t n  = view.size();
    auto stream      = cudf::get_default_stream();
    const int64_t now = std::chrono::duration_cast<std::chrono::seconds>(std::chrono::system_clock::now().time_since_epoch()).count();
    static const int32_t widths[6]          = {1, 8, 4, 1, 4, 4};
    static const cudf::type_id types[6]     = {cudf::type_id::UINT8, cudf::type_id::INT64, cudf::type_id::INT32, cudf::type_id::UINT8,
                                               cudf::type_id::INT32, cudf::type_id::INT32};
    std::vector<rmm::device_buffer> bufs;
    for (int i = 0; i < 6; ++i) bufs.emplace_back(static_cast<size_t>(n) * widths[i], stream);
    const int st = srj_cast_parse_timestamps(&in, &names, &t.fixed, &t.dst, default_timezone_index, default_epoch_day, now, platform, major, minor,
                                             patch, static_cast<uint8_t*>(bufs[0].data()), static_cast<int64_t*>(bufs[1].data()),
                                             static_cast<int32_t*>(bufs[2].data()), static_cast<uint8_t*>(bufs[3].data()),
                                             static_cast<int32_t*>(bufs[4].data()), static_cast<int32_t*>(bufs[5].data()), stream.value());
    if (throw_if_error(env, st)) return 0;
    std::vector<std::unique_ptr<cudf::column>> kids;
    for (int i = 0; i < 6; ++i)
      kids.push_back(std::make_unique<cudf::column>(cudf::data_type{types[i]}, static_cast<cudf::size_type>(n), std::move(bufs[i]),
                                                    rmm::device_buffer(0, stream), 0));
    return release_as_jlong(cudf::make_structs_column(static_cast<cudf::size_type>(n), std::move(kids), 0, rmm::device_buffer(0, stream), stream));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_CastStrings_parseDateStringsToDate(JNIEnv* env, jclass, jlong input_column)
{
  if (!input_column) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& view   = *reinterpret_cast<cudf::column_view const*>(input_column);
    const srj_column in = to_srj(view);
    const int64_t n     = view.size();
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(n) * 4, stream);
    rmm::device_buffer mask(static_cast<size_t>((n + 31) / 32) * 4, stream);
    int64_t nulls = 0;
    const int st  = srj_cast_parse_dates(&in, static_cast<int32_t*>(out.data()), static_cast<uint32_t*>(mask.data()), &nulls, stream.value());
    if (throw_if_error(env, st)) return 0;
    if (nulls == 0) mask = rmm::device_buffer(0, stream);                          // a mask only when some row is null
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::TIMESTAMP_DAYS}, static_cast<cudf::size_type>(n),
                                                           std::move(out), std::move(mask), static_cast<cudf::size_type>(nulls)));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
