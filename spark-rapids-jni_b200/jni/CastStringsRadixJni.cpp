// CastStringsRadixJni.cpp -- CastStrings' radix casts over libsrj_b200.so: fromLongToBinary, fromIntegersWithBase and
// bytesToHex of CastStrings.java (reference CastStringJni.cpp:168-182, 255-321).  Each takes one cudf::column_view* and
// returns a heap STRING cudf::column* with the input's null mask and null count:
//   fromLongToBinary     INT64 -> binary digits
//   fromIntegersWithBase INT8..UINT64, base 10 or 16 -> decimal / upper-case hex; another base throws the reference's
//                        com.nvidia.spark.rapids.jni.CastException on row 0
//   bytesToHex           STRING or LIST<UINT8> -> two upper-case hex digits a byte
// A null handle throws NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include <string>

#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

// CATCH_CAST_EXCEPTION (CastStringJni.cpp:39-60): CastException(String, int)
void throw_cast_error(JNIEnv* env, const std::string& msg, jint row)
{
  if (env->ExceptionCheck()) return;
  jclass cls = env->FindClass("com/nvidia/spark/rapids/jni/CastException");
  if (!cls) return;
  jmethodID ctor = env->GetMethodID(cls, "<init>", "(Ljava/lang/String;I)V");
  if (!ctor) return;
  jstring jmsg = env->NewStringUTF(msg.c_str());
  if (!jmsg) return;
  jobject ex = env->NewObject(cls, ctor, jmsg, row);
  if (ex) env->Throw(static_cast<jthrowable>(ex));
}

// sizes, chars, write: one STRING column from `in` (whose descriptor `in` describes view)
template <class Sizes, class Write>
jlong strings_from(JNIEnv* env, const cudf::column_view& view, const srj_column& in, int64_t ws_bytes, Sizes sizes, Write write)
{
  const int64_t n = in.size;
  auto stream     = cudf::get_default_stream();
  rmm::device_buffer offsets(static_cast<size_t>(n + 1) * 4, stream);
  rmm::device_buffer workspace(static_cast<size_t>(ws_bytes), stream);
  int64_t total = 0;
  int st        = sizes(static_cast<int32_t*>(offsets.data()), &total, workspace.data(), stream.value());
  if (throw_if_error(env, st)) return 0;
  rmm::device_buffer chars(static_cast<size_t>(total), stream);
  rmm::device_buffer mask = mask_like(in, stream);
  srj_column out{};
  out.type_id   = SRJ_STRING;
  out.size      = n;
  out.data      = chars.data();
  out.offsets   = static_cast<int32_t*>(offsets.data());
  out.null_mask = static_cast<uint32_t*>(mask.data());
  st            = write(&out, stream.value());
  if (throw_if_error(env, st)) return 0;
  auto offsets_col = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::INT32}, static_cast<cudf::size_type>(n + 1),
                                                    std::move(offsets), rmm::device_buffer{}, 0);
  return release_as_jlong(cudf::make_strings_column(static_cast<cudf::size_type>(n), std::move(offsets_col), std::move(chars),
                                                    view.null_count(), std::move(mask)));
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_CastStrings_fromLongToBinary(JNIEnv* env, jclass, jlong input_column)
{
  if (!input_column) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& view   = *reinterpret_cast<cudf::column_view const*>(input_column);
    const srj_column in = to_srj(view);
    return strings_from(
      env, view, in, srj_long_to_binary_workspace_bytes(in.size),
      [&](int32_t* offs, int64_t* total, void* ws, void* s) { return srj_long_to_binary_sizes(&in, offs, total, ws, s); },
      [&](const srj_column* out, void* s) { return srj_long_to_binary(&in, out, s); });
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_CastStrings_fromIntegersWithBase(JNIEnv* env, jclass, jlong input_column, jint base)
{
  if (!input_column) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }
  try {
    if (base != 10 && base != 16) {
      throw_cast_error(env, "Bases supported 10, 16; Actual: " + std::to_string(base), 0);
      return 0;
    }
    cudf::jni::auto_set_device(env);
    auto const& view   = *reinterpret_cast<cudf::column_view const*>(input_column);
    const srj_column in = to_srj(view);
    return strings_from(
      env, view, in, srj_integers_to_string_workspace_bytes(in.size),
      [&](int32_t* offs, int64_t* total, void* ws, void* s) { return srj_integers_to_string_sizes(&in, base, offs, total, ws, s); },
      [&](const srj_column* out, void* s) { return srj_integers_to_string(&in, base, out, s); });
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_CastStrings_bytesToHex(JNIEnv* env, jclass, jlong input_column)
{
  if (!input_column) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& view = *reinterpret_cast<cudf::column_view const*>(input_column);
    srj_column child{};
    const srj_column in = to_srj_any(view, &child);
    return strings_from(
      env, view, in, 0, [&](int32_t* offs, int64_t* total, void*, void* s) { return srj_bytes_to_hex_sizes(&in, offs, total, s); },
      [&](const srj_column* out, void* s) { return srj_bytes_to_hex(&in, out, s); });
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
