// NumberConverterJni.cpp -- com.nvidia.spark.rapids.jni.NumberConverter over libsrj_b200.so: the two natives of
// NumberConverter.java (reference NumberConverterJni.cpp).  `input` is a cudf::column_view* (STRING) when is_input_cv,
// else a cudf::string_scalar*; each base is a cudf::column_view* (INT32) when its flag is set, else the int itself.
// convert returns a heap STRING cudf::column* with a null mask only when it has nulls; isConvertOverflow returns whether
// a row overflows under Spark's ANSI rule.  A null handle throws NullPointerException, a null scalar input
// CudfException (the reference's CUDF_EXPECTS), C-ABI errors the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"
#ifndef SRJ_JNI_STUBS
#include <cudf/scalar/scalar.hpp>
#endif

using namespace srjshim;

namespace {

// the C-ABI arguments of one call: the input column or scalar bytes, and each base as a column or an int
struct ConvCall {
  srj_column in{}, from{}, to{};
  const srj_column *pin = nullptr, *pfrom = nullptr, *pto = nullptr;
  const uint8_t* scalar = nullptr;
  int32_t scalar_len = 0, from_int = 0, to_int = 0;
  int64_t rows = 0;
};

bool conv_call(JNIEnv* env, jlong input, jboolean is_input_cv, jlong from_base, jboolean is_from_cv, jlong to_base, jboolean is_to_cv,
               rmm::cuda_stream_view stream, ConvCall* c)
{
  if (!input) { throw_java(env, "java/lang/NullPointerException", "input column/scalar handle is null"); return false; }
  if (is_from_cv && !from_base) { throw_java(env, "java/lang/NullPointerException", "from_base column handle is null"); return false; }
  if (is_to_cv && !to_base) { throw_java(env, "java/lang/NullPointerException", "to_base column handle is null"); return false; }
  if (is_input_cv) {
    c->in  = to_srj(*reinterpret_cast<cudf::column_view const*>(input));
    c->pin = &c->in;
  } else {
    auto const& s = *reinterpret_cast<cudf::string_scalar const*>(input);
    c->scalar     = reinterpret_cast<const uint8_t*>(s.data());
    c->scalar_len = s.is_valid(stream) ? s.size() : -1;   // a null scalar is the C ABI's SRJ_EINVAL
  }
  if (is_from_cv) {
    c->from  = to_srj(*reinterpret_cast<cudf::column_view const*>(from_base));
    c->pfrom = &c->from;
  } else {
    c->from_int = static_cast<int32_t>(from_base);
  }
  if (is_to_cv) {
    c->to  = to_srj(*reinterpret_cast<cudf::column_view const*>(to_base));
    c->pto = &c->to;
  } else {
    c->to_int = static_cast<int32_t>(to_base);
  }
  c->rows = c->pin ? c->in.size : c->pfrom ? c->from.size : c->pto ? c->to.size : 0;
  return true;
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_NumberConverter_convert(JNIEnv* env, jclass, jlong input, jboolean is_input_cv,
                                                                                 jlong from_base, jboolean is_from_cv, jlong to_base,
                                                                                 jboolean is_to_cv)
{
  try {
    cudf::jni::auto_set_device(env);
    auto stream = cudf::get_default_stream();
    ConvCall c;
    if (!conv_call(env, input, is_input_cv, from_base, is_from_cv, to_base, is_to_cv, stream, &c)) return 0;
    const int64_t n = c.rows;
    rmm::device_buffer offsets(static_cast<size_t>(n + 1) * 4, stream);
    rmm::device_buffer mask(static_cast<size_t>((n + 31) / 32) * 4, stream);
    rmm::device_buffer workspace(static_cast<size_t>(srj_conv_workspace_bytes(n)), stream);
    int64_t nulls = 0, total = 0;
    int st = srj_conv_sizes(c.pin, c.scalar, c.scalar_len, c.pfrom, c.from_int, c.pto, c.to_int, static_cast<int32_t*>(offsets.data()),
                            static_cast<uint32_t*>(mask.data()), &nulls, &total, workspace.data(), stream.value());
    if (throw_if_error(env, st)) return 0;
    rmm::device_buffer chars(static_cast<size_t>(total), stream);
    st = srj_conv(c.pin, c.scalar, c.scalar_len, c.pfrom, c.from_int, c.pto, c.to_int, static_cast<const int32_t*>(offsets.data()),
                  static_cast<uint8_t*>(chars.data()), workspace.data(), stream.value());
    if (throw_if_error(env, st)) return 0;
    auto offsets_col = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::INT32}, static_cast<cudf::size_type>(n + 1),
                                                      std::move(offsets), rmm::device_buffer{}, 0);
    return release_as_jlong(cudf::make_strings_column(static_cast<cudf::size_type>(n), std::move(offsets_col), std::move(chars),
                                                      static_cast<cudf::size_type>(nulls), nulls ? std::move(mask) : rmm::device_buffer{}));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jboolean JNICALL Java_com_nvidia_spark_rapids_jni_NumberConverter_isConvertOverflow(JNIEnv* env, jclass, jlong input,
                                                                                             jboolean is_input_cv, jlong from_base,
                                                                                             jboolean is_from_cv, jlong to_base,
                                                                                             jboolean is_to_cv)
{
  try {
    cudf::jni::auto_set_device(env);
    auto stream = cudf::get_default_stream();
    ConvCall c;
    if (!conv_call(env, input, is_input_cv, from_base, is_from_cv, to_base, is_to_cv, stream, &c)) return 0;
    int32_t overflow = 0;
    const int st = srj_conv_overflow(c.pin, c.scalar, c.scalar_len, c.pfrom, c.from_int, c.pto, c.to_int, &overflow, stream.value());
    if (throw_if_error(env, st)) return 0;
    return overflow ? 1 : 0;
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
