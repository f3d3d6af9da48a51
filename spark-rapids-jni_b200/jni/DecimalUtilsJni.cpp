// DecimalUtilsJni.cpp -- com.nvidia.spark.rapids.jni.DecimalUtils over libsrj_b200.so: the five arithmetic natives of
// DecimalUtils.java (reference DecimalUtilsJni.cpp).  Inputs: two cudf::column_view* of DECIMAL128; output: a jlongArray
// of two heap cudf::column* -- BOOL8 overflow flags and the result (DECIMAL128 at the requested scale, INT64 for an
// integral divide) -- each with the AND of the input masks and its null count.  floatingPointToDecimal, the sixth
// native, is bound in DecimalUtilsCastJni.cpp.  A null handle throws NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

jlongArray binary(JNIEnv* env, jlong ha, jlong hb, int32_t op, jint scale, bool interim_cast)
{
  if (!ha || !hb) { throw_java(env, "java/lang/NullPointerException", "column is null"); return nullptr; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& va     = *reinterpret_cast<cudf::column_view const*>(ha);
    auto const& vb     = *reinterpret_cast<cudf::column_view const*>(hb);
    const srj_column a = to_srj(va), b = to_srj(vb);
    const int64_t n    = va.size();
    auto stream        = cudf::get_default_stream();
    const bool masked  = a.null_mask || b.null_mask;
    const size_t mask_bytes = masked ? static_cast<size_t>((n + 31) / 32) * 4 : 0;
    rmm::device_buffer ovf(static_cast<size_t>(n), stream);
    rmm::device_buffer out(static_cast<size_t>(n) * (op == SRJ_DECIMAL_INTEGER_DIVIDE ? 8 : 16), stream);
    rmm::device_buffer mask(mask_bytes, stream);
    int64_t nulls = 0;
    const int st  = srj_decimal128_binary(op, &a, &b, scale, interim_cast ? 1 : 0, static_cast<uint8_t*>(ovf.data()), out.data(),
                                          static_cast<uint32_t*>(mask.data()), &nulls, stream.value());
    if (throw_if_error(env, st)) return nullptr;
    rmm::device_buffer mask2 = masked ? rmm::device_buffer(mask.data(), mask_bytes, stream) : rmm::device_buffer();
    const auto rows          = static_cast<cudf::size_type>(n);
    const auto nc            = static_cast<cudf::size_type>(nulls);
    const cudf::data_type out_type = op == SRJ_DECIMAL_INTEGER_DIVIDE ? cudf::data_type{cudf::type_id::INT64}
                                                                      : cudf::data_type{cudf::type_id::DECIMAL128, scale};
    auto c0 = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::BOOL8}, rows, std::move(ovf), std::move(mask), nc);
    auto c1 = std::make_unique<cudf::column>(out_type, rows, std::move(out), std::move(mask2), nc);
    jlongArray arr = env->NewLongArray(2);
    if (!arr) return nullptr;
    const jlong handles[2] = {release_as_jlong(std::move(c0)), release_as_jlong(std::move(c1))};
    env->SetLongArrayRegion(arr, 0, 2, handles);
    return arr;
  } catch (...) {
    throw_from_exception(env);
  }
  return nullptr;
}

}  // namespace

extern "C" {

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_DecimalUtils_multiply128(JNIEnv* env, jclass, jlong a, jlong b, jint product_scale,
                                                                                      jboolean interim_cast)
{
  return binary(env, a, b, SRJ_DECIMAL_MULTIPLY, product_scale, interim_cast != 0);
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_DecimalUtils_divide128(JNIEnv* env, jclass, jlong a, jlong b, jint quotient_scale,
                                                                                    jboolean is_integer_divide)
{
  return binary(env, a, b, is_integer_divide ? SRJ_DECIMAL_INTEGER_DIVIDE : SRJ_DECIMAL_DIVIDE, quotient_scale, false);
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_DecimalUtils_remainder128(JNIEnv* env, jclass, jlong a, jlong b, jint remainder_scale)
{
  return binary(env, a, b, SRJ_DECIMAL_REMAINDER, remainder_scale, false);
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_DecimalUtils_add128(JNIEnv* env, jclass, jlong a, jlong b, jint target_scale)
{
  return binary(env, a, b, SRJ_DECIMAL_ADD, target_scale, false);
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_DecimalUtils_subtract128(JNIEnv* env, jclass, jlong a, jlong b, jint target_scale)
{
  return binary(env, a, b, SRJ_DECIMAL_SUBTRACT, target_scale, false);
}

}  // extern "C"
