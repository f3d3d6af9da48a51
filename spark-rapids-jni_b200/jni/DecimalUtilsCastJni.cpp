// DecimalUtilsCastJni.cpp -- DecimalUtils.floatingPointToDecimal over libsrj_b200.so (reference DecimalUtilsJni.cpp:118-137):
// Spark's CAST(float / double AS DECIMAL).  Together with DecimalUtilsJni.cpp this library defines all six natives of
// DecimalUtils.java; the JVM resolves natives from any translation unit of the loaded library.
// Input: a cudf::column_view* of FLOAT32 or FLOAT64, the output's cudf type id, precision and scale.  Output: a jlongArray
// of the heap cudf::column* of the decimal type, with a null mask only when it has nulls, and the smallest failing row
// (-1: none).  A null handle throws NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

using namespace srjshim;

extern "C" {

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_DecimalUtils_floatingPointToDecimal(JNIEnv* env, jclass, jlong j_input,
                                                                                                 jint output_type_id, jint precision,
                                                                                                 jint decimal_scale)
{
  if (!j_input) { throw_java(env, "java/lang/NullPointerException", "j_input is null"); return nullptr; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& view    = *reinterpret_cast<cudf::column_view const*>(j_input);
    const srj_column in = to_srj(view);
    const int64_t n     = view.size();
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer data(static_cast<size_t>(n) * static_cast<size_t>(size_of_type(output_type_id)), stream);
    rmm::device_buffer mask(static_cast<size_t>((n + 31) / 32) * 4, stream);
    int64_t nulls = 0, failure_row = -1;
    const int st = srj_float_to_fixed_point(&in, output_type_id, precision, decimal_scale, data.data(), static_cast<uint32_t*>(mask.data()),
                                            &nulls, &failure_row, stream.value());
    if (throw_if_error(env, st)) return nullptr;
    const cudf::data_type type(static_cast<cudf::type_id>(output_type_id), decimal_scale);
    auto col = std::make_unique<cudf::column>(type, static_cast<cudf::size_type>(n), std::move(data),
                                              nulls ? std::move(mask) : rmm::device_buffer{}, static_cast<cudf::size_type>(nulls));
    jlongArray arr = env->NewLongArray(2);
    if (!arr) return nullptr;
    const jlong out[2] = {release_as_jlong(std::move(col)), static_cast<jlong>(failure_row)};
    env->SetLongArrayRegion(arr, 0, 2, out);
    return arr;
  } catch (...) {
    throw_from_exception(env);
  }
  return nullptr;
}

}  // extern "C"
