// ArithmeticJni.cpp -- com.nvidia.spark.rapids.jni.Arithmetic over libsrj_b200.so: the two natives of Arithmetic.java:189-193
// (reference ArithmeticJni.cpp).  multiply's operands are each a cudf::column_view or, when its is*Cv flag is false, a
// cudf::scalar handle; round's input is a cudf::column_view.  Outputs (heap cudf::column*): the operands' type for multiply;
// for round the input's type, a decimal at scale -decimalPlaces (an empty input keeps its type, as the reference's
// empty_like).  An ANSI overflow throws ExceptionWithRowIndex(row) and returns no column; a null handle throws
// NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

#ifndef SRJ_JNI_STUBS
#include <cudf/scalar/scalar.hpp>
#endif

using namespace srjshim;

namespace {

// the C ABI reads a mask as nulls: a column without nulls goes without its mask
srj_column to_srj_nullable(const cudf::column_view& c)
{
  srj_column s = to_srj(c);
  if (c.null_count() == 0) s.null_mask = nullptr;
  return s;
}

template <typename T>
void* scalar_value(const cudf::scalar& s)
{
  return const_cast<T*>(static_cast<cudf::detail::fixed_width_scalar<T> const&>(s).data());
}

// an operand as srj_multiply takes it: a column, or a scalar's device value and device validity (never read on the host)
struct Operand {
  srj_column col{};
  const uint8_t* scalar_valid = nullptr;
};

Operand operand(jlong handle, bool is_cv)
{
  Operand o;
  if (is_cv) {
    o.col = to_srj_nullable(*reinterpret_cast<cudf::column_view const*>(handle));
    return o;
  }
  auto const& s  = *reinterpret_cast<cudf::scalar const*>(handle);
  o.col.type_id  = static_cast<int32_t>(s.type().id());
  o.col.scale    = s.type().scale();
  o.col.size     = 1;
  switch (s.type().id()) {                                     // another type has no value here: the C ABI rejects it
    case cudf::type_id::INT8: o.col.data = scalar_value<int8_t>(s); break;
    case cudf::type_id::INT16: o.col.data = scalar_value<int16_t>(s); break;
    case cudf::type_id::INT32: o.col.data = scalar_value<int32_t>(s); break;
    case cudf::type_id::INT64: o.col.data = scalar_value<int64_t>(s); break;
    case cudf::type_id::FLOAT32: o.col.data = scalar_value<float>(s); break;
    case cudf::type_id::FLOAT64: o.col.data = scalar_value<double>(s); break;
    default: break;
  }
  o.scalar_valid = reinterpret_cast<const uint8_t*>(s.validity_data());
  return o;
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Arithmetic_multiply(JNIEnv* env, jclass, jlong left, jboolean is_left_cv, jlong right,
                                                                             jboolean is_right_cv, jboolean ansi_enabled, jboolean is_try_mode)
{
  if (!left) { throw_java(env, "java/lang/NullPointerException", "left input is null"); return 0; }
  if (!right) { throw_java(env, "java/lang/NullPointerException", "right input is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    const Operand a = operand(left, is_left_cv), b = operand(right, is_right_cv);
    const srj_column& column = is_left_cv ? a.col : b.col;
    const int64_t rows       = column.size;
    auto stream              = cudf::get_default_stream();
    rmm::device_buffer data(static_cast<size_t>(rows) * static_cast<size_t>(size_of_type(column.type_id)), stream);
    rmm::device_buffer mask(static_cast<size_t>((rows + 31) / 32) * 4, stream);
    int64_t nulls = 0, error_row = -1;
    const int st = srj_multiply(&a.col, a.scalar_valid, &b.col, b.scalar_valid, ansi_enabled ? 1 : 0, is_try_mode ? 1 : 0, data.data(),
                                static_cast<uint32_t*>(mask.data()), &nulls, &error_row, stream.value());
    if (throw_if_error(env, st)) return 0;
    if (error_row >= 0) {
      throw_row_index(env, error_row, {&data, &mask});
      return 0;
    }
    const cudf::data_type type(static_cast<cudf::type_id>(column.type_id), column.scale);
    return release_as_jlong(std::make_unique<cudf::column>(type, static_cast<cudf::size_type>(rows), std::move(data),
                                                           nulls ? std::move(mask) : rmm::device_buffer{}, static_cast<cudf::size_type>(nulls)));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Arithmetic_round(JNIEnv* env, jclass, jlong input_ptr, jint decimal_places,
                                                                          jint rounding_method, jboolean is_ansi_mode)
{
  if (!input_ptr) { throw_java(env, "java/lang/NullPointerException", "input is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& input  = *reinterpret_cast<cudf::column_view const*>(input_ptr);
    const srj_column in = to_srj_nullable(input);
    const int64_t rows = in.size;
    auto stream        = cudf::get_default_stream();
    const cudf::type_id id = input.type().id();
    const bool decimal = id == cudf::type_id::DECIMAL32 || id == cudf::type_id::DECIMAL64 || id == cudf::type_id::DECIMAL128;
    const cudf::data_type type = decimal && rows > 0 ? cudf::data_type(id, -decimal_places) : input.type();
    rmm::device_buffer data(static_cast<size_t>(rows) * static_cast<size_t>(size_of_type(in.type_id)), stream);
    rmm::device_buffer mask = mask_like(in, stream);
    int64_t error_row       = -1;
    const int st = srj_round(&in, decimal_places, rounding_method, is_ansi_mode ? 1 : 0, data.data(),
                             in.null_mask ? static_cast<uint32_t*>(mask.data()) : nullptr, &error_row, stream.value());
    if (throw_if_error(env, st)) return 0;
    if (error_row >= 0) {
      throw_row_index(env, error_row, {&data, &mask});
      return 0;
    }
    return release_as_jlong(std::make_unique<cudf::column>(type, static_cast<cudf::size_type>(rows), std::move(data), std::move(mask),
                                                           in.null_mask ? input.null_count() : 0));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
