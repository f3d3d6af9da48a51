// IcebergTruncateJni.cpp -- com.nvidia.spark.rapids.jni.iceberg.IcebergTruncate over libsrj_b200.so: the native of
// IcebergTruncate.java (reference iceberg/IcebergTruncateJni.cpp).  Input: one cudf::column_view*; output: a heap
// cudf::column* of the input's type with the input's null mask and null count:
//   INT32, INT64, DECIMAL32/64/128 -> the same type and scale
//   STRING                         -> STRING (INT32 offsets child, chars)
//   LIST<UINT8>                    -> LIST<UINT8> (INT32 offsets child, non-nullable UINT8 child)
// Any other type throws IllegalArgumentException("Unsupported type for truncation"), as the reference's JNI does; a null
// handle throws NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

using namespace srjshim;

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_iceberg_IcebergTruncate_truncate(JNIEnv* env, jclass, jlong input_column, jint width)
{
  if (!input_column) { throw_java(env, "java/lang/NullPointerException", "input column is null"); return 0; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& view = *reinterpret_cast<cudf::column_view const*>(input_column);
    const auto type  = view.type().id();
    srj_column child{};
    const srj_column in = to_srj_any(view, &child);
    const int64_t n     = view.size();
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer mask = mask_like(in, stream);
    srj_column out{};
    out.type_id   = in.type_id;
    out.scale     = in.scale;
    out.size      = n;
    out.null_mask = static_cast<uint32_t*>(mask.data());
    switch (type) {
      case cudf::type_id::INT32:
      case cudf::type_id::INT64:
      case cudf::type_id::DECIMAL32:
      case cudf::type_id::DECIMAL64:
      case cudf::type_id::DECIMAL128: {
        rmm::device_buffer data(static_cast<size_t>(n) * size_of_type(in.type_id), stream);
        out.data     = data.data();
        const int st = srj_iceberg_truncate(&in, width, &out, stream.value());
        if (throw_if_error(env, st)) return 0;
        return release_as_jlong(std::make_unique<cudf::column>(view.type(), static_cast<cudf::size_type>(n), std::move(data), std::move(mask),
                                                               view.null_count()));
      }
      case cudf::type_id::STRING:
      case cudf::type_id::LIST: {
        rmm::device_buffer offsets(static_cast<size_t>(n + 1) * 4, stream);
        rmm::device_buffer workspace(static_cast<size_t>(srj_iceberg_truncate_workspace_bytes(n)), stream);
        int64_t total = 0;
        int st = srj_iceberg_truncate_sizes(&in, width, static_cast<int32_t*>(offsets.data()), &total, workspace.data(), stream.value());
        if (throw_if_error(env, st)) return 0;
        rmm::device_buffer bytes(static_cast<size_t>(total), stream);
        srj_column out_child{};
        out_child.type_id = SRJ_UINT8;
        out_child.size    = total;
        out_child.data    = bytes.data();
        out.offsets       = static_cast<int32_t*>(offsets.data());
        if (type == cudf::type_id::STRING) {
          out.data = bytes.data();
        } else {
          out.children     = &out_child;
          out.num_children = 1;
        }
        st = srj_iceberg_truncate(&in, width, &out, stream.value());
        if (throw_if_error(env, st)) return 0;
        auto offsets_col = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::INT32}, static_cast<cudf::size_type>(n + 1),
                                                          std::move(offsets), rmm::device_buffer{}, 0);
        if (type == cudf::type_id::STRING)
          return release_as_jlong(cudf::make_strings_column(static_cast<cudf::size_type>(n), std::move(offsets_col), std::move(bytes),
                                                            view.null_count(), std::move(mask)));
        auto bytes_col = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::UINT8}, static_cast<cudf::size_type>(total),
                                                        std::move(bytes), rmm::device_buffer{}, 0);
        return release_as_jlong(cudf::make_lists_column(static_cast<cudf::size_type>(n), std::move(offsets_col), std::move(bytes_col),
                                                        view.null_count(), std::move(mask)));
      }
      default: throw_java(env, "java/lang/IllegalArgumentException", "Unsupported type for truncation"); return 0;
    }
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
