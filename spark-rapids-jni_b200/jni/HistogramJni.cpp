// HistogramJni.cpp -- com.nvidia.spark.rapids.jni.Histogram over libsrj_b200.so: the two natives of Histogram.java:71-75
// (reference HistogramJni.cpp).  Inputs are cudf::column_view handles.  Outputs (heap cudf::column*):
//   createHistogramIfValid  -> STRUCT<T, INT64>, or LIST<STRUCT<T, INT64>> (one element per row with frequency > 0)
//   percentileFromHistogram -> FLOAT64 (rows * P, each null where its row is; rows when P is 0 or there is no element), or
//                              LIST<FLOAT64> (P per valid row, null rows empty)
// A null handle or array throws NullPointerException; C-ABI errors map to the classes of srj_jni_common.hpp.
#include "srj_jni_common.hpp"

#include <algorithm>

using namespace srjshim;

namespace {

// the C ABI reads a mask as nulls: a column without nulls goes without its mask
srj_column to_srj_nullable(const cudf::column_view& c)
{
  srj_column s = to_srj(c);
  if (c.null_count() == 0) s.null_mask = nullptr;
  return s;
}

std::unique_ptr<cudf::column> flat_column(cudf::data_type t, int64_t rows, rmm::device_buffer&& data, rmm::device_buffer&& mask, int64_t nulls)
{
  return std::make_unique<cudf::column>(t, static_cast<cudf::size_type>(rows), std::move(data),
                                        nulls ? std::move(mask) : rmm::device_buffer{}, static_cast<cudf::size_type>(nulls));
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Histogram_createHistogramIfValid(JNIEnv* env, jclass, jlong values_handle,
                                                                                        jlong frequencies_handle, jboolean output_as_lists)
{
  if (!values_handle) { throw_java(env, "java/lang/NullPointerException", "values_handle is null"); return 0; }
  if (!frequencies_handle) { throw_java(env, "java/lang/NullPointerException", "frequencies_handle is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& values = *reinterpret_cast<cudf::column_view const*>(values_handle);
    auto const& freqs  = *reinterpret_cast<cudf::column_view const*>(frequencies_handle);
    const srj_column v = to_srj_nullable(values), f = to_srj_nullable(freqs);
    const int32_t lists = output_as_lists ? 1 : 0;
    const int64_t rows  = values.size();
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer ws(static_cast<size_t>(srj_histogram_workspace_bytes(rows)), stream);
    int64_t n = 0, nulls = 0;
    int st = srj_histogram_create_size(&v, &f, lists, &n, &nulls, ws.data(), stream.value());
    if (throw_if_error(env, st)) return 0;
    const size_t width = static_cast<size_t>(size_of_type(v.type_id));
    rmm::device_buffer out_v(static_cast<size_t>(n) * width, stream), out_f(static_cast<size_t>(n) * 8, stream);
    const bool has_mask = !lists || v.null_mask;
    rmm::device_buffer mask(has_mask ? static_cast<size_t>(((lists ? n : rows) + 31) / 32) * 4 : 0, stream);
    rmm::device_buffer offsets(lists ? static_cast<size_t>(rows + 1) * 4 : 0, stream);
    st = srj_histogram_create(&v, &f, lists, out_v.data(), has_mask ? static_cast<uint32_t*>(mask.data()) : nullptr,
                              static_cast<int64_t*>(out_f.data()), lists ? static_cast<int32_t*>(offsets.data()) : nullptr, ws.data(),
                              stream.value());
    if (throw_if_error(env, st)) return 0;
    std::vector<std::unique_ptr<cudf::column>> children;
    children.push_back(flat_column(values.type(), n, std::move(out_v), std::move(mask), nulls));
    children.push_back(flat_column(cudf::data_type{cudf::type_id::INT64}, n, std::move(out_f), rmm::device_buffer{}, 0));
    auto structs = cudf::make_structs_column(static_cast<cudf::size_type>(n), std::move(children), 0, rmm::device_buffer{}, stream);
    if (!lists) return release_as_jlong(std::move(structs));
    if (rows == 0) {                                           // the fill call touches nothing for zero rows
      const int32_t zero = 0;
      if (!copy_from_host(offsets.data(), &zero, 4, stream)) { throw_java(env, "ai/rapids/cudf/CudaException", "offsets copy failed"); return 0; }
    }
    auto offsets_col = flat_column(cudf::data_type{cudf::type_id::INT32}, rows + 1, std::move(offsets), rmm::device_buffer{}, 0);
    return release_as_jlong(cudf::make_lists_column(static_cast<cudf::size_type>(rows), std::move(offsets_col), std::move(structs), 0,
                                                    rmm::device_buffer{}));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Histogram_percentileFromHistogram(JNIEnv* env, jclass, jlong input_handle,
                                                                                         jdoubleArray jpercentages, jboolean output_as_lists)
{
  if (!input_handle) { throw_java(env, "java/lang/NullPointerException", "input_handle is null"); return 0; }
  if (!jpercentages) { throw_java(env, "java/lang/NullPointerException", "jpercentages is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& input = *reinterpret_cast<cudf::column_view const*>(input_handle);
    std::vector<double> pct(static_cast<size_t>(env->GetArrayLength(jpercentages)));
    if (!pct.empty()) {
      jdouble* p = env->GetDoubleArrayElements(jpercentages, nullptr);
      std::copy(p, p + pct.size(), pct.begin());
      env->ReleaseDoubleArrayElements(jpercentages, p, JNI_ABORT);
    }
    const int32_t P = static_cast<int32_t>(pct.size());
    srj_column in{}, st{}, fields[2]{};
    in.type_id = static_cast<int32_t>(input.type().id());
    in.size    = input.size();
    if (input.type().id() == cudf::type_id::LIST) {
      cudf::lists_column_view const lv(input);
      in.offsets = const_cast<int32_t*>(lv.offsets().head<int32_t>()) + input.offset();   // a sliced view starts there
      cudf::column_view const child = lv.child();
      st                            = to_srj_nullable(child);
      for (int i = 0; i < 2 && i < child.num_children(); ++i) fields[i] = i == 0 ? to_srj(child.child(i)) : to_srj_nullable(child.child(i));
      st.children     = fields;
      st.num_children = child.num_children();
      in.children     = &st;
      in.num_children = 1;
    }
    const int32_t lists = output_as_lists ? 1 : 0;
    const int64_t rows  = in.size;
    auto stream         = cudf::get_default_stream();
    rmm::device_buffer ws(static_cast<size_t>(srj_percentile_workspace_bytes(rows, st.size, P)), stream);
    int64_t valid = 0, n = 0;
    int status = srj_percentile_from_histogram_size(&in, P, lists, &valid, &n, ws.data(), stream.value());
    if (throw_if_error(env, status)) return 0;
    // the mask has a bit per row of the list output, or per double of the flat output
    rmm::device_buffer out(static_cast<size_t>(n) * 8, stream), mask(static_cast<size_t>(((lists ? rows : n) + 31) / 32) * 4, stream);
    rmm::device_buffer offsets(lists ? static_cast<size_t>(rows + 1) * 4 : 0, stream);
    status = srj_percentile_from_histogram(&in, pct.data(), P, lists, static_cast<double*>(out.data()), static_cast<uint32_t*>(mask.data()),
                                           lists ? static_cast<int32_t*>(offsets.data()) : nullptr, ws.data(), stream.value());
    if (throw_if_error(env, status)) return 0;
    const int64_t nulls = rows - valid;
    if (!lists) return release_as_jlong(flat_column(cudf::data_type{cudf::type_id::FLOAT64}, n, std::move(out), std::move(mask),
                                                    rows ? nulls * (n / rows) : 0));
    if (rows == 0) return release_as_jlong(cudf::make_lists_column(0, flat_column(cudf::data_type{cudf::type_id::INT32}, 0, rmm::device_buffer{}, rmm::device_buffer{}, 0),
                                                                   flat_column(cudf::data_type{cudf::type_id::FLOAT64}, 0, std::move(out), rmm::device_buffer{}, 0),
                                                                   0, rmm::device_buffer{}));
    return release_as_jlong(cudf::make_lists_column(static_cast<cudf::size_type>(rows),
                                                    flat_column(cudf::data_type{cudf::type_id::INT32}, rows + 1, std::move(offsets), rmm::device_buffer{}, 0),
                                                    flat_column(cudf::data_type{cudf::type_id::FLOAT64}, n, std::move(out), rmm::device_buffer{}, 0),
                                                    static_cast<cudf::size_type>(nulls), nulls ? std::move(mask) : rmm::device_buffer{}));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
