// JoinPrimitivesJni.cpp -- com.nvidia.spark.rapids.jni.JoinPrimitives over libsrj_b200.so: six of the eight natives of
// JoinPrimitives.java (reference JoinPrimitivesJni.cpp).  nativeSortMergeInnerJoin and nativeFilterGatherMapsByAST are not
// defined (DESIGN 6).  Key tables arrive as cudf::table_view* handles, gather maps as (device address, byte length).  A pair
// of maps returns long[5] = {bytes, left address, left rmm::device_buffer*, right address, right rmm::device_buffer*}, one
// map long[3] = {bytes, address, rmm::device_buffer*}, as the reference's gather_maps_to_java / gather_single_map_to_java;
// getMatchedRows a heap cudf::column* (BOOL8, no null mask).  A null handle throws NullPointerException, a null address
// with a nonzero length or maps of differing lengths IllegalArgumentException (as the reference); a length that is not a
// multiple of 4 and the C ABI's errors map to the classes of srj_jni_common.hpp.
#include <memory>

#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

const char* kIllegalArg = "java/lang/IllegalArgumentException";

jlongArray to_java(JNIEnv* env, const jlong* v, jsize n)
{
  jlongArray out = env->NewLongArray(n);
  if (out) env->SetLongArrayRegion(out, 0, n, v);
  return out;
}

jlongArray pair_to_java(JNIEnv* env, std::unique_ptr<rmm::device_buffer> l, std::unique_ptr<rmm::device_buffer> r)
{
  const jlong v[5] = {static_cast<jlong>(l->size()), reinterpret_cast<jlong>(l->data()), reinterpret_cast<jlong>(l.get()),
                      reinterpret_cast<jlong>(r->data()), reinterpret_cast<jlong>(r.get())};
  jlongArray out = to_java(env, v, 5);
  if (out) {
    l.release();    // Java owns both buffers now
    r.release();
  }
  return out;
}

jlongArray single_to_java(JNIEnv* env, std::unique_ptr<rmm::device_buffer> m)
{
  const jlong v[3] = {static_cast<jlong>(m->size()), reinterpret_cast<jlong>(m->data()), reinterpret_cast<jlong>(m.get())};
  jlongArray out   = to_java(env, v, 3);
  if (out) m.release();
  return out;
}

// (address, byte length) of a gather map -> its entries; false when it threw
bool map_arg(JNIEnv* env, jlong addr, jlong bytes, const int32_t** map, int64_t* len)
{
  if (addr == 0 && bytes != 0) { throw_java(env, kIllegalArg, "buffer address is null but length is non-zero"); return false; }
  if (bytes < 0 || bytes % 4 != 0) { throw_java(env, "ai/rapids/cudf/CudfException", "gather map length is not a multiple of 4 bytes"); return false; }
  *map = reinterpret_cast<const int32_t*>(addr);
  *len = bytes / 4;
  return true;
}

std::unique_ptr<rmm::device_buffer> mask_ws(int64_t rows, rmm::cuda_stream_view stream)
{
  return std::make_unique<rmm::device_buffer>(static_cast<size_t>(srj_join_mask_workspace_bytes(rows)), stream);
}

jlongArray make_outer(JNIEnv* env, jlong la, jlong lb, jlong ra, jlong rb, jint left_size, jint right_size, bool full)
{
  const int32_t *lm = nullptr, *rm = nullptr;
  int64_t ln = 0, rn = 0;
  if (!map_arg(env, la, lb, &lm, &ln) || !map_arg(env, ra, rb, &rm, &rn)) return nullptr;
  if (lb != rb) { throw_java(env, kIllegalArg, "left and right gather maps must have the same length"); return nullptr; }
  cudf::jni::auto_set_device(env);
  auto stream = cudf::get_default_stream();
  auto lws = mask_ws(left_size, stream), rws = mask_ws(full ? right_size : 0, stream);
  if (throw_if_error(env, srj_join_mark(lm, ln, left_size, lws->data(), stream.value()))) return nullptr;
  if (full && throw_if_error(env, srj_join_mark(rm, rn, right_size, rws->data(), stream.value()))) return nullptr;
  const void* wss[2] = {lws->data(), rws->data()};
  int64_t matched[2] = {0, 0};
  if (throw_if_error(env, srj_join_matched_counts(wss, full ? 2 : 1, matched, stream.value()))) return nullptr;
  const int64_t lu = left_size - matched[0], ru = full ? right_size - matched[1] : 0;
  const size_t bytes = static_cast<size_t>(ln + lu + ru) * 4;
  auto ol = std::make_unique<rmm::device_buffer>(bytes, stream), orr = std::make_unique<rmm::device_buffer>(bytes, stream);
  if (throw_if_error(env, srj_join_make_outer(lm, rm, ln, left_size, right_size, lws->data(), lu, full ? rws->data() : nullptr, ru,
                                              static_cast<int32_t*>(ol->data()), static_cast<int32_t*>(orr->data()), stream.value())))
    return nullptr;
  return pair_to_java(env, std::move(ol), std::move(orr));
}

jlongArray semi_anti(JNIEnv* env, jlong addr, jlong bytes, jint size, bool semi)
{
  const int32_t* m = nullptr;
  int64_t n        = 0;
  if (!map_arg(env, addr, bytes, &m, &n)) return nullptr;
  cudf::jni::auto_set_device(env);
  auto stream = cudf::get_default_stream();
  auto ws     = mask_ws(size, stream);
  if (throw_if_error(env, srj_join_mark(m, n, size, ws->data(), stream.value()))) return nullptr;
  const void* wss[1] = {ws->data()};
  int64_t matched    = 0;
  if (throw_if_error(env, srj_join_matched_counts(wss, 1, &matched, stream.value()))) return nullptr;
  const int64_t count = semi ? matched : size - matched;
  auto out           = std::make_unique<rmm::device_buffer>(static_cast<size_t>(count) * 4, stream);
  if (count > 0 && throw_if_error(env, srj_join_compact(ws->data(), size, semi ? 1 : 0, static_cast<int32_t*>(out->data()), stream.value()))) return nullptr;
  return single_to_java(env, std::move(out));
}

}  // namespace

extern "C" {

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_JoinPrimitives_nativeHashInnerJoin(JNIEnv* env, jclass, jlong j_left_keys,
                                                                                                 jlong j_right_keys, jboolean j_nulls_equal)
{
  if (!j_left_keys) { throw_java(env, "java/lang/NullPointerException", "left keys table is null"); return nullptr; }
  if (!j_right_keys) { throw_java(env, "java/lang/NullPointerException", "right keys table is null"); return nullptr; }
  try {
    cudf::jni::auto_set_device(env);
    auto const* lt = reinterpret_cast<cudf::table_view const*>(j_left_keys);
    auto const* rt = reinterpret_cast<cudf::table_view const*>(j_right_keys);
    std::vector<srj_column> lc(lt->num_columns()), rc(rt->num_columns());
    for (int c = 0; c < lt->num_columns(); ++c) lc[c] = to_srj(lt->column(c));
    for (int c = 0; c < rt->num_columns(); ++c) rc[c] = to_srj(rt->column(c));
    auto stream = cudf::get_default_stream();
    rmm::device_buffer ws(static_cast<size_t>(srj_hash_join_workspace_bytes(lt->num_rows(), rt->num_rows())), stream);
    const int32_t nl = static_cast<int32_t>(lc.size()), nr = static_cast<int32_t>(rc.size()), eq = j_nulls_equal ? 1 : 0;
    int64_t pairs    = 0;
    if (throw_if_error(env, srj_hash_inner_join_size(lc.data(), nl, rc.data(), nr, eq, &pairs, ws.data(), stream.value()))) return nullptr;
    auto l = std::make_unique<rmm::device_buffer>(static_cast<size_t>(pairs) * 4, stream);
    auto r = std::make_unique<rmm::device_buffer>(static_cast<size_t>(pairs) * 4, stream);
    if (pairs > 0 && throw_if_error(env, srj_hash_inner_join(lc.data(), nl, rc.data(), nr, eq, static_cast<int32_t*>(l->data()),
                                                             static_cast<int32_t*>(r->data()), ws.data(), stream.value())))
      return nullptr;
    return pair_to_java(env, std::move(l), std::move(r));
  } catch (...) {
    throw_from_exception(env);
  }
  return nullptr;
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_JoinPrimitives_nativeMakeLeftOuter(JNIEnv* env, jclass, jlong j_left_address,
                                                                                                 jlong j_left_length, jlong j_right_address,
                                                                                                 jlong j_right_length, jint j_left_size,
                                                                                                 jint j_right_size)
{
  try {
    return make_outer(env, j_left_address, j_left_length, j_right_address, j_right_length, j_left_size, j_right_size, false);
  } catch (...) {
    throw_from_exception(env);
  }
  return nullptr;
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_JoinPrimitives_nativeMakeFullOuter(JNIEnv* env, jclass, jlong j_left_address,
                                                                                                 jlong j_left_length, jlong j_right_address,
                                                                                                 jlong j_right_length, jint j_left_size,
                                                                                                 jint j_right_size)
{
  try {
    return make_outer(env, j_left_address, j_left_length, j_right_address, j_right_length, j_left_size, j_right_size, true);
  } catch (...) {
    throw_from_exception(env);
  }
  return nullptr;
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_JoinPrimitives_nativeMakeSemi(JNIEnv* env, jclass, jlong j_address, jlong j_length,
                                                                                            jint j_size)
{
  try {
    return semi_anti(env, j_address, j_length, j_size, true);
  } catch (...) {
    throw_from_exception(env);
  }
  return nullptr;
}

JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_JoinPrimitives_nativeMakeAnti(JNIEnv* env, jclass, jlong j_address, jlong j_length,
                                                                                            jint j_size)
{
  try {
    return semi_anti(env, j_address, j_length, j_size, false);
  } catch (...) {
    throw_from_exception(env);
  }
  return nullptr;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_JoinPrimitives_nativeGetMatchedRows(JNIEnv* env, jclass, jlong j_address, jlong j_length,
                                                                                             jint j_size)
{
  try {
    const int32_t* m = nullptr;
    int64_t n        = 0;
    if (!map_arg(env, j_address, j_length, &m, &n)) return 0;
    cudf::jni::auto_set_device(env);
    auto stream = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(j_size > 0 ? j_size : 0), stream);
    if (throw_if_error(env, srj_join_matched_rows(m, n, j_size, static_cast<uint8_t*>(out.data()), stream.value()))) return 0;
    return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::BOOL8}, j_size, std::move(out), rmm::device_buffer(0, stream), 0));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
