// HashSha2Jni.cpp -- the rest of com.nvidia.spark.rapids.jni.Hash over libsrj_b200.so: sha224NullsPreserved,
// sha256NullsPreserved, sha384NullsPreserved, sha512NullsPreserved and hostCrc32 (reference hash/HashJni.cpp:81-157).
// Together with HashJni.cpp this library defines all nine natives of Hash.java:176-190; the JVM resolves natives
// from any translation unit of the loaded library.
// Input: one cudf::column_view* of type STRING; output: a heap cudf::column* STRING of lowercase hex digests with the
// input's null mask and null count.
#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

jlong sha2_nulls_preserved(JNIEnv* env, int32_t digest_bits, jlong column_handle)
{
  if (!column_handle) { throw_java(env, "java/lang/NullPointerException", "column handle is null"); return 0; }   // JNI_NULL_CHECK
  try {
    cudf::jni::auto_set_device(env);
    auto const& view   = *reinterpret_cast<cudf::column_view const*>(column_handle);
    const srj_column in = to_srj(view);
    const int64_t n     = view.size();
    auto stream         = cudf::get_default_stream();
    // the sizes call needs its workspace only when there is a mask to scan
    rmm::device_buffer offsets(static_cast<size_t>(n + 1) * 4, stream);
    rmm::device_buffer workspace(in.null_mask ? static_cast<size_t>(srj_sha2_workspace_bytes(n)) : 0, stream);
    int64_t total = 0;
    int st = srj_sha2_sizes(digest_bits, &in, static_cast<int32_t*>(offsets.data()), &total, in.null_mask ? workspace.data() : nullptr,
                            stream.value());
    if (throw_if_error(env, st)) return 0;
    rmm::device_buffer chars(static_cast<size_t>(total), stream);
    rmm::device_buffer mask(in.null_mask ? static_cast<size_t>((n + 31) / 32) * 4 : 0, stream);
    srj_column out{};
    out.type_id   = SRJ_STRING;
    out.size      = n;
    out.data      = total > 0 ? chars.data() : nullptr;
    out.null_mask = in.null_mask ? static_cast<uint32_t*>(mask.data()) : nullptr;
    out.offsets   = static_cast<int32_t*>(offsets.data());
    st = srj_sha2_hash(digest_bits, &in, &out, stream.value());
    if (throw_if_error(env, st)) return 0;
    auto offsets_col = std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::INT32}, static_cast<cudf::size_type>(n + 1),
                                                      std::move(offsets), rmm::device_buffer{}, 0);
    return release_as_jlong(cudf::make_strings_column(static_cast<cudf::size_type>(n), std::move(offsets_col), std::move(chars),
                                                      view.null_count(), std::move(mask)));
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Hash_sha224NullsPreserved(JNIEnv* env, jclass, jlong column_handle)
{
  return sha2_nulls_preserved(env, 224, column_handle);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Hash_sha256NullsPreserved(JNIEnv* env, jclass, jlong column_handle)
{
  return sha2_nulls_preserved(env, 256, column_handle);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Hash_sha384NullsPreserved(JNIEnv* env, jclass, jlong column_handle)
{
  return sha2_nulls_preserved(env, 384, column_handle);
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Hash_sha512NullsPreserved(JNIEnv* env, jclass, jlong column_handle)
{
  return sha2_nulls_preserved(env, 512, column_handle);
}

// Hash.hostCrc32(crc, address, len), HashJni.cpp:143-157: a NULL address only with len == 0, otherwise len > 0
// (IllegalArgumentException, JNI_ARG_CHECK); the CRC is zlib's crc32 computed on the host.
JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Hash_hostCrc32(JNIEnv* env, jclass, jlong crc, jlong buffer_handle, jint len)
{
  if (buffer_handle == 0 && len != 0) { throw_java(env, "java/lang/IllegalArgumentException", "len is not zero for empty buffer"); return 0; }
  if (buffer_handle != 0 && len <= 0) { throw_java(env, "java/lang/IllegalArgumentException", "len must be positive for non-empty buffer"); return 0; }
  try {
    uint32_t out = 0;
    const int st = srj_host_crc32(static_cast<uint32_t>(crc), reinterpret_cast<const void*>(buffer_handle), len, &out);
    if (throw_if_error(env, st)) return 0;
    return static_cast<jlong>(out);
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
