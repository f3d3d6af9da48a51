// BloomFilterJni.cpp -- com.nvidia.spark.rapids.jni.BloomFilter over libsrj_b200.so: the five natives of
// BloomFilter.java:112-118 (reference BloomFilterJni.cpp:27-117), with the reference's return conventions:
//   creategpu, merge     -> a heap cudf::list_scalar* whose child is the UINT8 bytes of the serialized filter
//   probe, probebuffer   -> a heap cudf::column* BOOL8 with a copy of the input's null mask and its null count
//   put                  -> 0, the filter's bytes updated in place
// A null handle throws NullPointerException; a bit count outside (0, INT32_MAX * 64] throws IllegalArgumentException
// (JNI_ARG_CHECK, BloomFilterJni.cpp:40-46); C-ABI errors map to the classes of srj_jni_common.hpp.
#ifndef SRJ_JNI_STUBS
#include <cudf/lists/lists_column_view.hpp>
#include <cudf/scalar/scalar.hpp>
#endif

#include "srj_jni_common.hpp"

using namespace srjshim;

namespace {

constexpr int64_t kMaxBits = static_cast<int64_t>(INT32_MAX) * 64;   // Spark's BitArray: at most INT32_MAX longs

jlong new_filter_scalar(rmm::device_buffer&& bytes, int64_t size, rmm::cuda_stream_view stream)
{
  cudf::column col(cudf::data_type{cudf::type_id::UINT8}, static_cast<cudf::size_type>(size), std::move(bytes), rmm::device_buffer{}, 0);
  return reinterpret_cast<jlong>(new cudf::list_scalar(std::move(col), true, stream));
}

jlong probe(JNIEnv* env, const uint8_t* filter, int64_t filter_bytes, jlong column_handle)
{
  auto const& view   = *reinterpret_cast<cudf::column_view const*>(column_handle);
  const srj_column in = to_srj(view);
  const int64_t n     = view.size();
  auto stream         = cudf::get_default_stream();
  rmm::device_buffer data(static_cast<size_t>(n), stream);
  rmm::device_buffer mask(in.null_mask ? static_cast<size_t>((n + 31) / 32) * 4 : 0, stream);
  const int st = srj_bloom_filter_probe(filter, filter_bytes, &in, static_cast<uint8_t*>(data.data()),
                                        in.null_mask ? static_cast<uint32_t*>(mask.data()) : nullptr, stream.value());
  if (throw_if_error(env, st)) return 0;
  return release_as_jlong(std::make_unique<cudf::column>(cudf::data_type{cudf::type_id::BOOL8}, static_cast<cudf::size_type>(n), std::move(data),
                                                         std::move(mask), view.null_count()));
}

}  // namespace

extern "C" {

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_BloomFilter_creategpu(JNIEnv* env, jclass, jint version, jint numHashes,
                                                                              jlong bloomFilterBits, jint seed)
{
  try {
    cudf::jni::auto_set_device(env);
    if (bloomFilterBits <= 0 || bloomFilterBits > kMaxBits) {
      throw_java(env, "java/lang/IllegalArgumentException",
                 "bloom filter bit count must be positive and less than or equal to the maximum supported size");
      return 0;
    }
    int32_t longs = 0;
    int64_t total = 0;
    int st        = srj_bloom_filter_sizes(version, numHashes, bloomFilterBits, &longs, &total);
    if (throw_if_error(env, st)) return 0;
    auto stream = cudf::get_default_stream();
    rmm::device_buffer buf(static_cast<size_t>(total), stream);
    st = srj_bloom_filter_init(version, numHashes, longs, seed, static_cast<uint8_t*>(buf.data()), stream.value());
    if (throw_if_error(env, st)) return 0;
    return new_filter_scalar(std::move(buf), total, stream);
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jint JNICALL Java_com_nvidia_spark_rapids_jni_BloomFilter_put(JNIEnv* env, jclass, jlong bloomFilter, jlong cv)
{
  if (!bloomFilter) { throw_java(env, "java/lang/NullPointerException", "bloom filter handle is null"); return 0; }
  if (!cv) { throw_java(env, "java/lang/NullPointerException", "column handle is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    // the scalar owns its bytes; view() is const only because cudf has no mutable list_scalar view
    cudf::column_view const bytes = reinterpret_cast<cudf::list_scalar*>(bloomFilter)->view();
    const srj_column in           = to_srj(*reinterpret_cast<cudf::column_view const*>(cv));
    const int st = srj_bloom_filter_put(const_cast<uint8_t*>(bytes.head<uint8_t>()), bytes.size(), &in, cudf::get_default_stream().value());
    throw_if_error(env, st);
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_BloomFilter_merge(JNIEnv* env, jclass, jlong bloomFilters)
{
  if (!bloomFilters) { throw_java(env, "java/lang/NullPointerException", "bloom filters handle is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    auto const& lists            = *reinterpret_cast<cudf::column_view const*>(bloomFilters);
    cudf::column_view const kids = cudf::lists_column_view(lists).child();
    const int32_t nfilters       = lists.size();
    const int64_t bytes          = kids.size();
    const int64_t out_bytes      = nfilters > 0 ? bytes / nfilters : 0;
    auto stream                  = cudf::get_default_stream();
    rmm::device_buffer out(static_cast<size_t>(out_bytes), stream);
    rmm::device_buffer workspace(static_cast<size_t>(srj_bloom_filter_merge_workspace_bytes()), stream);
    const int st = srj_bloom_filter_merge(kids.head<uint8_t>(), bytes, nfilters, static_cast<uint8_t*>(out.data()), workspace.data(),
                                          stream.value());
    if (throw_if_error(env, st)) return 0;
    return new_filter_scalar(std::move(out), out_bytes, stream);
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_BloomFilter_probe(JNIEnv* env, jclass, jlong bloomFilter, jlong cv)
{
  if (!bloomFilter) { throw_java(env, "java/lang/NullPointerException", "bloom filter handle is null"); return 0; }
  if (!cv) { throw_java(env, "java/lang/NullPointerException", "column handle is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    cudf::column_view const bytes = reinterpret_cast<cudf::list_scalar*>(bloomFilter)->view();
    return probe(env, bytes.head<uint8_t>(), bytes.size(), cv);
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

// probe(BaseDeviceMemoryBuffer, cv): the filter is `bloomFilterSize` bytes of device memory at address `bloomFilter`
JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_BloomFilter_probebuffer(JNIEnv* env, jclass, jlong bloomFilter, jlong bloomFilterSize,
                                                                                jlong cv)
{
  if (!cv) { throw_java(env, "java/lang/NullPointerException", "column handle is null"); return 0; }
  try {
    cudf::jni::auto_set_device(env);
    return probe(env, reinterpret_cast<const uint8_t*>(bloomFilter), bloomFilterSize, cv);
  } catch (...) {
    throw_from_exception(env);
  }
  return 0;
}

}  // extern "C"
