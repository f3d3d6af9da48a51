// bloom_filter.cu -- Spark's runtime-join bloom filter on the device (reference bloom_filter.cu, BloomFilter.java):
// init, put, probe and merge of the serialized V1 / V2 formats.
//
// Format (bloom_filter.hpp:32-49, bloom_filter.cu:154-172): big-endian int32 header {1, k, numLongs} (12 B, V1) or
// {2, k, seed, numLongs} (16 B, V2), then numLongs big-endian longs.  Bit p is bit p % 64 of long p / 64; in the
// little-endian uint32 view of the bit array that is bit (p % 32) ^ 24 of word (p / 32) ^ 1 (bloom_filter.cu:60-66).
// Every modulo is by bits = numLongs * 64.
//
// Element hashes (bloom_filter.cu:70-152, Spark's BloomFilterImpl / BloomFilterImplV2), all with Java int / long
// wrap-around, done here in unsigned arithmetic:
//   h1 = Murmur3_x86_32.hashLong(x, s), h2 = hashLong(x, h1); s = 0 (V1) or the header seed (V2)
//   V1: for i = 1..k:  c = (int32)(h1 + i * h2),  p = (c < 0 ? ~c : c) % bits
//   V2: c = (int64)h1 * INT32_MAX;  for i = 0..k-1:  c += (int64)h2,  p = (c < 0 ? ~c : c) % bits
//
// The modulo by the per-call constant `bits` uses a host-computed reciprocal (reciprocal.cuh: mod_v1 for V1's 31-bit
// dividends, mod_v2 for V2's 63-bit ones).  No division instruction or subroutine is left in the put / probe loops.
#include "check.hpp"
#include "common.cuh"
#include "hash_device.cuh"
#include "kernels.hpp"
#include "reciprocal.cuh"

namespace srj {

struct BloomHeader {
  int32_t version, num_hashes, seed, num_longs;   // seed is 0 for V1
};

namespace {

constexpr int kBloomThreads = 256;
constexpr int kRowsPerThread = 4;   // 2 x 16-byte key loads in, one 4-byte BOOL8 store out
constexpr int kHashChunk     = 8;   // word loads of one row issued together before any is tested

// The k bit positions of one key, produced one at a time (V1 state in 32 bits, V2 in 64).
template <int V>
struct Positions {
  uint64_t c, step;
  __device__ __forceinline__ Positions(int64_t key, uint32_t seed)
  {
    const uint32_t h1 = hash::mm_u64(static_cast<uint64_t>(key), V == 1 ? 0u : seed);
    const uint32_t h2 = hash::mm_u64(static_cast<uint64_t>(key), h1);
    if (V == 1) {
      c    = h1;
      step = h2;
    } else {
      c    = static_cast<uint64_t>(static_cast<int64_t>(static_cast<int32_t>(h1)) * INT32_MAX);
      step = static_cast<uint64_t>(static_cast<int64_t>(static_cast<int32_t>(h2)));
    }
  }
  // next position (V1: i = 1, 2, ...; V2: i = 0, 1, ...; both start by adding h2)
  __device__ __forceinline__ uint64_t next(uint64_t d, uint64_t m)
  {
    c += step;
    if (V == 1) {
      const uint32_t ci = static_cast<uint32_t>(c);
      const uint32_t x  = ci ^ static_cast<uint32_t>(static_cast<int32_t>(ci) >> 31);   // c < 0 ? ~c : c
      return mod_v1(x, static_cast<uint32_t>(d), static_cast<uint32_t>(m));
    } else {
      const uint64_t x = c ^ static_cast<uint64_t>(static_cast<int64_t>(c) >> 63);
      return mod_v2(x, d, m);
    }
  }
};

__device__ __forceinline__ uint64_t word_of(uint64_t p) { return (p >> 5) ^ 1u; }
__device__ __forceinline__ uint32_t bit_of(uint64_t p) { return 1u << ((static_cast<uint32_t>(p) & 31u) ^ 24u); }

// the kRowsPerThread keys of this thread (rows [r0, r0 + count)); 16-byte loads when the keys are 16-byte aligned
template <bool kVec>
__device__ __forceinline__ void load_keys(const int64_t* __restrict__ keys, int64_t r0, int count, int64_t (&k)[kRowsPerThread])
{
  if (kVec && count == kRowsPerThread) {
    const longlong2 a = __ldg(reinterpret_cast<const longlong2*>(keys + r0));
    const longlong2 b = __ldg(reinterpret_cast<const longlong2*>(keys + r0 + 2));
    k[0] = a.x; k[1] = a.y; k[2] = b.x; k[3] = b.y;
  } else {
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) k[j] = j < count ? __ldg(keys + r0 + j) : 0;
  }
}

// put: every valid row sets its k bits; atomicOr with the result unused compiles to RED.E.OR
template <int V, bool kVec>
__global__ void __launch_bounds__(kBloomThreads) bloom_put_kernel(uint32_t* __restrict__ words, uint64_t d, uint64_t m, int32_t k, uint32_t seed,
                                                                  const int64_t* __restrict__ keys, const uint32_t* __restrict__ mask, int64_t n)
{
  const int64_t r0 = (static_cast<int64_t>(blockIdx.x) * kBloomThreads + threadIdx.x) * kRowsPerThread;
  if (r0 >= n) return;
  const int count = static_cast<int>(tmin<int64_t>(kRowsPerThread, n - r0));
  int64_t key[kRowsPerThread];
  load_keys<kVec>(keys, r0, count, key);
  uint32_t valid = (1u << count) - 1u;                        // r0 is a multiple of 4: the rows share one mask word
  if (mask) valid &= __ldg(mask + (r0 >> 5)) >> (r0 & 31);
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    if (!((valid >> j) & 1u)) continue;
    Positions<V> pos(key[j], seed);
    for (int32_t i = 0; i < k; ++i) {
      const uint64_t p = pos.next(d, m);
      atomicOr(words + word_of(p), bit_of(p));
    }
  }
}

// probe: out[r] = all k bits of row r are set.  Per chunk of kHashChunk hashes, the word loads of all the thread's rows
// are issued (read-only path, L2-resident filter) before any is tested; a row whose chunk found a zero bit stops.
// Rows under nulls are computed like the others (their values are not part of the result).
template <int V, bool kVec>
__global__ void __launch_bounds__(kBloomThreads) bloom_probe_kernel(const uint32_t* __restrict__ words, uint64_t d, uint64_t m, int32_t k, uint32_t seed,
                                                                    const int64_t* __restrict__ keys, int64_t n, uint8_t* __restrict__ out)
{
  const int64_t r0 = (static_cast<int64_t>(blockIdx.x) * kBloomThreads + threadIdx.x) * kRowsPerThread;
  if (r0 >= n) return;
  const int count = static_cast<int>(tmin<int64_t>(kRowsPerThread, n - r0));
  int64_t key[kRowsPerThread];
  load_keys<kVec>(keys, r0, count, key);
  Positions<V> pos[kRowsPerThread] = {Positions<V>(key[0], seed), Positions<V>(key[1], seed), Positions<V>(key[2], seed),
                                      Positions<V>(key[3], seed)};
  uint32_t hit = 0xfu;                                        // bit j: row j still has every bit seen so far set
  for (int32_t i0 = 0; i0 < k && hit; i0 += kHashChunk) {
    uint32_t w[kRowsPerThread][kHashChunk], b[kRowsPerThread][kHashChunk];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
#pragma unroll
      for (int i = 0; i < kHashChunk; ++i) {
        b[j][i] = 0;
        w[j][i] = 0;
        if (i0 + i < k && ((hit >> j) & 1u)) {
          const uint64_t p = pos[j].next(d, m);
          b[j][i]          = bit_of(p);
          w[j][i]          = __ldg(words + word_of(p));
        }
      }
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
#pragma unroll
      for (int i = 0; i < kHashChunk; ++i)
        if ((w[j][i] & b[j][i]) != b[j][i]) hit &= ~(1u << j);
  }
  uint32_t packed = 0;
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) packed |= ((hit >> j) & 1u) << (8 * j);
  if (kVec && count == kRowsPerThread) {
    *reinterpret_cast<uint32_t*>(out + r0) = packed;
  } else {
    for (int j = 0; j < count; ++j) out[r0 + j] = static_cast<uint8_t>((packed >> (8 * j)) & 1u);
  }
}

// init: the big-endian header words, then zeros
__global__ void __launch_bounds__(kBloomThreads) bloom_init_kernel(uint32_t* __restrict__ buf, int64_t nwords, uint4 hdr, int hdr_words)
{
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kBloomThreads;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kBloomThreads + threadIdx.x; i < nwords; i += stride) {
    uint32_t v = 0;
    if (i < hdr_words) v = i == 0 ? hdr.x : i == 1 ? hdr.y : i == 2 ? hdr.z : hdr.w;
    buf[i] = v;
  }
}

// merge, header check: flag <- 1 when the header of any filter differs from the first one's
__global__ void __launch_bounds__(kBloomThreads) bloom_merge_check_kernel(const uint32_t* __restrict__ child, int64_t stride_words, int32_t nfilters,
                                                                          int hdr_words, int32_t* __restrict__ flag)
{
  const int64_t f = static_cast<int64_t>(blockIdx.x) * kBloomThreads + threadIdx.x + 1;
  if (f >= nfilters) return;
  bool same = true;
  for (int i = 0; i < hdr_words; ++i) same &= __ldg(child + f * stride_words + i) == __ldg(child + i);
  if (!same) *flag = 1;
}

// merge, bit arrays: dst[v] = OR over the filters of src_f[v], VW 32-bit words per access (16-byte accesses for VW = 4)
template <int VW>
struct Vec;
template <> struct Vec<1> { using T = uint32_t; __device__ static T orv(T a, T b) { return a | b; } };
template <> struct Vec<2> { using T = uint2; __device__ static T orv(T a, T b) { return make_uint2(a.x | b.x, a.y | b.y); } };
template <> struct Vec<4> {
  using T = uint4;
  __device__ static T orv(T a, T b) { return make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w); }
};

template <int VW>
__global__ void __launch_bounds__(kBloomThreads) bloom_merge_or_kernel(const uint8_t* __restrict__ src, int64_t stride_bytes, int32_t nfilters,
                                                                       int64_t nvec, uint8_t* __restrict__ dst)
{
  using T        = typename Vec<VW>::T;
  const int64_t v = static_cast<int64_t>(blockIdx.x) * kBloomThreads + threadIdx.x;
  if (v >= nvec) return;
  const T* s = reinterpret_cast<const T*>(src) + v;
  const int64_t sv = stride_bytes / static_cast<int64_t>(sizeof(T));
  T acc = __ldg(s);
  int32_t f = 1;
  for (; f + 4 <= nfilters; f += 4) {                          // four independent loads in flight per thread
    const T a = __ldg(s + f * sv), b = __ldg(s + (f + 1) * sv), c = __ldg(s + (f + 2) * sv), e = __ldg(s + (f + 3) * sv);
    acc = Vec<VW>::orv(acc, Vec<VW>::orv(Vec<VW>::orv(a, b), Vec<VW>::orv(c, e)));
  }
  for (; f < nfilters; ++f) acc = Vec<VW>::orv(acc, __ldg(s + f * sv));
  reinterpret_cast<T*>(dst)[v] = acc;
}

unsigned grid_for(int64_t threads) { return static_cast<unsigned>((threads + kBloomThreads - 1) / kBloomThreads); }

}  // namespace

// m with x % bits == x - mulhi(x, m) * bits, minus bits once more when that is >= bits (32-bit x for V1, 64-bit for V2)
static uint64_t bloom_reciprocal(int32_t version, uint64_t bits)
{
  return version == 1 ? reciprocal_v1(static_cast<uint32_t>(bits)) : reciprocal_v2(bits);
}

static int launch_bloom_init(const BloomHeader& h, uint8_t* buf, cudaStream_t stream)
{
  const int hdr_words = h.version == 1 ? 3 : 4;
  auto bswap          = [](int32_t v) { return __builtin_bswap32(static_cast<uint32_t>(v)); };
  const uint4 hdr     = h.version == 1 ? make_uint4(bswap(1), bswap(h.num_hashes), bswap(h.num_longs), 0u)
                                       : make_uint4(bswap(2), bswap(h.num_hashes), bswap(h.seed), bswap(h.num_longs));
  const int64_t nwords = hdr_words + 2 * static_cast<int64_t>(h.num_longs);
  const unsigned grid  = static_cast<unsigned>(tmin<int64_t>(grid_for(nwords), 16 * sm_count()));
  bloom_init_kernel<<<grid, kBloomThreads, 0, stream>>>(reinterpret_cast<uint32_t*>(buf), nwords, hdr, hdr_words);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_bloom_put(const BloomHeader& h, uint8_t* buf, const srj_column& in, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) return SRJ_OK;
  auto* words       = reinterpret_cast<uint32_t*>(buf + (h.version == 1 ? 12 : 16));
  const uint64_t d  = 64 * static_cast<uint64_t>(h.num_longs);
  const uint64_t m  = bloom_reciprocal(h.version, d);
  const auto* keys  = static_cast<const int64_t*>(in.data);
  const bool vec    = (reinterpret_cast<uintptr_t>(keys) & 15) == 0;
  const unsigned grid = grid_for((n + kRowsPerThread - 1) / kRowsPerThread);
  const uint32_t seed = static_cast<uint32_t>(h.seed);
#define SRJ_BLOOM_PUT(V, VEC) bloom_put_kernel<V, VEC><<<grid, kBloomThreads, 0, stream>>>(words, d, m, h.num_hashes, seed, keys, in.null_mask, n)
  if (h.version == 1) { if (vec) SRJ_BLOOM_PUT(1, true); else SRJ_BLOOM_PUT(1, false); }
  else                { if (vec) SRJ_BLOOM_PUT(2, true); else SRJ_BLOOM_PUT(2, false); }
#undef SRJ_BLOOM_PUT
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_bloom_probe(const BloomHeader& h, const uint8_t* buf, const srj_column& in, uint8_t* out, uint32_t* out_mask, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) return SRJ_OK;
  if (out_mask) {
    const size_t mask_bytes = static_cast<size_t>((n + 31) / 32) * 4;
    if (in.null_mask) SRJ_CUDA_TRY(cudaMemcpyAsync(out_mask, in.null_mask, mask_bytes, cudaMemcpyDeviceToDevice, stream));
    else SRJ_CUDA_TRY(cudaMemsetAsync(out_mask, 0xff, mask_bytes, stream));
  }
  const auto* words  = reinterpret_cast<const uint32_t*>(buf + (h.version == 1 ? 12 : 16));
  const uint64_t d   = 64 * static_cast<uint64_t>(h.num_longs);
  const uint64_t m   = bloom_reciprocal(h.version, d);
  const auto* keys   = static_cast<const int64_t*>(in.data);
  const bool vec     = (reinterpret_cast<uintptr_t>(keys) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0;
  const unsigned grid = grid_for((n + kRowsPerThread - 1) / kRowsPerThread);
  const uint32_t seed = static_cast<uint32_t>(h.seed);
#define SRJ_BLOOM_PROBE(V, VEC) bloom_probe_kernel<V, VEC><<<grid, kBloomThreads, 0, stream>>>(words, d, m, h.num_hashes, seed, keys, n, out)
  if (h.version == 1) { if (vec) SRJ_BLOOM_PROBE(1, true); else SRJ_BLOOM_PROBE(1, false); }
  else                { if (vec) SRJ_BLOOM_PROBE(2, true); else SRJ_BLOOM_PROBE(2, false); }
#undef SRJ_BLOOM_PROBE
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

// header copy, header check (*d_flag <- 1 on a mismatch) and the word-wise OR of `nfilters` filters `stride` bytes apart
static int launch_bloom_merge(const uint8_t* child, int64_t stride, int32_t nfilters, int hdr_bytes, uint8_t* out, int32_t* d_flag, cudaStream_t stream)
{
  SRJ_CUDA_TRY(cudaMemsetAsync(d_flag, 0, 4, stream));
  if (nfilters > 1) {
    bloom_merge_check_kernel<<<grid_for(nfilters - 1), kBloomThreads, 0, stream>>>(reinterpret_cast<const uint32_t*>(child), stride / 4, nfilters,
                                                                                   hdr_bytes / 4, d_flag);
    SRJ_CUDA_TRY(cudaGetLastError());
  }
  SRJ_CUDA_TRY(cudaMemcpyAsync(out, child, hdr_bytes, cudaMemcpyDeviceToDevice, stream));
  const uint8_t* src    = child + hdr_bytes;
  uint8_t* dst          = out + hdr_bytes;
  const int64_t nbytes  = stride - hdr_bytes;
  auto aligned = [&](int a) {
    return (reinterpret_cast<uintptr_t>(src) % a) == 0 && (reinterpret_cast<uintptr_t>(dst) % a) == 0 && stride % a == 0 && nbytes % a == 0;
  };
  if (aligned(16)) bloom_merge_or_kernel<4><<<grid_for(nbytes / 16), kBloomThreads, 0, stream>>>(src, stride, nfilters, nbytes / 16, dst);
  else if (aligned(8)) bloom_merge_or_kernel<2><<<grid_for(nbytes / 8), kBloomThreads, 0, stream>>>(src, stride, nfilters, nbytes / 8, dst);
  else bloom_merge_or_kernel<1><<<grid_for(nbytes / 4), kBloomThreads, 0, stream>>>(src, stride, nfilters, nbytes / 4, dst);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

static int bloom_hdr_bytes(int32_t version) { return version == 2 ? 16 : 12; }   // bloom_filter.hpp:59-63

static int bloom_check_params(const char* what, int32_t version, int32_t num_hashes, int64_t num_longs)
{
  if (version != 1 && version != 2) { set_error("%s: Bloom filter version must be 1 or 2 (got %d)", what, version); return SRJ_EINVAL; }
  if (num_hashes <= 0) { set_error("%s: Bloom filters must have a positive hash count", what); return SRJ_EINVAL; }
  if (num_longs <= 0) { set_error("%s: Bloom filters must have a positive number of bits", what); return SRJ_EINVAL; }
  if (bloom_hdr_bytes(version) + 8 * num_longs > INT32_MAX) { set_error("%s: Bloom filter buffer size exceeds int32 range", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

// bloom_filter.cu:189-236 + the size checks of put / probe (bloom_filter.cu:340, 459): parse the serialized header of a
// filter of `bytes` bytes at device address `buf` (one read-back, one stream synchronisation)
static int bloom_read_header(const char* what, const uint8_t* buf, int64_t bytes, BloomHeader* h, cudaStream_t stream)
{
  if (bytes < 12 || !buf) { set_error("%s: Encountered truncated bloom filter", what); return SRJ_EINVAL; }
  if (reinterpret_cast<uintptr_t>(buf) & 3) { set_error("%s: the filter buffer must be 4-byte aligned", what); return SRJ_EINVAL; }
  uint32_t raw[4] = {0, 0, 0, 0};
  SRJ_CUDA_TRY(cudaMemcpyAsync(raw, buf, static_cast<size_t>(std::min<int64_t>(bytes, 16)), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  const auto be = [](uint32_t v) { return static_cast<int32_t>(__builtin_bswap32(v)); };
  h->version    = be(raw[0]);
  if (h->version != 1 && h->version != 2) { set_error("%s: Unexpected bloom filter version %d", what, h->version); return SRJ_EINVAL; }
  const int hdr = bloom_hdr_bytes(h->version);
  if (bytes < hdr) { set_error("%s: Encountered truncated bloom filter header", what); return SRJ_EINVAL; }
  h->num_hashes = be(raw[1]);
  h->seed       = h->version == 2 ? be(raw[2]) : 0;
  h->num_longs  = h->version == 2 ? be(raw[3]) : be(raw[2]);
  if (h->num_longs <= 0) { set_error("%s: Invalid empty bloom filter size", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

static int bloom_check_input(const char* what, const srj_column* in)
{
  if (!in) { set_error("%s: input is null", what); return SRJ_EINVAL; }
  if (in->type_id != SRJ_INT64) { set_error("%s: bloom filters take one INT64 column (type id %d)", what, in->type_id); return SRJ_EUNSUPPORTED; }
  if (in->size < 0 || (in->size > 0 && !in->data)) { set_error("%s: bad input column", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

// put / probe: the buffer must be exactly one filter, and V1 indexes with 31-bit positions (bloom_filter.cu:340-359, 459-471)
static int bloom_check_filter(const char* what, const BloomHeader& h, int64_t bytes)
{
  if (bytes != bloom_hdr_bytes(h.version) + 8 * static_cast<int64_t>(h.num_longs)) {
    set_error("%s: Encountered invalid/mismatched bloom filter buffer data", what);
    return SRJ_EINVAL;
  }
  if (h.version == 1 && 64 * static_cast<int64_t>(h.num_longs) > INT32_MAX) { set_error("%s: V1 bloom filter bit count exceeds int32 range", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

int srj_bloom_filter_sizes(int32_t version, int32_t num_hashes, int64_t bits, int32_t* num_longs, int64_t* total_bytes)
{
  SRJ_API_RANGE();
  if (!num_longs || !total_bytes) { set_error("bloom_filter_sizes: bad argument"); return SRJ_EINVAL; }
  // BloomFilterJni.cpp:40-47: Spark's BitArray holds at most INT32_MAX longs
  if (bits > static_cast<int64_t>(INT32_MAX) * 64) {
    set_error("bloom_filter_sizes: bloom filter bit count must be positive and less than or equal to the maximum supported size");
    return SRJ_EINVAL;
  }
  const int64_t longs = bits > 0 ? (bits + 63) / 64 : 0;
  const int rc        = bloom_check_params("bloom_filter_sizes", version, num_hashes, longs);
  if (rc != SRJ_OK) return rc;
  *num_longs   = static_cast<int32_t>(longs);
  *total_bytes = bloom_hdr_bytes(version) + 8 * longs;
  return SRJ_OK;
}

int srj_bloom_filter_init(int32_t version, int32_t num_hashes, int32_t num_longs, int32_t seed, uint8_t* filter, void* stream)
{
  SRJ_API_RANGE();
  const int rc = bloom_check_params("bloom_filter_init", version, num_hashes, num_longs);
  if (rc != SRJ_OK) return rc;
  if (check_out("bloom_filter_init", "filter buffer", filter, 4) != SRJ_OK) return SRJ_EINVAL;
  return launch_bloom_init(BloomHeader{version, num_hashes, version == 2 ? seed : 0, num_longs}, filter, static_cast<cudaStream_t>(stream));
}

int srj_bloom_filter_put(uint8_t* filter, int64_t filter_bytes, const srj_column* input, void* stream)
{
  SRJ_API_RANGE();
  int rc = bloom_check_input("bloom_filter_put", input);
  if (rc != SRJ_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BloomHeader h{};
  if ((rc = bloom_read_header("bloom_filter_put", filter, filter_bytes, &h, st)) != SRJ_OK) return rc;
  if ((rc = bloom_check_filter("bloom_filter_put", h, filter_bytes)) != SRJ_OK) return rc;
  return launch_bloom_put(h, filter, *input, st);
}

int srj_bloom_filter_probe(const uint8_t* filter, int64_t filter_bytes, const srj_column* input, uint8_t* out, uint32_t* out_mask, void* stream)
{
  SRJ_API_RANGE();
  int rc = bloom_check_input("bloom_filter_probe", input);
  if (rc != SRJ_OK) return rc;
  if ((rc = check_out("bloom_filter_probe", "output", out, 1, input->size > 0)) != SRJ_OK) return rc;
  if ((rc = check_out("bloom_filter_probe", "output mask", out_mask, 1, input->size > 0 && input->null_mask)) != SRJ_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BloomHeader h{};
  if ((rc = bloom_read_header("bloom_filter_probe", filter, filter_bytes, &h, st)) != SRJ_OK) return rc;
  if ((rc = bloom_check_filter("bloom_filter_probe", h, filter_bytes)) != SRJ_OK) return rc;
  return launch_bloom_probe(h, filter, *input, out, out_mask, st);
}

int64_t srj_bloom_filter_merge_workspace_bytes(void) { return 16; }

// bloom_filter.cu:374-449.  The stride of the filters is known from the sizes alone (filters_bytes / num_filters), and the
// header size follows from it (12 + 8 * num_longs is 4 mod 8, 16 + 8 * num_longs is 0 mod 8), so the header check and
// the OR are enqueued before the first header is read back; header and flag then come back with one synchronisation and
// the checks run in the reference's order.  On an error `out` holds garbage.
int srj_bloom_filter_merge(const uint8_t* filters, int64_t filters_bytes, int32_t num_filters, uint8_t* out, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  const char* what = "bloom_filter_merge";
  if (num_filters <= 0 || filters_bytes < 0 || (filters_bytes > 0 && !filters)) { set_error("%s: bad argument", what); return SRJ_EINVAL; }
  if (filters_bytes < 12) { set_error("%s: Encountered truncated bloom filter", what); return SRJ_EINVAL; }
  if (!workspace || !out) { set_error("%s: the output and the workspace are needed", what); return SRJ_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(filters) | reinterpret_cast<uintptr_t>(out)) & 3) { set_error("%s: the buffers must be 4-byte aligned", what); return SRJ_EINVAL; }
  cudaStream_t st       = static_cast<cudaStream_t>(stream);
  const int64_t stride  = filters_bytes / num_filters;
  const bool launched   = stride * num_filters == filters_bytes && stride >= 16 && stride % 4 == 0 && stride <= INT32_MAX;
  auto* d_flag          = static_cast<int32_t*>(workspace);
  if (launched) {
    const int rc = launch_bloom_merge(filters, stride, num_filters, stride % 8 == 4 ? 12 : 16, out, d_flag, st);
    if (rc != SRJ_OK) return rc;
  }
  int32_t flag    = 0;
  uint32_t raw[4] = {0, 0, 0, 0};
  SRJ_CUDA_TRY(cudaMemcpyAsync(raw, filters, static_cast<size_t>(std::min<int64_t>(filters_bytes, 16)), cudaMemcpyDeviceToHost, st));
  if (launched) SRJ_CUDA_TRY(cudaMemcpyAsync(&flag, d_flag, 4, cudaMemcpyDeviceToHost, st));
  SRJ_CUDA_TRY(cudaStreamSynchronize(st));
  const auto be = [](uint32_t v) { return static_cast<int32_t>(__builtin_bswap32(v)); };
  const int32_t version = be(raw[0]);
  if (version != 1 && version != 2) { set_error("%s: Unexpected bloom filter version %d", what, version); return SRJ_EINVAL; }
  const int hdr = bloom_hdr_bytes(version);
  if (filters_bytes < hdr) { set_error("%s: Encountered truncated bloom filter header", what); return SRJ_EINVAL; }
  const int64_t num_longs = version == 2 ? be(raw[3]) : be(raw[2]);
  if (num_longs <= 0) { set_error("%s: Invalid empty bloom filter size", what); return SRJ_EINVAL; }
  if (filters_bytes != (hdr + 8 * num_longs) * num_filters) { set_error("%s: Encountered invalid/mismatched bloom filter buffer data", what); return SRJ_EINVAL; }
  if (hdr + 8 * num_longs > INT32_MAX) { set_error("%s: Bloom filter buffer size exceeds int32 range", what); return SRJ_EINVAL; }
  if (!launched || flag) { set_error("%s: Mismatch of bloom filter parameters", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

}  // extern "C"
