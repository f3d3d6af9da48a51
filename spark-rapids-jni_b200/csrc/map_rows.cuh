// map_rows.cuh -- the per-thread body of the fixed-width map kernels (iceberg.cu's ice_map_kernel, datetime.cu's
// dt_map_kernel, timezone.cu's grid-stride tz_convert_kernel / orc_tz_kernel), and RowWords, the aligned word reader of a
// STRING row.
#pragma once

#include <stdint.h>

#include "common.cuh"

namespace srj {

constexpr int kMapRows = 4;       // rows per thread

__device__ __forceinline__ int32_t ld_elem(const int32_t* p) { return __ldg(p); }
__device__ __forceinline__ int64_t ld_elem(const int64_t* p) { return __ldg(reinterpret_cast<const long long*>(p)); }

template <class T>
union RowBuf {
  T v[kMapRows];
  uint4 u[sizeof(T) * kMapRows / 16];
};

// One thread's rows [r0, r0 + kMapRows) of a map over n rows (r0 a multiple of kMapRows), loaded and stored with 16-byte
// accesses when vec (both buffers 16-byte aligned) and the thread owns a full group.  With Op::kNullsZero a null row gets
// Out{} instead of op(v).  Op supplies In, Out and a const operator().
template <class Op>
__device__ __forceinline__ void map_rows_at(int64_t r0, const typename Op::In* __restrict__ in, const uint32_t* __restrict__ mask,
                                            typename Op::Out* __restrict__ out, int64_t n, bool vec, const Op& op)
{
  using In         = typename Op::In;
  using Out        = typename Op::Out;
  if (r0 >= n) return;
  const int cnt = static_cast<int>(tmin<int64_t>(kMapRows, n - r0));
  RowBuf<In> a;
  if (vec && cnt == kMapRows) {
#pragma unroll
    for (int i = 0; i < static_cast<int>(sizeof(a.u) / 16); ++i) a.u[i] = __ldg(reinterpret_cast<const uint4*>(in + r0) + i);
  } else {
#pragma unroll
    for (int j = 0; j < kMapRows; ++j) a.v[j] = j < cnt ? ld_elem(in + r0 + j) : In{};
  }
  uint32_t valid = 0xfu;                                       // r0 is a multiple of 4: the rows share one mask word
  if (Op::kNullsZero && mask) valid = __ldg(mask + (r0 >> 5)) >> (r0 & 31);
  RowBuf<Out> b;
#pragma unroll
  for (int j = 0; j < kMapRows; ++j) b.v[j] = ((valid >> j) & 1u) ? op(a.v[j]) : Out{};
  if (vec && cnt == kMapRows) {
#pragma unroll
    for (int i = 0; i < static_cast<int>(sizeof(b.u) / 16); ++i) reinterpret_cast<uint4*>(out + r0)[i] = b.u[i];
  } else {
#pragma unroll
    for (int j = 0; j < kMapRows; ++j)
      if (j < cnt) out[r0 + j] = b.v[j];
  }
}

// One thread of a map over n rows, one group per thread: r0 = (block * kThreads + thread) * kMapRows.
template <int kThreads, class Op>
__device__ __forceinline__ void map_rows(const typename Op::In* __restrict__ in, const uint32_t* __restrict__ mask,
                                         typename Op::Out* __restrict__ out, int64_t n, bool vec, const Op& op)
{
  map_rows_at((static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) * kMapRows, in, mask, out, n, vec, op);
}

// The bytes [0, len) of a row starting at s: word(j) is aligned word j counted from the one holding s[0] (0 when it holds
// no byte of the row); at(a, b) is the 4 row bytes starting at the first byte of a.
struct RowWords {
  const uint32_t* aw;
  uint32_t sh;        // 8 * (s & 3)
  int32_t lim;        // (s & 3) + len: word j holds a row byte iff 4j < lim
  __device__ __forceinline__ RowWords(const uint8_t* s, int32_t len)
  {
    aw  = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(s) & ~uintptr_t{3});
    sh  = 8u * static_cast<uint32_t>(reinterpret_cast<uintptr_t>(s) & 3);
    lim = static_cast<int32_t>(reinterpret_cast<uintptr_t>(s) & 3) + len;
  }
  __device__ __forceinline__ uint32_t word(int32_t j) const { return 4 * j < lim ? __ldg(aw + j) : 0u; }
  __device__ __forceinline__ uint32_t at(uint32_t a, uint32_t b) const { return __funnelshift_r(a, b, sh); }
};

}  // namespace srj
