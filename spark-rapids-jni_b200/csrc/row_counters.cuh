// row_counters.cuh -- the two counters of null_counter() that a per-row kernel fills: counters[0] the null rows,
// counters[1] the smallest error row (kNoRow: none).  Each CTA adds to them with one atomic each, and the host resets
// them before the launch and reads both back after it with one synchronisation.
#pragma once
#include "common.cuh"
#include "kernels.hpp"

namespace srj {

constexpr unsigned long long kNoRow = ~0ull;   // the error counter's "none", read back as -1

// counters[0] += nulls and counters[1] = min(counters[1], first) over the CTA, one global atomic each
__device__ __forceinline__ void flush_counters(unsigned long long nulls, unsigned long long first, unsigned long long* counters)
{
  __shared__ unsigned long long s_nulls, s_first;
  if (threadIdx.x == 0) {
    s_nulls = 0;
    s_first = kNoRow;
  }
  __syncthreads();
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    nulls += __shfl_xor_sync(0xffffffffu, nulls, o);
    first = tmin(first, __shfl_xor_sync(0xffffffffu, first, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (nulls) atomicAdd(&s_nulls, nulls);
    if (first != kNoRow) atomicMin(&s_first, first);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_nulls) atomicAdd(counters, s_nulls);
    if (s_first != kNoRow) atomicMin(counters + 1, s_first);
  }
}

// the two counters: reset, and read back after the launch (one synchronisation)
inline int counters_reset(unsigned long long** d, cudaStream_t stream)
{
  int rc = null_counter(d);
  if (rc != SRJ_OK) return rc;
  SRJ_CUDA_TRY(cudaMemsetAsync(*d, 0, sizeof(unsigned long long), stream));
  SRJ_CUDA_TRY(cudaMemsetAsync(*d + 1, 0xff, sizeof(unsigned long long), stream));
  return SRJ_OK;
}

inline int counters_read(const unsigned long long* d, int64_t* nulls, int64_t* error_row, cudaStream_t stream)
{
  unsigned long long h[2];
  SRJ_CUDA_TRY(cudaMemcpyAsync(h, d, sizeof(h), cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  if (nulls) *nulls = static_cast<int64_t>(h[0]);
  *error_row = static_cast<int64_t>(h[1]);       // kNoRow reads as -1
  return SRJ_OK;
}

}  // namespace srj
