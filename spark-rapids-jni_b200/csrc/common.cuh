// common.cuh -- shared device helpers for the sm_90a row<->column kernels:
// mbarrier / TMA (1-D bulk async copy) PTX wrappers, warp utilities, error plumbing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/srj_b200.h"

namespace srj {

constexpr int kWarp = 32;

// ---- error plumbing (host) --------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
int sm_count();  // multiprocessors of the current device (grid caps of the grid-stride kernels)
#define SRJ_CUDA_TRY(expr)                                     \
  do {                                                         \
    cudaError_t _e = (expr);                                   \
    if (_e != cudaSuccess) return ::srj::cuda_fail(_e, #expr); \
  } while (0)

// ---- device: shared-memory address + mbarrier + bulk copies -----------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p)
{
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

// make mbarrier.init visible to the async (TMA) proxy before the first bulk copy signals it
__device__ __forceinline__ void fence_mbar_init()
{
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t tx_bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(tx_bytes)
               : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
  uint32_t ok;
  asm volatile(
    "{\n\t.reg .pred p;\n\t"
    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
    "selp.b32 %0, 1, 0, p;\n\t}"
    : "=r"(ok)
    : "r"(smem_u32(bar)), "r"(parity), "r"(0x200000u)  // suspend-time hint (ns): sleep in HW, do not spin
    : "memory");
  return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
  while (!mbar_try_wait(bar, parity)) {}  // try_wait suspends in hardware up to the hint; no software back-off
                                          // (a __nanosleep here wakes up later)
}

// Waiter that backs off between probes: for issue-bound kernels whose consumer warps finish unevenly
// (a spinning waiter steals issue slots from the warps still working).  Costs wake-up latency.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity, unsigned ns)
{
  while (!mbar_try_wait(bar, parity)) { __nanosleep(ns); }
}

// TMA 1-D bulk load global -> shared, completion counted in bytes on `bar` (SASS: UBLKCP).
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                 smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// TMA 1-D bulk store shared -> global (bulk async-group completion).
__device__ __forceinline__ void tma_store_1d(void* gdst, const void* smem_src, uint32_t bytes)
{
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read()
{
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all()
{
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// order generic-proxy smem writes before async-proxy (TMA store) reads
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void named_bar_sync(int id, int nthreads)
{
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

// streaming global stores / loads (data is touched once: keep it out of L1, evict-first in L2)
__device__ __forceinline__ void st_cs_u32(void* p, uint32_t v) { __stcs(reinterpret_cast<unsigned int*>(p), v); }

template <class T>
__host__ __device__ __forceinline__ T tmin(T a, T b) { return a < b ? a : b; }
template <class T>
__host__ __device__ __forceinline__ T tmax(T a, T b) { return a > b ? a : b; }

__host__ __device__ inline int64_t round_up64(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

}  // namespace srj
