// Shared device helpers for libgpk (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>

#include "../../include/gpk.h"

namespace gpk {

extern long long g_launch_count;  // defined in util.cu

#define GPK_CHECK_LAUNCH()                                   \
  do {                                                       \
    cudaError_t e__ = cudaGetLastError();                    \
    if (e__ != cudaSuccess) return -1000 - (int)e__;         \
  } while (0)

#define GPK_COUNT_LAUNCH() (++::gpk::g_launch_count)

// Lets `Kernel` launch with `bytes` of dynamic shared memory on the current device.  CUDA keeps this opt-in per kernel and
// per device, so the largest size set so far is remembered per device and the driver is called only for a larger
// request.  Returns 0, -1000 - cudaError, or GPK_ERR_UNSUPPORTED on a device ordinal above 63.
template <auto Kernel>
int opt_in_smem(int bytes) {
  static std::atomic<int> set[64];  // by device ordinal
  static std::mutex mu;             // never lowers a size another host thread has just set
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return -1000 - (int)e;
  if (dev >= 64) return GPK_ERR_UNSUPPORTED;
  if (bytes <= set[dev].load(std::memory_order_acquire)) return 0;
  std::lock_guard<std::mutex> lock(mu);
  if (bytes <= set[dev].load(std::memory_order_relaxed)) return 0;
  e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return -1000 - (int)e;
  set[dev].store(bytes, std::memory_order_release);
  return 0;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- cp.async (LDGSTS) 16-byte copies -------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// ---- mbarrier + 1-D bulk async copy (TMA engine, SASS: UBLKCP) -------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");  // the data the barrier guards must not be read before the wait
}
// ---- thread-block clusters: rank, cluster-wide barrier, remote mbarrier arrive, multicast TMA (SASS: UTMALDG.MULTICAST)
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster; orders the shared-memory writes before it (mbarrier inits included) for all
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;\n" ::: "memory");
}
// arrive on the mbarrier at `bar`'s shared-memory offset in CTA `rank` of the cluster (this CTA's own rank included).
// Default (CTA-scope release) semantics, as a consumer's release of a TMA pipeline stage needs: a cluster-scope release
// would put a MEMBAR.GPU, which waits for the thread's outstanding global reductions, in front of every arrive
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile(
      "{\n"
      ".reg .b32 remote;\n"
      "mapa.shared::cluster.u32 remote, %0, %1;\n"
      "mbarrier.arrive.shared::cluster.b64 _, [remote];\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(rank)
      : "memory");
}
// 3-D TMA box (tensor map `map`, a __grid_constant__ CUtensorMap) into `dst`'s offset in every CTA of `cta_mask`; each
// destination CTA's mbarrier at `bar`'s offset receives the box's bytes
__device__ __forceinline__ void tma_load_3d_multicast(void* dst, const void* map, int c0, int c1, int c2, uint64_t* bar,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3, "
      "%4}], [%5], %6;\n" ::"r"(smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---- fp64 tensor-core MMA (SASS: DMMA.8x8x4) --------------------------------------------------------
// D(8x8) += A(8x4, row) * B(4x8, col).  Lane l holds A[l/4][l%4], B[k=l%4][n=l/4], C[l/4][2*(l%4) + {0,1}].
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// The int8-slice emulation arguments (slices, ws, ws_bytes) of the fp64 entry points: slices 0 (fp64 tensor cores) or 5..8
// with a 1024-byte aligned scratch.  0 or GPK_ERR_ARG (gemm_oz.cu).
int oz_check_emulation(int32_t slices, const void* ws);

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace gpk
