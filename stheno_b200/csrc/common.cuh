// Shared helpers for libgpk (sm_90a only), and the host functions one translation unit calls in another.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>

#include "../../include/gpk.h"

namespace gpk {

extern long long g_launch_count;  // defined in util.cu

// a CUDA runtime result as a libgpk return code: 0, or -1000 - the cudaError_t (gpk.h)
inline int cuda_rc(cudaError_t e) { return e == cudaSuccess ? 0 : -1000 - (int)e; }

#define GPK_CHECK_LAUNCH()                                                  \
  do {                                                                      \
    if (const int rc__ = ::gpk::cuda_rc(cudaGetLastError())) return rc__; \
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
  if (const int rc = cuda_rc(cudaGetDevice(&dev))) return rc;
  if (dev >= 64) return GPK_ERR_UNSUPPORTED;
  if (bytes <= set[dev].load(std::memory_order_acquire)) return 0;
  std::lock_guard<std::mutex> lock(mu);
  if (bytes <= set[dev].load(std::memory_order_relaxed)) return 0;
  if (const int rc = cuda_rc(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes))) return rc;
  set[dev].store(bytes, std::memory_order_release);
  return 0;
}

// exp, sqrt, rsqrt and log of a T: the fp64 or the fp32 library function
template <typename T>
__device__ __forceinline__ T t_exp(T v) {
  return sizeof(T) == 8 ? (T)exp((double)v) : (T)expf((float)v);
}
template <typename T>
__device__ __forceinline__ T t_sqrt(T v) {
  return sizeof(T) == 8 ? (T)sqrt((double)v) : (T)sqrtf((float)v);
}
template <typename T>
__device__ __forceinline__ T t_rsqrt(T v) {
  return sizeof(T) == 8 ? (T)rsqrt((double)v) : (T)rsqrtf((float)v);
}
template <typename T>
__device__ __forceinline__ T t_log(T v) {
  return sizeof(T) == 8 ? (T)log((double)v) : (T)logf((float)v);
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

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- host functions that one translation unit calls in another ----------------------------------------------------------
// Each is defined in the file named above it, on the caller's stream, and returns 0 or a negative gpk.h error code unless
// its comment says otherwise.  (S, ws, ws_bytes) are the int8-slice emulation arguments of gpk.h's fp64 entry points; the
// fp32 overloads ignore them.

// kernel_matrix.cu: out[i][j] = k(x_i, y_j) for one problem, no noise or jitter, zero padded to multiples of 128
int kernel_rows(const gpk_kernel_desc* desc, const double* xg, int64_t xg_gstride, int64_t n, const double* yg,
                int64_t yg_gstride, int64_t n2, int32_t d, double* out, int64_t ldo, cudaStream_t stream);
int kernel_rows(const gpk_kernel_desc* desc, const float* xg, int64_t xg_gstride, int64_t n, const float* yg,
                int64_t yg_gstride, int64_t n2, int32_t d, float* out, int64_t ldo, cudaStream_t stream);

// util.cu: dot[r] = <V[r, :n_cols], b> and sq[r] = |V[r, :n_cols]|^2 for r < rows, one matrix; dot or sq may be null
int row_dot_sq(const double* V, int64_t ldv, int64_t rows, int64_t n_cols, const double* b, double* dot, double* sq,
               cudaStream_t stream);
int row_dot_sq(const float* V, int64_t ldv, int64_t rows, int64_t n_cols, const float* b, float* dot, float* sq,
               cudaStream_t stream);

// gemm.cu: C = beta C + alpha A B^T (gpk_gemm_nt_f64 / _f32)
int gemm_nt(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, int64_t a_bs, const double* B,
            int64_t ldb, int64_t b_bs, double beta, double* C, int64_t ldc, int64_t c_bs, int32_t lower, int32_t batch,
            int32_t S, void* ws, int64_t ws_bytes, cudaStream_t stream);
int gemm_nt(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t lda, int64_t a_bs, const float* B,
            int64_t ldb, int64_t b_bs, float beta, float* C, int64_t ldc, int64_t c_bs, int32_t lower, int32_t batch,
            int32_t S, void* ws, int64_t ws_bytes, cudaStream_t stream);
// gemm.cu: the in-situ event profile of the fp64 GEMMs (gpk_gemm_profile_*); kind 0 = DMMA, 1 = int8-slice emulation
bool prof_enabled();
void prof_begin(cudaStream_t stream, double flops, int kind);
void prof_end(cudaStream_t stream);

// potrf.cu: X L^T = B in place for one matrix (gpk_trsm_right_f64 / _f32)
int trsm_right(const double* L, int64_t ldl, int64_t n_pad, double* B, int64_t ldb, int64_t rows, int32_t S, void* ws,
               int64_t ws_bytes, cudaStream_t stream);
int trsm_right(const float* L, int64_t ldl, int64_t n_pad, float* B, int64_t ldb, int64_t rows, int32_t S, void* ws,
               int64_t ws_bytes, cudaStream_t stream);

// gemm_oz.cu: the emulation arguments of an fp64 entry point are valid: S = 0 (fp64 tensor cores), or 5..8 with a
// 1024-byte aligned scratch.  0 or GPK_ERR_ARG
int oz_check_emulation(int32_t S, const void* ws);
// gemm_oz.cu: scratch bytes of the S int8 slices of `rows` rows of K columns, with their row exponents
int64_t oz_ws_bytes(int64_t rows, int64_t K, int32_t S);
// gemm_oz.cu: slices of the rows x K panel P into ws, laid out for cap_rows rows
int oz_slice_panel(const double* P, int64_t ldp, int64_t rows, int64_t K, void* ws, int64_t cap_rows, int32_t S,
                   cudaStream_t stream);
// gemm_oz.cu: C[M x N] = beta C + alpha A B^T, A = sliced rows [rowA, rowA + M) of wsA, B = sliced rows [rowB, rowB + N) of wsB
int oz_gemm_sliced(int64_t M, int64_t N, int64_t K, double alpha, const void* wsA, int64_t capA, int64_t rowA,
                   const void* wsB, int64_t capB, int64_t rowB, double beta, double* C, int64_t ldc, int32_t lower,
                   int32_t S, cudaStream_t stream);
// gemm_oz.cu: gemm_nt on the int8 tensor cores.  1 = done, 0 = not applicable (the caller uses DMMA), < 0 = error
int gemm_nt_f64_emulated(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, const double* B,
                         int64_t ldb, double beta, double* C, int64_t ldc, int32_t lower, int32_t S, void* ws,
                         int64_t ws_bytes, cudaStream_t stream);

// gemm_tc32.cu: fp32 gemm_nt on the tensor cores (wgmma, 3xTF32).  1 = launched, 0 = shape not supported (the caller uses
// the FFMA kernel), < 0 = error
int gemm_nt_f32_tc(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t lda, int64_t a_bs, const float* B,
                   int64_t ldb, int64_t b_bs, float beta, float* C, int64_t ldc, int64_t c_bs, int32_t lower,
                   int32_t batch, cudaStream_t stream);
// gemm_tc32.cu: C[M x N] (fp64, lower tiles) -= P[0:M] P[0:N]^T, P = the M x K fp32 panel ws_rows (convert_panel_f32)
int syrk_f64_tf32x3(int64_t M, int64_t N, int64_t K, const float* ws_rows, double* C, int64_t ldc, cudaStream_t stream);
// gemm_tc32.cu: ws (rows x K, dense) = the fp64 panel P rounded to fp32
int convert_panel_f32(const double* P, int64_t ldp, int64_t rows, int64_t K, float* ws, cudaStream_t stream);

}  // namespace gpk
