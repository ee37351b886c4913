// fp32 GEMM  C = beta*C + alpha * A * B^T  on the Hopper tensor cores (wgmma.mma_async .tf32 + TMA), with fp32-level
// accuracy through the 3xTF32 split:   a = a_hi + a_lo  (a_hi = the 19 bits the TF32 datapath keeps, a_lo = a - a_hi)
//     a b  ~=  a_hi b_hi + a_hi b_lo + a_lo b_hi        (relative error ~2^-21, the fp32 FFMA kernel's is 2^-24)
//
// One 128 x 128 output tile per CTA, fp32 accumulators in registers, three warpgroups:
//   warpgroup 0     TMA producer (one thread): 128 x 32 fp32 tiles of A and B per k-block (cp.async.bulk.tensor.3d,
//                   SWIZZLE_128B, mbarrier complete_tx) into a 3-stage ring
//   warpgroups 1-2  consumers, rows 0-63 / 64-127 of the tile: as soon as a stage lands they write the low parts
//                   a - trunc_tf32(a) of both tiles next to it (element-wise, so the swizzled layout does not matter),
//                   fence.proxy.async, and after a barrier of both warpgroups issue 12 x wgmma m64n128k8
//                   -- (A, B), (A, B_lo), (A_lo, B) for each of the four 32-byte K slices -- straight from shared-memory
//                   descriptors; the stage goes back to the producer when the warpgroup's MMAs on it have completed.
//                   Epilogue: C read-modify-write from the accumulator registers.
// Used by the fp32 (batched) Cholesky for its trailing / panel updates (BASELINE config 3).  The fp64 default path
// cannot use this unit (no f64 wgmma); see DESIGN.md section 8.
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace gpk {

constexpr int TC_BM = 128, TC_BN = 128, TC_BK = 32;
constexpr int TC_TILE_BYTES = TC_BM * TC_BK * 4;  // 16 KB per A / B tile
constexpr int TC_GEMM_THREADS = 384;
constexpr int TC_STAGE_BYTES = 4 * TC_TILE_BYTES;  // A, A_lo, B, B_lo
constexpr int TC_STAGES = 3;
constexpr int TC_SMEM_BYTES = TC_STAGES * TC_STAGE_BYTES + 1024;

struct TcParams {
  float alpha, beta;
  void* C;  // float* or double* (CT of the kernel)
  int64_t ldc, c_bs;
  int32_t K, lower, tiles_m, tiles_n;
};

__device__ __forceinline__ void mbar_wait_parity(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "TCW_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra TCW_DONE;\n"
      "bra TCW_LOOP;\n"
      "TCW_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}

// Exact for every finite value, subnormals included.  For +-inf it is inf - inf = NaN, so a row holding an infinity comes out
// NaN (include/gpk.h, tests/test_fp32_route.py).
__device__ __forceinline__ float4 tf32_low_part(float4 v) {
  float4 lo;
  lo.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u);
  lo.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
  lo.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u);
  lo.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
  return lo;
}

// CT = type of C: float (fp32 problems) or double (opt-in mixed precision: fp64 matrix, fp32 operands -- the
// "tf32 where the user opts in" trailing update of the fp64 Cholesky).
template <typename CT>
__global__ void __launch_bounds__(TC_GEMM_THREADS, 1)
gemm_nt_f32_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                      const TcParams p) {
  int tm, tn;
  {
    const int GROUP = 8, per_group = GROUP * p.tiles_n, id = blockIdx.x;
    const int group = id / per_group, first_m = group * GROUP, gsize = min(p.tiles_m - first_m, GROUP);
    const int r = id - group * per_group;
    tm = first_m + r % gsize;
    tn = r / gsize;
  }
  if (p.lower && tn * TC_BN >= (tm + 1) * TC_BM) return;
  const int b = blockIdx.y;
  const int wg = threadIdx.x >> 7;

  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full_bar[TC_STAGES], empty_bar[TC_STAGES];

  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 256);  // every consumer thread, after its warpgroup's MMAs on the stage completed
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int KB = p.K / TC_BK;

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::);
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < KB; ++kb) {
        const int s = kb % TC_STAGES, it = kb / TC_STAGES;
        if (it > 0) mbar_wait_parity(&empty_bar[s], (it - 1) & 1);
        uint8_t* st = smem + s * TC_STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[s], 2 * TC_TILE_BYTES);
        tma_load_3d(st, &mapA, kb * TC_BK, tm * TC_BM, b, &full_bar[s]);
        tma_load_3d(st + 2 * TC_TILE_BYTES, &mapB, kb * TC_BK, tn * TC_BN, b, &full_bar[s]);
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::);
  const int t = threadIdx.x - 128;               // 0..255 over both consumer warpgroups
  const int tid = t & 127, wrow = 64 * (wg - 1);  // thread in the warpgroup, first tile row it owns
  float acc[64];
  for (int kb = 0; kb < KB; ++kb) {
    const int s = kb % TC_STAGES, it = kb / TC_STAGES;
    mbar_wait_parity(&full_bar[s], it & 1);
    float4* hiA = reinterpret_cast<float4*>(smem + s * TC_STAGE_BYTES);
    float4* loA = hiA + TC_TILE_BYTES / 16;
    float4* hiB = hiA + 2 * TC_TILE_BYTES / 16;
    float4* loB = hiB + TC_TILE_BYTES / 16;
#pragma unroll 4
    for (int i = t; i < TC_TILE_BYTES / 16; i += 256) {
      loA[i] = tf32_low_part(hiA[i]);
      loB[i] = tf32_low_part(hiB[i]);
    }
    fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
    asm volatile("bar.sync 1, 256;\n" ::: "memory");
    const uint32_t a_hi = smem_u32(smem + s * TC_STAGE_BYTES) + wrow * (TC_BK * 4), a_lo = a_hi + TC_TILE_BYTES;
    const uint32_t b_hi = smem_u32(smem + s * TC_STAGE_BYTES) + 2 * TC_TILE_BYTES, b_lo = b_hi + TC_TILE_BYTES;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {  // wgmma K = 8 tf32 = 32 bytes inside the 128-byte swizzle row
      const uint32_t off = ks * 32;
      wgmma_tf32_n128(acc, wgmma_desc<128>(a_hi + off), wgmma_desc<128>(b_hi + off), (kb > 0 || ks > 0) ? 1u : 0u);
      wgmma_tf32_n128(acc, wgmma_desc<128>(a_hi + off), wgmma_desc<128>(b_lo + off), 1u);
      wgmma_tf32_n128(acc, wgmma_desc<128>(a_lo + off), wgmma_desc<128>(b_hi + off), 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (kb > 0) mbar_arrive(&empty_bar[(kb - 1) % TC_STAGES]);
  }
  wgmma_wait<0>();
  // ---- epilogue: registers -> C (read-modify-write); registers 2j, 2j + 1 are adjacent columns of one row ----
  const int r_lo = 16 * (tid >> 5) + ((tid & 31) >> 2), c_lo = 2 * (tid & 3);
  CT* Ct = static_cast<CT*>(p.C) + (int64_t)b * p.c_bs + ((int64_t)tm * TC_BM + wrow + r_lo) * p.ldc + (int64_t)tn * TC_BN + c_lo;
  const float alpha = p.alpha, beta = p.beta;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    CT* cp = Ct + (int64_t)(8 * (j & 1)) * p.ldc + 8 * (j >> 1);
    if (sizeof(CT) == 4) {
      float2 v;
      v.x = alpha * acc[2 * j];
      v.y = alpha * acc[2 * j + 1];
      if (beta != 0.f) {
        const float2 o = *reinterpret_cast<float2*>(cp);
        v.x = fmaf(beta, o.x, v.x);
        v.y = fmaf(beta, o.y, v.y);
      }
      *reinterpret_cast<float2*>(cp) = v;
    } else {
      const double da = (double)alpha, db = (double)beta;
      double2 v;
      v.x = da * (double)acc[2 * j];
      v.y = da * (double)acc[2 * j + 1];
      if (beta != 0.f) {
        const double2 o = *reinterpret_cast<double2*>(cp);
        v.x = fma(db, o.x, v.x);
        v.y = fma(db, o.y, v.y);
      }
      *reinterpret_cast<double2*>(cp) = v;
    }
  }
}

// ---- host ------------------------------------------------------------------------------------------------------------
static bool make_map(CUtensorMap* m, const float* base, int64_t K, int64_t rows, int64_t ld, int64_t bs, int32_t batch,
                     int box_rows) {
  const EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return false;
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 4, (cuuint64_t)((batch > 1) ? bs : rows * ld) * 4};
  cuuint32_t box[3] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <typename CT>
static int launch_tc(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t lda, int64_t a_bs,
                     const float* B, int64_t ldb, int64_t b_bs, float beta, CT* C, int64_t ldc, int64_t c_bs, int32_t lower,
                     int32_t batch, cudaStream_t stream) {
  CUtensorMap mA, mB;
  if (!make_map(&mA, A, K, M, lda, a_bs, batch, TC_BM) || !make_map(&mB, B, K, N, ldb, b_bs, batch, TC_BN)) return 0;
  if (const int rc = opt_in_smem<gemm_nt_f32_tc_kernel<CT>>(TC_SMEM_BYTES)) return rc;
  TcParams p{alpha, beta, C, ldc, c_bs, (int32_t)K, lower, (int32_t)(M / TC_BM), (int32_t)(N / TC_BN)};
  dim3 grid((unsigned)(p.tiles_m * p.tiles_n), (unsigned)batch);
  gemm_nt_f32_tc_kernel<CT><<<grid, TC_GEMM_THREADS, TC_SMEM_BYTES, stream>>>(mA, mB, p);
  GPK_COUNT_LAUNCH();
  if (const int rc = cuda_rc(cudaGetLastError())) return rc;
  return 1;
}

int gemm_nt_f32_tc(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t lda, int64_t a_bs, const float* B,
                   int64_t ldb, int64_t b_bs, float beta, float* C, int64_t ldc, int64_t c_bs, int32_t lower,
                   int32_t batch, cudaStream_t stream) {
  if (K < 128 || K % TC_BK || M % TC_BM || N % TC_BN) return 0;
  if (lda % 4 || ldb % 4 || ldc % 4 || (batch > 1 && (a_bs % 4 || b_bs % 4))) return 0;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C)) % 16) return 0;
  return launch_tc<float>(M, N, K, alpha, A, lda, a_bs, B, ldb, b_bs, beta, C, ldc, c_bs, lower, batch, stream);
}

// ---- opt-in mixed precision for the fp64 Cholesky: trailing update C(fp64) -= P P^T with P rounded to fp32 and the
// product formed by the 3xTF32 tensor-core kernel above (north_star: "tf32/bf16 where the user opts in") ----------------
__global__ void f64_to_f32_panel_kernel(const double* __restrict__ src, int64_t lds, float* __restrict__ dst, int64_t rows,
                                        int64_t K) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * K) return;
  const int64_t r = idx / K, k = idx - r * K;
  dst[idx] = (float)src[r * lds + k];
}

// C[M x N] (lower tiles) -= P[0:M] P[0:N]^T, P = fp64 panel (M x K, ld = ldp) converted into ws (M x K floats).
int syrk_f64_tf32x3(int64_t M, int64_t N, int64_t K, const float* ws_rows, double* C, int64_t ldc, cudaStream_t stream) {
  if (K % TC_BK || M % TC_BM || N % TC_BN || K < 128) return GPK_ERR_ARG;
  const int rc = launch_tc<double>(M, N, K, -1.0f, ws_rows, K, 0, ws_rows, K, 0, 1.0f, C, ldc, 0, 1, 1, stream);
  return rc == 1 ? 0 : (rc < 0 ? rc : GPK_ERR_UNSUPPORTED);
}

int convert_panel_f32(const double* P, int64_t ldp, int64_t rows, int64_t K, float* ws, cudaStream_t stream) {
  const int64_t total = rows * K;
  if (total == 0) return 0;
  f64_to_f32_panel_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(P, ldp, ws, rows, K);
  GPK_COUNT_LAUNCH();
  return cuda_rc(cudaGetLastError());
}

}  // namespace gpk
