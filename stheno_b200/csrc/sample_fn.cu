// Random-feature evaluation for pathwise posterior samples (pathwise.py):
//
//   out[i][s] (+)= sum_j W[s][j] a_j cos(x_i . omega_j + b_j)
//
// x [n x d], omega [F x d] (already divided by each term's length scales), b, a [F], W [num x F].  The n x F feature matrix
// Phi is never written to global memory: each CTA owns a tile of rows and walks the features in blocks, forming that block's
// cosines in shared memory (or registers) and contracting them with the matching block of W on the spot.
//
//   * num >= 8, fp64: 64 rows x 32 columns per CTA, Phi tile in shared memory, contraction on the fp64 tensor cores (DMMA).
//   * otherwise (num < 8, or fp32): one row per thread, the cosines in registers, FMAs on the CUDA cores; 8 columns per CTA
//     in fp64 (num < 8 fits one), 32 in fp32.
// A CTA forms the cosines of its row tile once for the columns it owns: ceil(num / 32) n F cosines in all (n F in fp64 with
// num < 8), since every further tile of 32 samples recomputes them rather than holding more accumulators.
//
// Phases are formed in fp64 in both precisions (the fp32 products of x and omega are exact in fp64) and the cosine is a
// library one: at |x . omega| ~ 1e4, as short length scales give, an fp32 phase would already be off by ~1e-3.  The fp64
// variant takes cos of the phase; the fp32 variant reduces it to turns in [-1/2, 1/2] and takes cospi; its sums run in fp32.
#include <math.h>

#include "common.cuh"

namespace gpk {

namespace {

constexpr int kDC = 16;  // input dimensions staged in shared memory at a time

template <typename T>
__device__ __forceinline__ T feature_cos(double p);
template <>
__device__ __forceinline__ double feature_cos<double>(double p) {
  return cos(p);
}
template <>
__device__ __forceinline__ float feature_cos<float>(double p) {
  // p in turns, reduced in fp64 to [-1/2, 1/2] (off by ~|p| 2^-53 / 2 pi, far below fp32's resolution), then the fp64 cospi
  // rounded once: cosf / cospif keep a slow-path call that makes ptxas spill in this kernel
  const double t = p * 0.15915494309189535;
  return (float)cospi(2.0 * (t - rint(t)));
}

// ---- fp64, num >= 8: Phi tile in shared memory, DMMA contraction -------------------------------------------------------
constexpr int kTM = 64, kTN = 32, kFK = 32, kLD = kFK + 4;  // kLD: 8-byte words, conflict-free fragment reads

__global__ void __launch_bounds__(128) feature_eval_dmma_kernel(const double* __restrict__ x, int64_t ldx, int64_t n, int d,
                                                                const double* __restrict__ omega,
                                                                const double* __restrict__ b,
                                                                const double* __restrict__ amp, int64_t F,
                                                                const double* __restrict__ W, int64_t ldw, int num,
                                                                double* __restrict__ out, int64_t ldo, int accumulate) {
  __shared__ double phi[kTM][kLD];
  __shared__ double ws[kTN][kLD];
  __shared__ double xs[kTM][kDC + 1];
  __shared__ double om[kFK][kDC + 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * kTM;
  const int col0 = blockIdx.y * kTN;
  const int fk = tid & (kFK - 1);  // the feature of the block this thread forms cosines for
  double acc[2][4][2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

  for (int64_t f0 = 0; f0 < F; f0 += kFK) {
    // W a for this block (zero beyond num and F)
    for (int e = tid; e < kTN * kFK; e += 128) {
      const int c = e / kFK, k = e % kFK;
      const int64_t f = f0 + k;
      ws[c][k] = (col0 + c < num && f < F) ? W[(int64_t)(col0 + c) * ldw + f] * amp[f] : 0.0;
    }
    // phases p[q] of rows tid / 32 + 4 q for feature fk
    double p[kTM / 4];
#pragma unroll
    for (int q = 0; q < kTM / 4; ++q) p[q] = 0.0;
    for (int e0 = 0; e0 < d; e0 += kDC) {
      __syncthreads();
      for (int e = tid; e < kTM * kDC; e += 128) {
        const int r = e / kDC, c = e % kDC;
        xs[r][c] = (row0 + r < n && e0 + c < d) ? x[(row0 + r) * ldx + e0 + c] : 0.0;
      }
      for (int e = tid; e < kFK * kDC; e += 128) {
        const int k = e / kDC, c = e % kDC;
        om[k][c] = (f0 + k < F && e0 + c < d) ? omega[(f0 + k) * d + e0 + c] : 0.0;
      }
      __syncthreads();
      const int dc = d - e0 < kDC ? d - e0 : kDC;
      for (int c = 0; c < dc; ++c) {
        const double w = om[fk][c];
#pragma unroll
        for (int q = 0; q < kTM / 4; ++q) p[q] = fma(xs[(tid >> 5) + 4 * q][c], w, p[q]);
      }
    }
    const double bk = f0 + fk < F ? b[f0 + fk] : 0.0;
#pragma unroll
    for (int q = 0; q < kTM / 4; ++q) phi[(tid >> 5) + 4 * q][fk] = feature_cos<double>(p[q] + bk);
    __syncthreads();
    // warp w: rows 16 w .. 16 w + 15 (two 8-row blocks) x the 32 columns (four 8-column blocks)
#pragma unroll
    for (int kk = 0; kk < kFK; kk += 4) {
      const double a0 = phi[16 * warp + (lane >> 2)][kk + (lane & 3)];
      const double a1 = phi[16 * warp + 8 + (lane >> 2)][kk + (lane & 3)];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double bb = ws[8 * j + (lane >> 2)][kk + (lane & 3)];
        dmma884(acc[0][j][0], acc[0][j][1], a0, bb);
        dmma884(acc[1][j][0], acc[1][j][1], a1, bb);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int64_t r = row0 + 16 * warp + 8 * i + (lane >> 2);
    if (r >= n) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = col0 + 8 * j + 2 * (lane & 3) + h;
        if (c < num) {
          double* o = out + r * ldo + c;
          *o = accumulate ? *o + acc[i][j][h] : acc[i][j][h];
        }
      }
  }
}

// ---- CUDA-core FMAs: one row per thread, kNC columns per CTA (8 in fp64, 32 in fp32) ------------------------------------
constexpr int kRows = 128, kFB = 16;

template <typename T, int kNC>
__global__ void __launch_bounds__(kRows) feature_eval_fma_kernel(const T* __restrict__ x, int64_t ldx, int64_t n, int d,
                                                                 const T* __restrict__ omega, const T* __restrict__ b,
                                                                 const T* __restrict__ amp, int64_t F,
                                                                 const T* __restrict__ W, int64_t ldw, int num,
                                                                 T* __restrict__ out, int64_t ldo, int accumulate) {
  __shared__ double xs[kRows][kDC + 1];
  __shared__ double om[kFB][kDC + 1];
  __shared__ T ws[kNC][kFB];
  const int tid = threadIdx.x;
  const int64_t row0 = (int64_t)blockIdx.x * kRows, r = row0 + tid;
  const int col0 = blockIdx.y * kNC;
  const int nc = num - col0 < kNC ? num - col0 : kNC;
  T acc[kNC];
#pragma unroll
  for (int c = 0; c < kNC; ++c) acc[c] = T(0);

  for (int64_t f0 = 0; f0 < F; f0 += kFB) {
    double p[kFB];
#pragma unroll
    for (int k = 0; k < kFB; ++k) p[k] = 0.0;
    for (int e0 = 0; e0 < d; e0 += kDC) {
      __syncthreads();
      for (int e = tid; e < kRows * kDC; e += kRows) {
        const int rr = e / kDC, c = e % kDC;
        xs[rr][c] = (row0 + rr < n && e0 + c < d) ? (double)x[(row0 + rr) * ldx + e0 + c] : 0.0;
      }
      for (int e = tid; e < kFB * kDC; e += kRows) {
        const int k = e / kDC, c = e % kDC;
        om[k][c] = (f0 + k < F && e0 + c < d) ? (double)omega[(f0 + k) * d + e0 + c] : 0.0;
      }
      if (e0 == 0)
        for (int e = tid; e < kNC * kFB; e += kRows) {
          const int c = e / kFB, k = e % kFB;
          const int64_t f = f0 + k;
          ws[c][k] = (c < nc && f < F) ? W[(int64_t)(col0 + c) * ldw + f] * amp[f] : T(0);
        }
      __syncthreads();
      const int dc = d - e0 < kDC ? d - e0 : kDC;
      for (int c = 0; c < dc; ++c) {
        const double xv = xs[tid][c];
#pragma unroll
        for (int k = 0; k < kFB; ++k) p[k] = fma(xv, om[k][c], p[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < kFB; ++k) {
      const T v = feature_cos<T>(p[k] + (f0 + k < F ? (double)b[f0 + k] : 0.0));
#pragma unroll
      for (int c = 0; c < kNC; ++c) acc[c] = fma(ws[c][k], v, acc[c]);
    }
  }
  if (r >= n) return;
#pragma unroll
  for (int c = 0; c < kNC; ++c)
    if (c < nc) {
      T* o = out + r * ldo + col0 + c;
      *o = accumulate ? *o + acc[c] : acc[c];
    }
}

template <typename T>
int feature_eval(const T* x, int64_t ldx, int64_t n, int32_t d, const T* omega, const T* b, const T* amp, int64_t F,
                 const T* W, int64_t ldw, int32_t num, T* out, int64_t ldo, int32_t accumulate, void* stream) {
  if (!x || !omega || !b || !amp || !W || !out || n < 0 || d < 1 || F < 1 || num < 1) return GPK_ERR_ARG;
  if (ldx < d || ldw < F || ldo < num) return GPK_ERR_ARG;
  if (n == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  bool launched = false;
  if constexpr (sizeof(T) == 8) {
    if (num >= 8) {
      const int64_t ny = (num + kTN - 1) / kTN;
      if ((n + kTM - 1) / kTM > 0x7fffffff || ny > 65535) return GPK_ERR_UNSUPPORTED;
      dim3 grid((unsigned)((n + kTM - 1) / kTM), (unsigned)ny);
      feature_eval_dmma_kernel<<<grid, 128, 0, s>>>(x, ldx, n, d, omega, b, amp, F, W, ldw, num, out, ldo, accumulate);
      launched = true;
    }
  }
  if (!launched) {
    constexpr int kNC = sizeof(T) == 8 ? 8 : 32;
    const int64_t ny = (num + kNC - 1) / kNC;
    if ((n + kRows - 1) / kRows > 0x7fffffff || ny > 65535) return GPK_ERR_UNSUPPORTED;
    dim3 grid((unsigned)((n + kRows - 1) / kRows), (unsigned)ny);
    feature_eval_fma_kernel<T, kNC><<<grid, kRows, 0, s>>>(x, ldx, n, d, omega, b, amp, F, W, ldw, num, out, ldo, accumulate);
  }
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

}  // namespace

}  // namespace gpk

int gpk_feature_eval_f64(const double* x, int64_t ldx, int64_t n, int32_t d, const double* omega, const double* b,
                         const double* amp, int64_t F, const double* W, int64_t ldw, int32_t num, double* out, int64_t ldo,
                         int32_t accumulate, void* stream) {
  return gpk::feature_eval(x, ldx, n, d, omega, b, amp, F, W, ldw, num, out, ldo, accumulate, stream);
}
int gpk_feature_eval_f32(const float* x, int64_t ldx, int64_t n, int32_t d, const float* omega, const float* b,
                         const float* amp, int64_t F, const float* W, int64_t ldw, int32_t num, float* out, int64_t ldo,
                         int32_t accumulate, void* stream) {
  return gpk::feature_eval(x, ldx, n, d, omega, b, amp, F, W, ldw, num, out, ldo, accumulate, stream);
}
