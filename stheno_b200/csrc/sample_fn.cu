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

// ---- backward in x ------------------------------------------------------------------------------------------------------
//
//   grad_x[i][e] (+)= -sum_j c_ij sin(x_i . omega_j + b_j) omega_j[e],   c_ij = amp_j sum_s G[i][s] W[s][j]
//
// The forward's structure: a CTA owns kTM = 64 rows and walks the features in blocks of kFK = 32.  Per block it forms the
// phases (fp64, the forward's staging), writes -sin into a 64 x 32 tile `cs`, forms the coefficients c of the same tile by
// reducing over ALL samples in blocks of kSB, scales `cs` by them and contracts `cs` with the block's omega into the CTA's
// grad tile, which stays in registers over the whole feature loop.  A CTA covers up to kTD = 32 input dimensions of the
// gradient; wider inputs are split over gridDim.y, each split recomputing the phases, sines and c of its rows.
//   * kTC (fp64, num >= 8): both contractions on DMMA 8x8x4, the fragment pattern of feature_eval_dmma_kernel (warp = 16
//     rows x 32 columns; the grad contraction skips the 8-column blocks beyond the split's dimensions);
//   * otherwise: FMAs on the CUDA cores, sums in T.
// No atomics and no n x F buffer; a row of x or G holding a NaN reaches only its own row of grad_x.
constexpr int kSB = 16, kTD = 32, kSLD = kSB + 4;

template <typename T>
__device__ __forceinline__ T feature_sin(double p);
template <>
__device__ __forceinline__ double feature_sin<double>(double p) {
  return sin(p);
}
template <>
__device__ __forceinline__ float feature_sin<float>(double p) {
  // as feature_cos<float>: reduced to turns in fp64, the fp64 sinpi rounded once
  const double t = p * 0.15915494309189535;
  return (float)sinpi(2.0 * (t - rint(t)));
}

template <typename T, bool kTC>
__global__ void __launch_bounds__(128) feature_eval_bwd_kernel(const T* __restrict__ x, int64_t ldx, int64_t n, int d,
                                                               const T* __restrict__ omega, const T* __restrict__ b,
                                                               const T* __restrict__ amp, int64_t F,
                                                               const T* __restrict__ W, int64_t ldw, int num,
                                                               const T* __restrict__ G, int64_t ldg,
                                                               T* __restrict__ grad, int64_t ld, int accumulate) {
  // the phase staging (xs, om) and the sample staging (gs, ws) are never live together: one buffer holds either
  constexpr int kStage = (kTM + kFK) * (kDC + 1) * 8 > (kTM + kFK) * kSLD * (int)sizeof(T)
                             ? (kTM + kFK) * (kDC + 1) * 8 : (kTM + kFK) * kSLD * (int)sizeof(T);
  __shared__ __align__(16) unsigned char stage[kStage];
  __shared__ T cs[kTM][kLD];   // -sin, then c * -sin: rows x features of the block
  __shared__ T ot[kTD * kLD];  // omega of the block for this CTA's dimensions: [e][k] (kTC) or [k][e]
  double(*xs)[kDC + 1] = reinterpret_cast<double(*)[kDC + 1]>(stage);
  double(*om)[kDC + 1] = xs + kTM;
  T(*gs)[kSLD] = reinterpret_cast<T(*)[kSLD]>(stage);
  T* ws = reinterpret_cast<T*>(gs + kTM);  // W a of the block: [k][s] (kTC) or [s][k]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * kTM;
  const int d0 = blockIdx.y * kTD;
  const int dd = d - d0 < kTD ? d - d0 : kTD;  // dimensions of the gradient this CTA writes
  const int fk = lane;                          // the feature of the block this thread forms sines (and c, FMA) for
  double acc[2][4][2];  // kTC: the grad tile in DMMA fragments
  T g[16];              // FMA: outputs o = tid + 128 q of the 64 x dd tile
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
#pragma unroll
  for (int q = 0; q < 16; ++q) g[q] = T(0);

  for (int64_t f0 = 0; f0 < F; f0 += kFK) {
    // phases of rows warp + 4 q for feature fk, as the forward forms them
    {
      double p[kTM / 4];
#pragma unroll
      for (int q = 0; q < kTM / 4; ++q) p[q] = 0.0;
      for (int e0 = 0; e0 < d; e0 += kDC) {
        __syncthreads();
        for (int e = tid; e < kTM * kDC; e += 128) {
          const int r = e / kDC, c = e % kDC;
          xs[r][c] = (row0 + r < n && e0 + c < d) ? (double)x[(row0 + r) * ldx + e0 + c] : 0.0;
        }
        for (int e = tid; e < kFK * kDC; e += 128) {
          const int k = e / kDC, c = e % kDC;
          om[k][c] = (f0 + k < F && e0 + c < d) ? (double)omega[(f0 + k) * d + e0 + c] : 0.0;
        }
        __syncthreads();
        const int dc = d - e0 < kDC ? d - e0 : kDC;
        for (int c = 0; c < dc; ++c) {
          const double w = om[fk][c];
#pragma unroll
          for (int q = 0; q < kTM / 4; ++q) p[q] = fma(xs[warp + 4 * q][c], w, p[q]);
        }
      }
      const double bk = f0 + fk < F ? (double)b[f0 + fk] : 0.0;
#pragma unroll
      for (int q = 0; q < kTM / 4; ++q) cs[warp + 4 * q][fk] = -feature_sin<T>(p[q] + bk);
    }
    // c = G_tile (W a)_block^T, over every sample
    double c1[2][4][2];
    T cf[kTM / 4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) c1[i][j][0] = c1[i][j][1] = 0.0;
#pragma unroll
    for (int q = 0; q < kTM / 4; ++q) cf[q] = T(0);
    for (int s0 = 0; s0 < num; s0 += kSB) {
      __syncthreads();
      for (int e = tid; e < kTM * kSB; e += 128) {
        const int r = e / kSB, s = e % kSB;
        gs[r][s] = (row0 + r < n && s0 + s < num) ? G[(row0 + r) * ldg + s0 + s] : T(0);
      }
      for (int e = tid; e < kFK * kSB; e += 128) {
        const int s = e / kFK, k = e % kFK;
        const int64_t f = f0 + k;
        const T v = (s0 + s < num && f < F) ? W[(int64_t)(s0 + s) * ldw + f] * amp[f] : T(0);
        ws[kTC ? k * kSLD + s : s * kLD + k] = v;
      }
      __syncthreads();
      if constexpr (kTC) {
#pragma unroll
        for (int kk = 0; kk < kSB; kk += 4) {
          const double a0 = gs[16 * warp + (lane >> 2)][kk + (lane & 3)];
          const double a1 = gs[16 * warp + 8 + (lane >> 2)][kk + (lane & 3)];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const double bb = ws[(8 * j + (lane >> 2)) * kSLD + kk + (lane & 3)];
            dmma884(c1[0][j][0], c1[0][j][1], a0, bb);
            dmma884(c1[1][j][0], c1[1][j][1], a1, bb);
          }
        }
      } else {
        const int sc = num - s0 < kSB ? num - s0 : kSB;
        for (int s = 0; s < sc; ++s) {
          const T w = ws[s * kLD + fk];
#pragma unroll
          for (int q = 0; q < kTM / 4; ++q) cf[q] = fma(gs[warp + 4 * q][s], w, cf[q]);
        }
      }
    }
    // scale the sines by c (each thread its own elements; the sample loop's barriers ordered the sine writes before)
    if constexpr (kTC) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) cs[16 * warp + 8 * i + (lane >> 2)][8 * j + 2 * (lane & 3) + h] *= c1[i][j][h];
    } else {
#pragma unroll
      for (int q = 0; q < kTM / 4; ++q) cs[warp + 4 * q][fk] *= cf[q];
    }
    for (int e = tid; e < kTD * kFK; e += 128) {
      const int k = e / kTD, c = e % kTD;
      const T v = (f0 + k < F && c < dd) ? omega[(f0 + k) * d + d0 + c] : T(0);
      ot[kTC ? c * kLD + k : k * kLD + c] = v;
    }
    __syncthreads();
    // grad += cs omega_block (the barrier at the top of the next block's phase loop orders these reads before the writes)
    if constexpr (kTC) {
      const int nj = (dd + 7) / 8;
#pragma unroll
      for (int kk = 0; kk < kFK; kk += 4) {
        const double a0 = cs[16 * warp + (lane >> 2)][kk + (lane & 3)];
        const double a1 = cs[16 * warp + 8 + (lane >> 2)][kk + (lane & 3)];
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < nj) {
            const double bb = ot[(8 * j + (lane >> 2)) * kLD + kk + (lane & 3)];
            dmma884(acc[0][j][0], acc[0][j][1], a0, bb);
            dmma884(acc[1][j][0], acc[1][j][1], a1, bb);
          }
      }
    } else {
      const int no = kTM * dd;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const int o = tid + 128 * q;
        if (o < no) {
          const int r = o / dd, c = o - r * dd;
          T s = g[q];
#pragma unroll 8
          for (int k = 0; k < kFK; ++k) s = fma(cs[r][k], ot[k * kLD + c], s);
          g[q] = s;
        }
      }
    }
  }
  if constexpr (kTC) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t r = row0 + 16 * warp + 8 * i + (lane >> 2);
      if (r >= n) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int c = 8 * j + 2 * (lane & 3) + h;
          if (c < dd) {
            T* o = grad + r * ld + d0 + c;
            *o = accumulate ? *o + acc[i][j][h] : acc[i][j][h];
          }
        }
    }
  } else {
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int o = tid + 128 * q;
      if (o < kTM * dd) {
        const int64_t r = row0 + o / dd;
        const int c = o % dd;
        if (r < n) {
          T* p = grad + r * ld + d0 + c;
          *p = accumulate ? *p + g[q] : g[q];
        }
      }
    }
  }
}

template <typename T>
int feature_eval_bwd(const T* x, int64_t ldx, int64_t n, int32_t d, const T* omega, const T* b, const T* amp, int64_t F,
                     const T* W, int64_t ldw, int32_t num, const T* G, int64_t ldg, T* grad, int64_t ld,
                     int32_t accumulate, void* stream) {
  if (!x || !omega || !b || !amp || !W || !G || !grad || n < 0 || d < 1 || F < 1 || num < 1) return GPK_ERR_ARG;
  if (ldx < d || ldw < F || ldg < num || ld < d) return GPK_ERR_ARG;
  if (n == 0) return 0;
  const int64_t nx = (n + kTM - 1) / kTM, ny = (d + kTD - 1) / kTD;
  if (nx > 0x7fffffff || ny > 65535) return GPK_ERR_UNSUPPORTED;
  dim3 grid((unsigned)nx, (unsigned)ny);
  cudaStream_t s = (cudaStream_t)stream;
  bool launched = false;
  if constexpr (sizeof(T) == 8) {
    if (num >= 8) {
      feature_eval_bwd_kernel<T, true><<<grid, 128, 0, s>>>(x, ldx, n, d, omega, b, amp, F, W, ldw, num, G, ldg, grad, ld,
                                                            accumulate);
      launched = true;
    }
  }
  if (!launched)
    feature_eval_bwd_kernel<T, false><<<grid, 128, 0, s>>>(x, ldx, n, d, omega, b, amp, F, W, ldw, num, G, ldg, grad, ld,
                                                           accumulate);
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
int gpk_feature_eval_bwd_f64(const double* x, int64_t ldx, int64_t n, int32_t d, const double* omega, const double* b,
                             const double* amp, int64_t F, const double* W, int64_t ldw, int32_t num, const double* G,
                             int64_t ldg, double* grad_x, int64_t ld, int32_t accumulate, void* stream) {
  return gpk::feature_eval_bwd(x, ldx, n, d, omega, b, amp, F, W, ldw, num, G, ldg, grad_x, ld, accumulate, stream);
}
int gpk_feature_eval_bwd_f32(const float* x, int64_t ldx, int64_t n, int32_t d, const float* omega, const float* b,
                             const float* amp, int64_t F, const float* W, int64_t ldw, int32_t num, const float* G,
                             int64_t ldg, float* grad_x, int64_t ld, int32_t accumulate, void* stream) {
  return gpk::feature_eval_bwd(x, ldx, n, d, omega, b, amp, F, W, ldw, num, G, ldg, grad_x, ld, accumulate, stream);
}
