// Leave-one-out finish: the element-wise LOO predictive moments and log densities from c = diag Sigma^-1 and
// alpha = Sigma^-1 r, and the weights of their backward (stheno_b200/autograd.py, _KernelLoo).
#include <math.h>

#include "common.cuh"

namespace gpk {

// One CTA per (column cc, problem b).  Every thread walks its strided entries in order, the warps reduce by shuffles and
// thread 0 adds the warp sums in order: the log density is the same bit for bit from run to run.  fp64 in both precisions.
template <typename T>
__global__ void loo_finish_kernel(const T* __restrict__ c, int64_t c_bs, const T* __restrict__ alpha, int64_t lda,
                                  int64_t a_bs, const T* __restrict__ r, int64_t ldr, int64_t r_bs, int64_t n, int32_t k,
                                  T* __restrict__ mu, T* __restrict__ var, T* __restrict__ lp) {
  const int cc = blockIdx.x, b = blockIdx.y;
  const T* cb = c + (int64_t)b * c_bs;
  const T* ab = alpha + (int64_t)b * a_bs + (int64_t)cc * lda;
  const T* rb = r ? r + (int64_t)b * r_bs + (int64_t)cc * ldr : nullptr;
  T* mub = mu ? mu + ((int64_t)b * k + cc) * n : nullptr;
  T* varb = (var && cc == 0) ? var + (int64_t)b * n : nullptr;
  double t = 0.0;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
    const double cj = (double)cb[j], a = (double)ab[j];
    const double s = a / cj;
    if (mub) mub[j] = (T)((double)rb[j] - s);
    if (varb) varb[j] = (T)(1.0 / cj);
    t += log(cj) - a * s;
  }
  if (!lp) return;
  __shared__ double red[32];
  t = warp_sum(t);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double u = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) u += red[w];
    const double log2pi = 1.8378770664093454835606594728112;
    lp[(int64_t)b * k + cc] = (T)(0.5 * (u - (double)n * log2pi));
  }
}

// Backward weights, one thread per entry i, the columns in order:  P_i = sum_c g_c (1 + alpha_ci^2 / c_i) / (2 c_i),
// q_ci = g_c alpha_ci / c_i.  fp64 in both precisions.
template <typename T>
__global__ void loo_weights_kernel(const T* __restrict__ c, int64_t c_bs, const T* __restrict__ alpha, int64_t lda,
                                   int64_t a_bs, int64_t n, int32_t k, const T* __restrict__ g, T* __restrict__ P,
                                   T* __restrict__ q) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= n) return;
  const double ci = (double)c[(int64_t)b * c_bs + i];
  double p = 0.0;
  for (int cc = 0; cc < k; ++cc) {
    const double a = (double)alpha[(int64_t)b * a_bs + (int64_t)cc * lda + i];
    const double s = a / ci, gc = (double)g[(int64_t)b * k + cc];
    p += gc * (1.0 + a * s);
    if (q) q[((int64_t)b * k + cc) * n + i] = (T)(gc * s);
  }
  if (P) P[(int64_t)b * n + i] = (T)(p / (2.0 * ci));
}

template <typename T>
static int loo_finish(const T* c, int64_t c_bs, const T* alpha, int64_t lda, int64_t a_bs, const T* r, int64_t ldr,
                      int64_t r_bs, int64_t n, int32_t k, const T* g, T* mu, T* var, T* lp, T* P, T* q, int32_t batch,
                      void* stream) {
  if (!c || !alpha || n < 1 || k < 1 || batch < 1 || lda < n || (mu && (!r || ldr < n))) return GPK_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  if (g) {
    if (!P && !q) return 0;
    dim3 grid((unsigned)((n + 255) / 256), (unsigned)batch);
    loo_weights_kernel<T><<<grid, 256, 0, s>>>(c, c_bs, alpha, lda, a_bs, n, k, g, P, q);
  } else {
    if (!mu && !var && !lp) return 0;
    loo_finish_kernel<T><<<dim3((unsigned)k, (unsigned)batch), 512, 0, s>>>(c, c_bs, alpha, lda, a_bs, r, ldr, r_bs, n, k,
                                                                             mu, var, lp);
  }
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

}  // namespace gpk

extern "C" {

int gpk_loo_finish_f64(const double* c, int64_t c_bstride, const double* alpha, int64_t lda, int64_t a_bstride,
                       const double* r, int64_t ldr, int64_t r_bstride, int64_t n, int32_t k, const double* g, double* mu,
                       double* var, double* lp, double* P, double* q, int32_t batch, void* stream) {
  return gpk::loo_finish<double>(c, c_bstride, alpha, lda, a_bstride, r, ldr, r_bstride, n, k, g, mu, var, lp, P, q, batch,
                                 stream);
}
int gpk_loo_finish_f32(const float* c, int64_t c_bstride, const float* alpha, int64_t lda, int64_t a_bstride, const float* r,
                       int64_t ldr, int64_t r_bstride, int64_t n, int32_t k, const float* g, float* mu, float* var,
                       float* lp, float* P, float* q, int32_t batch, void* stream) {
  return gpk::loo_finish<float>(c, c_bstride, alpha, lda, a_bstride, r, ldr, r_bstride, n, k, g, mu, var, lp, P, q, batch,
                                stream);
}
}
