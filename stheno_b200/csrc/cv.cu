// Multi-fold cross-validation finish: the fold-wise predictive moments and log densities from the per-fold quantities of
// C = Sigma^-1 (stheno_b200/ops.py, Chol.cv), and the weights of their backward (stheno_b200/autograd.py, _KernelCV).
// Entries are in fold order: fold f holds the entries [offsets[f], offsets[f + 1]).
#include <math.h>

#include "common.cuh"

namespace gpk {

// One CTA per (column cc, problem b).  Every thread walks its strided entries in order, the warps reduce by shuffles,
// thread 0 adds the warp sums in order and then the folds' log-determinants in fold order: the log density is the same
// bit for bit from run to run.  fp64 in both precisions.
template <typename T>
__global__ void cv_finish_kernel(const int64_t* __restrict__ off, int32_t n_folds, const T* __restrict__ e, int64_t lde,
                                 int64_t e_bs, const T* __restrict__ z, int64_t ldz, int64_t z_bs, const T* __restrict__ v,
                                 int64_t v_bs, const T* __restrict__ ldet, int64_t ldet_bs, const T* __restrict__ r,
                                 int64_t ldr, int64_t r_bs, int64_t n, int32_t k, T* __restrict__ mu, T* __restrict__ var,
                                 T* __restrict__ lp) {
  const int cc = blockIdx.x, b = blockIdx.y;
  const T* eb = e ? e + (int64_t)b * e_bs + (int64_t)cc * lde : nullptr;
  const T* rb = r ? r + (int64_t)b * r_bs + (int64_t)cc * ldr : nullptr;
  const T* zb = z ? z + (int64_t)b * z_bs + (int64_t)cc * ldz : nullptr;
  const T* vb = v + (int64_t)b * v_bs;
  T* mub = mu ? mu + ((int64_t)b * k + cc) * n : nullptr;
  T* varb = (var && cc == 0) ? var + (int64_t)b * n : nullptr;
  double t = 0.0;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
    if (mub) mub[j] = (T)((double)rb[j] - (double)eb[j]);
    if (varb) varb[j] = vb[j];
    if (zb) {
      const double zj = (double)zb[j];
      t += zj * zj;
    }
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
    double s = 0.0;
    for (int f = 0; f < n_folds; ++f)
      s += (double)ldet[(int64_t)b * ldet_bs + f] - (double)(off[f + 1] - off[f]) * log2pi;
    lp[(int64_t)b * k + cc] = (T)(0.5 * (s - u));
  }
}

// Backward weights, one thread per entry i, the columns in order:  q_ci = g_c e_ci; and per fold the weight of C_II^-1 in
// P_I = s_f C_II^-1 + 1/2 sum_c q_cI e_cI^T, s_f = 1/2 sum_c g_c.  fp64 in both precisions.
template <typename T>
__global__ void cv_weights_kernel(int32_t n_folds, const T* __restrict__ e, int64_t lde, int64_t e_bs, int64_t n,
                                  int32_t k, const T* __restrict__ g, T* __restrict__ q, T* __restrict__ s) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  const T* gb = g + (int64_t)b * k;
  if (q && i < n) {
    for (int cc = 0; cc < k; ++cc)
      q[((int64_t)b * k + cc) * n + i] = (T)((double)gb[cc] * (double)e[(int64_t)b * e_bs + (int64_t)cc * lde + i]);
  }
  if (s && i < n_folds) {
    double w = 0.0;
    for (int cc = 0; cc < k; ++cc) w += (double)gb[cc];
    s[(int64_t)b * n_folds + i] = (T)(0.5 * w);
  }
}

template <typename T>
static int cv_finish(const int64_t* offsets, int32_t n_folds, const T* e, int64_t lde, int64_t e_bs, const T* z,
                     int64_t ldz, int64_t z_bs, const T* v, int64_t v_bs, const T* ldet, int64_t ldet_bs, const T* r,
                     int64_t ldr, int64_t r_bs, int64_t n, int32_t k, const T* g, T* mu, T* var, T* lp, T* q, T* s,
                     int32_t batch, void* stream) {
  if (n < 1 || k < 1 || batch < 1 || n_folds < 1 || n_folds > n) return GPK_ERR_ARG;
  const cudaStream_t st = (cudaStream_t)stream;
  if (g) {
    if (!q && !s) return 0;
    if (q && (!e || lde < n)) return GPK_ERR_ARG;
    dim3 grid((unsigned)((n + 255) / 256), (unsigned)batch);
    cv_weights_kernel<T><<<grid, 256, 0, st>>>(n_folds, e, lde, e_bs, n, k, g, q, s);
  } else {
    if (!mu && !var && !lp) return 0;
    if ((mu && (!e || !r || lde < n || ldr < n)) || (var && !v) || (lp && (!z || !ldet || !offsets || ldz < n)))
      return GPK_ERR_ARG;
    cv_finish_kernel<T><<<dim3((unsigned)k, (unsigned)batch), 512, 0, st>>>(
        offsets, n_folds, e, lde, e_bs, lp ? z : nullptr, ldz, z_bs, v, v_bs, ldet, ldet_bs, r, ldr, r_bs, n, k, mu, var,
        lp);
  }
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

}  // namespace gpk

extern "C" {

int gpk_cv_finish_f64(const int64_t* offsets, int32_t n_folds, const double* e, int64_t lde, int64_t e_bstride,
                      const double* z, int64_t ldz, int64_t z_bstride, const double* v, int64_t v_bstride,
                      const double* ldet, int64_t ldet_bstride, const double* r, int64_t ldr, int64_t r_bstride, int64_t n,
                      int32_t k, const double* g, double* mu, double* var, double* lp, double* q, double* s, int32_t batch,
                      void* stream) {
  return gpk::cv_finish<double>(offsets, n_folds, e, lde, e_bstride, z, ldz, z_bstride, v, v_bstride, ldet, ldet_bstride,
                                r, ldr, r_bstride, n, k, g, mu, var, lp, q, s, batch, stream);
}
int gpk_cv_finish_f32(const int64_t* offsets, int32_t n_folds, const float* e, int64_t lde, int64_t e_bstride,
                      const float* z, int64_t ldz, int64_t z_bstride, const float* v, int64_t v_bstride, const float* ldet,
                      int64_t ldet_bstride, const float* r, int64_t ldr, int64_t r_bstride, int64_t n, int32_t k,
                      const float* g, float* mu, float* var, float* lp, float* q, float* s, int32_t batch, void* stream) {
  return gpk::cv_finish<float>(offsets, n_folds, e, lde, e_bstride, z, ldz, z_bstride, v, v_bstride, ldet, ldet_bstride, r,
                               ldr, r_bstride, n, k, g, mu, var, lp, q, s, batch, stream);
}
}
