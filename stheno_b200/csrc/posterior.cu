// K3: posterior mean and marginal variance at a block of test points in ONE call (north_star "fused TRSM + GEMM for the
// posterior mean / var"; reference: PosteriorMean / PosteriorKernel behind stheno/model/observations.py:143-168, evaluated by
// mlkernels.mean_var_diag through stheno/model/fdd.py:72-74).
//
//   V^T = k(x*, x) L^-T          (K1 rows, built directly in the transposed form the right-side TRSM wants)
//   dot_i = <v_i, L^-1 (y - m(x))>   ->  posterior mean   = m(x*_i) + dot_i
//   sq_i  = |v_i|^2                  ->  marginal variance = k(x*_i, x*_i) - sq_i
//
// The test points are walked in chunks of `chunk` rows through a caller-provided workspace of chunk_pad x n_pad elements, so
// the cross-covariance K(x*, x) (m x n) is never held whole: device memory O(chunk n) whatever m is.  All of the n^2 m flops run
// in the tensor-core TRSM (DMMA, or the int8 emulation when the caller passes its slices and scratch).
//
// The sparse posterior (PseudoObs*: PosteriorKernel(z, K_z) + SubspaceKernel(z, A), observations.py:255-277) walks its test
// points the same way, with each K1 row solved twice -- against L_z (mean and the PosteriorKernel term) and against the factor
// L_S of the stored A + eps I (the SubspaceKernel term) -- and one reduction pass over both: O(chunk m_pad) device memory.
#include "common.cuh"

namespace gpk {

template <typename T>
static int posterior_marginals(const gpk_kernel_desc* desc, const T* xsg, int64_t xsg_gstride, int64_t m, const T* xg,
                               int64_t xg_gstride, int64_t n, int32_t d, const T* L, int64_t ldl, int64_t n_pad,
                               const T* half_y, T* dot, T* sq, int64_t chunk, T* ws, int64_t ws_elems, int32_t slices,
                               void* oz_ws, int64_t oz_ws_bytes, void* stream) {
  if (!desc || !xsg || !xg || !L || !ws || m < 0 || n < 1 || d < 1) return GPK_ERR_ARG;
  if (n_pad % 128 || n_pad < n || ldl < n_pad || chunk < 128 || chunk % 128) return GPK_ERR_ARG;
  if (ws_elems < chunk * n_pad || reinterpret_cast<uintptr_t>(ws) % 16) return GPK_ERR_ARG;
  if (!dot && !sq) return GPK_ERR_ARG;
  if (dot && !half_y) return GPK_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  for (int64_t a = 0; a < m; a += chunk) {
    const int64_t c = (m - a < chunk) ? m - a : chunk;
    const int64_t c_pad = (c + 127) / 128 * 128;
    if ((rc = kernel_rows(desc, xsg + a * d, xsg_gstride, c, xg, xg_gstride, n, d, ws, n_pad, s))) return rc;
    if ((rc = trsm_right(L, ldl, n_pad, ws, n_pad, c_pad, slices, oz_ws, oz_ws_bytes, s))) return rc;
    if ((rc = row_dot_sq(ws, n_pad, c, n_pad, half_y, dot ? dot + a : nullptr, sq ? sq + a : nullptr, s))) return rc;
  }
  return 0;
}

// Sparse (inducing-point) posterior marginals, per test point of a chunk (one warp per row, fp64 sums in both precisions):
//   dot[i] = <v_i, h>, sq_z[i] = |v_i|^2, sq_s[i] = |u_i|^2   (V, U: [c x m_pad], same ld; h zero padded; dot may be NULL)
template <typename T>
__global__ void sparse_post_rows_kernel(int64_t c, int64_t m_pad, const T* __restrict__ V, const T* __restrict__ U, int64_t ld,
                                        const T* __restrict__ h, T* __restrict__ dot, T* __restrict__ sq_z,
                                        T* __restrict__ sq_s) {
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= c) return;
  const int lane = threadIdx.x & 31;
  const T* v = V + i * ld;
  const T* u = U + i * ld;
  double sd = 0.0, sz = 0.0, ss = 0.0;
  for (int64_t j = lane; j < m_pad; j += 32) {
    const double vj = (double)v[j], uj = (double)u[j];
    sz = fma(vj, vj, sz);
    ss = fma(uj, uj, ss);
    if (dot) sd = fma(vj, (double)h[j], sd);
  }
  sd = warp_sum(sd);
  sz = warp_sum(sz);
  ss = warp_sum(ss);
  if (lane == 0) {
    if (dot) dot[i] = (T)sd;
    sq_z[i] = (T)sz;
    sq_s[i] = (T)ss;
  }
}

// Per chunk of test points: K1 rows k(x*_c, z) -> V, a device copy of them -> U (a copy rather than a second K1 launch: it
// costs 2 c m_pad elements of HBM traffic whatever the kernel expression, and both solves start from the same bits), right
// TRSM of V against L_z and of U against L_S, then the three row reductions.
template <typename T>
static int sparse_posterior_marginals(const gpk_kernel_desc* desc, const T* xsg, int64_t xsg_gstride, int64_t ns, const T* zg,
                                      int64_t zg_gstride, int64_t m, int32_t d, const T* Lz, int64_t ldlz, const T* LS,
                                      int64_t ldls, int64_t m_pad, const T* half_y, T* dot, T* sq_z, T* sq_s, int64_t chunk,
                                      T* ws, int64_t ws_elems, int32_t slices, void* oz_ws, int64_t oz_ws_bytes,
                                      void* stream) {
  if (!desc || !xsg || !zg || !Lz || !LS || !sq_z || !sq_s || !ws || ns < 0 || m < 1 || d < 1) return GPK_ERR_ARG;
  if (m_pad % 128 || m_pad < m || ldlz < m_pad || ldls < m_pad || chunk < 128 || chunk % 128) return GPK_ERR_ARG;
  if (ws_elems < gpk_sparse_posterior_ws_elems(chunk, m_pad)) return GPK_ERR_ARG;
  if (reinterpret_cast<uintptr_t>(ws) % 16) return GPK_ERR_ALIGN;
  if (dot && !half_y) return GPK_ERR_ARG;
  T* V = ws;
  T* U = ws + chunk * m_pad;
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  for (int64_t a = 0; a < ns; a += chunk) {
    const int64_t c = (ns - a < chunk) ? ns - a : chunk;
    const int64_t c_pad = (c + 127) / 128 * 128;
    if ((rc = kernel_rows(desc, xsg + a * d, xsg_gstride, c, zg, zg_gstride, m, d, V, m_pad, s))) return rc;
    if ((rc = cuda_rc(cudaMemcpyAsync(U, V, (size_t)(c_pad * m_pad) * sizeof(T), cudaMemcpyDeviceToDevice, s)))) return rc;
    if ((rc = trsm_right(Lz, ldlz, m_pad, V, m_pad, c_pad, slices, oz_ws, oz_ws_bytes, s))) return rc;
    if ((rc = trsm_right(LS, ldls, m_pad, U, m_pad, c_pad, slices, oz_ws, oz_ws_bytes, s))) return rc;
    sparse_post_rows_kernel<T><<<(unsigned)(c_pad / 8), 256, 0, s>>>(c, m_pad, V, U, m_pad, half_y, dot ? dot + a : nullptr,
                                                                    sq_z + a, sq_s + a);
    GPK_COUNT_LAUNCH();
    GPK_CHECK_LAUNCH();
  }
  return 0;
}

// Backward of the sparse marginals in the test inputs, per test point of a chunk (one warp per row): with the upstream
// gradients a_i of dot_i and b_i of the variance (k - sq_z) + sq_s, the rows of dL/dk(x*_i, z) are
// L_z^-T (a_i h - 2 b_i v_i) + L_S^-T (2 b_i u_i); this writes the two right-hand sides over V and U and zeroes the ragged rows.
template <typename T>
__global__ void sparse_post_rows_bwd_kernel(int64_t c, int64_t c_pad, int64_t m_pad, T* __restrict__ V, T* __restrict__ U,
                                            int64_t ld, const T* __restrict__ h, const T* __restrict__ a,
                                            const T* __restrict__ b) {
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= c_pad) return;
  const int lane = threadIdx.x & 31;
  T* v = V + i * ld;
  T* u = U + i * ld;
  if (i >= c) {
    for (int64_t j = lane; j < m_pad; j += 32) v[j] = u[j] = T(0);
    return;
  }
  // V and U are read only when b is given: without it the caller need not have formed them
  const double ai = a ? (double)a[i] : 0.0;
  const double b2 = b ? 2.0 * (double)b[i] : 0.0;
  for (int64_t j = lane; j < m_pad; j += 32) {
    double vj = a ? ai * (double)h[j] : 0.0;
    double uj = 0.0;
    if (b) {
      vj = fma(-b2, (double)v[j], vj);
      uj = b2 * (double)u[j];
    }
    v[j] = (T)vj;
    u[j] = (T)uj;
  }
}

template <typename T>
static int sparse_posterior_rows_bwd(int64_t c, int64_t m_pad, T* V, T* U, int64_t ld, const T* h, const T* a, const T* b,
                                     void* stream) {
  if (!V || !U || c < 1 || m_pad < 128 || m_pad % 128 || ld < m_pad) return GPK_ERR_ARG;
  if ((!a && !b) || (a && !h)) return GPK_ERR_ARG;
  const int64_t c_pad = (c + 127) / 128 * 128;
  sparse_post_rows_bwd_kernel<T><<<(unsigned)(c_pad / 8), 256, 0, (cudaStream_t)stream>>>(c, c_pad, m_pad, V, U, ld, h, a, b);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

}  // namespace gpk

extern "C" {
int gpk_sparse_posterior_rows_bwd_f64(int64_t c, int64_t m_pad, double* V, double* U, int64_t ld, const double* h,
                                      const double* a, const double* b, void* stream) {
  return gpk::sparse_posterior_rows_bwd<double>(c, m_pad, V, U, ld, h, a, b, stream);
}
int gpk_sparse_posterior_rows_bwd_f32(int64_t c, int64_t m_pad, float* V, float* U, int64_t ld, const float* h, const float* a,
                                      const float* b, void* stream) {
  return gpk::sparse_posterior_rows_bwd<float>(c, m_pad, V, U, ld, h, a, b, stream);
}
int64_t gpk_sparse_posterior_ws_elems(int64_t chunk, int64_t m_pad) { return 2 * ((chunk + 127) / 128 * 128) * m_pad; }
int gpk_sparse_posterior_marginals_f64(const gpk_kernel_desc* desc_host, const double* xsg, int64_t xsg_gstride, int64_t ns,
                                       const double* zg, int64_t zg_gstride, int64_t m, int32_t d, const double* Lz,
                                       int64_t ldlz, const double* LS, int64_t ldls, int64_t m_pad, const double* half_y,
                                       double* dot, double* sq_z, double* sq_s, int64_t chunk, double* ws, int64_t ws_elems,
                                       int32_t slices, void* oz_ws, int64_t oz_ws_bytes, void* stream) {
  return gpk::sparse_posterior_marginals<double>(desc_host, xsg, xsg_gstride, ns, zg, zg_gstride, m, d, Lz, ldlz, LS, ldls,
                                                 m_pad, half_y, dot, sq_z, sq_s, chunk, ws, ws_elems, slices, oz_ws,
                                                 oz_ws_bytes, stream);
}
int gpk_sparse_posterior_marginals_f32(const gpk_kernel_desc* desc_host, const float* xsg, int64_t xsg_gstride, int64_t ns,
                                       const float* zg, int64_t zg_gstride, int64_t m, int32_t d, const float* Lz, int64_t ldlz,
                                       const float* LS, int64_t ldls, int64_t m_pad, const float* half_y, float* dot,
                                       float* sq_z, float* sq_s, int64_t chunk, float* ws, int64_t ws_elems, void* stream) {
  return gpk::sparse_posterior_marginals<float>(desc_host, xsg, xsg_gstride, ns, zg, zg_gstride, m, d, Lz, ldlz, LS, ldls,
                                                m_pad, half_y, dot, sq_z, sq_s, chunk, ws, ws_elems, 0, nullptr, 0, stream);
}
int gpk_posterior_marginals_f64(const gpk_kernel_desc* desc_host, const double* xsg, int64_t xsg_gstride, int64_t m,
                                const double* xg, int64_t xg_gstride, int64_t n, int32_t d, const double* L, int64_t ldl,
                                int64_t n_pad, const double* half_y, double* dot, double* sq, int64_t chunk, double* ws,
                                int64_t ws_elems, int32_t slices, void* oz_ws, int64_t oz_ws_bytes, void* stream) {
  return gpk::posterior_marginals<double>(desc_host, xsg, xsg_gstride, m, xg, xg_gstride, n, d, L, ldl, n_pad, half_y, dot, sq,
                                          chunk, ws, ws_elems, slices, oz_ws, oz_ws_bytes, stream);
}
int gpk_posterior_marginals_f32(const gpk_kernel_desc* desc_host, const float* xsg, int64_t xsg_gstride, int64_t m,
                                const float* xg, int64_t xg_gstride, int64_t n, int32_t d, const float* L, int64_t ldl,
                                int64_t n_pad, const float* half_y, float* dot, float* sq, int64_t chunk, float* ws,
                                int64_t ws_elems, void* stream) {
  return gpk::posterior_marginals<float>(desc_host, xsg, xsg_gstride, m, xg, xg_gstride, n, d, L, ldl, n_pad, half_y, dot, sq,
                                         chunk, ws, ws_elems, 0, nullptr, 0, stream);
}
}
