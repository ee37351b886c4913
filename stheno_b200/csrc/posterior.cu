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
#include "common.cuh"

namespace gpk {

template <typename T>
struct PostAbi;
template <>
struct PostAbi<double> {
  static int km(const gpk_kernel_desc* d, const double* x, int64_t xg, int64_t n, const double* y, int64_t yg, int64_t n2, int32_t dim,
                double* out, int64_t ldo, void* s) {
    return gpk_kernel_matrix_f64(d, x, xg, 0, n, y, yg, 0, n2, dim, 0.0, nullptr, 0, 0.0, GPK_KM_PAD_ZERO, out, ldo, 0, 1, s);
  }
  static int trsm(const double* L, int64_t ldl, int64_t n, double* B, int64_t ldb, int64_t rows, int32_t S, void* ws,
                  int64_t ws_bytes, void* s) {
    return gpk_trsm_right_f64(L, ldl, 0, n, B, ldb, 0, rows, 1, S, ws, ws_bytes, s);
  }
  static int red(const double* V, int64_t ldv, int64_t rows, int64_t nc, const double* b, double* dot, double* sq, void* s) {
    return gpk_row_dot_sq_f64(V, ldv, 0, rows, nc, b, 0, dot, sq, 0, 1, s);
  }
};
template <>
struct PostAbi<float> {
  static int km(const gpk_kernel_desc* d, const float* x, int64_t xg, int64_t n, const float* y, int64_t yg, int64_t n2, int32_t dim,
                float* out, int64_t ldo, void* s) {
    return gpk_kernel_matrix_f32(d, x, xg, 0, n, y, yg, 0, n2, dim, 0.0, nullptr, 0, 0.0, GPK_KM_PAD_ZERO, out, ldo, 0, 1, s);
  }
  static int trsm(const float* L, int64_t ldl, int64_t n, float* B, int64_t ldb, int64_t rows, int32_t, void*, int64_t,
                  void* s) {
    return gpk_trsm_right_f32(L, ldl, 0, n, B, ldb, 0, rows, 1, s);
  }
  static int red(const float* V, int64_t ldv, int64_t rows, int64_t nc, const float* b, float* dot, float* sq, void* s) {
    return gpk_row_dot_sq_f32(V, ldv, 0, rows, nc, b, 0, dot, sq, 0, 1, s);
  }
};

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
  int rc;
  for (int64_t a = 0; a < m; a += chunk) {
    const int64_t c = (m - a < chunk) ? m - a : chunk;
    const int64_t c_pad = (c + 127) / 128 * 128;
    if ((rc = PostAbi<T>::km(desc, xsg + a * d, xsg_gstride, c, xg, xg_gstride, n, d, ws, n_pad, stream))) return rc;
    if ((rc = PostAbi<T>::trsm(L, ldl, n_pad, ws, n_pad, c_pad, slices, oz_ws, oz_ws_bytes, stream))) return rc;
    if ((rc = PostAbi<T>::red(ws, n_pad, c, n_pad, half_y, dot ? dot + a : nullptr, sq ? sq + a : nullptr, stream))) return rc;
  }
  return 0;
}

}  // namespace gpk

extern "C" {
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
