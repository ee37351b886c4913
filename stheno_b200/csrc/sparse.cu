// Streamed sparse (inducing-point) accumulation: one chunk of data points per call, K_zx is never held.
//
//   reference: AbstractPseudoObservations._compute, stheno/model/observations.py:279-336
//       :285  K_zx = k(z, x)              :301  W = L_z^-1 K_zx            :304-306 corr = diag K_x - colsum(W o W)
//       :308-313 trace part / FITC noise  :322  A = I + W K_n^-1 W^T       :327  prod = W K_n^-1 ybar
//       :334-336 the scalars of the ELBO
//   Round 1 materialised K_xz (8.6 GB at n = 262144, m = 4096), its transpose (8.6 GB) and one more copy.  Here the caller
//   walks the data in chunks of c points; per chunk (all stream-ordered, caller-provided workspace, no allocation):
//       K1 rows k(x_c, z) -> [c_pad, m_pad]  ->  right TRSM against L_z (rows are independent: the same tensor-core solve the
//       posterior uses)  ->  per-row |w_i|^2 (Q_ii)  ->  per-row scalars (corr, trace, FITC noise, 1/sqrt(K_n), ELBO sums)  ->
//       scaled transpose [m_pad, c_pad]  ->  A += W_s W_s^T (tensor-core SYRK on the lower tiles, K = c)  ->  prod += W_s ybar_s
//   so the m^2 n flops of the solve and of A both stay on the tensor cores and device memory is O(c m + m^2).
#include "common.cuh"

namespace gpk {

// per data point of the chunk: corr, method-specific noise, the scale 1/sqrt(K_n'), ybar scaled, and the three ELBO sums of
// each block of 256 points -> partial[k][blockIdx.x] (reduced by sparse_scalars_kernel: no atomics, so no run-to-run order)
template <typename T>
__global__ void sparse_rows_kernel(int64_t c, int64_t c_pad, const T* __restrict__ kdiag, const T* __restrict__ q,
                                   const T* __restrict__ kn, const T* __restrict__ ybar, int32_t method,
                                   T* __restrict__ rs, T* __restrict__ ybs, double* __restrict__ partial) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double s_log = 0.0, s_yy = 0.0, s_tr = 0.0;
  if (i < c_pad) {
    if (i < c) {
      double k = (double)kn[i];
      if (method != 2) {
        const double corr = (double)kdiag[i] - (double)q[i];  // :306
        if (method == 0) s_tr = corr / k;                     // :308-310  B.ratio(Diagonal(corr), K_n)
        else k += corr;                                       // :311-313
      }
      const double r = rsqrt(k);
      const double yb = (double)ybar[i];
      rs[i] = (T)r;
      ybs[i] = (T)(yb * r);
      s_log = log(6.283185307179586476925286766559 * k);      // :334
      s_yy = yb * yb / k;                                     // :335
    } else {
      rs[i] = T(0);
      ybs[i] = T(0);
    }
  }
  __shared__ double red[3][8];
  s_log = warp_sum(s_log);
  s_yy = warp_sum(s_yy);
  s_tr = warp_sum(s_tr);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) {
    red[0][w] = s_log;
    red[1][w] = s_yy;
    red[2][w] = s_tr;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[threadIdx.x][k];
    partial[threadIdx.x * (int64_t)gridDim.x + blockIdx.x] = s;
  }
}

// scalars[k] += sum_b partial[k][b] over the nb blocks of sparse_rows_kernel, one block of 256 threads summing in a fixed
// order: the same chunk adds the same bits on every run
template <typename T>
__global__ void sparse_scalars_kernel(const double* __restrict__ partial, int64_t nb, T* __restrict__ scalars) {
  __shared__ double red[8];
  for (int k = 0; k < 3; ++k) {
    double s = 0.0;
    for (int64_t b = threadIdx.x; b < nb; b += blockDim.x) s += partial[k * nb + b];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += red[w];
      scalars[k] += (T)t;
    }
    __syncthreads();
  }
}

// dst[j][i] = src[i][j] * rs[i]   (src: rows x cols, dst: cols x rows), 32 x 32 tiles through shared memory
template <typename T>
__global__ void transpose_scaled_kernel(const T* __restrict__ src, int64_t lds, int64_t rows, int64_t cols,
                                        const T* __restrict__ rs, T* __restrict__ dst, int64_t ldd) {
  __shared__ T tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t r0 = (int64_t)blockIdx.x * 32, c0 = (int64_t)blockIdx.y * 32;  // the long dimension (rows) on grid.x
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = r0 + i, cc = c0 + tx;
    tile[i][tx] = (r < rows && cc < cols) ? src[r * lds + cc] * rs[r] : T(0);
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = c0 + i, cc = r0 + tx;
    if (r < cols && cc < rows) dst[r * ldd + cc] = tile[tx][i];
  }
}

// acc[r] += <V[r, :n_cols], b>   (one warp per row)
template <typename T>
__global__ void row_dot_acc_kernel(const T* __restrict__ V, int64_t ldv, int64_t rows, int64_t n_cols,
                                   const T* __restrict__ b, T* __restrict__ acc) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const T* row = V + r * ldv;
  double s = 0.0;
  for (int64_t j = lane; j < n_cols; j += 32) s = fma((double)row[j], (double)b[j], s);
  s = warp_sum(s);
  if (lane == 0) acc[r] += (T)s;
}

// Backward of the streamed ELBO, per data point of a chunk (one warp per row; no atomics).  With s = A^-1 prod and the solved
// rows w_i (Wc) and u_i = A^-1 w_i (U):  beta_i = s.w_i, gamma_i = w_i.u_i, r_i = ybar_i - beta_i, kappa_i = K_n' (:311-313),
//   g_kappa = (r^2 + gamma - kappa) / (2 kappa^2),  dE/dybar_i = -r / kappa,
//   dE/dkn_i, dE/dkdiag_i, g_q by method (VFE: g_kappa + (kd - q) / (2 kn^2), -1 / (2 kn), 1 / (2 kn);  FITC: g_kappa, g_kappa,
//   -g_kappa;  DTC: g_kappa, -, 0),  and row i of U becomes g_i^T = ((-u_i + s r_i) / kappa + 2 g_q w_i)^T = dE/dw_i^T.
// Rows c .. c_pad - 1 of U are zeroed.  Padding columns of Wc, U and s are zero, so they stay zero.
template <typename T>
__global__ void sparse_rows_bwd_kernel(int64_t c, int64_t c_pad, int64_t m_pad, const T* __restrict__ Wc, int64_t ldw,
                                       T* __restrict__ U, int64_t ldu, const T* __restrict__ s, const T* __restrict__ q,
                                       const T* __restrict__ kdiag, const T* __restrict__ kn, const T* __restrict__ ybar,
                                       int32_t method, T* __restrict__ g_kn, T* __restrict__ g_kd, T* __restrict__ g_ybar) {
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= c_pad) return;
  const int lane = threadIdx.x & 31;
  T* u = U + i * ldu;
  if (i >= c) {
    for (int64_t j = lane; j < m_pad; j += 32) u[j] = T(0);
    return;
  }
  const T* w = Wc + i * ldw;
  double beta = 0.0, gamma = 0.0;
  for (int64_t j = lane; j < m_pad; j += 32) {
    const double wj = (double)w[j];
    beta = fma((double)s[j], wj, beta);
    gamma = fma(wj, (double)u[j], gamma);
  }
  beta = warp_sum(beta);
  gamma = warp_sum(gamma);
  const double sig = (double)kn[i], yb = (double)ybar[i];
  double kap = sig, qi = 0.0, kd = 0.0;
  if (method != 2) {
    qi = (double)q[i];
    kd = (double)kdiag[i];
    if (method == 1) kap += kd - qi;
  }
  const double r = yb - beta;
  const double g_kap = (r * r + gamma - kap) / (2.0 * kap * kap);
  double g_sig = g_kap, g_q = 0.0;
  if (method == 0) {
    g_sig += (kd - qi) / (2.0 * sig * sig);
    g_q = 0.5 / sig;
  } else if (method == 1) {
    g_q = -g_kap;
  }
  if (lane == 0) {
    g_kn[i] = (T)g_sig;
    g_ybar[i] = (T)(-r / kap);
    if (method == 0) g_kd[i] = (T)(-0.5 / sig);
    else if (method == 1) g_kd[i] = (T)g_kap;
  }
  const double inv = 1.0 / kap, two_gq = 2.0 * g_q;
  for (int64_t j = lane; j < m_pad; j += 32) {
    const double wj = (double)w[j];
    u[j] = (T)(fma((double)s[j], r, -(double)u[j]) * inv + two_gq * wj);
  }
}

static inline int64_t pad128(int64_t v) { return (v + 127) / 128 * 128; }

template <typename T>
static int sparse_accumulate(const gpk_kernel_desc* desc, const T* xg, int64_t xg_gstride, int64_t c, const T* zg,
                             int64_t zg_gstride, int64_t m, int32_t d, const T* Lz, int64_t ldl, int64_t m_pad,
                             const T* kdiag, const T* kn, const T* ybar, int32_t method, T* A, int64_t lda, T* prod,
                             T* scalars, T* ws, int64_t ws_elems, int32_t slices, void* oz_ws, int64_t oz_ws_bytes,
                             void* stream) {
  if (!desc || !xg || !zg || !Lz || !kn || !ybar || !A || !prod || !scalars || !ws) return GPK_ERR_ARG;
  if (c < 1 || m < 1 || d < 1 || m_pad % 128 || m_pad < m || ldl < m_pad || lda < m_pad) return GPK_ERR_ARG;
  if (method < 0 || method > 2 || (method != 2 && !kdiag)) return GPK_ERR_ARG;
  const int64_t c_pad = pad128(c);
  if (ws_elems < gpk_sparse_ws_elems(c, m_pad)) return GPK_ERR_ARG;
  if (reinterpret_cast<uintptr_t>(ws) % 16) return GPK_ERR_ALIGN;
  T* Wc = ws;                      // [c_pad][m_pad]
  T* WcT = Wc + c_pad * m_pad;     // [m_pad][c_pad]
  T* q = WcT + m_pad * c_pad;      // [c_pad]
  T* rs = q + c_pad;
  T* ybs = rs + c_pad;
  const int64_t nb = (c_pad + 255) / 256;  // blocks of sparse_rows_kernel
  double* partial = reinterpret_cast<double*>(ybs + c_pad);  // [3][nb]; 8-byte aligned: c_pad is a multiple of 128
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = kernel_rows(desc, xg, xg_gstride, c, zg, zg_gstride, m, d, Wc, m_pad, s))) return rc;           // :285
  if ((rc = trsm_right(Lz, ldl, m_pad, Wc, m_pad, c_pad, slices, oz_ws, oz_ws_bytes, s))) return rc;       // :301
  if (method != 2 && (rc = row_dot_sq(Wc, m_pad, c, m_pad, nullptr, nullptr, q, s))) return rc;           // :305
  sparse_rows_kernel<T><<<(unsigned)nb, 256, 0, s>>>(c, c_pad, kdiag, q, kn, ybar, method, rs, ybs, partial);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  sparse_scalars_kernel<T><<<1, 256, 0, s>>>(partial, nb, scalars);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  dim3 grid((unsigned)(c_pad / 32), (unsigned)(m_pad / 32)), block(32, 8);
  transpose_scaled_kernel<T><<<grid, block, 0, s>>>(Wc, m_pad, c_pad, m_pad, rs, WcT, c_pad);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  if ((rc = gemm_nt(m_pad, m_pad, c_pad, T(1), WcT, c_pad, 0, WcT, c_pad, 0, T(1), A, lda, 0, 1, 1, slices, oz_ws,
                    oz_ws_bytes, s)))  // :322
    return rc;
  row_dot_acc_kernel<T><<<(unsigned)((m_pad + 7) / 8), 256, 0, s>>>(WcT, c_pad, m_pad, c_pad, ybs, prod);       // :327
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

template <typename T>
static int sparse_rows_bwd(int64_t c, int64_t m_pad, const T* Wc, int64_t ldw, T* U, int64_t ldu, const T* s, const T* q,
                           const T* kdiag, const T* kn, const T* ybar, int32_t method, T* g_kn, T* g_kd, T* g_ybar,
                           void* stream) {
  if (!Wc || !U || !s || !kn || !ybar || !g_kn || !g_ybar) return GPK_ERR_ARG;
  if (c < 1 || m_pad < 128 || m_pad % 128 || ldw < m_pad || ldu < m_pad) return GPK_ERR_ARG;
  if (method < 0 || method > 2 || (method != 2 && (!q || !kdiag || !g_kd))) return GPK_ERR_ARG;
  const int64_t c_pad = pad128(c);
  sparse_rows_bwd_kernel<T><<<(unsigned)(c_pad / 8), 256, 0, (cudaStream_t)stream>>>(c, c_pad, m_pad, Wc, ldw, U, ldu, s, q, kdiag,
                                                                                    kn, ybar, method, g_kn, g_kd, g_ybar);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

}  // namespace gpk

extern "C" {

int gpk_sparse_rows_bwd_f64(int64_t c, int64_t m_pad, const double* Wc, int64_t ldw, double* U, int64_t ldu, const double* s,
                            const double* q, const double* kdiag, const double* kn, const double* ybar, int32_t method,
                            double* g_kn, double* g_kd, double* g_ybar, void* stream) {
  return gpk::sparse_rows_bwd<double>(c, m_pad, Wc, ldw, U, ldu, s, q, kdiag, kn, ybar, method, g_kn, g_kd, g_ybar, stream);
}
int gpk_sparse_rows_bwd_f32(int64_t c, int64_t m_pad, const float* Wc, int64_t ldw, float* U, int64_t ldu, const float* s,
                            const float* q, const float* kdiag, const float* kn, const float* ybar, int32_t method,
                            float* g_kn, float* g_kd, float* g_ybar, void* stream) {
  return gpk::sparse_rows_bwd<float>(c, m_pad, Wc, ldw, U, ldu, s, q, kdiag, kn, ybar, method, g_kn, g_kd, g_ybar, stream);
}

int64_t gpk_sparse_ws_elems(int64_t c, int64_t m_pad) {
  const int64_t c_pad = gpk::pad128(c);
  // Wc, WcT, q, rs, ybs, then the per-block ELBO sums: 3 doubles per 256 points (6 elements of either type)
  return 2 * c_pad * m_pad + 3 * c_pad + 6 * ((c_pad + 255) / 256);
}

int gpk_sparse_accumulate_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride, int64_t c,
                              const double* zg, int64_t zg_gstride, int64_t m, int32_t d, const double* Lz, int64_t ldl,
                              int64_t m_pad, const double* kdiag, const double* kn, const double* ybar, int32_t method,
                              double* A, int64_t lda, double* prod, double* scalars, double* ws, int64_t ws_elems,
                              int32_t slices, void* oz_ws, int64_t oz_ws_bytes, void* stream) {
  return gpk::sparse_accumulate<double>(desc_host, xg, xg_gstride, c, zg, zg_gstride, m, d, Lz, ldl, m_pad, kdiag, kn, ybar,
                                        method, A, lda, prod, scalars, ws, ws_elems, slices, oz_ws, oz_ws_bytes, stream);
}
int gpk_sparse_accumulate_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t c,
                              const float* zg, int64_t zg_gstride, int64_t m, int32_t d, const float* Lz, int64_t ldl,
                              int64_t m_pad, const float* kdiag, const float* kn, const float* ybar, int32_t method, float* A,
                              int64_t lda, float* prod, float* scalars, float* ws, int64_t ws_elems, void* stream) {
  return gpk::sparse_accumulate<float>(desc_host, xg, xg_gstride, c, zg, zg_gstride, m, d, Lz, ldl, m_pad, kdiag, kn, ybar,
                                       method, A, lda, prod, scalars, ws, ws_elems, 0, nullptr, 0, stream);
}
}
