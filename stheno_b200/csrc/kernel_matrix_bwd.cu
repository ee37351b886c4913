// K1-backward: contraction of an upstream gradient G = d(loss)/dK (symmetric, n x n) with dK/d(theta) WITHOUT
// materialising any n x n gradient tensor per hyper-parameter (SURVEY.md section 7 step 8).
//
// For K_ij = sum_t c_t prod_{f in t} phi_f(x_i^(g_f), x_j^(g_f))   (same points on both sides, x^(g) = x / l_g) it returns
//   term_sum[t]   = sum_ij G_ij prod_f phi_f(i, j)                       -> d loss / d c_t
//   grad_xg[g][i] = 2 sum_j G_ij sum_{t, f: g_f = g} c_t (prod_{f' != f} phi_f') d phi_f(x_i, x_j) / d x_i
//                                                                        -> d loss / d x^(g)_i  (chain rule to l_g and x
//                                                                           is left to torch autograd on x / l_g)
//   diag[i]       = G_ii                                                 -> d loss / d noise_i ; its sum for a scalar noise
//   param_sum[f]  = sum_ij G_ij c_t (prod_{f' != f} phi_f') d phi_f / d fac_param[f]
//                                                                        -> d loss / d alpha of an RQ factor f (optional)
// One CTA owns 64 rows and sweeps all column tiles; every thread keeps private partial sums for its 4 rows in shared
// memory and the 16 threads sharing a row are reduced once at the end.
//
// Reference: torch autograd through exp / cholesky / triangular_solve in readme_example13_optimisation_torch.py:46-53.
#include <algorithm>

#include "common.cuh"

namespace gpk {

constexpr int KB_TILE = 64;
constexpr int KB_THREADS = 256;
constexpr int KB_MAXF = 4;  // factors per term supported by the backward pass

struct KbParams {
  gpk_kernel_desc desc;
  const void* xg;
  int64_t xg_gstride, x_bstride;
  int64_t n;
  int32_t d;
  const void* G;
  int64_t ldg, g_bstride;
  void* term_sum;  // [batch][GPK_MAX_TERMS]
  void* grad_xg;   // [groups][batch][n][d]  (same strides as xg)
  void* diag;      // [batch][n]
  void* param_sum; // [batch][GPK_MAX_FACTORS] or NULL
};

// h(w) = log1p(w) - w / (1 + w) >= 0: d/da (1 + w)^-a = -(1 + w)^-a h(w) at fixed d2 (w = d2 / (2 a)).  The direct form
// cancels for small w (h ~ w^2 / 2).  With s = w / (2 + w), -log1p(-t) = 2 atanh(s) for t = w / (1 + w) = 2 s / (1 + s), so
//   h = 2 atanh(s) - t = 2 s^2 / (1 + s) + 2 s^3 sum_{j>=0} s^2j / (2j + 3),
// a sum of positive terms.  Up to w = 3 (s = 0.6) 36 terms of the series leave a remainder below 2^-55 h; above it the
// direct form loses at most a factor 2 to the subtraction.  The rounding of s (of 2 + w and of the division, together up
// to 2^-52 relative) would cost h up to 6 ulp: it is carried as ds (s + ds = w / (2 + w) to first order, from the exact
// error of the sum and the exact residual of the division) and added as dh/ds ds = 4 s ds / ((1 - s)(1 + s)^2).
// Against mpmath: at most 2.9 ulp for w in [1e-300, 1e300] (tests/_rq_model.py restates this operation for operation).
constexpr double RQ_H_SPLIT = 3.0;
constexpr int RQ_H_TERMS = 36;

__device__ __forceinline__ double rq_h(double w) {
  if (!(w <= RQ_H_SPLIT)) return log1p(w) - w / (1.0 + w);  // NaN stays NaN
  const double u2 = 2.0 + w, s = w / u2;
  const double e2 = w >= 2.0 ? 2.0 - (u2 - w) : w - (u2 - 2.0);  // Fast2Sum: 2 + w = u2 + e2 exactly
  const double ds = fma(-s, e2, fma(-s, u2, w)) / u2;
  const double s2 = s * s;
  double p = 1.0 / (2 * (RQ_H_TERMS - 1) + 3);
#pragma unroll
  for (int j = RQ_H_TERMS - 2; j >= 0; --j) p = fma(p, s2, 1.0 / (2 * j + 3));
  const double c = s2 * s;
  const double corr = 4.0 * s * ds / ((1.0 - s) * (1.0 + s) * (1.0 + s));
  return fma(c + c, p, (s2 + s2) / (1.0 + s)) + corr;
}

// d phi / d a = -phi h(w); 0 where phi is 0 (w = inf, or phi underflowed), where h may not be finite
__device__ __forceinline__ double rq_dphi_dalpha(double w, double phi) { return phi == 0.0 ? 0.0 : -phi * rq_h(w); }

// value and derivative w.r.t. the squared distance (for LINEAR: value = dot, dval = 1 marks d/d(dot)); with PARAM, also
// *dpar = d value / d param (nonzero for GPK_RQ only: d / d alpha)
template <typename T, bool PARAM = false>
__device__ __forceinline__ void eval_factor_grad(int kind, T d2, T dot, bool same_pt, int d, T& val, T& dval, double param = 0.0,
                                                 T* dpar = nullptr) {
  if constexpr (PARAM) *dpar = T(0);
  switch (kind) {
    case GPK_RQ: {  // v = (1 + d2 / (2 a))^-a ;  dv / d(d2) = -v / (2 (1 + d2 / (2 a)))
      const double a = param, u = 1.0 + (double)d2 / (2.0 * a);
      const double v = exp(-a * log(u));
      val = (T)v;
      dval = (T)(-0.5 * v / u);
      if constexpr (PARAM) *dpar = (T)rq_dphi_dalpha((double)d2 / (2.0 * a), v);
      return;
    }
    case GPK_EQ: {
      val = t_exp<T>(T(-0.5) * d2);
      dval = T(-0.5) * val;
      return;
    }
    case GPK_MATERN12: {
      // not differentiable at r = 0: coincident points get the subgradient 0, the value autograd gives through the
      // reference's |x - y| (d = 1) and sqrt(max(d2, 1e-30)) (d > 1)
      const bool flat = (d == 1) ? !(d2 > T(0)) : !(d2 > T(1e-30));
      T r = (d == 1) ? t_sqrt<T>(d2) : t_sqrt<T>(d2 > T(1e-30) ? d2 : T(1e-30));
      val = t_exp<T>(-r);
      dval = (same_pt || flat) ? T(0) : -val / (T(2) * r);
      return;
    }
    case GPK_MATERN32: {
      T r = (d == 1) ? t_sqrt<T>(d2) : t_sqrt<T>(d2 > T(1e-30) ? d2 : T(1e-30));
      T s = T(1.7320508075688772) * r;
      T e = t_exp<T>(-s);
      val = (T(1) + s) * e;
      dval = T(-1.5) * e;
      return;
    }
    case GPK_MATERN52: {
      T r = (d == 1) ? t_sqrt<T>(d2) : t_sqrt<T>(d2 > T(1e-30) ? d2 : T(1e-30));
      T s = T(2.23606797749979) * r;
      T e = t_exp<T>(-s);
      val = (T(1) + s + T(1.6666666666666667) * d2) * e;
      dval = T(-0.8333333333333334) * (T(1) + s) * e;
      return;
    }
    case GPK_LINEAR:
      val = dot;
      dval = T(1);
      return;
    case GPK_DELTA:
      val = same_pt ? T(1) : T(0);
      dval = T(0);
      return;
    default:
      val = T(1);
      dval = T(0);
      return;
  }
}

// The kinds with a shape parameter (fac_param) whose gradient param_sum forms
__device__ __forceinline__ bool kind_has_param(int kind) { return kind == GPK_RQ; }

// psum[f] += c for the factor f = f0 + q of a term.  A dynamic index into psum would put it in local memory: the compare
// against every slot keeps it in registers.
template <typename T>
__device__ __forceinline__ void add_param(T (&psum)[GPK_MAX_FACTORS], int f, T c) {
#pragma unroll
  for (int ff = 0; ff < GPK_MAX_FACTORS; ++ff)
    if (ff == f) psum[ff] += c;
}

// One atomic per parameter factor: block reduction of every thread's psum into out[0 .. GPK_MAX_FACTORS).  Called by all
// threads of the block.
template <typename T>
__device__ __forceinline__ void flush_params(const gpk_kernel_desc& desc, const T (&psum)[GPK_MAX_FACTORS], T* out) {
  __shared__ T pred[KB_THREADS / 32][GPK_MAX_FACTORS];
  const int tid = threadIdx.x;
#pragma unroll
  for (int f = 0; f < GPK_MAX_FACTORS; ++f) {
    const T v = warp_sum(psum[f]);
    if ((tid & 31) == 0) pred[tid >> 5][f] = v;
  }
  __syncthreads();
  if (tid < desc.term_begin[desc.n_terms] && kind_has_param(desc.fac_kind[tid])) {
    T s = T(0);
    for (int w = 0; w < KB_THREADS / 32; ++w) s += pred[w][tid];
    atomicAdd(out + tid, s);
  }
}

// The partial sums of grad_xg take 256 * G * 4 * d words of shared memory.  For wide inputs the launch is split over
// chunks of dimensions (blockIdx.z = chunk): every chunk evaluates the full distances and kernel values but keeps partial
// sums only for its dimensions [k0, k0 + dc); chunk 0 alone writes term_sum, diag and (PARAM) param_sum.
// The PARAM instantiation's parameter sums need more than the 128 registers ptxas aims for by default; the shared memory
// allows one CTA per SM whichever it is, so it may take them.
template <typename T, bool PARAM>
__global__ void __launch_bounds__(KB_THREADS, PARAM ? 1 : 0) kernel_matrix_bwd_kernel(const KbParams p, const int dc) {
  const int tile_r = blockIdx.x, b = blockIdx.y;
  const int d = p.d, G = p.desc.n_groups, nt = p.desc.n_terms;
  const int k0 = blockIdx.z * dc, k1 = min(d, k0 + dc);
  const bool first = blockIdx.z == 0;
  const int64_t r0 = (int64_t)tile_r * KB_TILE;
  extern __shared__ __align__(16) unsigned char kb_smem[];
  T* xs = reinterpret_cast<T*>(kb_smem);            // [G][64][d]   rows of this CTA
  T* yt = xs + (size_t)G * KB_TILE * d;              // [G][d][65]   current column tile, transposed
  T* part = yt + (size_t)G * d * (KB_TILE + 1);      // [256 threads][G][4 rows][dc]: sum_j of d K_ij / d x_ik, k in the chunk
  const T* xg = static_cast<const T*>(p.xg) + (int64_t)b * p.x_bstride;
  const T* Gm = static_cast<const T*>(p.G) + (int64_t)b * p.g_bstride;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int pstride = G * 4 * dc;
  T* mypart = part + (size_t)tid * pstride;
  for (int i = 0; i < pstride; ++i) mypart[i] = T(0);

  const int xr = (int)max((int64_t)0, min((int64_t)KB_TILE, p.n - r0));
  for (int g = 0; g < G; ++g)
    for (int i = tid; i < KB_TILE * d; i += KB_THREADS)
      xs[(size_t)g * KB_TILE * d + i] = (i < xr * d) ? xg[g * p.xg_gstride + r0 * d + i] : T(0);

  T tsum[GPK_MAX_TERMS];
#pragma unroll
  for (int t = 0; t < GPK_MAX_TERMS; ++t) tsum[t] = T(0);
  T psum[PARAM ? GPK_MAX_FACTORS : 1];
#pragma unroll
  for (int f = 0; f < (PARAM ? GPK_MAX_FACTORS : 1); ++f) psum[f] = T(0);

  const int n_ctiles = (int)((p.n + KB_TILE - 1) / KB_TILE);
  for (int tc = 0; tc < n_ctiles; ++tc) {
    const int64_t c0 = (int64_t)tc * KB_TILE;
    const int yr = (int)min((int64_t)KB_TILE, p.n - c0);
    __syncthreads();
    for (int idx = tid; idx < G * KB_TILE * d; idx += KB_THREADS) {
      const int g = idx / (KB_TILE * d), rem = idx - g * KB_TILE * d;
      const int c = rem / d, k = rem - c * d;
      yt[((size_t)g * d + k) * (KB_TILE + 1) + c] = (c < yr) ? xg[g * p.xg_gstride + (c0 + c) * d + k] : T(0);
    }
    __syncthreads();

#pragma unroll 1
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + ty * 4 + i;
#pragma unroll 1
      for (int j = 0; j < 4; ++j) {
        const int64_t c = c0 + tx + 16 * j;
        if (r >= p.n || c >= p.n) continue;
        const T gij = Gm[r * p.ldg + c];
        const bool same_pt = (r == c);
        for (int t = 0; t < nt; ++t) {
          const int f0 = p.desc.term_begin[t], f1 = p.desc.term_begin[t + 1];
          T val[KB_MAXF], dval[KB_MAXF], dpar[KB_MAXF];
          T prod = T(1);
#pragma unroll
          for (int q = 0; q < KB_MAXF; ++q) {
            val[q] = T(1);
            dval[q] = T(0);
            dpar[q] = T(0);
            if (f0 + q < f1) {
              const int g = p.desc.fac_group[f0 + q];
              const T* xr_ = xs + ((size_t)g * KB_TILE + ty * 4 + i) * d;
              const T* yc_ = yt + (size_t)g * d * (KB_TILE + 1) + tx + 16 * j;
              T d2 = T(0), dot = T(0);
              for (int k = 0; k < d; ++k) {
                const T xv = xr_[k], yv = yc_[(size_t)k * (KB_TILE + 1)];
                const T df = xv - yv;
                d2 = fma(df, df, d2);
                dot = fma(xv, yv, dot);
              }
              eval_factor_grad<T, PARAM>(p.desc.fac_kind[f0 + q], d2, dot, same_pt, d, val[q], dval[q],
                                         p.desc.fac_param[f0 + q], &dpar[q]);
              prod *= val[q];
            }
          }
#pragma unroll
          for (int tt = 0; tt < GPK_MAX_TERMS; ++tt)
            if (tt == t) tsum[tt] = fma(gij, prod, tsum[tt]);
          const T ct = (T)p.desc.coef[t];
          if constexpr (PARAM) {
            if (first) {
#pragma unroll
              for (int q = 0; q < KB_MAXF; ++q) {
                if (dpar[q] == T(0)) continue;
                T others = T(1);
#pragma unroll
                for (int q2 = 0; q2 < KB_MAXF; ++q2)
                  if (q2 != q) others *= val[q2];
                add_param(psum, f0 + q, gij * ct * others * dpar[q]);
              }
            }
          }
#pragma unroll
          for (int q = 0; q < KB_MAXF; ++q) {
            if (f0 + q >= f1 || dval[q] == T(0)) continue;
            T others = T(1);
#pragma unroll
            for (int q2 = 0; q2 < KB_MAXF; ++q2)
              if (q2 != q) others *= val[q2];
            const T wgt = gij * ct * others * dval[q];
            const int g = p.desc.fac_group[f0 + q];
            const int kind = p.desc.fac_kind[f0 + q];
            T* pp = mypart + ((size_t)g * 4 + i) * dc;  // pp[k - k0] for the dimensions k of this chunk
            const T* yc_ = yt + (size_t)g * d * (KB_TILE + 1) + tx + 16 * j;
            if (kind == GPK_LINEAR) {
              // d(dot)/dx_ik = x_jk ; factor 2 for the symmetric counterpart
              for (int k = k0; k < k1; ++k) pp[k - k0] = fma(T(2) * wgt, yc_[(size_t)k * (KB_TILE + 1)], pp[k - k0]);
            } else {
              // d(d2)/dx_ik = 2 (x_ik - x_jk) ; factor 2 for the symmetric counterpart.  The difference is formed per
              // pair: Matern-1/2's weight grows like 1/r for near-coincident points, and splitting it into
              // 4 wgt x_ik - 4 wgt x_jk would cancel catastrophically.
              const T* xr_ = xs + ((size_t)g * KB_TILE + ty * 4 + i) * d;
              for (int k = k0; k < k1; ++k)
                pp[k - k0] = fma(T(4) * wgt, xr_[k] - yc_[(size_t)k * (KB_TILE + 1)], pp[k - k0]);
            }
          }
        }
        if (first && same_pt && p.diag) static_cast<T*>(p.diag)[(int64_t)b * p.n + r] = gij;
      }
    }
  }
  __syncthreads();
  // reduce the 16 column-threads of every row and write this chunk's columns of grad_xg
  T* gout = static_cast<T*>(p.grad_xg) + (int64_t)b * p.x_bstride;
  const int w = k1 - k0;
  for (int idx = tid; idx < G * KB_TILE * w; idx += KB_THREADS) {
    const int g = idx / (KB_TILE * w), rem = idx - g * KB_TILE * w;
    const int row = rem / w, kk = rem - row * w;
    if (r0 + row >= p.n) continue;
    const int rty = row >> 2, ri = row & 3;
    T s = T(0);
    for (int t16 = 0; t16 < 16; ++t16) s += part[(size_t)(rty * 16 + t16) * pstride + ((size_t)g * 4 + ri) * dc + kk];
    gout[g * p.xg_gstride + (r0 + row) * d + k0 + kk] = s;
  }
  if (!first) return;
  // term sums: block reduction + one atomic per term
  __shared__ T red[8][GPK_MAX_TERMS];
#pragma unroll
  for (int t = 0; t < GPK_MAX_TERMS; ++t) {
    T v = warp_sum(tsum[t]);
    if ((tid & 31) == 0) red[tid >> 5][t] = v;
  }
  __syncthreads();
  if (tid < nt) {
    T s = T(0);
    for (int w = 0; w < 8; ++w) s += red[w][tid];
    atomicAdd(static_cast<T*>(p.term_sum) + (int64_t)b * GPK_MAX_TERMS + tid, s);
  }
  if constexpr (PARAM) flush_params(p.desc, psum, static_cast<T*>(p.param_sum) + (int64_t)b * GPK_MAX_FACTORS);
}

template <typename T>
static int launch_kernel_matrix_bwd(const gpk_kernel_desc* desc, const T* xg, int64_t xg_gstride, int64_t x_bstride,
                                    int64_t n, int32_t d, const T* G, int64_t ldg, int64_t g_bstride, T* term_sum,
                                    T* grad_xg, T* diag, T* param_sum, int32_t batch, void* stream) {
  if (!desc || !xg || !G || !term_sum || !grad_xg || n < 0 || d < 1 || batch < 1) return GPK_ERR_ARG;
  if (desc->n_terms < 0 || desc->n_terms > GPK_MAX_TERMS || desc->n_groups < 1 || desc->n_groups > GPK_MAX_GROUPS)
    return GPK_ERR_ARG;
  for (int t = 0; t < desc->n_terms; ++t)
    if (desc->term_begin[t + 1] - desc->term_begin[t] > KB_MAXF) return GPK_ERR_UNSUPPORTED;
  if (n == 0) return 0;
  KbParams p;
  p.desc = *desc;
  p.xg = xg;
  p.xg_gstride = xg_gstride;
  p.x_bstride = x_bstride;
  p.n = n;
  p.d = d;
  p.G = G;
  p.ldg = ldg;
  p.g_bstride = g_bstride;
  p.term_sum = term_sum;
  p.grad_xg = grad_xg;
  p.diag = diag;
  p.param_sum = param_sum;
  const int Gn = desc->n_groups;
  // input rows + transposed column tile (all d dimensions), then as many dimensions of partial sums as fit
  constexpr size_t kMaxSmem = 200 * 1024;
  const size_t rows_bytes = ((size_t)Gn * KB_TILE * d + (size_t)Gn * d * (KB_TILE + 1)) * sizeof(T);
  const size_t dim_bytes = (size_t)KB_THREADS * Gn * 4 * sizeof(T);
  if (rows_bytes + dim_bytes > kMaxSmem) return GPK_ERR_UNSUPPORTED;
  const size_t fit = (kMaxSmem - rows_bytes) / dim_bytes;
  const int dc = fit < (size_t)d ? (int)fit : d;
  const int chunks = (d + dc - 1) / dc;
  const size_t smem = rows_bytes + (size_t)dc * dim_bytes;
  // the same chunks with or without param_sum: its sums sit in registers, and every other output is formed as without it
  const auto kernel = param_sum ? kernel_matrix_bwd_kernel<T, true> : kernel_matrix_bwd_kernel<T, false>;
  if (const int rc = param_sum ? opt_in_smem<kernel_matrix_bwd_kernel<T, true>>((int)smem)
                               : opt_in_smem<kernel_matrix_bwd_kernel<T, false>>((int)smem))
    return rc;
  dim3 grid((unsigned)((n + KB_TILE - 1) / KB_TILE), (unsigned)batch, (unsigned)chunks);
  kernel<<<grid, KB_THREADS, smem, (cudaStream_t)stream>>>(p, dc);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

// ---- rectangular K1-backward: K_ij = k(a_i, b_j) for two different point sets ---------------------------------------------
// One launch contracts G with dK/d(a) over rows a (CTA = 64 rows sweeping every column); the column gradient is a second
// launch with the roles of a and b swapped and G read transposed.  G is given factored, G_ij = wr_i wc_j W_ij + u_i v_j
// (W, wr, wc, u, v each optional), so the mean-only gradient needs no rows x cols buffer.  There is no symmetry factor,
// and Delta between different objects is [r^2 < 1e-10] with gradient 0, like K1's forward.
struct KcParams {
  gpk_kernel_desc desc;
  const void* ag;  // rows:    [G][batch][na][d]
  int64_t a_gstride, a_bstride, na;
  const void* bg;  // columns: [G][batch][nb][d]
  int64_t b_gstride, b_bstride, nb;
  int32_t d;
  const void* W;  // W(i, j) = W[b * w_bstride + i * w_si + j * w_sj]
  int64_t w_si, w_sj, w_bstride;
  const void *wr, *u;  // [batch][na]
  const void *wc, *v;  // [batch][nb]
  void* term_sum;      // [batch][GPK_MAX_TERMS] or NULL
  void* grad;          // rows' gradient, accumulated, layout of ag; or NULL
  void* param_sum;     // [batch][GPK_MAX_FACTORS]; read only by the PARAM instantiation
};

template <typename T, bool PARAM = false>
__device__ __forceinline__ void eval_cross_factor_grad(int kind, T d2, T dot, int d, T& val, T& dval, double param,
                                                       T* dpar = nullptr) {
  if (kind == GPK_DELTA) {
    val = d2 < T(1e-10) ? T(1) : T(0);
    dval = T(0);
    if constexpr (PARAM) *dpar = T(0);
  } else {
    eval_factor_grad<T, PARAM>(kind, d2, dot, false, d, val, dval, param, dpar);
  }
}

template <typename T, bool PARAM>
__global__ void __launch_bounds__(KB_THREADS, 1) kernel_cross_bwd_kernel(const KcParams p, const int dc, const int nsplit) {
  const int tile_r = blockIdx.x, b = blockIdx.y;
  const int d = p.d, G = p.desc.n_groups, nt = p.desc.n_terms;
  const int chunk = blockIdx.z / nsplit, split = blockIdx.z - chunk * nsplit;
  const int k0 = chunk * dc, k1 = min(d, k0 + dc);
  const bool first = chunk == 0;
  const int64_t r0 = (int64_t)tile_r * KB_TILE;
  extern __shared__ __align__(16) unsigned char kb_smem[];
  T* xs = reinterpret_cast<T*>(kb_smem);        // [G][64][d]   rows of this CTA
  T* yt = xs + (size_t)G * KB_TILE * d;          // [G][d][65]   current column tile, transposed
  T* part = yt + (size_t)G * d * (KB_TILE + 1);  // [256 threads][G][4 rows][dc]
  const T* ag = static_cast<const T*>(p.ag) + (int64_t)b * p.a_bstride;
  const T* bg = static_cast<const T*>(p.bg) + (int64_t)b * p.b_bstride;
  const T* Wm = p.W ? static_cast<const T*>(p.W) + (int64_t)b * p.w_bstride : nullptr;
  const T* wr = p.wr ? static_cast<const T*>(p.wr) + (int64_t)b * p.na : nullptr;
  const T* u = p.u ? static_cast<const T*>(p.u) + (int64_t)b * p.na : nullptr;
  const T* wc = p.wc ? static_cast<const T*>(p.wc) + (int64_t)b * p.nb : nullptr;
  const T* v = p.v ? static_cast<const T*>(p.v) + (int64_t)b * p.nb : nullptr;
  const bool want_grad = p.grad != nullptr, want_terms = first && p.term_sum != nullptr;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int pstride = G * 4 * dc;
  T* mypart = part + (size_t)tid * pstride;
  if (want_grad)
    for (int i = 0; i < pstride; ++i) mypart[i] = T(0);

  const int xr = (int)max((int64_t)0, min((int64_t)KB_TILE, p.na - r0));
  for (int g = 0; g < G; ++g)
    for (int i = tid; i < KB_TILE * d; i += KB_THREADS)
      xs[(size_t)g * KB_TILE * d + i] = (i < xr * d) ? ag[g * p.a_gstride + r0 * d + i] : T(0);

  T tsum[GPK_MAX_TERMS];
#pragma unroll
  for (int t = 0; t < GPK_MAX_TERMS; ++t) tsum[t] = T(0);
  T psum[PARAM ? GPK_MAX_FACTORS : 1];
#pragma unroll
  for (int f = 0; f < (PARAM ? GPK_MAX_FACTORS : 1); ++f) psum[f] = T(0);

  // column split `split` of `nsplit` sweeps its share of the column tiles
  const int n_ctiles = (int)((p.nb + KB_TILE - 1) / KB_TILE);
  const int per = (n_ctiles + nsplit - 1) / nsplit;
  const int tc1 = min(n_ctiles, (split + 1) * per);
  for (int tc = split * per; tc < tc1; ++tc) {
    const int64_t c0 = (int64_t)tc * KB_TILE;
    const int yr = (int)min((int64_t)KB_TILE, p.nb - c0);
    __syncthreads();
    for (int idx = tid; idx < G * KB_TILE * d; idx += KB_THREADS) {
      const int g = idx / (KB_TILE * d), rem = idx - g * KB_TILE * d;
      const int c = rem / d, k = rem - c * d;
      yt[((size_t)g * d + k) * (KB_TILE + 1) + c] = (c < yr) ? bg[g * p.b_gstride + (c0 + c) * d + k] : T(0);
    }
    __syncthreads();

#pragma unroll 1
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + ty * 4 + i;
#pragma unroll 1
      for (int j = 0; j < 4; ++j) {
        const int64_t c = c0 + tx + 16 * j;
        if (r >= p.na || c >= p.nb) continue;
        T gij = T(0);
        if (Wm) gij = Wm[r * p.w_si + c * p.w_sj] * (wr ? wr[r] : T(1)) * (wc ? wc[c] : T(1));
        if (u && v) gij = fma(u[r], v[c], gij);
        if (gij == T(0)) continue;
        for (int t = 0; t < nt; ++t) {
          const int f0 = p.desc.term_begin[t], f1 = p.desc.term_begin[t + 1];
          T val[KB_MAXF], dval[KB_MAXF], dpar[KB_MAXF];
          T prod = T(1);
#pragma unroll
          for (int q = 0; q < KB_MAXF; ++q) {
            val[q] = T(1);
            dval[q] = T(0);
            dpar[q] = T(0);
            if (f0 + q < f1) {
              const int g = p.desc.fac_group[f0 + q];
              const T* xr_ = xs + ((size_t)g * KB_TILE + ty * 4 + i) * d;
              const T* yc_ = yt + (size_t)g * d * (KB_TILE + 1) + tx + 16 * j;
              T d2 = T(0), dot = T(0);
              for (int k = 0; k < d; ++k) {
                const T xv = xr_[k], yv = yc_[(size_t)k * (KB_TILE + 1)];
                const T df = xv - yv;
                d2 = fma(df, df, d2);
                dot = fma(xv, yv, dot);
              }
              eval_cross_factor_grad<T, PARAM>(p.desc.fac_kind[f0 + q], d2, dot, d, val[q], dval[q],
                                               p.desc.fac_param[f0 + q], &dpar[q]);
              prod *= val[q];
            }
          }
#pragma unroll
          for (int tt = 0; tt < GPK_MAX_TERMS; ++tt)
            if (tt == t) tsum[tt] = fma(gij, prod, tsum[tt]);
          if constexpr (PARAM) {
            if (first) {
              const T ctp = (T)p.desc.coef[t];
#pragma unroll
              for (int q = 0; q < KB_MAXF; ++q) {
                if (dpar[q] == T(0)) continue;
                T others = T(1);
#pragma unroll
                for (int q2 = 0; q2 < KB_MAXF; ++q2)
                  if (q2 != q) others *= val[q2];
                add_param(psum, f0 + q, gij * ctp * others * dpar[q]);
              }
            }
          }
          if (!want_grad) continue;
          const T ct = (T)p.desc.coef[t];
#pragma unroll
          for (int q = 0; q < KB_MAXF; ++q) {
            if (f0 + q >= f1 || dval[q] == T(0)) continue;
            T others = T(1);
#pragma unroll
            for (int q2 = 0; q2 < KB_MAXF; ++q2)
              if (q2 != q) others *= val[q2];
            const T wgt = gij * ct * others * dval[q];
            const int g = p.desc.fac_group[f0 + q];
            T* pp = mypart + ((size_t)g * 4 + i) * dc;
            const T* yc_ = yt + (size_t)g * d * (KB_TILE + 1) + tx + 16 * j;
            if (p.desc.fac_kind[f0 + q] == GPK_LINEAR) {
              for (int k = k0; k < k1; ++k) pp[k - k0] = fma(wgt, yc_[(size_t)k * (KB_TILE + 1)], pp[k - k0]);
            } else {
              // d(d2)/da_ik = 2 (a_ik - b_jk), the difference formed per pair (see kernel_matrix_bwd_kernel)
              const T* xr_ = xs + ((size_t)g * KB_TILE + ty * 4 + i) * d;
              for (int k = k0; k < k1; ++k)
                pp[k - k0] = fma(T(2) * wgt, xr_[k] - yc_[(size_t)k * (KB_TILE + 1)], pp[k - k0]);
            }
          }
        }
      }
    }
  }
  __syncthreads();
  if (want_grad) {
    T* gout = static_cast<T*>(p.grad) + (int64_t)b * p.a_bstride;
    const int w = k1 - k0;
    for (int idx = tid; idx < G * KB_TILE * w; idx += KB_THREADS) {
      const int g = idx / (KB_TILE * w), rem = idx - g * KB_TILE * w;
      const int row = rem / w, kk = rem - row * w;
      if (r0 + row >= p.na) continue;
      const int rty = row >> 2, ri = row & 3;
      T s = T(0);
      for (int t16 = 0; t16 < 16; ++t16) s += part[(size_t)(rty * 16 + t16) * pstride + ((size_t)g * 4 + ri) * dc + kk];
      T* o = gout + g * p.a_gstride + (r0 + row) * d + k0 + kk;
      if (nsplit > 1)
        atomicAdd(o, s);
      else
        *o += s;
    }
  }
  if (want_terms) {
    __shared__ T red[8][GPK_MAX_TERMS];
#pragma unroll
    for (int t = 0; t < GPK_MAX_TERMS; ++t) {
      T v_ = warp_sum(tsum[t]);
      if ((tid & 31) == 0) red[tid >> 5][t] = v_;
    }
    __syncthreads();
    if (tid < nt) {
      T s = T(0);
      for (int w = 0; w < 8; ++w) s += red[w][tid];
      atomicAdd(static_cast<T*>(p.term_sum) + (int64_t)b * GPK_MAX_TERMS + tid, s);
    }
  }
  if constexpr (PARAM)
    if (first) flush_params(p.desc, psum, static_cast<T*>(p.param_sum) + (int64_t)b * GPK_MAX_FACTORS);
}

// The prior-variance term: gdiag_i contracted with d k(a_i, a_i): adds to term_sum and, for Linear factors (the only kind
// whose diagonal depends on the point: d <a, a> / da = 2 a), to the rows' gradient.  One thread per point.  It adds nothing
// to param_sum: RQ's d phi / d alpha is exactly 0 at r = 0.
template <typename T>
__global__ void kernel_cross_bwd_diag_kernel(const gpk_kernel_desc desc, const T* ag, int64_t a_gstride, int64_t a_bstride,
                                             int64_t na, int32_t d, const T* gdiag, T* term_sum, T* grad) {
  const int b = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int nt = desc.n_terms;
  const T gi = i < na ? gdiag[(int64_t)b * na + i] : T(0);
  for (int t = 0; t < nt; ++t) {
    const int f0 = desc.term_begin[t], f1 = desc.term_begin[t + 1];
    T val[KB_MAXF], prod = T(1);
#pragma unroll
    for (int q = 0; q < KB_MAXF; ++q) {
      val[q] = T(1);
      if (f0 + q < f1 && i < na) {
        T dot = T(0);
        if (desc.fac_kind[f0 + q] == GPK_LINEAR) {
          const T* a = ag + desc.fac_group[f0 + q] * a_gstride + (int64_t)b * a_bstride + i * d;
          for (int k = 0; k < d; ++k) dot = fma(a[k], a[k], dot);
        }
        T dv;
        eval_cross_factor_grad<T>(desc.fac_kind[f0 + q], T(0), dot, d, val[q], dv, desc.fac_param[f0 + q]);
        prod *= val[q];
      }
    }
    if (term_sum) {
      const T s = warp_sum(gi * prod);
      if ((threadIdx.x & 31) == 0 && s != T(0)) atomicAdd(term_sum + (int64_t)b * GPK_MAX_TERMS + t, s);
    }
    if (!grad || i >= na) continue;
#pragma unroll
    for (int q = 0; q < KB_MAXF; ++q) {
      if (f0 + q >= f1 || desc.fac_kind[f0 + q] != GPK_LINEAR) continue;
      T others = T(1);
#pragma unroll
      for (int q2 = 0; q2 < KB_MAXF; ++q2)
        if (q2 != q) others *= val[q2];
      const T wgt = T(2) * gi * (T)desc.coef[t] * others;
      const int64_t off = desc.fac_group[f0 + q] * a_gstride + (int64_t)b * a_bstride + i * d;
      for (int k = 0; k < d; ++k) grad[off + k] = fma(wgt, ag[off + k], grad[off + k]);
    }
  }
}

template <typename T>
static int launch_cross_pass(const KcParams& p, int32_t batch, cudaStream_t stream) {
  if (p.na == 0 || p.nb == 0) return 0;
  const int Gn = p.desc.n_groups, d = p.d;
  constexpr size_t kMaxSmem = 200 * 1024;
  const size_t rows_bytes = ((size_t)Gn * KB_TILE * d + (size_t)Gn * d * (KB_TILE + 1)) * sizeof(T);
  const size_t dim_bytes = (size_t)KB_THREADS * Gn * 4 * sizeof(T);
  if (rows_bytes + dim_bytes > kMaxSmem) return GPK_ERR_UNSUPPORTED;
  // without a gradient output only term_sum is formed: one chunk, no partial sums
  const size_t fit = (kMaxSmem - rows_bytes) / dim_bytes;
  const int dc = p.grad ? (fit < (size_t)d ? (int)fit : d) : 1;
  const int chunks = p.grad ? (d + dc - 1) / dc : 1;
  const size_t smem = rows_bytes + (p.grad ? (size_t)dc * dim_bytes : 0);
  const bool param = p.param_sum != nullptr;
  if (const int rc = param ? opt_in_smem<kernel_cross_bwd_kernel<T, true>>((int)smem)
                           : opt_in_smem<kernel_cross_bwd_kernel<T, false>>((int)smem))
    return rc;
  // few rows (a handful of candidate points, a 4096-row chunk on 132 SMs) would leave SMs idle: the columns are then split
  // over CTAs until the grid holds about two CTAs per SM, and the row partials are added atomically
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t row_tiles = (p.na + KB_TILE - 1) / KB_TILE, n_ctiles = (p.nb + KB_TILE - 1) / KB_TILE;
  const int64_t base = row_tiles * batch * chunks;
  const int nsplit = (int)std::max<int64_t>(1, std::min<int64_t>(n_ctiles, (2 * sms + base - 1) / base));
  if ((int64_t)chunks * nsplit > 65535) return GPK_ERR_UNSUPPORTED;
  dim3 grid((unsigned)row_tiles, (unsigned)batch, (unsigned)(chunks * nsplit));
  const auto kernel = param ? kernel_cross_bwd_kernel<T, true> : kernel_cross_bwd_kernel<T, false>;
  kernel<<<grid, KB_THREADS, smem, stream>>>(p, dc, nsplit);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

template <typename T>
static int launch_kernel_cross_bwd(const gpk_kernel_desc* desc, const T* xsg, int64_t xsg_gstride, int64_t xs_bstride,
                                   int64_t m, const T* xg, int64_t xg_gstride, int64_t x_bstride, int64_t n, int32_t d,
                                   const T* W, int64_t ldw, int64_t w_bstride, const T* r, const T* u, const T* v,
                                   const T* gdiag, T* term_sum, T* grad_xsg, T* grad_xg, T* param_sum, int32_t batch,
                                   void* stream) {
  if (!desc || !xsg || !xg || m < 0 || n < 0 || d < 1 || batch < 1) return GPK_ERR_ARG;
  if ((u == nullptr) != (v == nullptr)) return GPK_ERR_ARG;
  if (desc->n_terms < 0 || desc->n_terms > GPK_MAX_TERMS || desc->n_groups < 1 || desc->n_groups > GPK_MAX_GROUPS)
    return GPK_ERR_ARG;
  for (int t = 0; t < desc->n_terms; ++t)
    if (desc->term_begin[t + 1] - desc->term_begin[t] > KB_MAXF) return GPK_ERR_UNSUPPORTED;
  const cudaStream_t st = (cudaStream_t)stream;
  KcParams p;
  p.desc = *desc;
  p.d = d;
  // rows = test points x*: term sums and their gradient
  p.ag = xsg, p.a_gstride = xsg_gstride, p.a_bstride = xs_bstride, p.na = m;
  p.bg = xg, p.b_gstride = xg_gstride, p.b_bstride = x_bstride, p.nb = n;
  p.W = W, p.w_si = ldw, p.w_sj = 1, p.w_bstride = w_bstride;
  p.wr = r, p.u = u, p.wc = nullptr, p.v = v;
  p.term_sum = term_sum, p.grad = grad_xsg, p.param_sum = param_sum;
  if ((W || u) && (term_sum || grad_xsg || param_sum))
    if (const int rc = launch_cross_pass<T>(p, batch, st)) return rc;
  // rows = points x: the columns' gradient, G read transposed
  if ((W || u) && grad_xg) {
    p.ag = xg, p.a_gstride = xg_gstride, p.a_bstride = x_bstride, p.na = n;
    p.bg = xsg, p.b_gstride = xsg_gstride, p.b_bstride = xs_bstride, p.nb = m;
    p.w_si = 1, p.w_sj = ldw;
    p.wr = nullptr, p.wc = r, p.u = v, p.v = u;
    p.term_sum = nullptr, p.grad = grad_xg, p.param_sum = nullptr;
    if (const int rc = launch_cross_pass<T>(p, batch, st)) return rc;
  }
  if (gdiag && m > 0 && (term_sum || grad_xsg)) {
    dim3 grid((unsigned)((m + 127) / 128), (unsigned)batch);
    kernel_cross_bwd_diag_kernel<T><<<grid, 128, 0, st>>>(*desc, xsg, xsg_gstride, xs_bstride, m, d, gdiag, term_sum,
                                                           grad_xsg);
    GPK_COUNT_LAUNCH();
    GPK_CHECK_LAUNCH();
  }
  return 0;
}

}  // namespace gpk

extern "C" {
int gpk_kernel_cross_bwd_f64(const gpk_kernel_desc* desc_host, const double* xsg, int64_t xsg_gstride,
                             int64_t xs_bstride, int64_t m, const double* xg, int64_t xg_gstride, int64_t x_bstride,
                             int64_t n, int32_t d, const double* W, int64_t ldw, int64_t w_bstride, const double* r,
                             const double* u, const double* v, const double* gdiag, double* term_sum, double* grad_xsg,
                             double* grad_xg, double* param_sum, int32_t batch, void* stream) {
  return gpk::launch_kernel_cross_bwd<double>(desc_host, xsg, xsg_gstride, xs_bstride, m, xg, xg_gstride, x_bstride, n, d,
                                              W, ldw, w_bstride, r, u, v, gdiag, term_sum, grad_xsg, grad_xg, param_sum,
                                              batch, stream);
}
int gpk_kernel_cross_bwd_f32(const gpk_kernel_desc* desc_host, const float* xsg, int64_t xsg_gstride, int64_t xs_bstride,
                             int64_t m, const float* xg, int64_t xg_gstride, int64_t x_bstride, int64_t n, int32_t d,
                             const float* W, int64_t ldw, int64_t w_bstride, const float* r, const float* u,
                             const float* v, const float* gdiag, float* term_sum, float* grad_xsg, float* grad_xg,
                             float* param_sum, int32_t batch, void* stream) {
  return gpk::launch_kernel_cross_bwd<float>(desc_host, xsg, xsg_gstride, xs_bstride, m, xg, xg_gstride, x_bstride, n, d,
                                             W, ldw, w_bstride, r, u, v, gdiag, term_sum, grad_xsg, grad_xg, param_sum,
                                             batch, stream);
}
int gpk_kernel_matrix_bwd_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride,
                              int64_t x_bstride, int64_t n, int32_t d, const double* G, int64_t ldg, int64_t g_bstride,
                              double* term_sum, double* grad_xg, double* diag, double* param_sum, int32_t batch,
                              void* stream) {
  return gpk::launch_kernel_matrix_bwd<double>(desc_host, xg, xg_gstride, x_bstride, n, d, G, ldg, g_bstride, term_sum,
                                               grad_xg, diag, param_sum, batch, stream);
}
int gpk_kernel_matrix_bwd_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t x_bstride,
                              int64_t n, int32_t d, const float* G, int64_t ldg, int64_t g_bstride, float* term_sum,
                              float* grad_xg, float* diag, float* param_sum, int32_t batch, void* stream) {
  return gpk::launch_kernel_matrix_bwd<float>(desc_host, xg, xg_gstride, x_bstride, n, d, G, ldg, g_bstride, term_sum,
                                              grad_xg, diag, param_sum, batch, stream);
}
}
