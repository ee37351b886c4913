/*
 * gpk.h -- C-ABI of libgpk: the H100 (sm_90a) kernels behind the Stheno GP-inference hot path.
 *
 * The reference (wesselb/stheno) has no FFI: its operator boundary is Python multiple dispatch into
 * `lab.B.*` / `matrix` / `mlkernels` (SURVEY.md section 8b).  Each entry point below names the reference
 * call site(s) whose arithmetic it replaces (paths relative to the reference tree).
 *
 * Conventions
 *   - All pointers are DEVICE pointers unless the parameter name ends in `_host`.
 *   - Matrices are ROW-MAJOR with an explicit leading dimension `ld` (in elements).
 *   - "Padded" matrices have their dimensions rounded up to a multiple of GPK_TILE (128); the padding of a
 *     matrix that will be factorised is the identity (1 on the diagonal, 0 elsewhere), padding of right-hand
 *     sides is 0.  `gpk_round_up(n)` gives the padded size.
 *   - Only the LOWER triangle of symmetric matrices / Cholesky factors is read or written.
 *   - Functions are stateless, re-entrant and stream-ordered on `stream` (a cudaStream_t passed as void*);
 *     they never allocate device memory and never synchronise the host.
 *   - Return value: 0 = launched OK; < 0 = bad argument (GPK_ERR_*) or a CUDA launch error (-1000 - cudaError).
 *     Numerical failure (non-positive pivot) is reported LAPACK-style through the device-side `info` word
 *     (index of the first bad pivot, 1-based; 0 = success) so that no host sync is forced.
 *   - `_f64` / `_f32` suffix = arithmetic type (double / float); everything is computed in that type, except the row
 *     reductions that say "fp64 sums in both precisions".
 *   - The one environment variable the library reads is GPK_NO_LOOKAHEAD, at every gpk_potrf_* call.  When it is set,
 *     the factorisation enqueues all its work on `stream` instead of factorising the next panel on side streams while
 *     the trailing update runs, so that CUDA events around a launch time that kernel alone.  It is meant for profiling:
 *     the factorisation is slower with it.
 */
#ifndef GPK_H_
#define GPK_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPK_TILE 128
#define GPK_VERSION 100

#define GPK_ERR_ARG (-1)
#define GPK_ERR_ALIGN (-2)
#define GPK_ERR_UNSUPPORTED (-3)

/* ---- kernel-expression descriptor -------------------------------------------------------------------
 * A kernel is flattened by the host into a sum of products:
 *     k(x, y) = sum_t coef[t] * prod_{f in term t} phi_{kind[f]}( x^(group[f]), y^(group[f]) )
 * where x^(g) = x / lengthscale_g is a pre-stretched copy of the inputs ("group" g), exactly as the
 * reference evaluates `k.stretch(l)` by dividing the inputs (mlkernels Stretched; call sites
 * stheno/model/fdd.py:79, stheno/model/observations.py:139,285,286).
 */
enum gpk_kind {
  GPK_EQ = 0,       /* exp(-r^2/2)                                  */
  GPK_MATERN12 = 1, /* exp(-r)                                      */
  GPK_MATERN32 = 2, /* (1 + sqrt3 r) exp(-sqrt3 r)                  */
  GPK_MATERN52 = 3, /* (1 + sqrt5 r + 5 r^2 / 3) exp(-sqrt5 r)      */
  GPK_LINEAR = 4,   /* <x, y>                                       */
  GPK_DELTA = 5,    /* same inputs: [i == j]; else [r^2 < 1e-10]    */
  GPK_ONE = 6,      /* 1                                            */
  GPK_RQ = 7        /* (1 + r^2 / (2 alpha))^-alpha, alpha = fac_param[f] (mlkernels RQ; README.md:1076-1088) */
};

#define GPK_MAX_TERMS 8
#define GPK_MAX_FACTORS 16
#define GPK_MAX_GROUPS 8

typedef struct gpk_kernel_desc {
  int32_t n_terms;
  int32_t n_groups;
  int32_t term_begin[GPK_MAX_TERMS + 1]; /* factors of term t: [term_begin[t], term_begin[t+1]) */
  int32_t fac_kind[GPK_MAX_FACTORS];
  int32_t fac_group[GPK_MAX_FACTORS];
  double coef[GPK_MAX_TERMS];
  double fac_param[GPK_MAX_FACTORS]; /* per-factor shape parameter (GPK_RQ: alpha); unused by the other kinds */
} gpk_kernel_desc;

/* flags for gpk_kernel_matrix_* */
#define GPK_KM_LOWER 1        /* x and y are the same points: write only tiles on/below the diagonal      */
#define GPK_KM_SAME 2         /* x and y are the same object (Delta -> [i == j]; diagonal terms apply)     */
#define GPK_KM_PAD_IDENTITY 4 /* fill rows/cols >= n up to the padded size with the identity               */
#define GPK_KM_PAD_ZERO 8     /* fill rows/cols >= n up to the padded size with zeros                      */

int gpk_version(void);
int64_t gpk_round_up(int64_t n);

/* K1: fused pairwise-distance + kernel evaluation (+ diagonal noise + Cholesky jitter).
 * Replaces `p.kernel(x)` / `B.add(K, noise)` / `B.reg` : stheno/model/fdd.py:79,
 * stheno/model/observations.py:139,285,286 and the `+ B.epsilon I` of every B.cholesky (README.md:820-830).
 *   xg: [n_groups][batch][n][d]  pre-stretched inputs (strides: xg_gstride, x_bstride, d)
 *   yg: same for the second argument (n2 points); may equal xg.
 *   out[b][i][j] (ld = ldo, batch stride = o_bstride), i < rows_out, j < cols_out where rows_out/cols_out are
 *   n / n2 rounded up to GPK_TILE when a PAD flag is given, else n / n2.
 *   Diagonal (only with GPK_KM_SAME): out[i][i] += noise_scalar (+ noise_vec[b][i] if non-NULL), then += jitter. */
int gpk_kernel_matrix_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride, int64_t x_bstride,
                          int64_t n, const double* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n2, int32_t d,
                          double noise_scalar, const double* noise_vec, int64_t nv_bstride, double jitter,
                          int32_t flags, double* out, int64_t ldo, int64_t o_bstride, int32_t batch, void* stream);
int gpk_kernel_matrix_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t x_bstride,
                          int64_t n, const float* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n2, int32_t d,
                          double noise_scalar, const float* noise_vec, int64_t nv_bstride, double jitter,
                          int32_t flags, float* out, int64_t ldo, int64_t o_bstride, int32_t batch, void* stream);

/* elwise: out[b][i] = k(x_i, y_i)  -- `k.elwise(x)` at stheno/model/fdd.py:66, observations.py:304. */
int gpk_kernel_diag_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride, int64_t x_bstride,
                        const double* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n, int32_t d, int32_t same,
                        double* out, int64_t o_bstride, int32_t batch, void* stream);
int gpk_kernel_diag_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t x_bstride,
                        const float* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n, int32_t d, int32_t same,
                        float* out, int64_t o_bstride, int32_t batch, void* stream);

/* K1-backward: contraction of an upstream gradient G = d(loss)/dK (symmetric n x n, ld = ldg) with dK/d(theta) for
 * K = k(x, x) (same points): term_sum[b][t] += sum_ij G_ij prod_f phi_f  (d loss / d coef_t; caller zeroes it; stride
 * GPK_MAX_TERMS), grad_xg[g][b][i][:] = d loss / d x^(g)_i (layout and strides of xg), diag[b][i] = G_ii (noise
 * gradient), and, optional (NULL: not formed),
 *   param_sum[b][f] += sum_ij G_ij coef_t prod_{f' != f in t} phi_f' d phi_f / d fac_param[f]   (stride GPK_MAX_FACTORS;
 *   caller zeroes it; 0 for kinds without a parameter; GPK_RQ: d loss / d alpha).  No n x n tensor per hyper-parameter is
 *   ever formed.  Replaces torch autograd through
 * exp / pw_dists2 in the reference's optimisation loop (readme_example13_optimisation_torch.py:46-53). */
int gpk_kernel_matrix_bwd_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride,
                              int64_t x_bstride, int64_t n, int32_t d, const double* G, int64_t ldg, int64_t g_bstride,
                              double* term_sum, double* grad_xg, double* diag, double* param_sum, int32_t batch,
                              void* stream);
int gpk_kernel_matrix_bwd_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t x_bstride,
                              int64_t n, int32_t d, const float* G, int64_t ldg, int64_t g_bstride, float* term_sum,
                              float* grad_xg, float* diag, float* param_sum, int32_t batch, void* stream);

/* Rectangular K1-backward: K_ij = k(x*_i, x_j) (m x n) for two DIFFERENT point sets (K1 without GPK_KM_SAME: Delta is
 * [r^2 < 1e-10] with gradient 0, no symmetry factor), upstream gradient given factored:
 *     G_ij = r_i W_ij + u_i v_j      W: [batch] x m x n (ld = ldw, batch stride w_bstride), r, u: [batch][m], v: [batch][n]
 * W, r, u, v may each be NULL (r = NULL: scale 1; an explicit dense G is W with r = NULL; u and v come together).
 * gdiag ([batch][m], may be NULL) adds the prior-variance term sum_i gdiag_i k(x*_i, x*_i).  Outputs, each accumulated (the
 * caller zeroes them) and each optional (NULL: not formed):
 *   term_sum[b][t] += sum_ij G_ij prod_f phi_f(i, j) (+ the gdiag term)        -> d loss / d coef_t
 *   grad_xsg[g][b][i][:] += d loss / d x*^(g)_i (layout of xsg)
 *   grad_xg[g][b][j][:] += d loss / d x^(g)_j (layout of xg; chunks of test points add up)
 *   param_sum[b][f] += as for gpk_kernel_matrix_bwd (the gdiag term adds nothing: RQ's d phi / d alpha is 0 at r = 0)
 * The posterior predictions' backward (autograd.py): G* = g_mu alpha^T - 2 diag(g_var) W with W = K* K^-1. */
int gpk_kernel_cross_bwd_f64(const gpk_kernel_desc* desc_host, const double* xsg, int64_t xsg_gstride,
                             int64_t xs_bstride, int64_t m, const double* xg, int64_t xg_gstride, int64_t x_bstride,
                             int64_t n, int32_t d, const double* W, int64_t ldw, int64_t w_bstride, const double* r,
                             const double* u, const double* v, const double* gdiag, double* term_sum, double* grad_xsg,
                             double* grad_xg, double* param_sum, int32_t batch, void* stream);
int gpk_kernel_cross_bwd_f32(const gpk_kernel_desc* desc_host, const float* xsg, int64_t xsg_gstride, int64_t xs_bstride,
                             int64_t m, const float* xg, int64_t xg_gstride, int64_t x_bstride, int64_t n, int32_t d,
                             const float* W, int64_t ldw, int64_t w_bstride, const float* r, const float* u,
                             const float* v, const float* gdiag, float* term_sum, float* grad_xsg, float* grad_xg,
                             float* param_sum, int32_t batch, void* stream);

/* fp64 emulation on the INT8 tensor cores (wgmma .s32.s8.s8; Ozaki splitting): every row of an operand is scaled by a
 * power of two and split error-free into `slices` signed 7-bit integers; the slice products are EXACT in int32 and are
 * recombined in fp64.  6 slices: 21 int8 GEMMs, product error ~2^-40 |a||b| (zero-mean); 7 slices: 28 GEMMs, ~2^-47.
 * The fp64 entry points gpk_potrf_f64, gpk_trsm_right_f64, gpk_gemm_nt_f64, gpk_posterior_marginals_f64,
 * gpk_sparse_posterior_marginals_f64 and gpk_sparse_accumulate_f64 take it as three trailing arguments (slices, ws, ws_bytes): slices = 0 keeps every product on
 * the fp64 tensor cores (ws may be NULL); slices = 5..8 with a caller-owned, 1024-byte aligned scratch `ws` runs the LARGE
 * GEMM-shaped updates of that call on the int8 tensor cores -- the trailing updates of a factorisation (batch 1,
 * n_pad >= 2048), and products of batch 1 with M, N, K >= 256 and M N K >= 1.5e9 (reductions longer than 65536 in several
 * exact passes) -- whenever `ws_bytes` covers them.  Everything else, and every update whose scratch is too small, stays on
 * the fp64 tensor cores.  The size queries give the scratch that makes every update of a call eligible, 0 when none is:
 *   gpk_gemm_nt_oz_ws_bytes     one product M x N x K
 *   gpk_trsm_right_oz_ws_bytes  the largest product of the recursive solve of `rows` right-hand sides (also the solve inside
 *                               gpk_posterior_marginals_f64 and gpk_sparse_posterior_marginals_f64 (rows = chunk) and
 *                               gpk_sparse_accumulate_f64 (rows = c_pad))
 *   gpk_potrf_oz_ws_bytes       a factorisation (the panel slices; from n_pad >= 4096 those of a pair of panels)
 * Calls that share a scratch buffer must be stream-ordered with respect to each other. */
int64_t gpk_gemm_nt_oz_ws_bytes(int64_t M, int64_t N, int64_t K, int32_t slices);
int64_t gpk_trsm_right_oz_ws_bytes(int64_t n_pad, int64_t rows, int32_t slices);
int64_t gpk_potrf_oz_ws_bytes(int64_t n_pad, int64_t extra_rows, int32_t slices);

/* GEMM  C = beta*C + alpha * A * B^T   (A: M x K, B: N x K, both K-contiguous; C: M x N).
 * M, N multiples of 128; K a multiple of 16; pointers 16-byte aligned; ld multiples of 2.
 * lower != 0: only tiles with (row tile >= col tile) are touched (SYRK-style trailing update, M >= N).
 * Replaces the BLAS-3 inside B.cholesky / B.iqf / B.mm (stheno/random.py:274-276,
 * stheno/model/observations.py:301,322,323). */
int gpk_gemm_nt_f64(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, int64_t a_bstride,
                    const double* B, int64_t ldb, int64_t b_bstride, double beta, double* C, int64_t ldc,
                    int64_t c_bstride, int32_t lower, int32_t batch, int32_t slices, void* ws, int64_t ws_bytes,
                    void* stream);
int gpk_gemm_nt_f32(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t lda, int64_t a_bstride,
                    const float* B, int64_t ldb, int64_t b_bstride, float beta, float* C, int64_t ldc,
                    int64_t c_bstride, int32_t lower, int32_t batch, void* stream);
/* gpk_gemm_nt_f32 runs on the wgmma tensor cores with the 3xTF32 split (a = hi + lo, hi = a & 0xFFFFE000; a b formed as
 * hi hi + hi lo + lo hi) when K >= 128, K % 32 == 0, every ld and batch stride is a multiple of 4 and the pointers are 16-byte
 * aligned, and on an fp32 FFMA kernel otherwise.  Where the two differ (measured on an H100 80GB HBM3 at a 700 W power limit):
 *   - error: FFMA is fp32 arithmetic.  3xTF32 on random normal operands gives max |err| / max(|A| |B|^T) = 3.1e-6 at K = 4096,
 *     4.3e-6 at 8192 and 6.1e-6 at 16384 (about 0.8 u sqrt(K), u = 2^-24); the worst case is (6 K + 48) u |alpha| |A| |B|^T.
 *   - subnormals: both keep subnormal operands and subnormal products (no flush to zero).
 *   - non-finite inputs: on 3xTF32 a row of A (B) holding a NaN or an infinity makes its whole row (column) of alpha A B^T NaN,
 *     where FFMA gives NaN or +-inf as fp32 does: the low part of +-inf is inf - inf = NaN.  (A low part of 0 would not give
 *     fp32's answer either: hi lo would be inf * 0 = NaN wherever the other operand is exact in TF32.)  The opt-in
 *     gpk_potrf_f64_tf32x3 below forms its trailing updates the same way. */

/* K2: blocked right-looking Cholesky, in place, lower, row-major.
 *   A: [(n_pad + extra_rows) x n_pad] (ld = lda): the first n_pad rows hold the (padded) SPD matrix; the
 *   `extra_rows` (multiple of 128, may be 0) rows below it hold right-hand sides b^T, one per row, which come out
 *   as (L^-1 b)^T -- the triangular solve of B.iqf_diag fused into the factorisation (stheno/random.py:276).
 *   logdet[b] += 2 sum log diag(L) (caller zeroes it); info[b] = first non-positive pivot (1-based) or 0.
 * Replaces B.cholesky + B.logdet: stheno/random.py:274, stheno/model/observations.py:300,334. */
int gpk_potrf_f64(double* A, int64_t lda, int64_t a_bstride, int64_t n_pad, int64_t extra_rows, double* logdet,
                  int32_t* info, int32_t batch, int32_t slices, void* ws, int64_t ws_bytes, void* stream);
int gpk_potrf_f32(float* A, int64_t lda, int64_t a_bstride, int64_t n_pad, int64_t extra_rows, float* logdet,
                  int32_t* info, int32_t batch, void* stream);

/* Opt-in mixed precision (BASELINE north_star: "tf32/bf16 where the user opts in"): same factorisation, but the
 * K >= 128 trailing updates of the fp64 matrix are formed from an fp32 copy of the panel by the wgmma 3xTF32 kernel
 * (fp32-level products, fp64 accumulation into the matrix).  `ws`: float workspace of >= (n_pad + extra_rows) * 512
 * elements.  Results agree with gpk_potrf_f64 to ~1e-6 relative, NOT to the 1e-10 parity bar: never the default. */
int gpk_potrf_f64_tf32x3(double* A, int64_t lda, int64_t a_bstride, int64_t n_pad, int64_t extra_rows, double* logdet,
                         int32_t* info, int32_t batch, float* ws, int64_t ws_elems, void* stream);

/* The emulated GEMM on its own, whatever its size: C = beta C + alpha A B^T (M % 128 == 0, N % 64 == 0, K a positive
 * multiple of 128), slices = 5..8.  `ws`: 1024-byte aligned, >= round_up(gpk_oz_ws_bytes(M, K, slices), 1024) +
 * gpk_oz_ws_bytes(N, K, slices) bytes.
 * Rows of every finite magnitude are scaled exactly (subnormal to near overflow); a row of A (B) holding a NaN or an
 * infinity makes its row (column) of alpha A B^T NaN, where fp64 gives NaN or +-inf.  Lower mode and beta as in
 * gpk_gemm_nt_f64: only the tiles that touch the lower triangle are read or written, for every beta. */
int64_t gpk_oz_ws_bytes(int64_t rows, int64_t K, int32_t slices);
int gpk_gemm_nt_f64_oz(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, const double* B,
                       int64_t ldb, double beta, double* C, int64_t ldc, int32_t lower, int32_t slices, void* ws,
                       int64_t ws_bytes, void* stream);

/* K3: X * L^T = B  in place (B: rows x n_pad, rows a multiple of 64; L: n_pad x n_pad lower).
 * Row r of the result is (L^-1 b_r)^T.  Replaces B.solve(L, .) / B.iqf:  stheno/model/observations.py:301 and
 * the PosteriorMean / PosteriorKernel evaluation behind observations.py:143-168. */
int gpk_trsm_right_f64(const double* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, double* B, int64_t ldb,
                       int64_t b_bstride, int64_t rows, int32_t batch, int32_t slices, void* ws, int64_t ws_bytes,
                       void* stream);
int gpk_trsm_right_f32(const float* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, float* B, int64_t ldb,
                       int64_t b_bstride, int64_t rows, int32_t batch, void* stream);

/* X * L = B in place (B: rows x n_pad): row r of the result is (L^-T b_r)^T.  Backward substitution used for
 * K^-1 b = L^-T L^-1 b (autograd, sampling from the posterior precision, B.solve with transposes). */
int gpk_trsm_right_t_f64(const double* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, double* B, int64_t ldb,
                         int64_t b_bstride, int64_t rows, int32_t batch, void* stream);
int gpk_trsm_right_t_f32(const float* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, float* B, int64_t ldb,
                         int64_t b_bstride, int64_t rows, int32_t batch, void* stream);

/* K4: log-marginal finish: out[b][c] = -0.5 * (logdet[b] + n * log(2 pi) + sum_j a[b][c][j]^2), c < k, where row c
 * of `a` (ld = lda) is (L^-1 (y_c - mu))^T.  fp64 sums in both precisions, rounded once.  stheno/random.py:272-279. */
int gpk_logpdf_finish_f64(const double* a, int64_t lda, int64_t a_bstride, int64_t n, int64_t n_cols, int32_t k,
                          const double* logdet, double* out, int32_t batch, void* stream);
int gpk_logpdf_finish_f32(const float* a, int64_t lda, int64_t a_bstride, int64_t n, int64_t n_cols, int32_t k,
                          const float* logdet, float* out, int32_t batch, void* stream);

/* Row reductions over V (rows x n_cols, ld = ldv):  dot[r] = sum_j V[r][j] * b[j] (b may be NULL),
 * sq[r] = sum_j V[r][j]^2 (sq may be NULL); fp64 sums in both precisions, rounded once.  Posterior mean  m(x*) + V b  and marginal variance
 * k(x*,x*) - sum V^2 (mlkernels mean_var_diag via stheno/model/fdd.py:72-74); B.matmul_diag at observations.py:305. */
int gpk_row_dot_sq_f64(const double* V, int64_t ldv, int64_t v_bstride, int64_t rows, int64_t n_cols,
                       const double* b, int64_t b_bstride, double* dot, double* sq, int64_t o_bstride,
                       int32_t batch, void* stream);
int gpk_row_dot_sq_f32(const float* V, int64_t ldv, int64_t v_bstride, int64_t rows, int64_t n_cols, const float* b,
                       int64_t b_bstride, float* dot, float* sq, int64_t o_bstride, int32_t batch, void* stream);

/* Layout helpers (padding, symmetrisation, transposition) -- the `B.dense`, `B.transpose`, `B.reg` plumbing.
 * gpk_pad_copy: dst[(rows_pad) x (cols_pad)] = src[rows x cols] (+ diag_add on the diagonal), padding = identity
 *   (pad_identity != 0) or zero.  gpk_symmetrize: mirror the lower triangle into the upper one (n x n).
 * gpk_transpose: dst[cols x rows] = src[rows x cols]^T. */
int gpk_pad_copy_f64(const double* src, int64_t lds, int64_t s_bstride, int64_t rows, int64_t cols, double* dst,
                     int64_t ldd, int64_t d_bstride, int64_t rows_pad, int64_t cols_pad, double diag_add,
                     int32_t pad_identity, int32_t batch, void* stream);
int gpk_pad_copy_f32(const float* src, int64_t lds, int64_t s_bstride, int64_t rows, int64_t cols, float* dst,
                     int64_t ldd, int64_t d_bstride, int64_t rows_pad, int64_t cols_pad, double diag_add,
                     int32_t pad_identity, int32_t batch, void* stream);
int gpk_symmetrize_f64(double* A, int64_t lda, int64_t a_bstride, int64_t n, int32_t batch, void* stream);
int gpk_symmetrize_f32(float* A, int64_t lda, int64_t a_bstride, int64_t n, int32_t batch, void* stream);
int gpk_transpose_f64(const double* src, int64_t lds, int64_t s_bstride, int64_t rows, int64_t cols, double* dst,
                      int64_t ldd, int64_t d_bstride, int32_t batch, void* stream);
int gpk_transpose_f32(const float* src, int64_t lds, int64_t s_bstride, int64_t rows, int64_t cols, float* dst,
                      int64_t ldd, int64_t d_bstride, int32_t batch, void* stream);

/* K3 in one call: posterior mean and marginal variance terms at m test points (PosteriorMean / PosteriorKernel behind
 * stheno/model/observations.py:143-168, mlkernels.mean_var_diag via stheno/model/fdd.py:72-74), batch 1:
 *   V^T = k(x*, x) L^-T (K1 rows + right TRSM);  dot[i] = <v_i, half_y>;  sq[i] = |v_i|^2
 * half_y = (L^-1 (y - m(x)))^T zero-padded to n_pad (dot may be NULL: variance only; sq may be NULL: mean only).
 * The caller adds the prior mean / subtracts sq from the prior variance.  Test points are processed in chunks of `chunk`
 * rows (multiple of 128) through `ws` (>= chunk * n_pad elements, 16-byte aligned): K(x*, x) is never held whole. */
int gpk_posterior_marginals_f64(const gpk_kernel_desc* desc_host, const double* xsg, int64_t xsg_gstride, int64_t m,
                                const double* xg, int64_t xg_gstride, int64_t n, int32_t d, const double* L, int64_t ldl,
                                int64_t n_pad, const double* half_y, double* dot, double* sq, int64_t chunk, double* ws,
                                int64_t ws_elems, int32_t slices, void* oz_ws, int64_t oz_ws_bytes, void* stream);
int gpk_posterior_marginals_f32(const gpk_kernel_desc* desc_host, const float* xsg, int64_t xsg_gstride, int64_t m,
                                const float* xg, int64_t xg_gstride, int64_t n, int32_t d, const float* L, int64_t ldl,
                                int64_t n_pad, const float* half_y, float* dot, float* sq, int64_t chunk, float* ws,
                                int64_t ws_elems, void* stream);

/* The same for a sparse (inducing-point) posterior, PosteriorKernel(z, K_z) + SubspaceKernel(z, A) with PosteriorMean(z, K_z, mu)
 * (stheno/model/observations.py:255-277), batch 1, at ns test points:
 *   V^T = k(x*, z) L_z^-T,  U^T = k(x*, z) L_S^-T   (K1 rows once, copied on the device, two right TRSMs)
 *   dot[i] = <v_i, half_y>;  sq_z[i] = |v_i|^2;  sq_s[i] = |u_i|^2   (fp64 sums in both precisions)
 * Lz: padded lower factor of K_z + eps I; LS: that of the stored A (= L_z A L_z^T) + eps I; half_y = (L_z^-1 (mu - m_z(z)))^T
 * zero-padded to m_pad (dot may be NULL: variances only; sq_z and sq_s are always written).  The caller forms
 * mean = m(x*) + dot and variance = (k(x*, x*) - sq_z) + sq_s.  Test points are walked in chunks of `chunk` rows (multiple of
 * 128) through `ws` (>= gpk_sparse_posterior_ws_elems(chunk, m_pad) elements, 16-byte aligned): device memory
 * O(chunk m_pad) whatever ns is.  The emulation scratch of the fp64 entry point: gpk_trsm_right_oz_ws_bytes(m_pad, chunk). */
int64_t gpk_sparse_posterior_ws_elems(int64_t chunk, int64_t m_pad);
int gpk_sparse_posterior_marginals_f64(const gpk_kernel_desc* desc_host, const double* xsg, int64_t xsg_gstride, int64_t ns,
                                       const double* zg, int64_t zg_gstride, int64_t m, int32_t d, const double* Lz,
                                       int64_t ldlz, const double* LS, int64_t ldls, int64_t m_pad, const double* half_y,
                                       double* dot, double* sq_z, double* sq_s, int64_t chunk, double* ws, int64_t ws_elems,
                                       int32_t slices, void* oz_ws, int64_t oz_ws_bytes, void* stream);
int gpk_sparse_posterior_marginals_f32(const gpk_kernel_desc* desc_host, const float* xsg, int64_t xsg_gstride, int64_t ns,
                                       const float* zg, int64_t zg_gstride, int64_t m, int32_t d, const float* Lz, int64_t ldlz,
                                       const float* LS, int64_t ldls, int64_t m_pad, const float* half_y, float* dot,
                                       float* sq_z, float* sq_s, int64_t chunk, float* ws, int64_t ws_elems, void* stream);

/* Backward of gpk_sparse_posterior_marginals in the test inputs, the per-test-point step of one chunk of `c` points (rows;
 * c_pad = round_up(c)).  In: V, U [c_pad x m_pad] (same ld) the solved rows v_i^T = k(x*_i, z) L_z^-T and
 * u_i^T = k(x*_i, z) L_S^-T as the forward leaves them, h [m_pad] = half_y (zero padded), a [c] the upstream gradient of
 * dot (mean) and b [c] that of the variance (k - sq_z) + sq_s; either of a and b may be NULL (zero), not both; h may be
 * NULL when a is.  In place:
 *   row i of V <- a_i h - 2 b_i v_i,   row i of U <- 2 b_i u_i;   rows c .. c_pad - 1 of V and U are zeroed.
 * V and U are read only when b is given (without it they may hold anything: V becomes a_i h, U zero).
 * The caller finishes dL/dk(x*_i, z) = L_z^-T (row i of V) + L_S^-T (row i of U) with two transposed solves and contracts
 * it with dk/dx* in the rectangular K1-backward (gpk_kernel_cross_bwd).  One warp per row, fp64 arithmetic in both
 * precisions. */
int gpk_sparse_posterior_rows_bwd_f64(int64_t c, int64_t m_pad, double* V, double* U, int64_t ld, const double* h,
                                      const double* a, const double* b, void* stream);
int gpk_sparse_posterior_rows_bwd_f32(int64_t c, int64_t m_pad, float* V, float* U, int64_t ld, const float* h, const float* a,
                                      const float* b, void* stream);

/* Streamed sparse (inducing-point) accumulation -- AbstractPseudoObservations._compute, stheno/model/observations.py:279-336,
 * one chunk of `c` data points per call; K_zx (8.6 GB at n = 262144, m = 4096) is never held.  Per chunk, stream-ordered:
 *   W_c^T = k(x_c, z) L_z^-T  (:285, :301; rows = data points, [c_pad x m_pad], c_pad = round_up(c))
 *   corr_i = kdiag_i - |w_i|^2 (:304-306);  method 0 (VFE): scalars[2] += sum corr_i / kn_i (:308-310);
 *   method 1 (FITC): kn_i += corr_i (:311-313);  method 2 (DTC): neither (kdiag may be NULL)
 *   A    += W diag(1/kn) W^T   (:322; lower 128-tiles of the m_pad x m_pad accumulator, the caller starts it at I)
 *   prod += W diag(1/kn) ybar  (:327);  scalars[0] += sum log(2 pi kn_i) (:334);  scalars[1] += sum ybar_i^2 / kn_i (:335)
 * xg / zg: pre-stretched inputs [n_groups][c or m][d] (group strides given); Lz: padded lower factor of K_z + eps I
 * (gpk_potrf); ws: 16-byte aligned workspace of gpk_sparse_ws_elems(c, m_pad) elements.  The m^2 c flops of the solve and of
 * the accumulation run on the tensor cores (the int8 emulation of those (slices, oz_ws, oz_ws_bytes) admits:
 * gpk_gemm_nt_oz_ws_bytes(m_pad, m_pad, c_pad) covers the accumulation, gpk_trsm_right_oz_ws_bytes(m_pad, c_pad) the solve). */
int64_t gpk_sparse_ws_elems(int64_t c, int64_t m_pad);
int gpk_sparse_accumulate_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride, int64_t c,
                              const double* zg, int64_t zg_gstride, int64_t m, int32_t d, const double* Lz, int64_t ldl,
                              int64_t m_pad, const double* kdiag, const double* kn, const double* ybar, int32_t method,
                              double* A, int64_t lda, double* prod, double* scalars, double* ws, int64_t ws_elems,
                              int32_t slices, void* oz_ws, int64_t oz_ws_bytes, void* stream);
int gpk_sparse_accumulate_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t c,
                              const float* zg, int64_t zg_gstride, int64_t m, int32_t d, const float* Lz, int64_t ldl,
                              int64_t m_pad, const float* kdiag, const float* kn, const float* ybar, int32_t method, float* A,
                              int64_t lda, float* prod, float* scalars, float* ws, int64_t ws_elems, void* stream);

/* Backward of the streamed ELBO, the per-data-point step of one chunk of `c` points (rows; c_pad = round_up(c), layouts of
 * gpk_sparse_accumulate).  In: Wc [c_pad x m_pad] (ld ldw) the solved rows w_i^T = k(x_i, z) L_z^-T, U [c_pad x m_pad]
 * (ld ldu) the rows u_i^T = w_i^T A^-1, s [m_pad] = A^-1 prod (zero padded), q_i = |w_i|^2, kdiag, kn, ybar [c] (q and kdiag
 * NULL for DTC).  With beta_i = s.w_i, gamma_i = w_i.u_i, kappa_i = kn_i (+ kdiag_i - q_i for FITC), r_i = ybar_i - beta_i,
 * g_kappa_i = (r_i^2 + gamma_i - kappa_i) / (2 kappa_i^2):
 *   g_ybar_i = dE/dybar_i = -r_i / kappa_i;   g_kn_i = dE/dkn_i;   g_kd_i = dE/dkdiag_i (not written for DTC);
 *   row i of U <- g_i^T, g_i = dE/dw_i = (s r_i - u_i) / kappa_i + 2 g_q,i w_i;  rows c .. c_pad - 1 of U are zeroed.
 *   method 0 (VFE): g_kn = g_kappa + (kdiag - q) / (2 kn^2), g_kd = -1 / (2 kn), g_q = 1 / (2 kn)
 *   method 1 (FITC): g_kn = g_kd = g_kappa, g_q = -g_kappa;   method 2 (DTC): g_kn = g_kappa, g_q = 0
 * One warp per row, fp64 accumulation in both precisions, no atomics. */
int gpk_sparse_rows_bwd_f64(int64_t c, int64_t m_pad, const double* Wc, int64_t ldw, double* U, int64_t ldu, const double* s,
                            const double* q, const double* kdiag, const double* kn, const double* ybar, int32_t method,
                            double* g_kn, double* g_kd, double* g_ybar, void* stream);
int gpk_sparse_rows_bwd_f32(int64_t c, int64_t m_pad, const float* Wc, int64_t ldw, float* U, int64_t ldu, const float* s,
                            const float* q, const float* kdiag, const float* kn, const float* ybar, int32_t method,
                            float* g_kn, float* g_kd, float* g_ybar, void* stream);

/* Random-feature evaluation of a pathwise function sample (stheno_b200/pathwise.py):
 *   out[i][s] = (accumulate ? out[i][s] : 0) + sum_j W[s][j] amp[j] cos(x_i . omega[j] + b[j]),   i < n, s < num
 * x: [n x d] (ld = ldx), omega: [F x d] dense (already divided by the length scales), b, amp: [F], W: [num x F] (ld = ldw),
 * out: [n x num] (ld = ldo).  The n x F feature matrix is never written to memory: feature blocks are formed in shared memory
 * or registers and contracted at once, on the fp64 tensor cores (DMMA) for the fp64 entry point with num >= 8 and by
 * CUDA-core FMAs otherwise.  The phase x . omega + b is formed in fp64 in both precisions and its cosine is the library one
 * (full accuracy at large arguments); the fp32 entry point sums in fp32.  A row of x holding a NaN gives a NaN row. */
int gpk_feature_eval_f64(const double* x, int64_t ldx, int64_t n, int32_t d, const double* omega, const double* b,
                         const double* amp, int64_t F, const double* W, int64_t ldw, int32_t num, double* out, int64_t ldo,
                         int32_t accumulate, void* stream);
int gpk_feature_eval_f32(const float* x, int64_t ldx, int64_t n, int32_t d, const float* omega, const float* b,
                         const float* amp, int64_t F, const float* W, int64_t ldw, int32_t num, float* out, int64_t ldo,
                         int32_t accumulate, void* stream);

/* Measurement helper (bench.py): runs a register-resident fp64 tensor-core (DMMA) loop on every SM and returns the
 * achieved TFLOP/s -- the denominator of the fp64 roofline -- or a negative error code.  Synchronises the device. */
double gpk_probe_dmma_tflops(void);

/* In-situ timing of the dominant kernel (the fp64 tensor-core GEMM) for bench.py's roofline leg: while enabled every
 * launch is bracketed by CUDA events on its own stream; read() (after the caller synchronised the device) returns the
 * summed durations, the summed ALGORITHMIC flops (2*128*128*K per computed tile) and the launch count.
 * enable(0/1) also clears the record. */
void gpk_gemm_profile_enable(int32_t on);
int gpk_gemm_profile_read_kind(int32_t kind, double* total_ms, double* total_flops, int64_t* launches); /* 0 DMMA, 1 int8 emulation, -1 all */
int gpk_gemm_profile_read(double* total_ms_host, double* total_flops_host, int64_t* launches_host);

/* Test helper (no GPU needed): the tile order of the emulated GEMM evaluated on the host -- tile index t of a launch with
 * tiles_m x tiles_n tiles (128 x 64; `lower`: only the tiles touching the lower triangle; `band`: tile rows per band) ->
 * (*tm, *tn).  Returns the number of tiles of the launch. */
int32_t gpk_debug_oz_tile(int32_t lower, int32_t tiles_m, int32_t tiles_n, int32_t band, int32_t t, int32_t* tm, int32_t* tn);

/* Measurement helper (tools/time_leaf_phases.py): while `buf` (>= 16 int64, device memory) is set, every leaf-Cholesky launch
 * records clock64() at its phase boundaries there; NULL switches it off.  Synchronises the device. */
int gpk_debug_leaf_phase_clock(void* buf16_int64);

/* Number of kernels this library has launched since load / the last reset (bench.py's `gpu_launches`). */
int64_t gpk_launch_count(void);
void gpk_launch_count_reset(void);

#ifdef __cplusplus
}
#endif
#endif /* GPK_H_ */
